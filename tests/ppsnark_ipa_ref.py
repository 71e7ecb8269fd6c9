"""ppsnark with the IPA evaluation engine (ipa_pc.rs:64-100) composed from the oracle's pieces.  TEST INFRASTRUCTURE
ONLY: oracle/ppsnark_ref.py's prove_core / verify_core and batched commitment with oracle/pyref.py's ipa_prove /
ipa_verify, the way oracle/snark_ref.py composes spartan::snark with the IPA (its prove_ipa / verify_ipa)."""
from oracle import ppsnark_ref as pr
from oracle.pyref import eq_evals, ipa_prove, ipa_verify


def prove_ipa(p, curve, ck_pts, ck_c, S, spark, U, W, vk_digest, S_comm):
    """RelaxedR1CSSNARK::prove of ppsnark.rs with EvaluationEngine::prove of provider/ipa_pc.rs:64-77: prove_core
    over the Pedersen key `ck_pts` (r = 0), then the inner-product argument between the batched polynomial and the
    eq table of r_inner_batched, on the batched commitment sum_i c^i C_i.  ck_c: the key's extra generator."""
    out = pr.prove_core(p, lambda v: curve.msm_naive(v, ck_pts[:len(v)]), S, spark, U, W, vk_digest)
    C = pr.batch_commitment(p, curve, pr.comm_vec_of(U, S_comm, out), out["batch_challenge"])
    out["eval_arg"] = ipa_prove(curve, ck_pts, ck_c, C, eq_evals(p, out["r_inner_batched"]), out["batched_eval"],
                                out["batched_poly"], out["transcript"])
    return out


class _CurveWithMsm:
    """`curve` whose msm_naive over exactly n points is `msm`: in ipa_verify that is the n-point ck_hat; its other two
    MSMs have 2 log n + 1 and 2 points, never n for n >= 4"""

    def __init__(self, curve, msm, n: int):
        self._curve, self._msm, self._n = curve, msm, n

    def __getattr__(self, name):
        return getattr(self._curve, name)

    def msm_naive(self, scalars, bases):
        return self._msm(scalars, bases) if len(bases) == self._n else self._curve.msm_naive(scalars, bases)


def verify_ipa(p, curve, ck_pts, ck_c, num_cons, num_vars, N, U, S_comm, vk_digest, proof, msm=None) -> bool:
    """RelaxedR1CSSNARK::verify of ppsnark.rs with the IPA engine's verify (ipa_pc.rs:80-100, 286-396): verify_core,
    the batched commitment and evaluation, then ipa_verify.  `msm(scalars, points) -> point`, if given, computes the
    verifier's N-point MSM (large keys pass the C oracle's); the default is curve.msm_naive."""
    holder = {}
    try:
        pr.verify_core(p, num_cons, num_vars, N, U, vk_digest, proof, holder)
    except AssertionError:
        return False
    tr = holder["tr"]
    eval_vec = [proof[k] for k in pr.EVAL_ORDER]
    tr.absorb_bytes(b"e", pr.scalars_bytes(eval_vec))
    c = tr.squeeze(b"c")
    C = pr.batch_commitment(p, curve, pr.comm_vec_of(U, S_comm, proof), c)
    e = sum(pow(c, i, p) * v for i, v in enumerate(eval_vec)) % p
    L_vec, R_vec, a_hat = proof["eval_arg"]
    if msm is not None:
        assert N >= 4
        curve = _CurveWithMsm(curve, msm, N)
    return ipa_verify(curve, ck_pts, ck_c, C, eq_evals(p, proof["r_inner_batched"]), e, L_vec, R_vec, a_hat, tr)
