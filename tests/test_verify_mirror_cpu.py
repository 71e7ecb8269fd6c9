"""The product's verifier (nova_b200.snark.verify_core / verify, nova_b200.ipa.InnerProductArgument.verify,
spartan.SumcheckProof.verify) on the CPU: the library is replaced by tests/emulated_device.py plus the verifier entries
of tests/emulated_verify.py, and the verdicts are compared with the oracle's restated verifier
(oracle/snark_ref.verify_ipa) on proofs the oracle made -- accepted, and rejected with the reference's error kind
whenever a proof field is altered."""
import gc

import pytest

import emulated_verify
from oracle import snark_ref as sr
from oracle.ppsnark_ref import random_instance
from oracle.pyref import CURVES, Keccak256Transcript, SplitMix64, eq_evals
from snark_parity import csr, pack


@pytest.fixture()
def emu():
    import nova_b200
    emulated_verify.install()
    yield nova_b200
    gc.collect()
    emulated_verify.uninstall()


CASES = {}


def case(cid, num_cons=8, num_vars=8, num_io=2):
    """an oracle S2 proof (snark + IPA) of a random satisfying instance, its key and shape; cached per parameters"""
    key = (cid, num_cons, num_vars, num_io)
    if key not in CASES:
        c = CURVES[cid]
        p = c.q
        rng = SplitMix64(7700 + 10 * cid + num_io + num_cons)
        S, W, u, X = random_instance(p, rng, num_cons, num_vars, num_io)
        n_key = max(num_cons, num_vars)
        pts = c.bases_arith(n_key + 1, k0=515)
        ck_pts, ck_c = pts[:n_key], pts[n_key]
        U = dict(comm_W=c.msm_naive(W["W"], ck_pts[:num_vars]), comm_E=c.msm_naive(W["E"], ck_pts[:num_cons]), u=u, X=X)
        proof = sr.prove_ipa(p, c, ck_pts, ck_c, S, U, W, 321)
        proof.pop("transcript")
        CASES[key] = (S, U, proof, ck_pts, ck_c)
    return CASES[key]


def device_shape(nb, cid, S, num_io):
    from nova_b200 import spartan as sp
    c = CURVES[cid]
    mats = {}
    for name in "ABC":
        d, idx, ptr = csr(S[name], S["num_cons"])
        mats[name] = sp.SparseMatrix(c.scalar_field, pack(c.q, d), idx, ptr, S["num_vars"] + 1 + num_io)
    return dict(num_cons=S["num_cons"], num_vars=S["num_vars"], **mats)


def key(nb, cid, ck_pts, ck_c):
    c = CURVES[cid]
    return nb.CommitmentKey(nb.Curve(cid), b"".join(c.affine_bytes(P) for P in ck_pts), c.affine_bytes(ck_c))


def oracle_verdict(cid, S, U, proof, ck_pts, ck_c):
    c = CURVES[cid]
    try:
        return bool(sr.verify_ipa(c.q, c, ck_pts, ck_c, S, U, 321, proof))
    except (AssertionError, ZeroDivisionError):
        return False


def mirror(nb, cid, S, num_io, U, proof, ck):
    """None if the mirror accepts, else the error kind it raised"""
    from nova_b200 import snark
    tr = Keccak256Transcript(CURVES[cid].q, b"RelaxedR1CSSNARK")
    try:
        snark.verify(nb.Curve(cid), device_shape(nb, cid, S, num_io), U, 321, proof, tr, ee="ipa", ck=ck)
    except ValueError as e:
        return str(e)
    return None


@pytest.mark.parametrize("num_io", [0, 1, 3])
@pytest.mark.parametrize("cid", [0, 1, 2, 3])
def test_verify_accepts_oracle_proofs(emu, cid, num_io):
    S, U, proof, ck_pts, ck_c = case(cid, num_io=num_io)
    ck = key(emu, cid, ck_pts, ck_c)
    assert oracle_verdict(cid, S, U, proof, ck_pts, ck_c)
    assert mirror(emu, cid, S, num_io, U, proof, ck) is None
    from nova_b200 import snark
    c = CURVES[cid]
    tr = Keccak256Transcript(c.q, b"RelaxedR1CSSNARK")
    got = snark.verify_core(emu.Curve(cid), device_shape(emu, cid, S, num_io), U, 321, proof, tr)
    assert got == sr.verify_core(c.q, c, S, U, 321, proof)
    assert got == (proof["batched_c"], proof["batched_x"], proof["batched_e"])


def tampered(proof, field, p):
    q = dict(proof)
    if field == "sc_outer":
        q["sc_proof_outer"] = [list(x) for x in proof["sc_proof_outer"]]
        q["sc_proof_outer"][1][0] = (q["sc_proof_outer"][1][0] + 1) % p
    elif field == "sc_inner":
        q["sc_proof_inner"] = [list(x) for x in proof["sc_proof_inner"]]
        q["sc_proof_inner"][0][-1] = (q["sc_proof_inner"][0][-1] + 1) % p
    elif field == "sc_batch":
        q["sc_proof_batch"] = [list(x) for x in proof["sc_proof_batch"]]
        q["sc_proof_batch"][-1][0] = (q["sc_proof_batch"][-1][0] + 1) % p
    elif field == "claims_outer":
        a, b, c = proof["claims_outer"]
        q["claims_outer"] = (a, (b + 1) % p, c)
    elif field in ("eval_E", "eval_W"):
        q[field] = (proof[field] + 1) % p
    elif field == "evals_batch":
        q["evals_batch"] = [proof["evals_batch"][0], (proof["evals_batch"][1] + 1) % p]
    else:
        L_vec, R_vec, a_hat = proof["eval_arg"]
        L_vec, R_vec = list(L_vec), list(R_vec)
        if field == "L_vec":
            L_vec[0] = R_vec[1]
        elif field == "R_vec":
            R_vec[-1] = L_vec[0]
        elif field == "a_hat":
            a_hat = (a_hat + 1) % p
        q["eval_arg"] = (L_vec, R_vec, a_hat)
    return q


@pytest.mark.parametrize("field,kind", [
    ("sc_outer", "InvalidSumcheckProof"), ("sc_inner", "InvalidSumcheckProof"), ("sc_batch", "InvalidSumcheckProof"),
    ("claims_outer", "InvalidSumcheckProof"), ("eval_E", "InvalidSumcheckProof"), ("eval_W", "InvalidSumcheckProof"),
    ("evals_batch", "InvalidSumcheckProof"), ("L_vec", "InvalidPCS"), ("R_vec", "InvalidPCS"), ("a_hat", "InvalidPCS"),
    ("comm_W", "InvalidSumcheckProof")])
@pytest.mark.parametrize("cid", [1, 3])
def test_tampered_proofs_rejected_as_the_reference_does(emu, cid, field, kind):
    S, U, proof, ck_pts, ck_c = case(cid)
    c = CURVES[cid]
    ck = key(emu, cid, ck_pts, ck_c)
    if field == "comm_W":  # a different instance: the transcript changes, the proof no longer opens
        U = dict(U, comm_W=c.add(U["comm_W"], ck_pts[0]))
        bad = proof
    else:
        bad = tampered(proof, field, c.q)
    got = mirror(emu, cid, S, 2, U, bad, ck)
    assert not oracle_verdict(cid, S, U, bad, ck_pts, ck_c)
    assert got == kind


def test_length_and_round_errors(emu):
    """every InvalidInputLength / InvalidSumcheckProof path that does not need a wrong proof value"""
    cid = 2
    S, U, proof, ck_pts, ck_c = case(cid)
    p = CURVES[cid].q
    ck = key(emu, cid, ck_pts, ck_c)
    L_vec, R_vec, a_hat = proof["eval_arg"]
    bad = {
        "outer rounds": dict(proof, sc_proof_outer=proof["sc_proof_outer"][:-1]),
        "inner rounds": dict(proof, sc_proof_inner=proof["sc_proof_inner"] + [[1, 2]]),
        "batch rounds": dict(proof, sc_proof_batch=proof["sc_proof_batch"][1:]),
        "outer degree": dict(proof, sc_proof_outer=[list(x) + [0] for x in proof["sc_proof_outer"]]),
        "inner degree": dict(proof, sc_proof_inner=[list(x) + [5] for x in proof["sc_proof_inner"]]),
    }
    for name, q in bad.items():
        assert mirror(emu, cid, S, 2, U, q, ck) == "InvalidSumcheckProof", name
        assert not oracle_verdict(cid, S, U, q, ck_pts, ck_c), name
    for name, arg in {"L_vec short": (L_vec[:-1], R_vec[:-1], a_hat), "R_vec short": (L_vec, R_vec[:-1], a_hat),
                      "L_vec long": (list(L_vec) + [L_vec[0]], R_vec, a_hat)}.items():
        q = dict(proof, eval_arg=arg)
        assert mirror(emu, cid, S, 2, U, q, ck) == "InvalidInputLength", name
        assert not oracle_verdict(cid, S, U, q, ck_pts, ck_c), name
    # 32 rounds is the reference's limit, whatever the lengths match
    from nova_b200 import ipa
    with pytest.raises(ValueError, match="InvalidInputLength"):
        ipa.InnerProductArgument.verify(emu.Curve(cid), ck, U["comm_W"], [0] * 3, 0, [None] * 32, [None] * 32, 0,
                                        Keccak256Transcript(p, b"t"))


def test_ipa_key_checks_and_engines(emu):
    import nova_b200 as nb
    from nova_b200 import ipa, snark
    cid = 3
    S, U, proof, ck_pts, ck_c = case(cid)
    c = CURVES[cid]
    tr = lambda: Keccak256Transcript(c.q, b"RelaxedR1CSSNARK")
    no_h = nb.CommitmentKey(nb.Curve(cid), b"".join(c.affine_bytes(P) for P in ck_pts))
    short = nb.CommitmentKey(nb.Curve(cid), b"".join(c.affine_bytes(P) for P in ck_pts[:4]), c.affine_bytes(ck_c))
    shape = device_shape(emu, cid, S, 2)
    for bad in (None, no_h, short):
        with pytest.raises(ValueError, match="IPA"):
            snark.verify(nb.Curve(cid), shape, U, 321, proof, tr(), ee="ipa", ck=bad)
        with pytest.raises(ValueError, match="IPA"):
            ipa.verify_at_point(nb.Curve(cid), bad, proof["batched_c"], proof["batched_x"], proof["batched_e"],
                                proof["eval_arg"], tr())
    for ee in ("hyperkzg", "mercury", "nope"):
        with pytest.raises(ValueError):
            snark.verify(nb.Curve(cid), shape, U, 321, proof, tr(), ee=ee, ck=short)


def test_zero_challenge_is_internal_error(emu, monkeypatch):
    """a zero round challenge makes batch_invert fail (InternalError), as in the reference"""
    from nova_b200 import ipa
    cid = 1
    S, U, proof, ck_pts, ck_c = case(cid)
    p = CURVES[cid].q
    ck = key(emu, cid, ck_pts, ck_c)

    class ZeroAfterU(Keccak256Transcript):
        def squeeze(self, label):
            v = super().squeeze(label)
            self.n = getattr(self, "n", 0) + 1
            return 0 if self.n == 3 else v  # r0, then the first two round challenges: the second is zero
    L_vec, R_vec, a_hat = proof["eval_arg"]
    with pytest.raises(ValueError, match="InternalError"):
        ipa.InnerProductArgument.verify(emu.Curve(cid), ck, proof["batched_c"], proof["batched_x"], proof["batched_e"],
                                        L_vec, R_vec, a_hat, ZeroAfterU(p, b"t"))


@pytest.mark.parametrize("L", [1, 2, 5])
def test_b_hat_closed_form(L):
    """<eq(x), s> = prod r^-1 prod ((1 - x) + x r^2), the form the verifier uses, against the O(n) inner product"""
    import verify_ref
    from oracle.pyref import FIELD_MODULUS, from_mont_bytes
    fid = 3
    p = FIELD_MODULUS[fid]
    rng = SplitMix64(40 + L)
    r, x = [rng.field(p) for _ in range(L)], [rng.field(p) for _ in range(L)]
    s_raw = verify_ref.ipa_s(fid, r)
    s = [from_mont_bytes(p, s_raw[k:k + 32]) for k in range(0, len(s_raw), 32)]
    closed = 1
    for xj, rj in zip(x, r):
        closed = closed * pow(rj, -1, p) * ((1 - xj) + xj * rj * rj) % p
    assert closed == sum(a * b for a, b in zip(eq_evals(p, x), s)) % p


def test_multi_evaluate_host_form_and_errors(emu):
    from nova_b200 import spartan as sp
    from nova_b200.native import B200_E_ARG, B200_E_HANDLE, B200_E_RANGE, B200Error, lib
    cid = 0
    S, U, proof, ck_pts, ck_c = case(cid)
    c = CURVES[cid]
    p = c.q
    shape = device_shape(emu, cid, S, 2)
    rng = SplitMix64(5)
    rx, ry = [rng.field(p) for _ in range(3)], [rng.field(p) for _ in range(4)]
    Tx, Ty = eq_evals(p, rx), eq_evals(p, ry)
    want = [sum(Tx[r] * Ty[col] * v for (r, col, v) in S[k]) % p for k in "ABC"]
    got = sp.R1CSShape(shape["A"], shape["B"], shape["C"]).multi_evaluate(rx, ry)
    assert got == want
    import ctypes
    from nova_b200.provider import _cbuf
    from nova_b200 import fields
    out = ctypes.create_string_buffer(96)
    hs = lambda *h: (ctypes.c_uint64 * 3)(*h)
    A, B = shape["A"].handle, shape["B"].handle
    r3, r2 = _cbuf(fields.pack(c.scalar_field, rx)), _cbuf(fields.pack(c.scalar_field, ry[:2]))
    assert lib().b200_r1cs_eval(hs(A, 987654, B), 3, r3, 3, r3, 3, out) == B200_E_HANDLE
    assert lib().b200_r1cs_eval(hs(A, B, A), 0, r3, 3, r3, 3, out) == B200_E_ARG
    assert lib().b200_r1cs_eval(hs(A, B, A), 4, r3, 3, r3, 3, out) == B200_E_ARG
    assert lib().b200_r1cs_eval(hs(A, B, A), 3, r3, 3, r2, 2, out) == B200_E_RANGE  # 4 entries of T_y, 11 columns
    assert out.raw == bytes(96)


def test_cpp_mirror_verifier_wrappers_compile_and_link():
    """R1CSShape::multi_evaluate, R1CSShapeDev::multi_evaluate and ipa_s (include/nova_b200.hpp) instantiate and link
    against the library"""
    import subprocess
    import verify_ref
    out = subprocess.check_output([verify_ref.cpp_mirror(), "--compile-check"], text=True)
    assert "verify_mirror_test" in out
