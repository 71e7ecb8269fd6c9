"""Host-side mirror of spartan::snark::RelaxedR1CSSNARK::prove up to the evaluation argument
(src/spartan/snark.rs:113-256; SURVEY.md §3.5, §8a row a32), every O(N) step on the device:

  z = (W, u, X), (Az, Bz, Cz) = S.multiply_vec(z)                 snark.rs:131-147   b200_spmv_dev x3
  poly_uCz_E = u*Cz + E                                            snark.rs:148-150   b200_axpy_dev
  outer sum-check  prove_cubic_with_three_inputs                   snark.rs:159-166   b200_sumcheck_cubic3 *
  claim_Cz = Cz(r_x), eval_E = E(r_x)                              snark.rs:170-171   b200_mle_eval_dev
  evals_rx, compute_eval_table_sparse, A + r B + r^2 C             snark.rs:181-195   b200_eq_table_dev,
                                                                                      b200_spmv_t_dev x3, b200_rlc_dev
  inner sum-check  prove_quad_prod over (poly_ABC, poly_z)         snark.rs:202-208   b200_sumcheck_quad_prod *
  eval_W = W(r_y[1..])                                             snark.rs:218       b200_mle_eval_dev
  batch_eval_reduce -> (C, x, e) and the batched polynomial        spartan/mod.rs:377-432

  * `device_transcript=True` runs each of the two sum-check loops as ONE call with the Keccak transcript
    on the device (csrc/capi_sumcheck.inc); False keeps the per-round host transcript (the D2H ->
    algebra -> H2D path).  Both produce identical prover messages.

W, E and the batched opening polynomial stay resident; the caller hands the result to the evaluation
argument (spartan.hyperkzg_prove_resident).  The transcript object is passed in and advanced exactly
as E::TE is in the reference (needs `absorb_bytes`, `squeeze` and the serialisable fields `round`,
`state`, `buf`).

verify_core / verify restate RelaxedR1CSSNARK::verify (snark.rs:259-396): the sum-check checks and the batch
evaluation claim are O(log N) host algebra; the three R1CS matrix evaluations (multi_evaluate, snark.rs:325-355),
the verifier's only O(nnz) step, run on the device (b200_eq_table_dev x2, b200_r1cs_eval_dev), and with the IPA
evaluation engine so do the opening's tensor vector and its n-point commitment (ipa.InnerProductArgument.verify).
"""
from __future__ import annotations

from . import fields
from .native import check, lib
from .ppsnark import View, _as_dev, _mle_eval, _rlc_dev, commitment_transcript_bytes, dev_scalar, dev_zeros, to_repr
from .provider import CommitmentKey, Curve, DlogGroup, _cbuf
from .spartan import DeviceVec, R1CSShape, SumcheckProof


def _affine_bytes(curve: Curve, P) -> bytes:
    if P is None:
        return bytes(64)
    fid = curve.base_field
    return fields.to_mont_bytes(fid, P[0]) + fields.to_mont_bytes(fid, P[1])


def prove_core(curve, ck: CommitmentKey | None, S: dict, U: dict, W: dict, vk_digest: int, transcript,
               device_transcript: bool = True, timings: dict | None = None):
    """S: dict(num_cons, num_vars, A, B, C) with A/B/C `spartan.SparseMatrix` (regular shape: powers of
    two, num_io < num_vars).  U: dict(comm_W, comm_E (affine or None), u, X: ints).  W: dict(W, E) as
    Montgomery bytes or DeviceVec.  Returns the proof fields of RelaxedR1CSSNARK (without eval_arg), the
    joint opening claim (batched_c, batched_x, batched_e) and the batched polynomial (DeviceVec)."""
    import time
    curve = Curve(curve)
    t_last = [time.perf_counter()]

    def mark(name):
        if timings is not None:
            check(lib().b200_sync())
            now = time.perf_counter()
            timings[name] = timings.get(name, 0.0) + now - t_last[0]
            t_last[0] = now
    fid = curve.scalar_field
    p = fields.MODULUS[fid]
    num_cons, num_vars = S["num_cons"], S["num_vars"]
    nrx, nry = num_cons.bit_length() - 1, num_vars.bit_length()
    assert 1 << nrx == num_cons and 1 << (nry - 1) == num_vars and len(U["X"]) < num_vars
    tr = transcript
    tr.absorb_bytes(b"vk", to_repr(vk_digest % p))
    tr.absorb_bytes(b"U", commitment_transcript_bytes(U["comm_W"]) + commitment_transcript_bytes(U["comm_E"])
                    + to_repr(U["u"] % p) + b"".join(to_repr(x % p) for x in U["X"]))
    Wd, Ed = _as_dev(W["W"]), _as_dev(W["E"])
    # poly_z = (W, u, X) zero-extended to 2 * num_vars (snark.rs:197-200); also the SpMV input
    z = dev_zeros(2 * num_vars)
    check(lib().b200_memcpy_d2d(z.ptr, Wd.ptr, 32 * num_vars, None))
    check(lib().b200_memcpy_h2d(View(z, num_vars).ptr, _cbuf(fields.pack(fid, [U["u"]] + list(U["X"]))),
                                32 * (1 + len(U["X"]))))
    tau = [tr.squeeze(b"t") for _ in range(nrx)]
    Az, Bz, Cz = (DeviceVec(32 * num_cons) for _ in range(3))
    for M, out in ((S["A"], Az), (S["B"], Bz), (S["C"], Cz)):
        check(lib().b200_spmv_dev(M.handle, z.ptr, None, out.ptr, None, None))
    u_dev = dev_scalar(fid, U["u"])
    uCz_E = DeviceVec(32 * num_cons)
    check(lib().b200_axpy_dev(fid, Ed.ptr, Cz.ptr, u_dev.ptr, num_cons, uCz_E.ptr, None))  # E + u*Cz
    mark("spmv")
    outer = (SumcheckProof.prove_cubic_with_three_inputs_device if device_transcript
             else SumcheckProof.prove_cubic_with_three_inputs)
    sc_outer, r_x, claims_outer = outer(fid, 0, tau, Az, Bz, uCz_E, tr)
    claim_Az, claim_Bz = claims_outer[0], claims_outer[1]
    rx_dev = DeviceVec.from_bytes(fields.pack(fid, r_x))
    claim_Cz = _mle_eval(fid, Cz, nrx, rx_dev)
    eval_E = _mle_eval(fid, Ed, nrx, rx_dev)
    tr.absorb_bytes(b"claims_outer", b"".join(to_repr(x) for x in (claim_Az, claim_Bz, claim_Cz, eval_E)))
    mark("outer_sumcheck")
    r = tr.squeeze(b"r")
    claim_inner_joint = (claim_Az + r * claim_Bz + r * r * claim_Cz) % p
    evals_rx = DeviceVec(32 * num_cons)
    check(lib().b200_eq_table_dev(fid, rx_dev.ptr, nrx, evals_rx.ptr, None))
    tabs = [DeviceVec(32 * 2 * num_vars) for _ in range(3)]  # compute_eval_table_sparse, spartan/mod.rs:497-534
    for M, out in zip((S["A"], S["B"], S["C"]), tabs):
        check(lib().b200_spmv_t_dev(M.handle, evals_rx.ptr, 2 * num_vars, out.ptr, None))
    poly_ABC = DeviceVec(32 * 2 * num_vars)
    _rlc_dev(fid, tabs, [1, r, r * r % p], 2 * num_vars, poly_ABC)
    mark("eval_tables")
    inner = SumcheckProof.prove_quad_prod_device if device_transcript else SumcheckProof.prove_quad_prod
    sc_inner, r_y, _ = inner(fid, claim_inner_joint, nry, poly_ABC, z, tr)
    eval_W = _mle_eval(fid, Wd, nry - 1, DeviceVec.from_bytes(fields.pack(fid, r_y[1:])))
    tr.absorb_bytes(b"w", to_repr(eval_W))
    mark("inner_sumcheck")
    # batch_eval_reduce (spartan/mod.rs:377-432)
    u_vec = [(U["comm_W"], r_y[1:], eval_W), (U["comm_E"], r_x, eval_E)]
    num_rounds = [len(x) for (_, x, _) in u_vec]
    rho = tr.squeeze(b"r")
    powers = [pow(rho, i, p) for i in range(len(u_vec))]
    sc_batch, r_b, evals_batch = SumcheckProof.prove_batch_eval(fid, [e for (_, _, e) in u_vec], num_rounds,
                                                                [Wd, Ed], [x for (_, x, _) in u_vec], powers, tr)
    tr.absorb_bytes(b"l", b"".join(to_repr(x) for x in evals_batch))
    c = tr.squeeze(b"c")
    nmax = len(r_b)
    batched_e, coeffs = 0, []
    for i, (ev, nv) in enumerate(zip(evals_batch, num_rounds)):  # PolyEvalInstance::batch_diff_size, mod.rs:304-344
        lag = 1
        for rr in r_b[:nmax - nv]:
            lag = lag * (1 - rr) % p
        g = pow(c, i, p)
        coeffs.append(g)
        batched_e = (batched_e + g * lag * ev) % p
    # C = sum_i c^i C_i : a two-term MSM over the commitments themselves
    batched_c = DlogGroup(curve).vartime_multiscalar_mul(
        fields.pack(fid, coeffs), b"".join(_affine_bytes(curve, cm) for (cm, _, _) in u_vec))
    size_max = max(num_vars, num_cons)
    batched_poly = DeviceVec(32 * size_max)  # PolyEvalWitness::batch_diff_size, mod.rs:165-222
    _rlc_dev(fid, [Wd, Ed], coeffs, size_max, batched_poly, lens=[num_vars, num_cons])
    mark("batch_eval_reduce")
    return dict(sc_proof_outer=sc_outer, claims_outer=(claim_Az, claim_Bz, claim_Cz), eval_E=eval_E,
                sc_proof_inner=sc_inner, eval_W=eval_W, sc_proof_batch=sc_batch, evals_batch=evals_batch,
                r_x=r_x, r_y=r_y, batched_c=batched_c, batched_x=r_b, batched_e=batched_e, batched_poly=batched_poly)


def prove(curve, ck: CommitmentKey, S: dict, U: dict, W: dict, vk_digest: int, transcript, device_transcript: bool = True,
          timings: dict | None = None, ee: str = "hyperkzg"):
    """The whole RelaxedR1CSSNARK::prove (snark.rs:113-256): prove_core, then EE::prove on the batched claim with
    the same transcript; `ck` must be the key the commitments in U were made with.
      ee = "hyperkzg": hyperkzg.rs:926-1116 (primary curve, S1)       -> eval_arg = (com, w, v)
      ee = "ipa":      ipa_pc.rs:64-77, 174-285 (secondary curve, S2) -> eval_arg = (L_vec, R_vec, a_hat);
                       `ck` must carry the generator ck_c as its blinding base.
      ee = "mercury":  mercury.rs:891-1268 (BN254, HyperKZG key)      -> eval_arg = mercury.EvaluationArgument,
                       on the batched claim (batched_c, batched_x, batched_e)."""
    proof = prove_core(curve, ck, S, U, W, vk_digest, transcript, device_transcript, timings)
    if ee == "hyperkzg":
        from .spartan import hyperkzg_prove
        proof["eval_arg"] = hyperkzg_prove(curve, ck, proof["batched_poly"], proof["batched_x"], transcript, timings)
    elif ee == "mercury":
        from .mercury import mercury_prove
        proof["eval_arg"] = mercury_prove(curve, ck, proof["batched_poly"], proof["batched_x"], transcript, timings,
                                          comm=proof["batched_c"], eval_=proof["batched_e"])
    elif ee == "ipa":
        from .ipa import prove_at_point
        proof["eval_arg"] = prove_at_point(curve, ck, proof["batched_c"], proof["batched_x"], proof["batched_e"],
                                           proof["batched_poly"], transcript)
    else:
        raise ValueError(f"unknown evaluation engine {ee!r}")
    return proof


def _eq_evaluate(p, a, b) -> int:
    """EqPolynomial::evaluate (polys/eq.rs:38-47): prod (a_i b_i + (1 - a_i)(1 - b_i))"""
    out = 1
    for x, y in zip(a, b):
        out = out * (x * y + (1 - x) * (1 - y)) % p
    return out


def _sparse_poly_evaluate(p, num_vars, Z, r) -> int:
    """SparsePolynomial::evaluate (polys/multilinear.rs:207-225) of the public IO (u, X) at r."""
    assert len(r) == num_vars
    nvz = (max(len(Z), 1) - 1).bit_length()  # log2 of next_power_of_two(len(Z))
    assert num_vars - 1 - nvz >= 0, "public IO too long for the shape"
    k = num_vars - 1 - nvz
    tail = r[k:]  # Z pairs with the first len(Z) entries of eq(tail), each a product over its bits
    partial = 0
    for i, z in enumerate(Z):
        chi = 1
        for j, x in enumerate(tail):
            chi = chi * (x if (i >> (len(tail) - 1 - j)) & 1 else 1 - x) % p
        partial += z * chi
    common = 1
    for x in r[:k]:
        common = common * (1 - x) % p
    return common * partial % p


def verify_core(curve, S: dict, U: dict, vk_digest: int, proof: dict, transcript, timings: dict | None = None):
    """RelaxedR1CSSNARK::verify (snark.rs:259-396) up to EE::verify, with batch_eval_verify (spartan/mod.rs:436-480):
    re-derives every challenge, checks both sum-checks' final claims -- the inner one against the three matrix
    evaluations, computed on the device -- and the batch-evaluation claim.  S, U, vk_digest as in prove_core; `proof`
    the fields prove_core returns (sc_proof_outer, claims_outer, eval_E, sc_proof_inner, eval_W, sc_proof_batch,
    evals_batch); `transcript` fresh, labelled b"RelaxedR1CSSNARK", and advanced to where EE::verify starts.
    Returns the joint claim (C, x, e) for any evaluation engine; a failed check raises
    ValueError("InvalidSumcheckProof").  `timings` (optional): "sumcheck_checks", "eq_tables", "matrix_eval",
    "batch_eval_verify" in seconds."""
    from .ipa import _marker
    mark = _marker(timings)
    curve = Curve(curve)
    fid = curve.scalar_field
    p = fields.MODULUS[fid]
    num_cons, num_vars = S["num_cons"], S["num_vars"]
    nrx, nry = num_cons.bit_length() - 1, num_vars.bit_length()
    assert 1 << nrx == num_cons and 1 << (nry - 1) == num_vars and len(U["X"]) < num_vars
    u = U["u"] % p
    tr = transcript
    tr.absorb_bytes(b"vk", to_repr(vk_digest % p))
    tr.absorb_bytes(b"U", commitment_transcript_bytes(U["comm_W"]) + commitment_transcript_bytes(U["comm_E"])
                    + to_repr(u) + b"".join(to_repr(x % p) for x in U["X"]))
    tau = [tr.squeeze(b"t") for _ in range(nrx)]
    claim_outer_final, r_x = SumcheckProof.verify(fid, proof["sc_proof_outer"], 0, nrx, 3, tr)
    cAz, cBz, cCz = (x % p for x in proof["claims_outer"])
    eval_E, eval_W = proof["eval_E"] % p, proof["eval_W"] % p
    if claim_outer_final != _eq_evaluate(p, tau, r_x) * (cAz * cBz - u * cCz - eval_E) % p:
        raise ValueError("InvalidSumcheckProof")  # snark.rs:283-288
    tr.absorb_bytes(b"claims_outer", b"".join(to_repr(x) for x in (cAz, cBz, cCz, eval_E)))
    r = tr.squeeze(b"r")
    claim_inner_final, r_y = SumcheckProof.verify(fid, proof["sc_proof_inner"], (cAz + r * cBz + r * r * cCz) % p,
                                                  nry, 2, tr)
    eval_X = _sparse_poly_evaluate(p, nry - 1, [u] + [x % p for x in U["X"]], r_y[1:])
    eval_Z = ((1 - r_y[0]) * eval_W + r_y[0] * eval_X) % p
    mark("sumcheck_checks")
    T_x, T_y = DeviceVec(32 * num_cons), DeviceVec(32 << nry)
    rx_dev, ry_dev = DeviceVec.from_bytes(fields.pack(fid, r_x)), DeviceVec.from_bytes(fields.pack(fid, r_y))
    check(lib().b200_eq_table_dev(fid, rx_dev.ptr, nrx, T_x.ptr, None))
    check(lib().b200_eq_table_dev(fid, ry_dev.ptr, nry, T_y.ptr, None))
    mark("eq_tables")
    evA, evB, evC = R1CSShape(S["A"], S["B"], S["C"]).multi_evaluate_dev(T_x, num_cons, T_y, 1 << nry)
    mark("matrix_eval")
    if claim_inner_final != (evA + r * evB + r * r * evC) * eval_Z % p:
        raise ValueError("InvalidSumcheckProof")  # snark.rs:355-358
    tr.absorb_bytes(b"w", to_repr(eval_W))
    # batch_eval_verify (spartan/mod.rs:436-480) over the claims W(r_y[1..]) = eval_W and E(r_x) = eval_E
    u_vec = [(U["comm_W"], r_y[1:], eval_W), (U["comm_E"], r_x, eval_E)]
    evals_batch = [x % p for x in proof["evals_batch"]]
    if len(evals_batch) != len(u_vec):
        raise ValueError("InvalidInputLength")  # the reference's assert_eq (mod.rs:445)
    rho = tr.squeeze(b"r")
    powers = [pow(rho, i, p) for i in range(len(u_vec))]
    num_rounds = [len(x) for (_, x, _) in u_vec]
    nmax = max(num_rounds)
    claim_batch_final, r_b = SumcheckProof.verify_batch(fid, proof["sc_proof_batch"], [e for (_, _, e) in u_vec],
                                                        num_rounds, powers, 2, tr)
    expected = sum(_eq_evaluate(p, r_b[nmax - len(x):], x) * ev * k
                   for (_, x, _), ev, k in zip(u_vec, evals_batch, powers)) % p
    if claim_batch_final != expected:
        raise ValueError("InvalidSumcheckProof")  # mod.rs:471-473
    tr.absorb_bytes(b"l", b"".join(to_repr(x) for x in evals_batch))
    c = tr.squeeze(b"c")
    batched_e, coeffs = 0, []
    for i, (ev, nv) in enumerate(zip(evals_batch, num_rounds)):  # PolyEvalInstance::batch_diff_size, mod.rs:304-344
        lag = 1
        for rr in r_b[:nmax - nv]:
            lag = lag * (1 - rr) % p
        coeffs.append(pow(c, i, p))
        batched_e = (batched_e + coeffs[i] * lag * ev) % p
    batched_c = DlogGroup(curve).vartime_multiscalar_mul(
        fields.pack(fid, coeffs), b"".join(_affine_bytes(curve, cm) for (cm, _, _) in u_vec))
    mark("batch_eval_verify")
    return batched_c, r_b, batched_e


def verify(curve, S: dict, U: dict, vk_digest: int, proof: dict, transcript, ee: str = "ipa",
           ck: CommitmentKey | None = None, timings: dict | None = None):
    """The whole RelaxedR1CSSNARK::verify (snark.rs:259-396): verify_core, then EE::verify on the joint claim with the
    same transcript.  Returns None on success (the reference's Ok(())); a failed check raises ValueError with the
    reference's error kind (InvalidSumcheckProof, InvalidInputLength, InternalError, InvalidPCS).
      ee = "ipa": ipa_pc.rs:80-100, 286-396; `ck` is the Pedersen key registered with h = ck_c, at least
                  max(num_cons, num_vars) bases (checked before any device work).
    HyperKZG and Mercury end in a pairing check, which stays with the caller: take verify_core's claim."""
    if ee in ("hyperkzg", "mercury"):
        raise ValueError(f"ee={ee!r}: the pairing check is not done here; run verify_core and check its claim")
    if ee != "ipa":
        raise ValueError(f"unknown evaluation engine {ee!r}")
    from .ipa import check_key, verify_at_point
    check_key(ck, max(S["num_cons"], S["num_vars"]))
    C, x, e = verify_core(curve, S, U, vk_digest, proof, transcript, timings)
    verify_at_point(curve, ck, C, x, e, proof["eval_arg"], transcript, timings)
