#!/usr/bin/env python3
"""RelaxedR1CSSNARK::verify with the IPA evaluation engine (spartan/snark.rs:259-396 + provider/ipa_pc.rs:286-396, the
S2 verifier of CompressedSNARK on every non-BN254 half) on one GPU, on the synthetic shape of tools/spark_ipa_replay.py
(2^LOG2CONS constraints, 2^(LOG2CONS+1) witness variables, about 3.9 entries per row over A, B, C).

    python tools/verify_replay.py [--log2cons 12,16,20] [--curves 1,3] [--reps 3] [--check]

Per (curve, size), after one proof by snark.prove(ee="ipa") and one warm-up verification, best of --reps:
  verify     snark.verify(ee="ipa") split into its phases: the host sum-check checks, the two eq tables, the matrix
             evaluation (b200_r1cs_eval_dev), the batch-evaluation check with its 2-point MSM, the IPA's transcript
             scalars, s (b200_ipa_s_dev), the n-point commitment (b200_commit_dev) and the (2L+1)-point host MSM
  r1cs_ab    the fused matrix evaluation against the composition it replaces: per matrix b200_spmv_dev with z = T_y,
             then b200_sc_eval_dev form 11 (dot) with T_x -- both checked equal
  cpu        the same matrix evaluation (tests/verify_oracle.c, rows over all host cores) and the n-point MSM (the C
             oracle's MSM, all cores), once
--check also runs a tampered proof (a_hat + 1) and requires InvalidPCS.  One JSON line per (curve, size).
"""
import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np

from mercury_replay import gpu_info
from spark_ipa_replay import build, key_for

VK_DIGEST = 4321


def prove(inst, ck):
    import nova_b200 as nb
    from nova_b200 import ppsnark as dp, snark
    from nova_b200.transcript import Keccak256Transcript
    S, curve = inst["S"], inst["curve"]
    U = dict(comm_W=dp.commit_dev(curve, ck, inst["W"], S["num_vars"]),
             comm_E=dp.commit_dev(curve, ck, inst["E"], S["num_cons"]), u=inst["u"], X=inst["X"])
    tr = Keccak256Transcript(inst["p"], b"RelaxedR1CSSNARK")
    proof = snark.prove(curve, ck, S, U, dict(W=inst["W"], E=inst["E"]), VK_DIGEST, tr, ee="ipa")
    proof.pop("batched_poly").free()
    nb.lib().b200_sync()
    return U, proof


def verify(inst, ck, U, proof, timings=None):
    from nova_b200 import snark
    from nova_b200.transcript import Keccak256Transcript
    tr = Keccak256Transcript(inst["p"], b"RelaxedR1CSSNARK")
    snark.verify(inst["curve"], inst["S"], U, VK_DIGEST, proof, tr, ee="ipa", ck=ck, timings=timings)


def r1cs_ab(inst, reps):
    """(fused seconds, composed seconds), best of reps; both results checked equal"""
    from nova_b200 import spartan as sp
    from nova_b200.native import check, lib
    L = lib()
    S, fid, p = inst["S"], inst["fid"], inst["p"]
    rng = np.random.default_rng(3)
    nrx, nry = S["num_cons"].bit_length() - 1, S["num_vars"].bit_length()
    from nova_b200 import fields
    rx = sp.DeviceVec.from_bytes(fields.pack(fid, [int(x) for x in rng.integers(1, 1 << 62, size=nrx)]))
    ry = sp.DeviceVec.from_bytes(fields.pack(fid, [int(x) for x in rng.integers(1, 1 << 62, size=nry)]))
    Tx, Ty = sp.DeviceVec(32 << nrx), sp.DeviceVec(32 << nry)
    check(L.b200_eq_table_dev(fid, rx.ptr, nrx, Tx.ptr, None))
    check(L.b200_eq_table_dev(fid, ry.ptr, nry, Ty.ptr, None))
    shape = sp.R1CSShape(S["A"], S["B"], S["C"])
    Mz = sp.DeviceVec(32 << nrx)
    dot = sp.DeviceVec(96)

    def fused():
        return shape.multi_evaluate_dev(Tx, 1 << nrx, Ty, 1 << nry)

    def composed():
        for k, M in enumerate((S["A"], S["B"], S["C"])):
            check(L.b200_spmv_dev(M.handle, Ty.ptr, None, Mz.ptr, None, None))
            check(L.b200_sc_eval_dev(fid, 11, Mz.ptr, Tx.ptr, None, 1 << nrx, None, None, 0,
                                     ctypes.c_void_p(dot.ptr.value + 32 * k), None))
        return fields.unpack(fid, dot.to_bytes(96))

    out = {}
    for name, fn in (("fused", fused), ("composed", composed)):
        res = fn()
        best = float("inf")
        for _ in range(reps):
            check(L.b200_sync())
            t0 = time.perf_counter()
            fn()
            check(L.b200_sync())
            best = min(best, time.perf_counter() - t0)
        out[name] = (best, res)
    assert out["fused"][1] == out["composed"][1], "fused and composed matrix evaluations differ"
    return out["fused"][0], out["composed"][0], (Tx, Ty, nrx, nry)


def cpu_side(inst, ck, tables):
    """the matrix evaluation and the n-point MSM on the C oracle over all host cores (seconds)"""
    import verify_ref
    from oracle import coracle as co
    rows, cols, vals = inst["host"]
    S, fid, cid = inst["S"], inst["fid"], int(inst["curve"])
    Tx, Ty, nrx, nry = tables
    tx, ty = Tx.to_bytes(32 << nrx), Ty.to_bytes(32 << nry)
    ncores = os.cpu_count() or 1
    t_mat, off = 0.0, 0
    for v in vals:
        n = len(v)
        r, c = rows[off:off + n], cols[off:off + n]
        off += n
        indptr = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=S["num_cons"]))]).tolist()
        t0 = time.perf_counter()
        verify_ref.r1cs_eval(fid, v.tobytes(), c.tolist(), indptr, tx, ty, nthreads=ncores)
        t_mat += time.perf_counter() - t0
    n = S["num_vars"]
    bases = ck.export_bases(0, n)
    scalars = co.gen_scalars(fid, 11, n)
    t0 = time.perf_counter()
    co.msm(cid, scalars, bases)
    return t_mat, time.perf_counter() - t0, ncores


def run(cid, log2cons, reps=3, check_tamper=False):
    import nova_b200 as nb
    nb.lib().b200_init(0)
    inst = build(cid, log2cons)
    ck = key_for(inst["curve"], inst["S"]["num_vars"])
    U, proof = prove(inst, ck)
    verify(inst, ck, U, proof)  # warm-up; raises if the proof is rejected
    best, best_t = float("inf"), None
    for _ in range(reps):
        t = {}
        t0 = time.perf_counter()
        verify(inst, ck, U, proof, t)
        dt = time.perf_counter() - t0
        if dt < best:
            best, best_t = dt, t
    res = dict(curve=cid, log2cons=log2cons, nnz=sum(m.nnz for m in (inst["S"]["A"], inst["S"]["B"], inst["S"]["C"])),
               verify_ms=round(1e3 * best, 3), phases_ms={k: round(1e3 * v, 3) for k, v in best_t.items()})
    fused, composed, tables = r1cs_ab(inst, reps)
    res.update(r1cs_fused_ms=round(1e3 * fused, 3), r1cs_composed_ms=round(1e3 * composed, 3))
    t_mat, t_msm, ncores = cpu_side(inst, ck, tables)
    res.update(cpu_r1cs_ms=round(1e3 * t_mat, 1), cpu_msm_ms=round(1e3 * t_msm, 1), cpu_cores=ncores)
    if check_tamper:
        L_vec, R_vec, a_hat = proof["eval_arg"]
        try:
            verify(inst, ck, U, dict(proof, eval_arg=(L_vec, R_vec, (a_hat + 1) % inst["p"])))
            res["tamper"] = "accepted"
        except ValueError as e:
            res["tamper"] = str(e)
        assert res["tamper"] == "InvalidPCS", res["tamper"]
    res.update(gpu_info())
    ck.release()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2cons", default="12,16,20")
    ap.add_argument("--curves", default="1,3")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check", action="store_true")
    a = ap.parse_args()
    for cid in (int(c) for c in a.curves.split(",")):
        for lg in (int(x) for x in a.log2cons.split(",")):
            print(json.dumps(run(cid, lg, a.reps, a.check)), flush=True)


if __name__ == "__main__":
    main()
