#!/usr/bin/env python3
"""ppsnark + IPA (RelaxedR1CSSNARK of spartan/ppsnark.rs over provider/ipa_pc.rs, the engine of every non-BN254
half) on one GPU, on a synthetic shape with a sha256-circuit-like profile (tools/ppsnark_replay.synth_matrix):
2^LOG2CONS constraints, 2^(LOG2CONS+1) witness variables, about 3.9 entries per row over A, B, C, so
N = 2^(LOG2CONS+2).

    python tools/spark_ipa_replay.py [--log2cons 16] [--curve 1] [--reps 3] [--check]

Timed, best of --reps after one warm-up run:
  setup      nova_b200.ppsnark.setup: SparkRepr.from_shape (b200_spark_repr_dev) and the seven shape commitments;
             once, against the host path it replaces: SparkRepr.from_numpy (host arrays, np.bincount, upload) and
             the seven commitments by the C oracle's multi-threaded MSM on the CPU
  prove      ppsnark.prove(ee="ipa"): the phases of prove_core, then the IPA opening split into the batched
             commitment, b_vec (eq table), the inner products, the scalar vectors + the two N-point commitments
             per round, and the folds.
The key is a synthetic Pedersen key (k0 + i) G with ck_c = (k0 + N) G; the transcript is the reference's Keccak
transcript (nova_b200.transcript).  --check verifies the last proof with the restated verifier
(tests/ppsnark_ipa_ref.verify_ipa) with S_comm, U and the verifier's N-point MSM from the C oracle.
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
import numpy as np

from mercury_replay import gpu_info
from ppsnark_replay import synth_matrix

VK_DIGEST = 1234
K0 = 0x5EED  # CommitmentKey.setup_synthetic's default


def build(curve_id: int, log2cons: int, seed: int = 5) -> dict:
    """Registered matrices, a satisfying relaxed instance (E = Az o Bz - u Cz) resident on the device, and the host
    arrays SparkRepr.from_numpy takes."""
    import nova_b200 as nb
    from nova_b200 import fields, ppsnark as dp, spartan as sp
    from nova_b200.native import check, lib
    L = lib()
    curve = nb.Curve(curve_id)
    fid = curve.scalar_field
    p = fields.MODULUS[fid]
    rng = np.random.default_rng(seed)
    num_cons, num_vars, num_io = 1 << log2cons, 2 << log2cons, 2
    ncols = num_vars + 1 + num_io
    table = np.frombuffer(b"".join(fields.to_mont_bytes(fid, v) for v in (1, p - 1, 2)), dtype=np.uint64).reshape(3, 4)
    mats, rows_all, cols_all, vals = {}, [], [], []
    for name, extra in (("A", 0.5), ("B", 0.3), ("C", 0.1)):
        r, idx, ptr, codes = synth_matrix(rng, num_cons, ncols, extra)
        v = np.ascontiguousarray(table[codes])
        h = ctypes.c_uint64(0)
        check(L.b200_spmv_register(fid, v.ctypes.data_as(ctypes.c_void_p), idx.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)),
                                   ptr.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)), num_cons, ncols, ctypes.byref(h)))
        mm = sp.SparseMatrix.__new__(sp.SparseMatrix)
        mm.fid, mm.rows, mm.cols, mm.nnz, mm.handle = fid, num_cons, ncols, len(idx), h.value
        mats[name] = mm
        rows_all.append(r)
        cols_all.append(idx.astype(np.uint32))
        vals.append(v)
    bits = rng.integers(0, 2, size=num_vars, dtype=np.uint64)  # witness: bits, 10 % of them replaced by wide values
    Wd = dp.dev_from_u64(fid, bits)
    wb = np.frombuffer(Wd.to_bytes(), dtype=np.uint64).reshape(num_vars, 4).copy()
    sel = np.flatnonzero(rng.random(num_vars) < 0.1)
    wb[sel] = np.frombuffer(b"".join(fields.to_mont_bytes(fid, int(x)) for x in rng.integers(1, 1 << 62, size=len(sel))),
                            dtype=np.uint64).reshape(-1, 4)
    check(L.b200_memcpy_h2d(Wd.ptr, wb.ctypes.data_as(ctypes.c_void_p), 32 * num_vars))
    u = int(rng.integers(1, 1 << 62))
    X = [int(rng.integers(1, 1 << 62)) for _ in range(num_io)]
    z = sp.DeviceVec(32 * ncols)
    check(L.b200_memcpy_d2d(z.ptr, Wd.ptr, 32 * num_vars, None))
    tail = fields.pack(fid, [u] + X)
    check(L.b200_memcpy_h2d(dp.View(z, num_vars).ptr, ctypes.create_string_buffer(tail, len(tail)), len(tail)))
    Az, Bz, Cz = (sp.DeviceVec(32 * num_cons) for _ in range(3))
    for name, out in (("A", Az), ("B", Bz), ("C", Cz)):
        check(L.b200_spmv_dev(mats[name].handle, z.ptr, None, out.ptr, None, None))
    Ed, zero, u_dev = sp.DeviceVec(32 * num_cons), dp.dev_zeros(num_cons), dp.dev_scalar(fid, u)
    check(L.b200_cross_term_dev(fid, Az.ptr, Bz.ptr, Cz.ptr, zero.ptr, None, u_dev.ptr, num_cons, Ed.ptr, None))
    check(L.b200_sync())
    return dict(curve=curve, fid=fid, p=p, S=dict(num_cons=num_cons, num_vars=num_vars, **mats), W=Wd, E=Ed, u=u, X=X,
                host=(np.concatenate(rows_all), np.concatenate(cols_all), vals))


def key_for(curve, N: int):
    """Pedersen key (k0 + i) G, i < N, with ck_c = (k0 + N) G as its blinding generator"""
    import nova_b200 as nb
    return nb.CommitmentKey.setup_synthetic(curve, N, K0, with_h=True)


def oracle_check(inst: dict, ck, spark, S_comm: dict, U: dict, proof: dict) -> dict:
    """The restated verifier on `proof`, with S_comm, U and the verifier's N-point MSM from the C oracle; also
    whether the device's S_comm and U equal the C oracle's."""
    from nova_b200 import fields
    from oracle import coracle as co
    from oracle.pyref import CURVES
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import ppsnark_ipa_ref as ipr
    cid, fid, p, N, S = int(inst["curve"]), inst["fid"], inst["p"], spark.N, inst["S"]
    c = CURVES[cid]
    bases = ck.export_bases(0, N)
    commit = lambda raw: c.affine_from_bytes(co.msm(cid, raw, bases[:2 * len(raw)]))  # 32-byte scalars, 64-byte bases
    S_comm_o = {k: commit(getattr(spark, k).to_bytes(32 * N)) for k in S_comm}
    U_o = dict(U, comm_W=commit(inst["W"].to_bytes(32 * S["num_vars"])),
               comm_E=commit(inst["E"].to_bytes(32 * S["num_cons"])))
    ck_pts = [c.affine_from_bytes(bases[64 * i:64 * i + 64]) for i in range(N)]
    ck_c = c.mul(K0 + N, c.gen)
    msm = lambda scalars, _pts: commit(fields.pack(fid, scalars))  # ipa_verify's ck_hat over all N bases
    ok = ipr.verify_ipa(p, c, ck_pts, ck_c, S["num_cons"], S["num_vars"], N, U_o, S_comm_o, VK_DIGEST, proof, msm=msm)
    return {"S_comm_equal": S_comm_o == S_comm, "U_equal": U_o == U, "verified": bool(ok)}


def run(log2cons=16, curve_id=1, reps=3, check_proof=False):
    from nova_b200 import ppsnark as dp
    from nova_b200.native import check, lib
    from nova_b200.transcript import Keccak256Transcript
    check(lib().b200_init(0))
    inst = build(curve_id, log2cons)
    curve, fid, p, S = inst["curve"], inst["fid"], inst["p"], inst["S"]
    # device setup (first call warms the pool and the key's workspace; both timed calls are after it)
    spark = dp.SparkRepr.from_shape(fid, S)
    N = spark.N
    ck = key_for(curve, N)
    dp.setup(curve, ck, S)
    check(lib().b200_sync())
    t0 = time.perf_counter()
    spark = dp.SparkRepr.from_shape(fid, S)
    check(lib().b200_sync())
    t1 = time.perf_counter()
    spark, S_comm = dp.setup(curve, ck, S)
    check(lib().b200_sync())
    t2 = time.perf_counter()
    # the host path: numpy + upload, then the seven commitments on the CPU
    from oracle import coracle as co
    rows, cols, vals = inst["host"]
    t3 = time.perf_counter()
    host = dp.SparkRepr.from_numpy(fid, rows, cols, vals, S["num_cons"], S["num_vars"])
    check(lib().b200_sync())
    t4 = time.perf_counter()
    bases = ck.export_bases(0, N)
    vecs = [getattr(host, k).to_bytes(32 * N) for k in dp.SHAPE_COMMITMENTS]
    t5 = time.perf_counter()
    for v in vecs:
        co.msm(int(curve), v, bases)
    t6 = time.perf_counter()
    same = all(getattr(host, k).to_bytes() == getattr(spark, k).to_bytes()
               for k in dp.SHAPE_COMMITMENTS + ("row_idx", "col_idx"))
    U = dict(comm_W=dp.commit_dev(curve, ck, inst["W"], S["num_vars"]), comm_E=dp.commit_dev(curve, ck, inst["E"], S["num_cons"]),
             u=inst["u"], X=inst["X"])
    runs, proof = [], None
    for rep in range(reps + 1):  # rep 0 warms up
        tm = {}
        t7 = time.perf_counter()
        proof = dp.prove(curve, ck, S, spark, U, dict(W=inst["W"], E=inst["E"]), VK_DIGEST,
                         Keccak256Transcript(p, b"RelaxedR1CSSNARK"), timings=tm, ee="ipa", S_comm=S_comm)
        check(lib().b200_sync())
        tm["total"] = time.perf_counter() - t7
        if rep or not reps:
            runs.append(tm)
    best = min(runs, key=lambda t: t["total"])
    ms = {k: round(v * 1e3, 3) for k, v in best.items()}
    ipa = round(sum(v for k, v in ms.items() if k.startswith("ipa")), 3)
    out = {"workload": f"ppsnark + IPA, sha256-like synthetic shape, {curve.name}", "num_cons": S["num_cons"],
           "num_vars": S["num_vars"], "nnz": int(len(rows)), "N": N, **gpu_info(), "reps": reps,
           "setup_ms": {"device_from_shape": round((t1 - t0) * 1e3, 3), "device_setup_total": round((t2 - t1) * 1e3, 3),
                        "host_from_numpy": round((t4 - t3) * 1e3, 3),
                        "host_commit_cpu": round((t6 - t5) * 1e3, 3), "cpu_threads": co.ncores(),
                        "same_vectors": bool(same)},
           "prove_ms": ms, "ipa_ms": ipa, "ipa_share": round(ipa / ms["total"], 3),
           "totals_over_reps_ms": [round(t["total"] * 1e3, 3) for t in runs]}
    if check_proof:
        t8 = time.time()
        out["check"] = oracle_check(inst, ck, spark, S_comm, U, proof)
        out["check_s"] = round(time.time() - t8, 1)
    ck.release()
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2cons", type=int, default=16)
    ap.add_argument("--curve", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check", action="store_true")
    a = ap.parse_args()
    res = run(a.log2cons, a.curve, a.reps, a.check)
    print(json.dumps(res))
    if a.check and not all(res["check"].values()):
        sys.exit(1)
