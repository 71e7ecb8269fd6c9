#!/usr/bin/env python3
"""NeutronNova's fold against Nova's on the same shape, on one GPU: the device restatement of the reference's
bench_nifs_inner (src/neutron/nifs.rs:533-720, generate_sample_r1cs).

    python tools/neutron_replay.py [--log2n 20] [--reps 3] [--check]

The shape is x * x = x on every variable, num_vars = num_cons = N = 2^LOG2N, num_io = 1, X = [0]; the witness is
random bits.  Each timed Neutron step commits the witness with commit_small on its u8 values (b200_msm_small) plus
the blind, then runs nova_b200.neutron.nifs_prove from the default running pair with a fresh Poseidon RO2 (the
reference's `neutron_nifs_simple_N`).  Each timed Nova step commits the witness over its field elements and runs
nova_b200.r1cs.nifs_prove against a sampled random relaxed pair (`nova_nifs_simple_N`); its challenge is a
Poseidon squeeze over comm_T on the host.  The shape, key, witness and the relaxed pair are resident before the
clock starts; every timed step ends in a device synchronise.

Reported per Neutron phase: commit_W, E_comm_E (split table and its commitment), spmv (the six SpMVs), evals (the
five sums), folds (the two witness folds), host_ro (random oracle and O(1) algebra).  `evals_kernel_ms` times the
evals pass alone over EVALS_REPS back-to-back launches; `evals_product_bound_ms` is the least time its 10 field
products per row could take at the multiplier's measured peak (MUL_RATE_GPS, DESIGN.md §4).
--check verifies the last Neutron fold: the oracle's restated NIFS::verify reproduces U, the device is_sat holds,
its sum equals the C oracle's, a tampered T is rejected, and the last Nova fold satisfies is_sat_relaxed.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MUL_RATE_GPS = 58.2  # G field products/s of the multiplier on the H100 (DESIGN.md §4)
EVALS_REPS = 20      # back-to-back launches of the evals pass for its kernel time


def gpu_info():
    """name and power limit of GPU 0 (read-only query)"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit": power}
    except Exception:
        return {"gpu": "unknown", "power_limit": "unknown"}


def _identity_shape(nb, fid, n):
    from nova_b200 import fields, r1cs, spartan as sp
    one = fields.to_mont_bytes(fid, 1) * n
    M = sp.SparseMatrix(fid, one, range(n), range(n + 1), n + 2)
    return r1cs.R1CSShape(nb.Curve(0), M, M, M, n, n, 1)


def run(log2n=20, reps=3, check_proof=False):
    import ctypes

    import numpy as np

    import nova_b200 as nb
    from nova_b200 import fields, neutron as ne, r1cs, spartan as sp
    from nova_b200.native import check, lib
    from nova_b200.poseidon import PoseidonRO
    from nova_b200.ppsnark import dev_from_u64
    from nova_b200.provider import _jac_to_affine
    from oracle import coracle as co
    from oracle.pyref import SplitMix64
    L = lib()
    check(L.b200_init(0))
    n = 1 << log2n
    curve = nb.Curve(0)
    fid = curve.scalar_field
    p = fields.MODULUS[fid]
    t0 = time.time()
    rng = SplitMix64(2024)
    bases = co.gen_bases(0, n + 1)
    ck = nb.CommitmentKey(curve, bases[:64 * n], bases[64 * n:])
    S = _identity_shape(nb, fid, n)
    st = ne.Structure(S)
    w = np.frombuffer(rng.bytes(n), dtype=np.uint8) & 1
    W = r1cs.R1CSWitness(dev_from_u64(fid, w), rng.field(p))
    x = [0]
    f_U, f_W = ne.FoldedInstance.default(st), ne.FoldedWitness.default(st)
    assert ne.is_sat(ck, st, f_U, f_W)
    ce = nb.CommitmentEngine(curve)
    r_W_bytes = fields.to_mont_bytes(fid, W.r_W)
    w_u8 = np.ascontiguousarray(w)

    def commit_small():
        """CE::commit_small(ck, w, r_W) on the u8 witness: msm_small over ck[..n] (b200_msm_small) plus r_W h"""
        jac = ctypes.create_string_buffer(96)
        check(L.b200_msm_small(ck.handle, 0, w_u8.ctypes.data_as(ctypes.c_void_p), 1, n, 0, jac))
        return ce._plus_blind(ck, _jac_to_affine(curve, jac.raw), r_W_bytes)
    # Nova: a sampled random relaxed pair (r1cs/mod.rs:786-831)
    Z = co.gen_scalars(fid, 31, n + 2)
    r_U, r_Wn = r1cs.sample_random_instance_witness(ck, S, Z, rng.field(p), rng.field(p))
    check(L.b200_sync())
    setup_s = time.time() - t0

    def challenge(comm_T):
        ro = PoseidonRO(curve.base_field)
        for c in ((0, 0) if comm_T is None else comm_T):
            ro.absorb(c)
        return ro.squeeze(128) % p

    neutron_runs, nova_runs, last = [], [], None
    for rep in range(reps + 1):  # rep 0 warms up (allocations, pools, Poseidon constants)
        tm = {}
        t1 = time.perf_counter()
        comm_W = commit_small()
        tm["commit_W"] = time.perf_counter() - t1
        U2 = r1cs.R1CSInstance(comm_W, x)
        r_E = rng.field(p)
        nifs, (U, Wf) = ne.nifs_prove(ck, PoseidonRO(fid), 0, st, f_U, f_W, U2, W, r_E, timings=tm)
        check(L.b200_sync())
        tm["total"] = time.perf_counter() - t1
        t2 = time.perf_counter()
        comm_W_nova = S._commit(ck, W.W, n, W.r_W)
        U2n = r1cs.R1CSInstance(comm_W_nova, x)
        _, (Un, Wn) = r1cs.nifs_prove(ck, S, r_U, r_Wn, U2n, W, rng.field(p), challenge)
        check(L.b200_sync())
        t_nova = time.perf_counter() - t2
        if rep:
            neutron_runs.append(tm)
            nova_runs.append(t_nova)
        last = (nifs, U2, U, Wf, Un, Wn)
    best = min(neutron_runs, key=lambda t: t["total"])
    ms = {k: round(v * 1e3, 3) for k, v in best.items()}
    # the evals pass alone: EVALS_REPS launches on resident vectors (the running pair against the incoming one)
    z = S._z(W.W, 1, x)
    abc = S.multiply_vec_dev(z)
    sums = sp.DeviceVec(32 * 5)
    Ef = last[3].E
    check(L.b200_sync())
    t4 = time.perf_counter()
    for _ in range(EVALS_REPS):
        check(L.b200_neutron_evals_dev(fid, Ef.ptr, *(v.ptr for v in abc), Ef.ptr, *(v.ptr for v in abc), st.left,
                                       st.right, sums.ptr, None))
    check(L.b200_sync())
    evals_kernel_ms = (time.perf_counter() - t4) * 1e3 / EVALS_REPS
    bound_ms = 10 * n / (MUL_RATE_GPS * 1e9) * 1e3  # 10 products per row (prove_helper's five comb_func)
    out = {"workload": f"NeutronNova vs Nova NIFS::prove, BN254, x*x = x, 2^{log2n} constraints, random bits",
           "log2n": log2n, "left": st.left, "right": st.right, "setup_s": round(setup_s, 2), "reps": reps,
           **gpu_info(), "neutron_ms": ms,
           "nova_ms": round(min(nova_runs) * 1e3, 3),
           "neutron_totals_ms": [round(t["total"] * 1e3, 3) for t in neutron_runs],
           "nova_totals_ms": [round(t * 1e3, 3) for t in nova_runs],
           "evals_kernel_ms": round(evals_kernel_ms, 4), "evals_product_bound_ms": round(bound_ms, 4),
           "evals_share_of_product_bound": round(bound_ms / evals_kernel_ms, 3),
           "comm_E_points": st.left + st.right,
           "digest": [U.T % (1 << 64), last[0].poly[5] % (1 << 64), U.comm_E[0] % (1 << 64)]}
    if check_proof:
        from oracle import neutron_ref as nr
        from oracle.poseidon_ref import PoseidonRO as OracleRO
        from oracle.pyref import FIELD_MODULUS
        nifs, U2, U, Wf, Un, Wn = last
        t3 = time.time()
        U1o = nr.FoldedInstance(None, None, 0, 0, [0])
        Uo = nr.nifs_verify(0, p, nr.NIFS(nifs.comm_E, list(nifs.poly)), OracleRO(FIELD_MODULUS[fid]), 0, U1o,
                            nr.R1CSInstance(U2.comm_W, U2.X))
        same_U = Uo is not None and (Uo.comm_W, Uo.comm_E, Uo.T, Uo.u, Uo.X) == (U.comm_W, U.comm_E, U.T, U.u, U.X)
        sat = ne.is_sat(ck, st, U, Wf)
        # the is_sat sum by the C oracle: Az = Bz = Cz = W for this shape (z = (W, u, X), identity on W)
        Wb, Eb = Wf.W.to_bytes(32 * n), Wf.E.to_bytes(32 * (st.left + st.right))
        E = fields.unpack(fid, Eb)
        sum_c = nr.evals_raw(fid, st.left, st.right, E, Wb, Wb, Wb, E, Wb, Wb, Wb)[0]
        tampered = ne.is_sat(ck, st, ne.FoldedInstance(U.comm_W, U.comm_E, (U.T + 1) % p, U.u, U.X), Wf)
        nova_sat = S.is_sat_relaxed(ck, Un, Wn)
        out["check_detail"] = {"verify_reproduces_U": bool(same_U), "is_sat": bool(sat),
                               "sum_matches_c_oracle": sum_c == U.T, "tampered_T_rejected": not tampered,
                               "nova_is_sat_relaxed": bool(nova_sat)}
        out["check"] = all(out["check_detail"].values())
        out["check_s"] = round(time.time() - t3, 1)
    ck.release()
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check", action="store_true")
    a = ap.parse_args()
    if not 8 <= a.log2n <= 22:
        ap.error("--log2n runs from 8 (a CPU-sized run) to 22")
    res = run(a.log2n, a.reps, a.check)
    print(json.dumps(res))
    if a.check and not res["check"]:
        sys.exit(1)
