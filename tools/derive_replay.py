#!/usr/bin/env python3
"""ck_derive_by_address (traits/commitment.rs:177-194) on one GPU, against the path a Rust shim would otherwise take.

    python tools/derive_replay.py [--sizes 20:16,20:20,22:16,22:22] [--reps 3] [--check]

For each m:table_size pair (log2), over a synthetic key of m bases (k0 + i) G on BN254 and uniform random addresses:
  device     b200_ck_derive_by_address, best of --reps after one warm-up: the wall time of the call (synchronised
             host clock; it returns once the key is built), and from torch.profiler the device time of the derivation's
             kernels (checks, address stage, radix passes, bucket accumulation and fix-up, affine output) and of the
             table expansion of the derived key (k_expand_key), separately
  shim       once: b200_ck_export_bases of the whole key, the reference loop restated serially in C
             (tests/derive_oracle.c: one XYZZ mixed addition per address, then the normalisation), b200_ck_register
--check compares the derived bases (b200_ck_export_bases) with the C restatement's, byte for byte.  The GPU name and
power limit are read in the same run and printed with every line.
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

from mercury_replay import gpu_info


def _device_split(fn):
    """(expansion ms, other kernels ms) of the kernels fn launches, from torch.profiler's CUDA activity"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    expand = other = 0.0
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        if "k_expand_key" in ev.name:
            expand += us
        elif "Memset" not in ev.name and "Memcpy" not in ev.name:
            other += us
    return expand / 1e3, other / 1e3


def run_one(log2m, log2t, reps, check, info):
    import numpy as np
    import torch  # noqa: F401  (CUDA context for the profiler)

    import derive_ref
    import nova_b200 as nb
    from nova_b200.native import c_u64, check as ok, lib
    L = lib()
    m, table_size = 1 << log2m, 1 << log2t
    ck = nb.CommitmentKey.setup_synthetic(nb.Curve(0), m)
    addrs = np.random.default_rng(log2m * 100 + log2t).integers(0, table_size, m).astype(np.uint64)
    arr = addrs.ctypes.data_as(ctypes.POINTER(c_u64))
    ce = nb.CommitmentEngine(0)

    def derive():
        out, bad = ctypes.c_uint64(0), ctypes.c_size_t(0)
        ok(L.b200_ck_derive_by_address(ck.handle, arr, m, table_size, 0, ctypes.byref(out), ctypes.byref(bad)))
        return nb.CommitmentKey.from_handle(nb.Curve(0), out.value, None, None, table_size)

    derive().release()  # warm-up: pool growth, first launches
    walls = []
    for _ in range(reps):
        t0 = time.perf_counter()
        d = derive()
        walls.append((time.perf_counter() - t0) * 1e3)
        d.release()
    expand_ms, derive_kernels_ms = _device_split(lambda: derive().release())

    t0 = time.perf_counter()
    bases = ck.export_bases()
    t_export = time.perf_counter() - t0
    t0 = time.perf_counter()
    ref = derive_ref.derive(0, bases, addrs.tolist(), table_size)
    t_loop = time.perf_counter() - t0
    t0 = time.perf_counter()
    shim = nb.CommitmentKey(nb.Curve(0), ref)
    t_register = time.perf_counter() - t0
    shim.release()
    res = {"m": f"2^{log2m}", "table_size": f"2^{log2t}", **info, "reps": reps,
           "device_call_ms": round(min(walls), 2), "device_derive_kernels_ms": round(derive_kernels_ms, 2),
           "device_expand_ms": round(expand_ms, 2),
           "shim_export_ms": round(t_export * 1e3, 1), "shim_c_loop_ms": round(t_loop * 1e3, 1),
           "shim_register_ms": round(t_register * 1e3, 1),
           "shim_total_ms": round((t_export + t_loop + t_register) * 1e3, 1)}
    if check:
        d = ce.ck_derive_by_address(ck, addrs.tolist(), table_size)
        res["check"] = "ok" if d.export_bases() == ref else "MISMATCH"
        d.release()
    ck.release()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20:16,20:20,22:16,22:22", help="log2(m):log2(table_size),...")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check", action="store_true")
    a = ap.parse_args()
    from nova_b200.native import check, lib
    check(lib().b200_init(0))
    info = gpu_info()
    failed = False
    for pair in a.sizes.split(","):
        lm, lt = (int(x) for x in pair.split(":"))
        res = run_one(lm, lt, a.reps, a.check, info)
        failed |= res.get("check") == "MISMATCH"
        print(json.dumps(res), flush=True)
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
