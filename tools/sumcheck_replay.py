#!/usr/bin/env python3
"""Times the two sum-check round loops of spartan::snark (sumcheck.rs:199-242, 446-507) on
device-resident polynomials, two ways:

  host   : per round  reduce kernel -> D2H -> host algebra + Keccak (Python here, Rust in production)
           -> H2D challenge -> bind kernels                      (SumcheckProof.prove_*)
  device : every round's reduce / round kernel / binds enqueued back to back, one D2H at the end
           (b200_sumcheck_quad_prod / b200_sumcheck_cubic3, csrc/capi_sumcheck.inc)

and a streamed witness commit against the one-shot commit.  Torch-free (ctypes only) so it starts
in seconds on a fresh box.  Prints one JSON line per measurement.

  python tools/sumcheck_replay.py [--log-n 20] [--reps 3]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import nova_b200 as nb  # noqa: E402
from nova_b200 import fields, spartan  # noqa: E402
from nova_b200.native import check, lib  # noqa: E402


class Transcript:
    """Minimal stand-in with the serialisable fields of Keccak256Transcript; the host loop needs real
    challenges, so it hashes with hashlib's SHA3 (NOT the reference's Keccak padding -- timing only)."""

    def __init__(self, p):
        import hashlib
        self._h = hashlib
        self.p, self.round, self.state, self.buf = p, 0, bytes(64), b""

    def absorb_bytes(self, label, b):
        self.buf += label + b

    def squeeze(self, label):
        inp = self.buf + b"NoDS" + self.round.to_bytes(8, "little") + self.state + label
        out = self._h.sha3_256(inp + b"\0").digest() + self._h.sha3_256(inp + b"\1").digest()
        self.round, self.state, self.buf = self.round + 1, out, b""
        return int.from_bytes(out, "little") % self.p


def rand_vec(fid, n, seed):
    import random
    r = random.Random(seed)
    p = fields.MODULUS[fid]
    # cheap pseudo-random residues (values do not matter for timing)
    return b"".join(r.getrandbits(250).to_bytes(32, "little") for _ in range(n)) if n <= 1 << 16 else \
        (b"".join(r.getrandbits(250).to_bytes(32, "little") for _ in range(1 << 16)) * (n >> 16))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    check(lib().b200_init(0))
    fid, l = 0, a.log_n
    p = fields.MODULUS[fid]
    n = 1 << l
    A, B, C = (rand_vec(fid, n, s) for s in (1, 2, 3))
    taus = [(12345 + 7 * i) % p for i in range(l)]

    def timed(name, fn):
        best = None
        for _ in range(a.reps):
            dA, dB, dC = (spartan.DeviceVec.from_bytes(x) for x in (A, B, C))
            check(lib().b200_sync())
            t0 = time.perf_counter()
            fn(dA, dB, dC)
            check(lib().b200_sync())
            dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
            for v in (dA, dB, dC):
                v.free()
        print(json.dumps({"what": name, "log_n": l, "ms": round(best * 1e3, 3), "ms_per_round": round(best * 1e3 / l, 4)}),
              flush=True)

    timed("cubic3_device_transcript",
          lambda dA, dB, dC: spartan.SumcheckProof.prove_cubic_with_three_inputs_device(fid, 5, taus, dA, dB, dC, Transcript(p)))
    timed("quad_prod_device_transcript",
          lambda dA, dB, dC: spartan.SumcheckProof.prove_quad_prod_device(fid, 5, l, dA, dB, Transcript(p)))

    timed("cubic3_host_transcript_python",
          lambda dA, dB, dC: spartan.SumcheckProof.prove_cubic_with_three_inputs(fid, 5, taus, dA, dB, dC, Transcript(p)))

    # streamed witness commit vs one-shot commit (chunks of 2^16 scalars)
    ck = nb.CommitmentKey.setup_synthetic(nb.Curve(0), n)
    eng = nb.CommitmentEngine(0)
    eng.commit(ck, A, None)
    t0 = time.perf_counter()
    for _ in range(a.reps):
        whole = eng.commit(ck, A, None)
    t_whole = (time.perf_counter() - t0) / a.reps
    step = 32 << 16
    t0 = time.perf_counter()
    for _ in range(a.reps):
        ws = nb.WitnessStream(ck, n)
        for off in range(0, len(A), step):
            ws.append(A[off:off + step])
        streamed = ws.finish(None)
        ws.release()
    t_stream = (time.perf_counter() - t0) / a.reps
    print(json.dumps({"what": "commit_one_shot_vs_streamed", "log_n": l, "one_shot_ms": round(t_whole * 1e3, 3),
                      "streamed_ms_incl_begin_release": round(t_stream * 1e3, 3), "equal": whole == streamed}), flush=True)


if __name__ == "__main__":
    main()
