"""Inner-product argument prover (src/provider/ipa_pc.rs:174-285) on the device.

The reference folds the commitment key every round (`ck.fold`, pedersen.rs:484-497) and commits
over the folded key.  Here the ORIGINAL key stays registered (window tables resident) and the fold
weights move into the scalars (include/nova_b200.h, "inner-product argument"): per round two
device inner products, one kernel building the two scalar vectors, two `b200_commit_dev` calls whose
blinding slot carries the `c * r0 * ck_c` term, and three element-wise kernels (fold a, fold b,
update weights).  L_vec, R_vec and a_hat are group / field elements, hence identical to the
reference's.  The host keeps the transcript and the O(1) algebra.

The verifier (ipa_pc.rs:286-396) keeps the transcript, the O(log n) scalars and the (2L+1)-point left-hand side on
the host; its n-entry tensor vector s (b200_ipa_s_dev, scaled by a_hat) and the n-point commitment to it
(b200_commit_dev, with the ck_c terms in the blinding slot) run on the device.
"""
from __future__ import annotations

import ctypes
import time

from . import fields
from .native import check, lib
from .provider import CommitmentKey, Curve, DlogGroup, _jac_to_affine
from .spartan import DeviceVec


def commitment_transcript_bytes(P) -> bytes:
    """pedersen.rs:107-117."""
    if P is None:
        return bytes(64) + b"\x01"
    return int(P[0]).to_bytes(32, "little") + int(P[1]).to_bytes(32, "little") + b"\x00"


class InnerProductArgument:
    @staticmethod
    def prove(curve, ck: CommitmentKey, comm_a, b_vec: bytes, c_claim: int, a_vec: bytes, transcript,
              timings: dict | None = None):
        """`ck` must be registered over the n bases with `h = ck_c` (the single generator the reference
        keeps in `ck_c`).  b_vec / a_vec are Montgomery field-element vectors of n = 2^l entries.
        `timings`, if given, receives wall-clock seconds summed over the rounds for "ipa_inner_products",
        "ipa_commit" (the scalar vectors and the two n-point commitments) and "ipa_fold"."""
        mark = _marker(timings)
        curve = Curve(curve)
        fid = curve.scalar_field
        q = fields.MODULUS[fid]
        size = lambda v: v.nbytes if isinstance(v, DeviceVec) else len(v)
        n = size(b_vec) // 32
        if size(a_vec) != size(b_vec):
            raise ValueError("InvalidInputLength")  # ipa_pc.rs:187-189
        assert n and n & (n - 1) == 0 and n <= len(ck) and ck.has_h
        L = lib()
        transcript.absorb_bytes(b"NoDS", b"IPA")
        transcript.absorb_bytes(b"U", commitment_transcript_bytes(comm_a) + int(c_claim % q).to_bytes(32, "little"))
        r0 = transcript.squeeze(b"r")
        def working(v):  # the folds overwrite both vectors: resident inputs are copied device-to-device
            if not isinstance(v, DeviceVec):
                return DeviceVec.from_bytes(v)
            c = DeviceVec(32 * n)
            check(L.b200_memcpy_d2d(c.ptr, v.ptr, 32 * n, None))
            return c
        a, b = working(a_vec), working(b_vec)
        w, sL, sR = DeviceVec(32 * n), DeviceVec(32 * n), DeviceVec(32 * n)
        a2, b2 = DeviceVec(16 * n), DeviceVec(16 * n)
        out = DeviceVec(96 * 2)
        ip = DeviceVec(64)
        check(L.b200_ipa_weights_dev(fid, w.ptr, n, 0, None, None, None))  # w := 1
        L_vec, R_vec = [], []
        nk = n
        off = lambda v, elems: ctypes.c_void_p(v.ptr.value + 32 * elems)
        while nk > 1:
            h = nk // 2
            # c_L = <a_L, b_R>, c_R = <a_R, b_L>
            check(L.b200_sc_eval_dev(fid, 11, a.ptr, off(b, h), None, h, None, None, 0, ip.ptr, None))
            check(L.b200_sc_eval_dev(fid, 11, off(a, h), b.ptr, None, h, None, None, 0, off(ip, 1), None))
            c_L, c_R = fields.unpack(fid, ip.to_bytes(64))
            mark("ipa_inner_products")
            check(L.b200_ipa_scalars_dev(fid, a.ptr, w.ptr, n, nk, sL.ptr, sR.ptr, None))
            blind = DeviceVec.from_bytes(fields.pack(fid, [c_L * r0 % q, c_R * r0 % q]))
            check(L.b200_commit_dev(ck.handle, sL.ptr, n, blind.ptr, out.ptr, None))
            check(L.b200_commit_dev(ck.handle, sR.ptr, n, off(blind, 1), ctypes.c_void_p(out.ptr.value + 96), None))
            raw = out.to_bytes(192)
            Lk, Rk = _jac_to_affine(curve, raw[:96]), _jac_to_affine(curve, raw[96:])
            mark("ipa_commit")
            transcript.absorb_bytes(b"L", commitment_transcript_bytes(Lk))
            transcript.absorb_bytes(b"R", commitment_transcript_bytes(Rk))
            r = transcript.squeeze(b"r")
            ri = pow(r, -1, q)
            rr = DeviceVec.from_bytes(fields.pack(fid, [r, ri]))
            check(L.b200_fold_halves_dev(fid, a.ptr, nk, rr.ptr, off(rr, 1), a2.ptr, None))  # a_L r + r^-1 a_R
            check(L.b200_fold_halves_dev(fid, b.ptr, nk, off(rr, 1), rr.ptr, b2.ptr, None))  # b_L r^-1 + r b_R
            check(L.b200_ipa_weights_dev(fid, w.ptr, n, nk, rr.ptr, off(rr, 1), None))
            check(L.b200_sync())
            a, a2 = a2, a
            b, b2 = b2, b
            L_vec.append(Lk)
            R_vec.append(Rk)
            nk = h
            mark("ipa_fold")
        a_hat = fields.unpack(fid, a.to_bytes(32))[0]
        return L_vec, R_vec, a_hat


    @staticmethod
    def verify(curve, ck: CommitmentKey, comm_a, point: list, c: int, L_vec, R_vec, a_hat: int, transcript,
               timings: dict | None = None):
        """InnerProductArgument::verify (ipa_pc.rs:286-396) for the instance (comm_a, b_vec = eq(point), c) that
        EvaluationEngine::verify builds (ipa_pc.rs:80-100); n = 2^len(point).  Returns None; raises
        ValueError("InvalidInputLength") (the reference's length checks, in its order), ValueError("InternalError")
        (a zero round challenge) or ValueError("InvalidPCS") (the final equation fails).  `ck` must be registered
        with h = ck_c and hold at least n bases (checked before any device work).

        The reference's check  sum r_k^2 L_k + sum r_k^-2 R_k + P  ==  a_hat ck_hat + a_hat b_hat (r0 ck_c),  with
        P = comm_a + c (r0 ck_c) and ck_hat = <s, ck>, is tested here with the c (r0 ck_c) term moved to the right:
            sum r_k^2 L_k + sum r_k^-2 R_k + comm_a  ==  commit(ck, a_hat s, blind = r0 (a_hat b_hat - c)),
        the same group equation; the right side is one n-point b200_commit_dev and ck_c is never needed on the host.
        b_hat = <eq(point), s> = prod r_k^-1 prod ((1 - x_k) + x_k r_k^2) in O(log n).  `timings` (optional):
        "ipa_scalars", "ipa_s", "ipa_commit", "ipa_host_msm" in seconds."""
        mark = _marker(timings)
        curve = Curve(curve)
        fid = curve.scalar_field
        q = fields.MODULUS[fid]
        n = 1 << len(point)
        check_key(ck, n)  # ck.split_at(n) (ipa_pc.rs:294) panics on a shorter key
        transcript.absorb_bytes(b"NoDS", b"IPA")
        if n != 1 << len(L_vec) or len(L_vec) != len(R_vec) or len(L_vec) >= 32:
            raise ValueError("InvalidInputLength")  # ipa_pc.rs:297-303
        transcript.absorb_bytes(b"U", commitment_transcript_bytes(comm_a) + int(c % q).to_bytes(32, "little"))
        r0 = transcript.squeeze(b"r")
        rs = []
        for Lk, Rk in zip(L_vec, R_vec):
            transcript.absorb_bytes(b"L", commitment_transcript_bytes(Lk))
            transcript.absorb_bytes(b"R", commitment_transcript_bytes(Rk))
            rs.append(transcript.squeeze(b"r"))
        if any(r % q == 0 for r in rs):
            raise ValueError("InternalError")  # batch_invert (spartan/mod.rs:130-132)
        r_inv = [pow(r, -1, q) for r in rs]
        b_hat = 1
        for x, r, ri in zip(point, rs, r_inv):
            b_hat = b_hat * ri % q * ((1 - x) + x * r % q * r) % q
        a_hat %= q
        mark("ipa_scalars")
        L = lib()
        s = DeviceVec(32 * n)
        rd, rid = DeviceVec.from_bytes(fields.pack(fid, rs)), DeviceVec.from_bytes(fields.pack(fid, r_inv))
        scale = DeviceVec.from_bytes(fields.to_mont_bytes(fid, a_hat))
        check(L.b200_ipa_s_dev(fid, rd.ptr, rid.ptr, len(rs), scale.ptr, s.ptr, None))
        mark("ipa_s")
        blind = DeviceVec.from_bytes(fields.to_mont_bytes(fid, r0 * (a_hat * b_hat - c) % q))
        out = DeviceVec(96)
        check(L.b200_commit_dev(ck.handle, s.ptr, n, blind.ptr, out.ptr, None))
        rhs = _jac_to_affine(curve, out.to_bytes(96))
        mark("ipa_commit")
        from .snark import _affine_bytes
        scalars = [r * r % q for r in rs] + [ri * ri % q for ri in r_inv] + [1]
        lhs = DlogGroup(curve).vartime_multiscalar_mul(
            fields.pack(fid, scalars), b"".join(_affine_bytes(curve, P) for P in list(L_vec) + list(R_vec) + [comm_a]))
        mark("ipa_host_msm")
        if lhs != rhs:
            raise ValueError("InvalidPCS")  # ipa_pc.rs:378-388


def check_key(ck: CommitmentKey | None, n: int):
    """The key an IPA opening of n = 2^l entries needs: registered with h = ck_c and at least n bases."""
    if ck is None or not ck.has_h:
        raise ValueError("the IPA needs a key registered with h = ck_c")
    if len(ck) < n:
        raise ValueError(f"the IPA over {n} entries needs a key of at least {n} bases, not {len(ck)}")


def verify_at_point(curve, ck: CommitmentKey, comm, point: list, eval_: int, eval_arg, transcript,
                    timings: dict | None = None):
    """EvaluationEngine::verify (ipa_pc.rs:80-100): eval_arg = (L_vec, R_vec, a_hat) opens `comm` at `point` to
    `eval_`.  Returns None or raises ValueError as InnerProductArgument.verify does."""
    L_vec, R_vec, a_hat = eval_arg
    InnerProductArgument.verify(curve, ck, comm, point, eval_, L_vec, R_vec, a_hat, transcript, timings)


def prove_at_point(curve, ck: CommitmentKey, comm, point: list, eval_: int, poly, transcript,
                   timings: dict | None = None):
    """EvaluationEngine::prove (ipa_pc.rs:64-77): the inner-product argument between `poly` (2^len(point)
    Montgomery elements, bytes or DeviceVec) and b_vec = EqPolynomial::new(point).evals(), built on the device.
    `timings`: "ipa_b_vec" and the phases of InnerProductArgument.prove."""
    mark = _marker(timings)
    fid = Curve(curve).scalar_field
    b_vec = DeviceVec(32 << len(point))
    x_dev = DeviceVec.from_bytes(fields.pack(fid, point))
    check(lib().b200_eq_table_dev(fid, x_dev.ptr, len(point), b_vec.ptr, None))
    mark("ipa_b_vec")
    return InnerProductArgument.prove(curve, ck, comm, b_vec, eval_, poly, transcript, timings)


def _marker(timings: dict | None):
    """mark(name) adds the seconds since the previous mark to timings[name], the device synchronised first;
    a no-op without `timings`"""
    last = [time.perf_counter()]

    def mark(name):
        if timings is not None:
            check(lib().b200_sync())
            now = time.perf_counter()
            timings[name] = timings.get(name, 0.0) + now - last[0]
            last[0] = now
    return mark
