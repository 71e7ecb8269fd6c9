"""Host-side mirror of the reference's provider surface for the hot path.

Names follow the reference so the parity tests read like its own tests:

  DlogGroup.vartime_multiscalar_mul / batch_vartime_multiscalar_mul /
  vartime_multiscalar_mul_small(_with_max_num_bits)        src/provider/traits.rs:77-117
  CommitmentEngine.commit / batch_commit / commit_small / commit_sparse_binary
                                                           src/provider/pedersen.rs:263-427,
                                                           src/provider/hyperkzg.rs:584-783
  cross_term (commit_T's T), fold_witness                   src/r1cs/mod.rs:578-664, 1044-1107
  bind_poly_var_top                                         src/spartan/polys/multilinear.rs:65-84

Vectors cross this layer as raw bytes in the FFI layout (32 B Montgomery field elements,
64 B affine points); group results come back as affine (x, y) integer tuples or None for the
identity -- the single Jacobian->affine normalisation per result is done here with Python
integers (it is O(1) per call, the reference does it in `affine()`, traits.rs:285-289).
Length mismatches raise AssertionError like the reference's `assert_eq!` (msm.rs:226).
"""
from __future__ import annotations

import ctypes
import enum

from . import fields
from .native import B200Error, c_size_t, c_u64, check, lib


class Curve(enum.IntEnum):
    BN254_G1 = 0
    GRUMPKIN = 1
    PALLAS = 2
    VESTA = 3

    @property
    def base_field(self) -> int:
        return (fields.BN254_FQ, fields.BN254_FR, fields.PALLAS_FP, fields.PALLAS_FQ)[int(self)]

    @property
    def scalar_field(self) -> int:
        return (fields.BN254_FR, fields.BN254_FQ, fields.PALLAS_FQ, fields.PALLAS_FP)[int(self)]


# curve generators (halo2curves): G1 (1,2); Grumpkin (1, sqrt(-16)); Pallas/Vesta (-1, 2)
GENERATORS = {
    0: (1, 2),
    1: (1, 0x0000000000000002CF135E7506A45D632D270D45F1181294833FC48D823F272C),
    2: (fields.MODULUS[fields.PALLAS_FP] - 1, 2),
    3: (fields.MODULUS[fields.PALLAS_FQ] - 1, 2),
}


def _cbuf(b):
    if b is None:
        return None
    return (ctypes.c_char * len(b)).from_buffer_copy(b) if len(b) else (ctypes.c_char * 1)()


def _jac_to_affine(curve: Curve, jac: bytes):
    fid = curve.base_field
    p = fields.MODULUS[fid]
    x, y, z = (fields.from_mont_bytes(fid, jac[i:i + 32]) for i in (0, 32, 64))
    if z == 0:
        return None
    zi = pow(z, -1, p)
    return (x * zi * zi % p, y * zi * zi * zi % p)


class CommitmentKey:
    """Device-resident `CommitmentKey{ck, h}` (pedersen.rs:32-38 / hyperkzg.rs:76-84)."""

    def __init__(self, curve: Curve, bases: bytes, h: bytes | None = None, window_bits: int = 0):
        assert len(bases) % 64 == 0 and len(bases) > 0
        self.curve = Curve(curve)
        self.n = len(bases) // 64
        handle = c_u64(0)
        check(lib().b200_ck_register(int(curve), _cbuf(bases), self.n, _cbuf(h) if h else None,
                                     window_bits, ctypes.byref(handle)))
        self.handle = handle.value
        self.has_h = h is not None
        # the host keeps `ck.ck` / `ck.h` as the reference does (pedersen.rs:32-38): commit_sparse gathers
        # bases on the host (pedersen.rs:418-420) and the `+ h * r` terms are commitment-sized host work
        self.bases, self.h = bases, h

    @classmethod
    def from_handle(cls, curve: "Curve", handle: int, bases: bytes | None, h: bytes | None, n: int) -> "CommitmentKey":
        """Wrap a key the library has already registered (e.g. through b200_ck_register_checked)."""
        self = cls.__new__(cls)
        self.curve, self.n, self.handle, self.has_h = Curve(curve), n, handle, h is not None
        self.bases, self.h = bases, h
        return self

    @classmethod
    def setup_synthetic(cls, curve: "Curve", n: int, k0: int = 0x5EED, with_h: bool = False,
                        window_bits: int = 0) -> "CommitmentKey":
        """Test/bench key bases[i] = (k0+i)*G built on the device (cf. hyperkzg.rs:357-376)."""
        self = cls.__new__(cls)
        self.curve = Curve(curve)
        self.n = n
        self.has_h = with_h
        gen = GENERATORS[int(curve)]
        fid = self.curve.base_field
        g = fields.to_mont_bytes(fid, gen[0]) + fields.to_mont_bytes(fid, gen[1])
        handle = c_u64(0)
        check(lib().b200_ck_setup_synthetic(int(curve), _cbuf(g), k0, n, int(with_h), window_bits,
                                            ctypes.byref(handle)))
        self.handle = handle.value
        self.bases, self.h = None, None  # built on the device: no host copy
        return self

    @classmethod
    def setup_tau(cls, curve: "Curve", n: int, tau: int, window_bits: int = 0) -> "CommitmentKey":
        """Test/bench SRS ck[i] = [tau^i] G built on the device (hyperkzg.rs:357-376 `setup_from_rng`)."""
        self = cls.__new__(cls)
        self.curve = Curve(curve)
        self.n, self.has_h = n, False
        gen = GENERATORS[int(curve)]
        fid = self.curve.base_field
        g = fields.to_mont_bytes(fid, gen[0]) + fields.to_mont_bytes(fid, gen[1])
        handle = c_u64(0)
        check(lib().b200_ck_setup_tau(int(curve), _cbuf(g), _cbuf(fields.to_mont_bytes(self.curve.scalar_field, tau)),
                                      n, window_bits, ctypes.byref(handle)))
        self.handle = handle.value
        self.bases, self.h = None, None
        return self

    def export_bases(self, offset: int = 0, n: int | None = None) -> bytes:
        """ck[offset .. offset + n) as affine Montgomery bytes (the layout `CommitmentKey(curve, bases)` takes)."""
        n = self.n - offset if n is None else n
        out = ctypes.create_string_buffer(64 * n)
        check(lib().b200_ck_export_bases(self.handle, offset, n, out))
        return out.raw

    @staticmethod
    def validate(curve: "Curve", bases: bytes):
        """CommitmentKey::new's on-curve loop (hyperkzg.rs:113-119) on the device: returns None if
        every base is on the curve, else the index of the first one that is not
        (-> NovaError::InvalidCommitmentKey in the Rust shim)."""
        bad = c_size_t(0)
        check(lib().b200_ck_validate(int(curve), _cbuf(bases), len(bases) // 64, ctypes.byref(bad)))
        return None if bad.value == ctypes.c_size_t(-1).value else bad.value

    def __len__(self):
        return self.n

    def release(self):
        if self.handle:
            check(lib().b200_ck_release(self.handle))
            self.handle = 0

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class DlogGroup:
    """`DlogGroupExt` for one curve (src/provider/traits.rs:77-117)."""

    def __init__(self, curve: Curve):
        self.curve = Curve(curve)

    def vartime_multiscalar_mul(self, scalars: bytes, bases) -> tuple | None:
        """msm(scalars, bases) (msm.rs:225).  `bases` is a CommitmentKey (uses ck[..n]) or raw
        affine bytes (one-shot key, pedersen.rs:418-420)."""
        n = len(scalars) // 32
        out = ctypes.create_string_buffer(96)
        if isinstance(bases, CommitmentKey):
            assert n <= len(bases), "scalars and bases length mismatch"
            check(lib().b200_msm(bases.handle, 0, _cbuf(scalars), n, out))
        else:
            assert len(bases) == 64 * n, "scalars and bases length mismatch"  # msm.rs:226
            check(lib().b200_msm_adhoc(int(self.curve), _cbuf(bases), _cbuf(scalars), n, out))
        return _jac_to_affine(self.curve, out.raw)

    def batch_vartime_multiscalar_mul(self, scalars: list, ck: CommitmentKey) -> list:
        """traits.rs:82-90: vector k uses bases[..len(scalars[k])]."""
        k = len(scalars)
        bufs = [_cbuf(s) for s in scalars]
        ptrs = (ctypes.c_void_p * max(k, 1))(*[ctypes.cast(b, ctypes.c_void_p) for b in bufs])
        lens = (c_size_t * max(k, 1))(*[len(s) // 32 for s in scalars])
        out = ctypes.create_string_buffer(96 * max(k, 1))
        check(lib().b200_msm_batch(ck.handle, ptrs, lens, k, out))
        return [_jac_to_affine(self.curve, out.raw[96 * j:96 * j + 96]) for j in range(k)]

    def vartime_multiscalar_mul_small(self, scalars, ck: CommitmentKey, elem_bytes: int = 8,
                                      max_num_bits: int = 0, base_offset: int = 0):
        """msm_small / msm_small_with_max_num_bits (msm.rs:469-503) on integer scalars, over
        ck[base_offset .. base_offset + len(scalars))."""
        n = len(scalars)
        assert base_offset + n <= len(ck)
        raw = b"".join(int(s).to_bytes(elem_bytes, "little") for s in scalars)
        out = ctypes.create_string_buffer(96)
        check(lib().b200_msm_small(ck.handle, base_offset, _cbuf(raw), elem_bytes, n, max_num_bits, out))
        return _jac_to_affine(self.curve, out.raw)

    def batch_vartime_multiscalar_mul_small(self, scalars: list, ck: CommitmentKey, elem_bytes: int = 8) -> list:
        """traits.rs:105-116 default: one msm_small per vector over bases[..len]."""
        return [self.vartime_multiscalar_mul_small(v, ck, elem_bytes) for v in scalars]

    def batch_add(self, ck: CommitmentKey, one_indices) -> tuple | None:
        """msm.rs:689-708."""
        m = len(one_indices)
        idx = (c_u64 * max(m, 1))(*one_indices)
        out = ctypes.create_string_buffer(96)
        check(lib().b200_msm_indices(ck.handle, idx, m, out))
        return _jac_to_affine(self.curve, out.raw)


class CommitmentEngine:
    """`CommitmentEngineTrait` for Pedersen / HyperKZG commitments (same MSM + r*h shape:
    pedersen.rs:263-270, hyperkzg.rs:584-591)."""

    def __init__(self, curve: Curve):
        self.curve = Curve(curve)
        self.group = DlogGroup(curve)

    def commit(self, ck: CommitmentKey, v: bytes, r: bytes | None = None):
        n = len(v) // 32
        assert len(ck) >= n  # pedersen.rs:264
        out = ctypes.create_string_buffer(96)
        check(lib().b200_commit(ck.handle, _cbuf(v), n, _cbuf(r) if r else None, out))
        return _jac_to_affine(self.curve, out.raw)

    def batch_commit(self, ck: CommitmentKey, vs: list):
        """traits/commitment.rs:94-104 default / hyperkzg.rs:594-612 with r = 0."""
        return self.group.batch_vartime_multiscalar_mul(vs, ck)

    def commit_small(self, ck: CommitmentKey, v, elem_bytes: int = 8, r: bytes | None = None):
        """pedersen.rs:272-283 / hyperkzg.rs commit_small: msm_small + h * r."""
        return self._plus_blind(ck, self.group.vartime_multiscalar_mul_small(v, ck, elem_bytes), r)

    def batch_commit_small(self, ck: CommitmentKey, vs: list, elem_bytes: int = 8):
        """hyperkzg.rs batch_commit_small with r = 0."""
        return self.group.batch_vartime_multiscalar_mul_small(vs, ck, elem_bytes)

    def _plus_blind(self, ck: CommitmentKey, P, r: bytes | None):
        """P + h * r: the commitment-sized term the reference adds on the host (pedersen.rs:281, 300-302)."""
        fid = self.curve.scalar_field
        if not r or fields.from_mont_bytes(fid, r) == 0:
            return P
        assert ck.h is not None, "key has no blinding generator on the host"
        bf = self.curve.base_field
        Pb = bytes(64) if P is None else fields.to_mont_bytes(bf, P[0]) + fields.to_mont_bytes(bf, P[1])
        return self.group.vartime_multiscalar_mul(fields.to_mont_bytes(fid, 1) + r, Pb + ck.h)

    def commit_sparse_binary(self, ck: CommitmentKey, non_zero_indices, r: bytes | None = None):
        """pedersen.rs:396-409: batch_add over the key + h * r."""
        return self._plus_blind(ck, self.group.batch_add(ck, non_zero_indices), r)

    def commit_small_range(self, ck: CommitmentKey, v, r: bytes | None, lo: int, hi: int, max_num_bits: int,
                           elem_bytes: int = 8):
        """pedersen.rs:285-305: msm_small_with_max_num_bits(v[lo..hi], ck[lo..hi]) + h * r."""
        assert hi <= len(ck) and hi <= len(v)
        P = self.group.vartime_multiscalar_mul_small(v[lo:hi], ck, elem_bytes, max_num_bits, base_offset=lo)
        return self._plus_blind(ck, P, r)

    def ck_derive_by_address(self, ck: CommitmentKey, addresses, table_size: int, window_bits: int = 0) -> CommitmentKey:
        """traits/commitment.rs:177-194 (pedersen.rs:360-382, hyperkzg.rs:731-749): the key of table_size bases with
        derived[j] = sum of ck[i] over the i < len(addresses) with addresses[i] = j, built on the device.  Then
        commit(derived, T) == commit(ck, T[addresses]).  The new key has no host copy of its bases; its h is ck's.
        Errors raise B200Error with .code (B200_E_POINT, B200_E_RANGE, B200_E_INDEX, ...) and .first_bad."""
        m = len(addresses)
        arr = (c_u64 * max(m, 1))(*addresses)
        return self._derived(ck, lambda out, bad: lib().b200_ck_derive_by_address(
            ck.handle, arr, m, table_size, window_bits, out, bad), table_size)

    def ck_derive_by_address_dev(self, ck: CommitmentKey, d_addresses, m: int, table_size: int, window_bits: int = 0,
                                 stream=None) -> CommitmentKey:
        """The same from m u32 addresses in device memory (a device pointer), on `stream` (None: the library's)."""
        return self._derived(ck, lambda out, bad: lib().b200_ck_derive_by_address_dev(
            ck.handle, d_addresses, m, table_size, window_bits, out, bad, stream), table_size)

    def _derived(self, ck: CommitmentKey, call, table_size: int) -> CommitmentKey:
        out, bad = c_u64(0), c_size_t(-1)
        rc = call(ctypes.byref(out), ctypes.byref(bad))
        if rc:
            err = B200Error(rc, lib().b200_last_error().decode())
            err.first_bad = None if bad.value == ctypes.c_size_t(-1).value else bad.value
            raise err
        key = CommitmentKey.from_handle(self.curve, out.value, None, ck.h, table_size)
        key.has_h = ck.has_h
        return key

    def commit_sparse(self, ck: CommitmentKey, indices, scalars: bytes, r: bytes | None = None):
        """pedersen.rs:411-427: gather ck[indices] on the host, one MSM over the gathered bases (+ h * r as
        one more pair)."""
        assert len(indices) * 32 == len(scalars)  # pedersen.rs:417
        assert ck.bases is not None, "key has no host copy of its bases"
        bases = b"".join(ck.bases[64 * i:64 * i + 64] for i in indices)
        fid = self.curve.scalar_field
        if r and fields.from_mont_bytes(fid, r):
            assert ck.h is not None
            scalars, bases = scalars + r, bases + ck.h
        return self.group.vartime_multiscalar_mul(scalars, bases)


class WitnessStream:
    """Streamed witness hand-off (SURVEY.md §8f-2): `append` every finished prefix of
    `aux_assignment` while synthesis is still running (witness_cs.rs:93-103 only appends), then
    `finish(r_W)` returns commit(ck, W, r_W) exactly as frontend/r1cs.rs:40-50 would.  The chunk
    copies and the MSM's digit/histogram stage overlap with the host's work."""

    def __init__(self, ck: CommitmentKey, num_vars: int):
        self.ck, self.n = ck, num_vars
        h = c_u64(0)
        check(lib().b200_witness_begin(ck.handle, num_vars, ctypes.byref(h)))
        self.handle = h.value
        self._keep = []  # chunk buffers must outlive the asynchronous copies
        self.d_witness = None

    def append(self, scalars: bytes):
        assert len(scalars) % 32 == 0
        buf = _cbuf(scalars)
        self._keep.append(buf)
        check(lib().b200_witness_append(self.handle, buf, len(scalars) // 32))

    def finish(self, r: bytes | None = None):
        out = ctypes.create_string_buffer(96)
        dw = ctypes.c_void_p()
        check(lib().b200_witness_finish(self.handle, _cbuf(r) if r else None, out, ctypes.byref(dw)))
        self._keep.clear()
        self.d_witness = dw
        return _jac_to_affine(self.ck.curve, out.raw)

    def reset(self):
        """Re-arm for the next step's witness (same num_vars); keeps the device workspace."""
        check(lib().b200_witness_reset(self.handle))
        self._keep.clear()
        self.d_witness = None

    def release(self):
        if self.handle:
            check(lib().b200_witness_release(self.handle))
            self.handle = 0

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


# ---- R1CS witness field arithmetic ------------------------------------------------------------
def cross_term(fid: int, az: bytes, bz: bytes, cz: bytes, e1: bytes, u: bytes,
               e2: bytes | None = None) -> bytes:
    """T of commit_T / commit_T_relaxed (r1cs/mod.rs:614-620, 650-657)."""
    n = len(az) // 32
    assert len(bz) == len(az) == len(cz) == len(e1) and (e2 is None or len(e2) == len(az))
    out = ctypes.create_string_buffer(max(32 * n, 1))
    check(lib().b200_cross_term(fid, _cbuf(az), _cbuf(bz), _cbuf(cz), _cbuf(e1),
                                _cbuf(e2) if e2 is not None else None, _cbuf(u), n, out))
    return out.raw[:32 * n]


def fold_witness(fid: int, a: bytes, b: bytes, r: bytes) -> bytes:
    """a + r*b  (RelaxedR1CSWitness::fold, r1cs/mod.rs:1058-1069)."""
    n = len(a) // 32
    if len(a) != len(b):
        raise ValueError("InvalidWitnessLength")  # r1cs/mod.rs:1054-1056
    out = ctypes.create_string_buffer(max(32 * n, 1))
    check(lib().b200_axpy(fid, _cbuf(a), _cbuf(b), _cbuf(r), n, out))
    return out.raw[:32 * n]


def vec_add(fid: int, a: bytes, b: bytes) -> bytes:
    n = len(a) // 32
    assert len(a) == len(b)
    out = ctypes.create_string_buffer(max(32 * n, 1))
    check(lib().b200_vec_add(fid, _cbuf(a), _cbuf(b), n, out))
    return out.raw[:32 * n]


def bind_poly_var_top(fid: int, z: bytes, r: bytes) -> bytes:
    """multilinear.rs:65-84: returns the bound polynomial of half the length."""
    n = len(z) // 32
    buf = _cbuf(z)
    check(lib().b200_bind_top(fid, buf, n, _cbuf(r)))
    return bytes(buf[:32 * (n // 2)])


class MultiGpuCommitmentKey:
    """A commitment key sharded block-cyclically over the GPUs of ONE process (b200_mgpu_*): `commit` is the single
    call a `CommitmentEngine::commit` / `vartime_multiscalar_mul` makes, the library fans it out over the devices
    and exchanges the partial sums over NVLink inside the reduction kernels (include/nova_b200.h)."""

    def __init__(self, curve: "Curve", bases: bytes, h: bytes | None = None, devices=None, ndev: int | None = None,
                 window_bits: int = 0):
        L = lib()
        devs = list(devices) if devices is not None else list(range(ndev or 1))
        arr = (ctypes.c_int * len(devs))(*devs)
        check(L.b200_mgpu_init(len(devs), arr))
        self.curve, self.n, self.has_h = Curve(curve), len(bases) // 64, h is not None
        handle = c_u64(0)
        check(L.b200_mgpu_ck_register(int(curve), _cbuf(bases), self.n, _cbuf(h) if h else None, window_bits,
                                      ctypes.byref(handle)))
        self.handle = handle.value

    def commit(self, v: bytes, r: bytes | None = None):
        """-> affine point (x, y) as integers, or None for the identity"""
        out = ctypes.create_string_buffer(96)
        check(lib().b200_mgpu_commit(self.handle, _cbuf(v), len(v) // 32, _cbuf(r) if r else None, out))
        return _jac_to_affine(self.curve, out.raw)

    def release(self):
        if self.handle:
            check(lib().b200_mgpu_ck_release(self.handle))
            self.handle = 0

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass
