"""Host-side mirror of the R1CS / Spartan / HyperKZG prover pieces on the hot path.

Same names and argument meaning as the reference:

  SparseMatrix, R1CSShape.multiply_vec / multiply_vec_pair     src/r1cs/sparse.rs, src/r1cs/mod.rs:407-471
  EqPolynomial.evals_from_points                               src/spartan/polys/eq.rs:54-73
  MultilinearPolynomial.evaluate_with / bind_poly_var_top      src/spartan/polys/multilinear.rs:65-127
  batch_invert                                                 src/spartan/mod.rs:54-145
  UniPoly                                                      src/spartan/polys/univariate.rs:89-205
  EqSumCheckInstance, SumcheckProof.prove_quad_prod /
  prove_cubic_with_three_inputs                                src/spartan/sumcheck.rs:199-242, 446-507, 593-1251
  hyperkzg_prove_core (fold, batch commit, 3-point evals, batch polynomial, quotients)
                                                               src/provider/hyperkzg.rs:926-1116

The O(N) work runs on the device through the C ABI; this layer keeps exactly what the Rust host
would keep: O(1) field algebra per round (Python integers), the transcript interface and control
flow.  Polynomials stay RESIDENT on the device across sum-check rounds (`DeviceVec`).
"""
from __future__ import annotations

import ctypes

from . import fields
from .native import B200Error, c_size_t, c_u64, check, lib
from .provider import CommitmentKey, Curve, DlogGroup, _cbuf, _jac_to_affine

(SC_QUAD_PROD, SC_LINEAR, SC_QUADRATIC, SC_CUBIC, SC_EQ_CUBIC3, SC_EQ_CUBIC2, SC_EQ_QUAD1, SC_EQ_CUBIC3_M1,
 SC_EQ_CUBIC2_M1, SC_EQ_QUAD1_M1, SC_DOT_EQ) = range(11)
SC_NOUT = {0: 2, 1: 2, 2: 2, 3: 3, 4: 2, 5: 2, 6: 1, 7: 1, 8: 1, 9: 1, 10: 1}


class DeviceVec:
    """A vector of field elements resident in HBM (b200_dev_alloc)."""

    def __init__(self, nbytes: int):
        self.nbytes = nbytes
        p = ctypes.c_void_p()
        check(lib().b200_dev_alloc(max(nbytes, 1), ctypes.byref(p)))
        self.ptr = p

    @classmethod
    def from_bytes(cls, b: bytes) -> "DeviceVec":
        v = cls(len(b))
        if b:
            check(lib().b200_memcpy_h2d(v.ptr, _cbuf(b), len(b)))
        return v

    def to_bytes(self, nbytes: int | None = None) -> bytes:
        n = self.nbytes if nbytes is None else nbytes
        out = ctypes.create_string_buffer(max(n, 1))
        if n:
            check(lib().b200_memcpy_d2h(out, self.ptr, n))
        return out.raw[:n]

    def free(self):
        if self.ptr:
            lib().b200_dev_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


# ---------------------------------------------------------------------------------------------
# sparse matrices / R1CS shape
# ---------------------------------------------------------------------------------------------
class SparseMatrix:
    """CSR `SparseMatrix{data, indices, indptr, cols}` (sparse.rs:235-247), device resident."""

    def __init__(self, fid: int, data: bytes, indices, indptr, cols: int):
        self.fid, self.rows, self.cols, self.nnz = fid, len(indptr) - 1, cols, int(indptr[-1])
        ia = (c_u64 * max(len(indices), 1))(*indices)
        ip = (c_u64 * len(indptr))(*indptr)
        h = c_u64(0)
        check(lib().b200_spmv_register(fid, _cbuf(data), ia, ip, self.rows, cols, ctypes.byref(h)))
        self.handle = h.value

    def multiply_vec(self, z: bytes) -> bytes:
        return R1CSShape._multi([self], z, None)[0][0]

    def multiply_transpose(self, rx: bytes, out_len: int) -> bytes:
        """M^T rx padded to out_len: one matrix of compute_eval_table_sparse (spartan/mod.rs:497-534)."""
        assert len(rx) == 32 * self.rows  # spartan/mod.rs:501
        out = ctypes.create_string_buffer(max(32 * out_len, 1))
        check(lib().b200_spmv_t(self.handle, _cbuf(rx), out_len, out))
        return out.raw[:32 * out_len]

    def release(self):
        if self.handle:
            lib().b200_spmv_release(self.handle)
            self.handle = 0

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class R1CSShape:
    def __init__(self, A: SparseMatrix, B: SparseMatrix, C: SparseMatrix):
        self.A, self.B, self.C = A, B, C

    @staticmethod
    def _multi(mats, z1: bytes, z2: bytes | None):
        k = len(mats)
        zlen = len(z1) // 32
        hs = (c_u64 * k)(*[m.handle for m in mats])
        o1 = [ctypes.create_string_buffer(max(32 * m.rows, 1)) for m in mats]
        o2 = [ctypes.create_string_buffer(max(32 * m.rows, 1)) for m in mats] if z2 is not None else None
        p1 = (ctypes.c_void_p * k)(*[ctypes.cast(b, ctypes.c_void_p) for b in o1])
        p2 = (ctypes.c_void_p * k)(*[ctypes.cast(b, ctypes.c_void_p) for b in o2]) if o2 else None
        rc = lib().b200_spmv_multi(hs, k, _cbuf(z1), _cbuf(z2) if z2 is not None else None, zlen, p1, p2)
        if rc == 1 and b"InvalidWitnessLength" in lib().b200_last_error():
            raise ValueError("InvalidWitnessLength")  # r1cs/mod.rs:411-413
        check(rc)
        r1 = [b.raw[:32 * m.rows] for b, m in zip(o1, mats)]
        r2 = [b.raw[:32 * m.rows] for b, m in zip(o2, mats)] if o2 else None
        return r1, r2

    def multiply_vec(self, z: bytes):
        """(Az, Bz, Cz) — r1cs/mod.rs:407-431."""
        r, _ = self._multi([self.A, self.B, self.C], z, None)
        return tuple(r)

    def multiply_vec_pair(self, z1: bytes, z2: bytes):
        """((Az1,Bz1,Cz1),(Az2,Bz2,Cz2)) — r1cs/mod.rs:435-471."""
        r1, r2 = self._multi([self.A, self.B, self.C], z1, z2)
        return tuple(r1), tuple(r2)

    def _handles(self):
        return (c_u64 * 3)(self.A.handle, self.B.handle, self.C.handle)

    def multi_evaluate(self, r_x: list, r_y: list) -> list:
        """[A(r_x, r_y), B(r_x, r_y), C(r_x, r_y)] = sum over each matrix's entries of eq(r_x)[row] eq(r_y)[col] val
        (multi_evaluate of RelaxedR1CSSNARK::verify, spartan/snark.rs:325-355).  r_x, r_y: the points as integers;
        both eq tables are built on the device (b200_r1cs_eval)."""
        fid = self.A.fid
        out = ctypes.create_string_buffer(96)
        check(lib().b200_r1cs_eval(self._handles(), 3, _cbuf(fields.pack(fid, r_x)), len(r_x),
                                   _cbuf(fields.pack(fid, r_y)), len(r_y), out))
        return fields.unpack(fid, out.raw)

    def multi_evaluate_dev(self, T_x: "DeviceVec", tx_len: int, T_y: "DeviceVec", ty_len: int) -> list:
        """The same on resident eq tables T_x (tx_len entries >= rows) and T_y (ty_len entries >= cols)."""
        out = _small_buf("r1cs_eval", 96)
        check(lib().b200_r1cs_eval_dev(self._handles(), 3, T_x.ptr, tx_len, T_y.ptr, ty_len, out.ptr, None))
        return fields.unpack(self.A.fid, out.to_bytes(96))


# ---------------------------------------------------------------------------------------------
# polynomials
# ---------------------------------------------------------------------------------------------
def eq_evals_from_points(fid: int, r: bytes) -> bytes:
    ell = len(r) // 32
    out = ctypes.create_string_buffer(32 << ell)
    check(lib().b200_eq_table(fid, _cbuf(r), ell, out))
    return out.raw


def evaluate_with(fid: int, Z: bytes, r: bytes) -> bytes:
    ell = len(r) // 32
    assert len(Z) == 32 << ell  # multilinear.rs:90
    out = ctypes.create_string_buffer(32)
    check(lib().b200_mle_eval(fid, _cbuf(Z), ell, _cbuf(r), out))
    return out.raw


def gather(table: bytes, indices) -> bytes:
    """out[i] = table[indices[i]] (L_row / L_col, spartan/ppsnark.rs:236-250)."""
    n = len(indices)
    idx = (c_u64 * max(n, 1))(*indices)
    out = ctypes.create_string_buffer(max(32 * n, 1))
    check(lib().b200_gather(_cbuf(table), len(table) // 32, idx, n, out))
    return out.raw[:32 * n]


def batch_invert(fid: int, v: bytes) -> bytes:
    """Raises ValueError("InternalError") on a zero element (spartan/mod.rs:98-100)."""
    n = len(v) // 32
    out = ctypes.create_string_buffer(max(32 * n, 1))
    rc = lib().b200_batch_invert(fid, _cbuf(v), n, out)
    if rc == 6:
        raise ValueError("InternalError")
    check(rc)
    return out.raw[:32 * n]


def rlc(fid: int, polys: list, coeffs: bytes, n: int) -> bytes:
    k = len(polys)
    bufs = [_cbuf(p) for p in polys]
    ptrs = (ctypes.c_void_p * max(k, 1))(*[ctypes.cast(b, ctypes.c_void_p) for b in bufs])
    lens = (c_size_t * max(k, 1))(*[len(p) // 32 for p in polys])
    out = ctypes.create_string_buffer(max(32 * n, 1))
    check(lib().b200_rlc(fid, ptrs, lens, k, _cbuf(coeffs), n, out))
    return out.raw[:32 * n]


def kzg_fold(fid: int, p: bytes, x: bytes) -> bytes:
    n = len(p) // 32
    out = ctypes.create_string_buffer(max(16 * n, 1))
    check(lib().b200_kzg_fold(fid, _cbuf(p), n, _cbuf(x), out))
    return out.raw[:16 * n]


def poly_eval(fid: int, f: bytes, us: bytes) -> bytes:
    n, nu = len(f) // 32, len(us) // 32
    out = ctypes.create_string_buffer(32 * nu)
    check(lib().b200_poly_eval(fid, _cbuf(f), n, _cbuf(us), nu, out))
    return out.raw


def poly_div(fid: int, f: bytes, u: bytes) -> bytes:
    n = len(f) // 32
    assert n > 0  # hyperkzg.rs:966
    out = ctypes.create_string_buffer(max(32 * (n - 1), 1))
    check(lib().b200_poly_div(fid, _cbuf(f), n, _cbuf(u), out))
    return out.raw[:32 * (n - 1)]


# ---------------------------------------------------------------------------------------------
# sum-check (host keeps O(1) algebra on Python integers; device does the sums and binds)
# ---------------------------------------------------------------------------------------------
class UniPoly:
    """polys/univariate.rs:89-154; transcript bytes :177-190 (non-evm)."""

    def __init__(self, p, coeffs):
        self.p, self.coeffs = p, [c % p for c in coeffs]

    @classmethod
    def from_evals_deg2(cls, p, ev):
        c, abc, a = ev
        return cls(p, [c, abc - a - c, a])

    @classmethod
    def from_evals_deg3(cls, p, ev):
        d, abcd, a, m1 = ev
        b = ((abcd + m1) * pow(2, -1, p) - d) % p
        return cls(p, [d, abcd - a - d - b, b, a])

    @classmethod
    def from_evals(cls, p, ev):
        """UniPoly::from_evals (univariate.rs:58-85): the polynomial of degree < len(ev) through (x, ev[x]),
        x = 0, 1, ...  The reference solves the Vandermonde system by Gaussian elimination; the interpolant is
        unique, so Lagrange's formula gives the same coefficients."""
        n = len(ev)
        coeffs = [0] * n
        for i, y in enumerate(ev):
            num, den = [1], 1  # prod_{m != i} (X - m) / (i - m), coefficients lowest first
            for m in range(n):
                if m != i:
                    num = [(a - m * b) % p for a, b in zip([0] + num, num + [0])]
                    den = den * (i - m) % p
            k = y * pow(den, -1, p) % p
            coeffs = [(c + k * a) % p for c, a in zip(coeffs, num)]
        return cls(p, coeffs)

    def evaluate(self, r):
        acc, pw = self.coeffs[0], r
        for c in self.coeffs[1:]:
            acc = (acc + pw * c) % self.p
            pw = pw * r % self.p
        return acc

    def compress(self):
        return [self.coeffs[0]] + self.coeffs[2:]

    def to_transcript_bytes(self):
        return b"".join(int(c).to_bytes(32, "little") for c in self.compress())


_SMALL = {}


def _small_buf(name: str, nbytes: int) -> "DeviceVec":
    """Persistent few-byte device buffers (round results, the current challenge): allocating and
    freeing them every sum-check round costs more than the round's kernels once the tables are
    short (cudaFree synchronises the device)."""
    v = _SMALL.get(name)
    if v is None or v.nbytes < nbytes or not v.ptr:
        v = _SMALL[name] = DeviceVec(nbytes)
    return v


def _challenge_dev(fid: int, r_int: int) -> "DeviceVec":
    rdev = _small_buf("challenge", 32)
    check(lib().b200_memcpy_h2d(rdev.ptr, _cbuf(fields.to_mont_bytes(fid, r_int)), 32))
    return rdev


def mle_eval_multi_dev(fid: int, vecs: list, ell: int, r_dev: "DeviceVec") -> list:
    """MultilinearPolynomial::multi_evaluate_with (multilinear.rs:129-180) on device-resident polynomials of
    2^ell entries: one pair of sqrt-sized eq tables for all of them, one read-back of the k values."""
    k = len(vecs)
    if k == 0:
        return []
    ptrs = (ctypes.c_void_p * k)(*[v.ptr.value for v in vecs])
    out = DeviceVec(32 * k)
    check(lib().b200_mle_eval_multi_dev(fid, ptrs, k, ell, r_dev.ptr, out.ptr, None))
    return fields.unpack(fid, out.to_bytes(32 * k))


def commit_many_dev(curve, ck: CommitmentKey, vecs: list, lens: list) -> list:
    """CE::batch_commit with r = 0 on device-resident vectors (b200_commit_many_dev: the MSMs are
    spread over the key's lanes so short ones overlap) -> affine points / None."""
    k = len(vecs)
    if k == 0:
        return []
    ptrs = (ctypes.c_void_p * k)(*[v.ptr.value for v in vecs])
    lns = (c_size_t * k)(*lens)
    out = _small_buf("commit_many", 96 * max(k, 32))
    check(lib().b200_commit_many_dev(ck.handle, ptrs, lns, k, out.ptr, None))
    raw = out.to_bytes(96 * k)
    return [_jac_to_affine(Curve(curve), raw[96 * j:96 * j + 96]) for j in range(k)]


def _sc_eval_dev(fid, form, A, B, C, length, eq_left, eq_right, shift) -> list:
    out = _small_buf("sc_out", 96)
    check(lib().b200_sc_eval_dev(fid, form, A.ptr, B.ptr if B else None, C.ptr if C else None, length,
                                 eq_left.ptr if eq_left else None, eq_right.ptr if eq_right else None,
                                 shift, out.ptr, None))
    raw = out.to_bytes(32 * SC_NOUT[form])
    return fields.unpack(fid, raw)


def _bind_dev(fid, Z: DeviceVec, length: int, r_int: int):
    check(lib().b200_bind_top_dev(fid, Z.ptr, length, _challenge_dev(fid, r_int).ptr, None))


def _bind_all(fid, polys, length, r_dev):
    """bind_poly_var_top of several tables of one length with the same challenge: ONE launch (b200_bind_top_multi_dev)"""
    polys = list(polys)
    ptrs = (ctypes.c_void_p * len(polys))(*[Z.ptr.value for Z in polys])
    check(lib().b200_bind_top_multi_dev(fid, ptrs, len(polys), length, r_dev.ptr, None))


def _resident(x) -> DeviceVec:
    """a DeviceVec as it is (the caller's table is bound in place), bytes uploaded into a new one"""
    return x if isinstance(x, DeviceVec) else DeviceVec.from_bytes(x)


class EqSumCheckInstance:
    """sumcheck.rs:593-1251.  The sqrt-sized eq tables are built on the host exactly as in `new`
    (:606-664) and uploaded once; per-round sums run on the device."""

    def __init__(self, fid: int, taus: list):
        p = fields.MODULUS[fid]
        self.fid, self.p = fid, p
        l = len(taus)
        self.init_num_vars, self.first_half = l, l // 2
        self.second_half = l - self.first_half
        self.round, self.taus, self.eval_eq_left = 1, list(taus), 1

        def compute(ts):
            res = [[1]]
            for t in ts:
                prev = res[-1]
                hi = [v * t % p for v in prev]
                res.append([(a - b) % p for a, b in zip(prev, hi)] + hi)
            return res

        # built on first use: the one-call loops (b200_sumcheck_batched / b200_sumcheck_cubic3) build their own on the device
        self._compute, self._left, self._right = compute, None, None
        self.eq_tau_0_a_inf = [((1 - t) % p, (2 * t - 1) % p, (2 - 3 * t) % p) for t in taus]

    def _build_tables(self):
        taus, fid = self.taus, self.fid
        left = list(reversed(taus[1:self.first_half])) if self.first_half >= 1 else []
        right = list(reversed(taus[self.first_half:]))
        self._left = [DeviceVec.from_bytes(fields.pack(fid, t)) for t in self._compute(left)]
        self._right = [DeviceVec.from_bytes(fields.pack(fid, t)) for t in self._compute(right)]

    def _tables(self):
        if self._left is None:
            self._build_tables()
        if self.round < self.first_half:  # poly_eqs_first_half, sumcheck.rs:1233-1246
            return self._left[self.first_half - self.round], self._right[self.second_half], self.second_half
        return None, self._right[self.init_num_vars - self.round], 0  # :1248-1251

    def evaluation_points(self, t0, tinf, claim, t_m1):
        """(s(0), lead, s(-1)) of the eq-weighted claim `claim` from the sums t(0), t(inf) of its inner polynomial
        (tinf = 0 when that polynomial is linear).  s(-1) comes from t(1), which the claim determines unless this
        round's tau is 0 (sumcheck.rs:696-698); then `t_m1()` is called for the third sum t(-1)
        (sumcheck.rs:1082-1213)."""
        p, q = self.p, self.eval_eq_left
        e0, slope, em1 = self.eq_tau_0_a_inf[self.round - 1]
        s0 = e0 * q * t0 % p
        l1p = (e0 + slope) * q % p
        if l1p == 0:
            tm1 = t_m1()
        else:
            t1 = (claim - s0) * pow(l1p, -1, p) % p
            tm1 = 2 * tinf + 2 * t0 - t1
        return s0, slope * q * tinf % p, em1 * q * (tm1 % p) % p

    def evaluation_points_cubic_with_three_inputs(self, A, B, C, length, claim):
        """sumcheck.rs:900-966 (+ fall-back :1082-1178)."""
        L, R, sh = self._tables()
        t0, tinf = _sc_eval_dev(self.fid, SC_EQ_CUBIC3, A, B, C, length, L, R, sh)
        return self.evaluation_points(t0, tinf, claim,
                                      lambda: _sc_eval_dev(self.fid, SC_EQ_CUBIC3_M1, A, B, C, length, L, R, sh)[0])

    def evaluation_points_quadratic_with_one_input(self, A, length, claim):
        """sumcheck.rs:1039-1080 (+ fall-back :1180-1213)."""
        L, R, sh = self._tables()
        (t0,) = _sc_eval_dev(self.fid, SC_EQ_QUAD1, A, None, None, length, L, R, sh)
        return self.evaluation_points(t0, 0, claim,
                                      lambda: _sc_eval_dev(self.fid, SC_EQ_QUAD1_M1, A, None, None, length, L, R, sh)[0])

    def bound(self, r):
        tau = self.taus[self.round - 1]
        self.eval_eq_left = self.eval_eq_left * (1 - tau - r + 2 * r * tau) % self.p
        self.round += 1


def update_claim(p, claim, evals, r):
    """SumcheckProof::update_claim (sumcheck.rs:68-75)."""
    e0, c3, em1 = evals
    e1 = (claim - e0) % p
    half = pow(2, -1, p)
    a1 = ((e1 - em1) * half - c3) % p
    a2 = ((e1 + em1) * half - e0) % p
    return (e0 + r * (a1 + r * (a2 + r * c3))) % p


class SumcheckProof:
    @staticmethod
    def verify(fid, polys, claim, num_rounds, degree_bound, transcript):
        """SumcheckProof::verify (sumcheck.rs:87-127): `polys` are the compressed round polynomials (the coefficients
        without the linear term, CompressedUniPoly::decompress restores it from the running claim).  Returns (the
        final claim, the challenges); a wrong number of rounds or a degree above the bound raises
        ValueError("InvalidSumcheckProof")."""
        p = fields.MODULUS[fid]
        if len(polys) != num_rounds:
            raise ValueError("InvalidSumcheckProof")
        e, rs = claim % p, []
        for cp in polys:
            if not 1 <= len(cp) <= degree_bound:  # decompressed degree = len(cp); an empty message has no c0
                raise ValueError("InvalidSumcheckProof")
            poly = UniPoly(p, [cp[0], e - 2 * cp[0] - sum(cp[1:])] + list(cp[1:]))
            transcript.absorb_bytes(b"p", poly.to_transcript_bytes())
            r = transcript.squeeze(b"c")
            rs.append(r)
            e = poly.evaluate(r)
        return e, rs

    @staticmethod
    def verify_batch(fid, polys, claims, num_rounds, coeffs, degree_bound, transcript):
        """SumcheckProof::verify_batch (sumcheck.rs:131-161): instances of different sizes, each claim scaled by
        2^(n - n_i) for the padding and combined with `coeffs`, then `verify` over n = max n_i rounds."""
        p = fields.MODULUS[fid]
        assert len(claims) == len(num_rounds) == len(coeffs)
        nmax = max(num_rounds)
        claim = sum(c * pow(2, nmax - nr, p) * k for c, nr, k in zip(claims, num_rounds, coeffs)) % p
        return SumcheckProof.verify(fid, polys, claim, nmax, degree_bound, transcript)

    @staticmethod
    def prove_batch_eval(fid, claims, num_rounds, polys: list, eq_points: list, coeffs, transcript):
        """sumcheck.rs:251-351: batched evaluation claims of different sizes; polynomials resident on
        the device, one `eq_quad1` reduction per active instance per round."""
        p = fields.MODULUS[fid]
        k = len(claims)
        assert len(num_rounds) == k and len(polys) == k and len(eq_points) == k and len(coeffs) == k
        for i in range(k):
            if not isinstance(polys[i], DeviceVec):
                assert len(polys[i]) == 32 << num_rounds[i], f"poly size mismatch at index {i}"
            assert len(eq_points[i]) == num_rounds[i], f"eq_point length mismatch at index {i}"
        nmax = max(num_rounds)

        def working_copy(P, n):  # the loop binds in place; resident inputs are copied device-to-device
            if not isinstance(P, DeviceVec):
                return DeviceVec.from_bytes(P)
            v = DeviceVec(32 * n)
            check(lib().b200_memcpy_d2d(v.ptr, P.ptr, 32 * n, None))
            return v
        dev = [working_copy(P, 1 << nr) for P, nr in zip(polys, num_rounds)]
        lens = [1 << nr for nr in num_rounds]
        eqs = [EqSumCheckInstance(fid, pts) for pts in eq_points]
        running = list(claims)
        e = sum(claims[i] * pow(2, nmax - num_rounds[i], p) * coeffs[i] for i in range(k)) % p
        rs, out = [], []
        for cur in range(nmax):
            rem = nmax - cur
            evals = []
            for i in range(k):
                if rem <= num_rounds[i]:
                    e0, _, em1 = eqs[i].evaluation_points_quadratic_with_one_input(dev[i], lens[i], running[i])
                    evals.append((e0, 0, em1))
                else:
                    sc = pow(2, rem - num_rounds[i] - 1, p) * claims[i] % p
                    evals.append((sc, 0, sc))
            c0 = sum(evals[i][0] * coeffs[i] for i in range(k)) % p
            cm1 = sum(evals[i][2] * coeffs[i] for i in range(k)) % p
            c1 = (e - c0) % p
            quad = (c1 + cm1 - 2 * c0) * pow(2, -1, p) % p
            poly = UniPoly.from_evals_deg2(p, [c0, c1, quad])
            transcript.absorb_bytes(b"p", poly.to_transcript_bytes())
            r = transcript.squeeze(b"c")
            rs.append(r)
            for i in range(k):
                if rem <= num_rounds[i]:
                    running[i] = update_claim(p, running[i], evals[i], r)
                    _bind_dev(fid, dev[i], lens[i], r)
                    lens[i] //= 2
                    eqs[i].bound(r)
            e = poly.evaluate(r)
            out.append(poly.compress())
        finals = [fields.unpack(fid, d.to_bytes(32))[0] for d in dev]
        return out, rs, finals

    @staticmethod
    def prove_quad_prod(fid, claim, num_rounds, poly_A, poly_B, transcript):
        """sumcheck.rs:199-242 -> (compressed polys, challenges r, [A(r), B(r)]).  poly_A / poly_B: bytes (uploaded)
        or DeviceVec of 2^num_rounds entries (bound in place)."""
        p = fields.MODULUS[fid]
        length = 1 << num_rounds if isinstance(poly_A, DeviceVec) else len(poly_A) // 32
        A, B = _resident(poly_A), _resident(poly_B)
        rs, polys = [], []
        for _ in range(num_rounds):
            e0, bc = _sc_eval_dev(fid, SC_QUAD_PROD, A, B, None, length, None, None, 0)
            poly = UniPoly.from_evals_deg2(p, [e0, (claim - e0) % p, bc])
            transcript.absorb_bytes(b"p", poly.to_transcript_bytes())
            r = transcript.squeeze(b"c")
            rs.append(r)
            polys.append(poly.compress())
            claim = poly.evaluate(r)
            _bind_dev(fid, A, length, r)
            _bind_dev(fid, B, length, r)
            length //= 2
        return polys, rs, fields.unpack(fid, A.to_bytes(32)) + fields.unpack(fid, B.to_bytes(32))

    @staticmethod
    def prove_cubic_with_three_inputs(fid, claim, taus, poly_A, poly_B, poly_C, transcript):
        """sumcheck.rs:446-507.  poly_A / poly_B / poly_C: bytes (uploaded) or DeviceVec of 2^len(taus) entries
        (bound in place)."""
        p = fields.MODULUS[fid]
        length = 1 << len(taus) if isinstance(poly_A, DeviceVec) else len(poly_A) // 32
        A, B, C = (_resident(x) for x in (poly_A, poly_B, poly_C))
        eq = EqSumCheckInstance(fid, taus)
        rs, polys = [], []
        for _ in range(len(taus)):
            e0, lead, em1 = eq.evaluation_points_cubic_with_three_inputs(A, B, C, length, claim)
            poly = UniPoly.from_evals_deg3(p, [e0, (claim - e0) % p, lead, em1])
            transcript.absorb_bytes(b"p", poly.to_transcript_bytes())
            r = transcript.squeeze(b"c")
            rs.append(r)
            polys.append(poly.compress())
            claim = poly.evaluate(r)
            _bind_all(fid, (A, B, C), length, _challenge_dev(fid, r))
            eq.bound(r)
            length //= 2
        finals = [fields.unpack(fid, Z.to_bytes(32))[0] for Z in (A, B, C)]
        return polys, rs, finals


    @staticmethod
    def prove_batched_cubic(fid, claim, taus, polys_A: list, polys_B: list, polys_C: list, alphas, transcript):
        """sumcheck.rs:513-577: sum_x eq(tau, x) sum_i alpha_i (A_i B_i - C_i)(x) over K instance triples.
        The inner polynomial is linear in the instances, so t(0), t(inf) (and t(-1) in a tau = 0 round) are
        the alpha-combinations of the K single-instance reductions (form eq_cubic3), one launch pair each,
        all read back at once.  -> (compressed polys, r, [[A_i(r), B_i(r), C_i(r)]])."""
        p = fields.MODULUS[fid]
        k = len(polys_A)
        if k == 0:
            raise ValueError("InvalidNumInstances")  # sumcheck.rs:524-526
        assert k == len(polys_B) == len(polys_C) == len(alphas) and k <= 16
        dev = [[P if isinstance(P, DeviceVec) else DeviceVec.from_bytes(P) for P in V] for V in (polys_A, polys_B, polys_C)]
        length = 1 << len(taus)
        eq = EqSumCheckInstance(fid, taus)
        out = _small_buf("batched_cubic_sums", 96 * 16)
        rs, polys = [], []

        def sums(form, nout):
            L, R, sh = eq._tables()
            for i in range(k):
                dst = ctypes.c_void_p(out.ptr.value + 96 * i)
                check(lib().b200_sc_eval_dev(fid, form, dev[0][i].ptr, dev[1][i].ptr, dev[2][i].ptr, length,
                                             L.ptr if L else None, R.ptr, sh, dst, None))
            raw = out.to_bytes(96 * k)
            per = [fields.unpack(fid, raw[96 * i:96 * i + 32 * nout]) for i in range(k)]
            return [sum(a * v[c] for a, v in zip(alphas, per)) % p for c in range(nout)]
        for _ in range(len(taus)):
            t0, tinf = sums(SC_EQ_CUBIC3, 2)
            e0, lead, em1 = eq.evaluation_points(t0, tinf, claim, lambda: sums(SC_EQ_CUBIC3_M1, 1)[0])  # tau = 0: :838-890
            poly = UniPoly.from_evals_deg3(p, [e0, (claim - e0) % p, lead, em1])
            transcript.absorb_bytes(b"p", poly.to_transcript_bytes())
            r = transcript.squeeze(b"c")
            rs.append(r)
            polys.append(poly.compress())
            claim = poly.evaluate(r)
            r_dev = _challenge_dev(fid, r)
            for V in dev:
                for Z in V:
                    check(lib().b200_bind_top_dev(fid, Z.ptr, length, r_dev.ptr, None))
            eq.bound(r)
            length //= 2
        finals = [[fields.unpack(fid, dev[c][i].to_bytes(32))[0] for c in range(3)] for i in range(k)]
        return polys, rs, finals

    # ---- the same two loops with the transcript on the device (SURVEY.md §8f-3) --------------------
    # One FFI call each: every round's reduction, round algebra + Keccak and binds are enqueued back
    # to back (csrc/capi_sumcheck.inc); the host reads the proof once.  `transcript` is any object
    # with the serialisable fields of Keccak256Transcript (keccak.rs:19-27): `round`, `state`
    # (64 bytes) and `buf` (bytes absorbed since the last squeeze); it is advanced in place.
    @staticmethod
    def _device_loop(fid, transcript, call, num_rounds, ncoef, nfinals):
        tr = (ctypes.c_ubyte * 72)()
        ctypes.memmove(tr, int(transcript.round).to_bytes(8, "little") + bytes(transcript.state), 72)
        pending = bytes(transcript.buf)
        polys = ctypes.create_string_buffer(32 * ncoef * num_rounds)
        rs = ctypes.create_string_buffer(32 * num_rounds)
        finals = ctypes.create_string_buffer(32 * nfinals)
        check(call(tr, _cbuf(pending) if pending else None, len(pending), polys, rs, finals))
        raw = bytes(tr)
        transcript.round = int.from_bytes(raw[:8], "little")
        transcript.state = raw[8:72]
        transcript.buf = b""
        coeffs = [int.from_bytes(polys.raw[32 * i:32 * i + 32], "little") for i in range(ncoef * num_rounds)]
        return ([coeffs[ncoef * j:ncoef * (j + 1)] for j in range(num_rounds)], fields.unpack(fid, rs.raw),
                fields.unpack(fid, finals.raw))

    @staticmethod
    def prove_quad_prod_device(fid, claim, num_rounds, poly_A, poly_B, transcript):
        """sumcheck.rs:199-242 through b200_sumcheck_quad_prod.  poly_A / poly_B: bytes (uploaded) or
        DeviceVec (bound in place)."""
        A, B = _resident(poly_A), _resident(poly_B)
        cl = _cbuf(fields.to_mont_bytes(fid, claim))
        return SumcheckProof._device_loop(
            fid, transcript,
            lambda tr, pend, plen, polys, rs, fin: lib().b200_sumcheck_quad_prod(
                fid, cl, num_rounds, A.ptr, B.ptr, tr, pend, plen, polys, rs, fin),
            num_rounds, 2, 2)

    @staticmethod
    def prove_cubic_with_three_inputs_device(fid, claim, taus, poly_A, poly_B, poly_C, transcript):
        """sumcheck.rs:446-507 through b200_sumcheck_cubic3 (eq tables, 1/tau and the tau = 0
        fall-back are handled inside the library)."""
        A, B, C = (_resident(x) for x in (poly_A, poly_B, poly_C))
        cl = _cbuf(fields.to_mont_bytes(fid, claim))
        tb = _cbuf(fields.pack(fid, taus))
        return SumcheckProof._device_loop(
            fid, transcript,
            lambda tr, pend, plen, polys, rs, fin: lib().b200_sumcheck_cubic3(
                fid, cl, tb, len(taus), A.ptr, B.ptr, C.ptr, tr, pend, plen, polys, rs, fin),
            len(taus), 3, 3)


# ---------------------------------------------------------------------------------------------
# HyperKZG prover core (hyperkzg.rs:1076-1116 with the transcript challenges r, q given)
# ---------------------------------------------------------------------------------------------
def hyperkzg_prove_resident(curve, ck: CommitmentKey, P: "DeviceVec", x: list, r, q,
                            timings: dict | None = None, on_w=None):
    """The same on a polynomial that is already in HBM: folds, commitments, the 3-point
    evaluations, the batch polynomial and the three quotients never leave the device; the host
    receives ell-1 + 3 points and 3*ell scalars.  Returns (com, v, w, polys) with `polys` the
    resident fold chain.  `timings` (optional) receives seconds per phase.
    `r` / `q` are the two challenges, or callables `r(com)` / `q(v)` that derive them from the messages
    produced so far (the transcript steps of hyperkzg.rs:1099-1107, 1060); `on_w(w)` sees the quotient
    commitments (verifier_second_challenge, :1068-1070)."""
    import time
    fid = Curve(curve).scalar_field
    p = fields.MODULUS[fid]
    ell = len(x)
    n = 1 << ell
    L = lib()
    t_last = [time.perf_counter()]

    def mark(name):
        if timings is not None:
            check(L.b200_sync())
            now = time.perf_counter()
            timings[name] = timings.get(name, 0.0) + now - t_last[0]
            t_last[0] = now
    polys, lens = [P], [n]
    for i in range(ell - 1):  # Phase 1: fold (hyperkzg.rs:1083-1095)
        xi = DeviceVec.from_bytes(fields.to_mont_bytes(fid, x[ell - i - 1]))
        nxt = DeviceVec(16 * lens[i])
        check(L.b200_kzg_fold_dev(fid, polys[i].ptr, lens[i], xi.ptr, nxt.ptr, None))
        polys.append(nxt)
        lens.append(lens[i] // 2)
    mark("fold")
    com = commit_many_dev(curve, ck, polys[1:], lens[1:])  # :1099-1100 batch_commit(polys[1..])
    mark("commit_folds")
    if callable(r):
        r = r(com)
    u = [r % p, (-r) % p, r * r % p]  # :1105-1106
    us = DeviceVec.from_bytes(fields.pack(fid, u))
    ev = DeviceVec(96 * ell)
    check(L.b200_poly_eval_many_dev(fid, (ctypes.c_void_p * ell)(*[v_.ptr.value for v_ in polys]), (c_size_t * ell)(*lens), ell,
                                    us.ptr, 3, ev.ptr, None))  # :1048-1056, the short polynomials in one launch
    evb = ev.to_bytes(96 * ell)
    v = [fields.unpack(fid, evb[96 * i:96 * i + 96]) for i in range(ell)]
    mark("evals")
    if callable(q):
        q = q(v)
    assert ell <= 32, "rlc of more than 32 polynomials"
    qd = DeviceVec.from_bytes(fields.pack(fid, [pow(q, k, p) for k in range(ell)]))  # batch_challenge_powers
    ptrs = (ctypes.c_void_p * ell)(*[v_.ptr.value for v_ in polys])
    lns = (c_size_t * ell)(*lens)
    Bpoly = DeviceVec(32 * n)
    check(L.b200_rlc_dev(fid, ptrs, lns, ell, qd.ptr, n, Bpoly.ptr, None))  # :1028-1040
    mark("batch_poly")
    hs = []
    for t, ut in enumerate(u):  # :1062-1065: w_t = commit(B / (X - u_t))
        ud = DeviceVec.from_bytes(fields.to_mont_bytes(fid, ut))
        h = DeviceVec(32 * max(n - 1, 1))
        check(L.b200_poly_div_dev(fid, Bpoly.ptr, n, ud.ptr, h.ptr, None))
        hs.append((h, ud))
    mark("quotients")
    w = commit_many_dev(curve, ck, [h for h, _ in hs], [n - 1] * 3)
    mark("commit_quotients")
    if on_w is not None:
        on_w(w)
    return com, v, w, polys


def _commitment_bytes(P) -> bytes:
    """Commitment::to_transcript_bytes (hyperkzg.rs:233-248): x || y || is_infinity."""
    if P is None:
        return bytes(64) + b"\x01"
    return int(P[0]).to_bytes(32, "little") + int(P[1]).to_bytes(32, "little") + b"\x00"


def hyperkzg_prove(curve, ck: CommitmentKey, P: "DeviceVec", x: list, transcript, timings: dict | None = None):
    """EvaluationEngine::prove (hyperkzg.rs:926-1116) with the transcript: r = H(com), q = H(v), and the second
    verifier challenge squeezed after W so that the transcript ends in the verifier's state.
    -> EvaluationArgument (com, w, v)."""
    def r_of(com):  # compute_challenge, :861-865
        transcript.absorb_bytes(b"c", b"".join(_commitment_bytes(C) for C in com))
        return transcript.squeeze(b"c")

    def q_of(v):    # get_batch_challenge, :869-880
        transcript.absorb_bytes(b"v", b"".join(int(e).to_bytes(32, "little") for row in v for e in row))
        return transcript.squeeze(b"r")

    def after_w(w):  # verifier_second_challenge, :891-898
        transcript.absorb_bytes(b"W", b"".join(_commitment_bytes(C) for C in w))
        transcript.squeeze(b"d")
    com, v, w, _ = hyperkzg_prove_resident(curve, ck, P, x, r_of, q_of, timings, after_w)
    return com, w, v


def hyperkzg_prove_core(curve, ck: CommitmentKey, hat_P: bytes, x: list, r: int, q: int):
    """Returns (com[ell-1], v[ell][3], w[3]) for challenges r (evaluation points r, -r, r^2) and q
    (batching).  `x` is the evaluation point as integers."""
    assert len(hat_P) // 32 == 1 << len(x)  # hyperkzg.rs:1078
    com, v, w, _ = hyperkzg_prove_resident(curve, ck, DeviceVec.from_bytes(hat_P), x, r, q)
    return com, v, w


class DeviceSumcheckEngine:
    """Local engine of `sharding.sharded_prove_cubic_with_three_inputs` on one GPU: tables resident
    in HBM, sums through b200_sc_eval_sharded_dev, binds through b200_bind_top_dev."""

    def __init__(self, fid: int):
        self.fid = fid
        self.p = fields.MODULUS[fid]

    def upload(self, b: bytes) -> DeviceVec:
        return DeviceVec.from_bytes(b)

    def download(self, h: DeviceVec, n_elems: int) -> bytes:
        return h.to_bytes(32 * n_elems)

    def download_canonical(self, h: DeviceVec) -> bytes:
        return fields.from_mont_bytes(self.fid, h.to_bytes(32)).to_bytes(32, "little")

    def eq_tables(self, taus):
        inst = EqSumCheckInstance(self.fid, taus)

        class _T:
            def tables(_, rnd):
                inst.round = rnd
                return inst._tables()
        return _T()

    def sc_eval(self, form, A, B, C, local_len, left, right, shift, id_mul, id_add):
        out = DeviceVec(96)
        check(lib().b200_sc_eval_sharded_dev(self.fid, form, A.ptr, B.ptr, C.ptr, local_len,
                                             left.ptr if left else None, right.ptr, shift, id_mul, id_add,
                                             out.ptr, None))
        return fields.unpack(self.fid, out.to_bytes(32 * SC_NOUT[form]))

    def bind(self, h, local_len, r):
        _bind_dev(self.fid, h, local_len, r)
