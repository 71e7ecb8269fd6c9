"""CPU restatement of NeutronNova's folding scheme (src/neutron/nifs.rs, src/neutron/relation.rs) on Python
integers, with SpMV, commitments and the large sums taken from the C oracle.  TEST INFRASTRUCTURE ONLY.

  split_evals / evals         PowPolynomial (spartan/polys/power.rs:32-86)
  prove_helper                NIFS::prove_helper (nifs.rs:29-186), in its incremental form
  from_evals                  UniPoly::from_evals by gaussian_elimination (spartan/polys/univariate.rs:58-85, 218-262)
  to_bignat_repr, absorb_*    Commitment::absorb_in_ro2 (pedersen.rs:141-156, gadgets/utils.rs:107),
                              R1CSInstance::absorb_in_ro2 (r1cs/mod.rs:967-975), UniPoly (univariate.rs:207-213)
  pad                         R1CSShape::pad (r1cs/mod.rs:668-730) and R1CSWitness::pad (:874-879)
  Structure, is_sat           Structure::new / is_sat (relation.rs:52-116)
  FoldedInstance / Witness    default and fold (relation.rs:119-198)
  nifs_prove / nifs_verify    NIFS::prove / verify (nifs.rs:200-343)

A shape is `Shape(fid, num_cons, num_vars, num_io, A, B, C)` with each matrix in CSR form
(data: list of ints, indices, indptr); z = (W, u, X).  A commitment key is `(curve_id, bases, h)`: bases the
64-byte affine points, h the blinding generator.  Commitments are affine tuples, None for the identity.
`ro` is any object with absorb(int) / squeeze(num_bits, start_with_one) over the scalar field
(oracle.poseidon_ref.PoseidonRO in use).

`evals_raw` is the same sum as `prove_helper` before its rho factors, composed from the C oracle's vector passes
(axpy, cross_term, and the eq-weighted dot product of sc_eval with the split table as its two eq factors), for
sizes where the literal Python loop is too slow."""
from collections import namedtuple
from dataclasses import dataclass, field

from . import coracle as co
from .pyref import CURVES, FIELD_MODULUS, from_mont_bytes, mont_bytes

NUM_CHALLENGE_BITS = 128                  # constants.rs:4
BN_LIMB_WIDTH, BN_N_LIMBS = 64, 4         # constants.rs:10-13

Shape = namedtuple("Shape", "fid num_cons num_vars num_io A B C")


def _pack(p, xs):
    return b"".join(mont_bytes(p, x) for x in xs)


def _ints(p, b):
    return [from_mont_bytes(p, b[i:i + 32]) for i in range(0, len(b), 32)]


# ---- power polynomial (power.rs) ---------------------------------------------------------------------------
def evals(p, tau, ell):
    """PowPolynomial::evals: tau^k for k < 2^ell"""
    out, x = [], 1
    for _ in range(1 << ell):
        out.append(x)
        x = x * tau % p
    return out


def split_evals(p, tau, left, right):
    """PowPolynomial::split_evals(len_left, len_right), literally: `right[1]` panics when right = 1."""
    lv = [1]
    while len(lv) < left:
        lv.append(lv[-1] * tau % p)
    left_last_times_t = lv[left - 1] * tau % p
    rv = [1] * right
    rv[0] = 1
    if right < 2:
        raise IndexError("split_evals indexes right[1] (power.rs:79): right must be at least 2")
    rv[1] = left_last_times_t
    for i in range(2, right):
        rv[i] = rv[i - 1] * left_last_times_t % p
    return lv + rv


# ---- univariate polynomials (univariate.rs) ----------------------------------------------------------------
def gaussian_elimination(p, matrix):
    size = len(matrix)
    assert size == len(matrix[0]) - 1
    div = lambda a, b: a * pow(b, -1, p) % p
    for i in range(size - 1):
        for j in range(i, size - 1):  # echelon
            if matrix[i][i] % p:
                factor = div(matrix[j + 1][i], matrix[i][i])
                for k in range(i, size + 1):
                    matrix[j + 1][k] = (matrix[j + 1][k] - factor * matrix[i][k]) % p
    for i in range(size - 1, 0, -1):  # eliminate
        if matrix[i][i] % p:
            for j in range(i, 0, -1):
                factor = div(matrix[j - 1][i], matrix[i][i])
                for k in range(size, -1, -1):
                    matrix[j - 1][k] = (matrix[j - 1][k] - factor * matrix[i][k]) % p
    return [div(matrix[i][size], matrix[i][i]) for i in range(size)]


def from_evals(p, ev):
    """UniPoly::from_evals: the interpolant through (x, ev[x]), x = 0 .. len-1, by Gaussian elimination"""
    n = len(ev)
    if n == 1:
        return [ev[0] % p]
    matrix = []
    for i in range(n):
        row = [1, i % p]
        for j in range(2, n):
            row.append(row[j - 1] * i % p)
        row.append(ev[i] % p)
        matrix.append(row)
    return gaussian_elimination(p, matrix)


def uni_eval(p, coeffs, r):
    """UniPoly::evaluate"""
    acc, pw = coeffs[0], r
    for c in coeffs[1:]:
        acc = (acc + pw * c) % p
        pw = pw * r % p
    return acc


# ---- RO2 absorption ----------------------------------------------------------------------------------------
def to_bignat_repr(x):
    """BN_N_LIMBS little-endian limbs of BN_LIMB_WIDTH bits of a base-field element"""
    return [(x >> (BN_LIMB_WIDTH * k)) & ((1 << BN_LIMB_WIDTH) - 1) for k in range(BN_N_LIMBS)]


def absorb_commitment(ro, P):
    """Commitment::absorb_in_ro2: limbs of x, limbs of y, then the infinity flag; the identity is (0, 0, true)"""
    x, y, inf = (0, 0, 1) if P is None else (P[0], P[1], 0)
    for limb in to_bignat_repr(x) + to_bignat_repr(y):
        ro.absorb(limb)
    ro.absorb(inf)


def absorb_r1cs_instance(ro, U2):
    absorb_commitment(ro, U2.comm_W)
    for x in U2.X:
        ro.absorb(x)


# ---- shape (r1cs/mod.rs) ------------------------------------------------------------------------------------
def _pow2(n):
    return n > 0 and n & (n - 1) == 0


def is_regular_shape(S):
    return _pow2(S.num_cons) and _pow2(S.num_vars) and S.num_io < S.num_vars


def pad(S):
    """R1CSShape::pad: num_cons = num_vars = the next power of two of max(num_vars, num_cons, num_io); the
    columns of u and X move up by the padding, new rows are empty."""
    if is_regular_shape(S):
        return S
    m = 1
    while m < max(S.num_vars, S.num_cons, S.num_io):
        m *= 2
    if S.num_vars == m:
        return S._replace(num_cons=m, num_vars=m)

    def apply_pad(M):
        data, idx, ptr = M
        idx = [c + (m - S.num_vars) if c >= S.num_vars else c for c in idx]
        return list(data), idx, list(ptr) + [ptr[-1]] * (m - S.num_cons)
    return Shape(S.fid, m, m, S.num_io, apply_pad(S.A), apply_pad(S.B), apply_pad(S.C))


def pad_witness(S, W):
    """R1CSWitness::pad"""
    return list(W) + [0] * (S.num_vars - len(W))


def multiply_vec(S, z):
    """(Az, Bz, Cz) by the C oracle's SpMV"""
    p = FIELD_MODULUS[S.fid]
    assert len(z) == S.num_vars + 1 + S.num_io, "InvalidWitnessLength"
    zb = _pack(p, z)
    return [_ints(p, co.spmv(S.fid, _pack(p, d), i, pt, zb)) for (d, i, pt) in (S.A, S.B, S.C)]


# ---- commitments ---------------------------------------------------------------------------------------------
def commit(ck, fid, v, r):
    """CE::commit(ck, v, r) = MSM(v, ck[..len]) + r h"""
    cid, bases, h = ck
    p = FIELD_MODULUS[fid]
    return CURVES[cid].affine_from_bytes(co.msm(cid, _pack(p, list(v) + [r]), bases[:64 * len(v)] + h))


def lincomb(cid, terms):
    c = CURVES[cid]
    acc = None
    for k, P in terms:
        acc = c.add(acc, c.mul(k, P))
    return acc


# ---- relation (relation.rs) -----------------------------------------------------------------------------------
@dataclass
class Structure:
    S: Shape
    ell: int
    left: int
    right: int

    @classmethod
    def new(cls, S):
        S = pad(S)
        ell = (S.num_cons - 1).bit_length()  # num_cons.next_power_of_two().log_2()
        return cls(S, ell, 1 << ((ell + 1) // 2), 1 << (ell // 2))


@dataclass
class R1CSInstance:
    comm_W: tuple
    X: list


@dataclass
class R1CSWitness:
    W: list
    r_W: int = 0


@dataclass
class FoldedInstance:
    comm_W: tuple
    comm_E: tuple
    T: int
    u: int
    X: list

    @classmethod
    def default(cls, st):
        return cls(None, None, 0, 0, [0] * st.S.num_io)

    def fold(self, cid, p, U2, comm_E, r_b, T_out):
        one_m = (1 - r_b) % p
        return FoldedInstance(lincomb(cid, [(one_m, self.comm_W), (r_b, U2.comm_W)]),
                              lincomb(cid, [(one_m, self.comm_E), (r_b, comm_E)]), T_out % p,
                              (one_m * self.u + r_b) % p,
                              [(one_m * x1 + r_b * x2) % p for x1, x2 in zip(self.X, U2.X)])


@dataclass
class FoldedWitness:
    W: list
    r_W: int
    E: list
    r_E: int

    @classmethod
    def default(cls, st):
        return cls([0] * st.S.num_vars, 0, [0] * (st.left + st.right), 0)

    def fold(self, p, W2, E2, r_E2, r_b):
        one_m = (1 - r_b) % p
        return FoldedWitness([(w1 + r_b * (w2 - w1)) % p for w1, w2 in zip(self.W, W2.W)],
                             (one_m * self.r_W + r_b * W2.r_W) % p,
                             [(e1 + r_b * (e2 - e1)) % p for e1, e2 in zip(self.E, E2)],
                             (one_m * self.r_E + r_b * r_E2) % p)


@dataclass
class NIFS:
    comm_E: tuple
    poly: list = field(default_factory=list)


def prove_helper_raw(p, left, right, e1, Az1, Bz1, Cz1, e2, Az2, Bz2, Cz2):
    """the five sums of prove_helper before the rho factors, in the reference's loop order and incremental form"""
    assert len(e1) == left + right and len(e2) == left + right
    assert all(len(v) == left * right for v in (Az1, Bz1, Cz1, Az2, Bz2, Cz2))
    comb = lambda c1, c2, c3, c4: c1 * (c2 * c3 - c4) % p
    tot = [0] * 5
    f1, f2 = e1[left:], e2[left:]
    for i in range(right):
        ii = [0] * 5
        for j in range(left):
            k = i * left + j
            ii[0] += comb(e1[j], Az1[k], Bz1[k], Cz1[k])
            pe, pa, pb, pc = (2 * e2[j] - e1[j], 2 * Az2[k] - Az1[k], 2 * Bz2[k] - Bz1[k], 2 * Cz2[k] - Cz1[k])
            ii[1] += comb(pe, pa, pb, pc)
            for t in (2, 3, 4):
                pe, pa, pb, pc = (pe + e2[j] - e1[j], pa + Az2[k] - Az1[k], pb + Bz2[k] - Bz1[k],
                                  pc + Cz2[k] - Cz1[k])
                ii[t] += comb(pe, pa, pb, pc)
        tot[0] += f1[i] * ii[0]
        pf = 2 * f2[i] - f1[i]
        tot[1] += pf * ii[1]
        for t in (2, 3, 4):
            pf = pf + f2[i] - f1[i]
            tot[t] += pf * ii[t]
    return [x % p for x in tot]


def rho_factors(p, rho):
    """(1 - rho), (3 rho - 1), (5 rho - 2), (7 rho - 3), (9 rho - 4)"""
    return [(1 - rho) % p, (3 * rho - 1) % p, (5 * rho - 2) % p, (7 * rho - 3) % p, (9 * rho - 4) % p]


def prove_helper(p, rho, left, right, *vecs):
    return [s * f % p for s, f in zip(prove_helper_raw(p, left, right, *vecs), rho_factors(p, rho))]


def evals_raw(fid, left, right, e1, az1, bz1, cz1, e2, az2, bz2, cz2):
    """prove_helper_raw on Montgomery bytes (e1, e2: lists of ints; the n-vectors: bytes) from the C oracle:
    V_t = V1 + t (V2 - V1) by axpy, Az_t Bz_t - Cz_t by cross_term (E = 0, u = 1), and
    sum_k f_t[k >> log2(left)] e_t[k & (left - 1)] g_t[k] by the eq-weighted dot product.  left: a power of two."""
    p = FIELD_MODULUS[fid]
    assert _pow2(left)
    n = left * right
    zero, one, m1 = bytes(32 * n), mont_bytes(p, 1), mont_bytes(p, p - 1)
    diffs = [co.axpy(fid, v2, v1, m1) for v1, v2 in ((az1, az2), (bz1, bz2), (cz1, cz2))]
    out = []
    for t in (0, 2, 3, 4, 5):
        tb = mont_bytes(p, t)
        a, b, c = (co.axpy(fid, v1, d, tb) for v1, d in zip((az1, bz1, cz1), diffs))
        g = co.cross_term(fid, a, b, c, zero, None, one)
        et = [(x1 + t * (x2 - x1)) % p for x1, x2 in zip(e1, e2)]
        out.append(from_mont_bytes(p, co.sc_eval(fid, 10, g, eq_left=_pack(p, et[left:]), eq_right=_pack(p, et[:left]),
                                                 shift=left.bit_length() - 1)))
    return out


# ---- NIFS (nifs.rs) ---------------------------------------------------------------------------------------------
def _challenges_after_E(p, ro, pp_digest, U2):
    ro.absorb(pp_digest)
    absorb_r1cs_instance(ro, U2)
    return ro.squeeze(NUM_CHALLENGE_BITS, False)


def _finish(p, ro, poly, rho):
    for c in poly:
        ro.absorb(c)
    r_b = ro.squeeze(NUM_CHALLENGE_BITS, False)
    eq_rho_r_b = ((1 - rho) * (1 - r_b) + rho * r_b) % p
    if eq_rho_r_b == 0:
        raise ZeroDivisionError("eq(rho, r_b) is zero (nifs.rs:282 unwrap)")
    return r_b, uni_eval(p, poly, r_b) * pow(eq_rho_r_b, -1, p) % p


def nifs_prove(ck, ro, pp_digest, st, U1, W1, U2, W2, r_E, sums=None):
    """NIFS::prove with the blind r_E supplied.  `sums(e1, Az1, Bz1, Cz1, e2, Az2, Bz2, Cz2)` may replace the
    literal prove_helper_raw (e.g. by evals_raw).  -> (NIFS, (U, W))"""
    S = st.S
    fid, cid = S.fid, ck[0]
    p = FIELD_MODULUS[fid]
    if len(U1.X) != S.num_io or len(U2.X) != S.num_io or len(W2.W) != S.num_vars:
        raise ValueError("InvalidInputLength")
    tau = _challenges_after_E(p, ro, pp_digest, U2)
    E = split_evals(p, tau, st.left, st.right)
    comm_E = commit(ck, fid, E, r_E)
    absorb_commitment(ro, comm_E)
    rho = ro.squeeze(NUM_CHALLENGE_BITS, False)
    T = (1 - rho) * U1.T % p
    Az1, Bz1, Cz1 = multiply_vec(S, W1.W + [U1.u] + U1.X)
    Az2, Bz2, Cz2 = multiply_vec(S, W2.W + [1] + U2.X)
    raw = (sums or (lambda *v: prove_helper_raw(p, st.left, st.right, *v)))(W1.E, Az1, Bz1, Cz1, E, Az2, Bz2, Cz2)
    e0, e2, e3, e4, e5 = [s * f % p for s, f in zip(raw, rho_factors(p, rho))]
    poly = from_evals(p, [e0, (T - e0) % p, e2, e3, e4, e5])
    r_b, T_out = _finish(p, ro, poly, rho)
    U = U1.fold(cid, p, U2, comm_E, r_b, T_out)
    W = W1.fold(p, W2, E, r_E, r_b)
    return NIFS(comm_E, poly), (U, W)


def nifs_verify(cid, p, nifs, ro, pp_digest, U1, U2):
    """NIFS::verify -> the folded instance, or None where the reference returns InvalidSumcheckProof"""
    _challenges_after_E(p, ro, pp_digest, U2)
    absorb_commitment(ro, nifs.comm_E)
    rho = ro.squeeze(NUM_CHALLENGE_BITS, False)
    T = (1 - rho) * U1.T % p
    if (nifs.poly[0] + sum(nifs.poly)) % p != T:
        return None
    r_b, T_out = _finish(p, ro, nifs.poly, rho)
    return U1.fold(cid, p, U2, nifs.comm_E, r_b, T_out)


def is_sat_sum(st, U, W):
    """sum_k E2[i] E1[j] (Az Bz - Cz) of Structure::is_sat (literal outer product)"""
    p = FIELD_MODULUS[st.S.fid]
    Az, Bz, Cz = multiply_vec(st.S, W.W + [U.u] + U.X)
    E1, E2 = W.E[:st.left], W.E[st.left:]
    return sum(E2[i] * E1[j] * (Az[i * st.left + j] * Bz[i * st.left + j] - Cz[i * st.left + j])
               for i in range(st.right) for j in range(st.left)) % p


def is_sat(ck, st, U, W, sat_sum=None):
    """Structure::is_sat: the sum equals U.T and both commitments open"""
    fid = st.S.fid
    s = is_sat_sum(st, U, W) if sat_sum is None else sat_sum
    if s != U.T:
        return False
    return commit(ck, fid, W.W, W.r_W) == U.comm_W and commit(ck, fid, W.E, W.r_E) == U.comm_E
