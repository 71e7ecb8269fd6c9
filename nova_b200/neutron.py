"""Device-resident mirror of NeutronNova's folding scheme (src/neutron/, `feature = "experimental"`):

  Structure::new / is_sat                    neutron/relation.rs:52-116
  FoldedInstance / FoldedWitness (+ fold)    neutron/relation.rs:119-198
  NIFS::prove / NIFS::verify                 neutron/nifs.rs:200-343

One fold keeps every vector of size n in HBM:  z1, z2 -> 6 SpMVs -> the five sums of prove_helper in one pass
(b200_neutron_evals_dev) -> two witness folds (b200_lerp_dev).  The power polynomial's split table E
(b200_pow_split_evals_dev, left + right ~ 2 sqrt(n) entries) is the only vector that is committed, so a fold has no
n-point MSM.  The host reads back the five sums and comm_E and keeps the O(1) algebra: the random oracle (RO2 over
the scalar field, passed in), the rho factors, the degree-5 interpolation, T_out, and the instance fold.
"""
from __future__ import annotations

import time
from collections import namedtuple
from dataclasses import dataclass

from . import fields
from .native import check, lib
from .ppsnark import dev_scalar, dev_zeros
from .provider import Curve
from .r1cs import R1CSShape, _lincomb
from .spartan import DeviceVec, UniPoly

NUM_CHALLENGE_BITS = 128               # constants.rs:4
BN_LIMB_WIDTH, BN_N_LIMBS = 64, 4      # constants.rs:10-13

NIFS = namedtuple("NIFS", ["comm_E", "poly"])  # nifs.rs:21-24 (poly: the six coefficients, lowest first)


def absorb_commitment(ro, P):
    """Commitment::absorb_in_ro2 (pedersen.rs:141-156): x and y as BN_N_LIMBS limbs of BN_LIMB_WIDTH bits
    (to_bignat_repr, gadgets/utils.rs:107), then the infinity flag; the identity (None) is (0, 0, true)."""
    x, y, inf = (0, 0, 1) if P is None else (P[0], P[1], 0)
    mask = (1 << BN_LIMB_WIDTH) - 1
    for c in (x, y):
        for k in range(BN_N_LIMBS):
            ro.absorb((c >> (BN_LIMB_WIDTH * k)) & mask)
    ro.absorb(inf)


def _absorb_instance(ro, U2):
    """R1CSInstance::absorb_in_ro2 (r1cs/mod.rs:967-975)"""
    absorb_commitment(ro, U2.comm_W)
    for x in U2.X:
        ro.absorb(x)


def _pow2(n: int) -> bool:
    return n > 0 and n & (n - 1) == 0


class Structure:
    """Structure::new (relation.rs:52-68) over a device-resident r1cs.R1CSShape: n = num_cons = 2^ell rows split
    as left = 2^ceil(ell/2), right = 2^floor(ell/2).  The reference pads the shape first; padding is a host CSR
    transformation that is not done here, so the shape must already be regular (R1CSShape::is_regular_shape,
    r1cs/mod.rs:399-404: num_cons and num_vars powers of two, num_io < num_vars), which is what pad() returns.
    ell must be at least 2: for ell <= 1, right = 1 and the reference's split_evals panics."""

    def __init__(self, S: R1CSShape):
        if not (_pow2(S.num_cons) and _pow2(S.num_vars) and S.num_io < S.num_vars):
            raise ValueError(f"shape is not regular (num_cons {S.num_cons}, num_vars {S.num_vars}, "
                             f"num_io {S.num_io}): pad it first (R1CSShape::pad)")
        self.S = S
        self.ell = S.num_cons.bit_length() - 1
        if self.ell < 2:
            raise ValueError(f"a structure needs at least 4 constraints, got {S.num_cons}")
        self.left, self.right = 1 << ((self.ell + 1) // 2), 1 << (self.ell // 2)

    @property
    def fid(self) -> int:
        return self.S.fid


@dataclass
class FoldedInstance:          # relation.rs:42-48
    comm_W: tuple | None
    comm_E: tuple | None
    T: int
    u: int
    X: list

    @classmethod
    def default(cls, S: Structure):  # relation.rs:161-169
        return cls(None, None, 0, 0, [0] * S.S.num_io)


@dataclass
class FoldedWitness:           # relation.rs:29-37
    W: DeviceVec
    r_W: int
    E: DeviceVec
    r_E: int

    @classmethod
    def default(cls, S: Structure):  # relation.rs:121-128
        return cls(dev_zeros(S.S.num_vars), 0, dev_zeros(S.left + S.right), 0)


def _nbytes(v):
    return getattr(v, "nbytes", None)


def _check_sizes(S: Structure, U1, W1, U2, W2):
    """the reference's length checks (prove_helper's asserts, multiply_vec's InvalidWitnessLength)"""
    sh = S.S
    if len(U1.X) != sh.num_io or len(U2.X) != sh.num_io:
        raise ValueError("InvalidInputLength")
    for v, n in ((W1.W, sh.num_vars), (W1.E, S.left + S.right), (W2.W, sh.num_vars)):
        if _nbytes(v) is not None and _nbytes(v) != 32 * n:
            raise ValueError(f"InvalidWitnessLength: a vector of {_nbytes(v) // 32} entries where {n} are needed")


def rho_factors(p: int, rho: int) -> list:
    """the common factors of prove_helper (nifs.rs:172-185): (1 - rho), (3 rho - 1), (5 rho - 2), (7 rho - 3),
    (9 rho - 4) for the evaluations at 0, 2, 3, 4, 5"""
    return [(1 - rho) % p, (3 * rho - 1) % p, (5 * rho - 2) % p, (7 * rho - 3) % p, (9 * rho - 4) % p]


def _evals_dev(S: Structure, e1, abc1, e2, abc2) -> list:
    """the five raw sums of prove_helper (before the rho factors) on resident vectors"""
    out = DeviceVec(32 * 5)
    check(lib().b200_neutron_evals_dev(S.fid, e1.ptr, *(v.ptr for v in abc1), e2.ptr, *(v.ptr for v in abc2),
                                       S.left, S.right, out.ptr, None))
    return fields.unpack(S.fid, out.to_bytes(32 * 5))


def _t_out(p: int, poly: UniPoly, rho: int, r_b: int) -> int:
    """poly(r_b) / ((1 - rho)(1 - r_b) + rho r_b); the reference unwraps the inverse (nifs.rs:281-282)"""
    eq_rho_r_b = ((1 - rho) * (1 - r_b) + rho * r_b) % p
    if eq_rho_r_b == 0:
        raise ValueError("eq(rho, r_b) is zero: T_out is undefined (nifs.rs:282)")
    return poly.evaluate(r_b) * pow(eq_rho_r_b, -1, p) % p


def fold_instance(curve, U1: FoldedInstance, U2, comm_E, r_b: int, T_out: int) -> FoldedInstance:
    """FoldedInstance::fold (relation.rs:172-197): every field becomes (1 - r_b) old + r_b new, u = (1 - r_b) u1 + r_b"""
    curve = Curve(curve)
    p = fields.MODULUS[curve.scalar_field]
    one_m = (1 - r_b) % p
    return FoldedInstance(_lincomb(curve, [(one_m, U1.comm_W), (r_b, U2.comm_W)]),
                          _lincomb(curve, [(one_m, U1.comm_E), (r_b, comm_E)]), T_out % p,
                          (one_m * U1.u + r_b) % p, [(one_m * a + r_b * b) % p for a, b in zip(U1.X, U2.X)])


def fold_witness(S: Structure, W1: FoldedWitness, W2, E: DeviceVec, r_E: int, r_b: int) -> FoldedWitness:
    """FoldedWitness::fold (relation.rs:131-156): W1 + r_b (W2 - W1), E1 + r_b (E - E1) on the device, blinds on the
    host.  Writes new vectors: W1 is left as it is."""
    fid, p = S.fid, fields.MODULUS[S.fid]
    L = lib()
    rd = dev_scalar(fid, r_b)
    nv, ne = S.S.num_vars, S.left + S.right
    W, E_out = DeviceVec(32 * nv), DeviceVec(32 * ne)
    check(L.b200_lerp_dev(fid, W1.W.ptr, W2.W.ptr, rd.ptr, nv, W.ptr, None))
    check(L.b200_lerp_dev(fid, W1.E.ptr, E.ptr, rd.ptr, ne, E_out.ptr, None))
    check(L.b200_sync())  # rd must outlive the launches
    one_m = (1 - r_b) % p
    return FoldedWitness(W, (one_m * W1.r_W + r_b * W2.r_W) % p, E_out, (one_m * W1.r_E + r_b * r_E) % p)


def nifs_prove(ck, ro, pp_digest: int, S: Structure, U1: FoldedInstance, W1: FoldedWitness, U2, W2, r_E: int,
               timings: dict | None = None):
    """NIFS::prove (nifs.rs:200-289).  `ro`: a fresh RO2 over the scalar field (absorb(int) /
    squeeze(num_bits, start_with_one)), e.g. poseidon.PoseidonRO(scalar field).  U2, W2: r1cs.R1CSInstance /
    R1CSWitness with W2.W resident.  r_E: the blind of comm_E (random in the reference).
    `timings` (optional) receives seconds per phase: "E_comm_E", "spmv", "evals", "folds", "host_ro" (the random
    oracle and the O(1) algebra).  -> (NIFS(comm_E, poly), (U, W)).
    Raises ValueError on a length mismatch or a zero denominator for T_out, where the reference panics."""
    sh = S.S
    fid, p = S.fid, fields.MODULUS[S.fid]
    _check_sizes(S, U1, W1, U2, W2)
    L = lib()
    t_last = [time.perf_counter()]

    def mark(name):
        if timings is not None:
            check(L.b200_sync())
            now = time.perf_counter()
            timings[name] = timings.get(name, 0.0) + now - t_last[0]
            t_last[0] = now

    ro.absorb(pp_digest)
    _absorb_instance(ro, U2)
    tau = ro.squeeze(NUM_CHALLENGE_BITS, False)
    mark("host_ro")
    ne = S.left + S.right
    E = DeviceVec(32 * ne)
    tau_d = dev_scalar(fid, tau)
    check(L.b200_pow_split_evals_dev(fid, tau_d.ptr, S.left, S.right, E.ptr, None))
    comm_E = sh._commit(ck, E, ne, r_E)  # reads the commitment back: tau_d is no longer needed
    mark("E_comm_E")
    absorb_commitment(ro, comm_E)
    rho = ro.squeeze(NUM_CHALLENGE_BITS, False)
    T = (1 - rho) * U1.T % p
    mark("host_ro")
    z1, z2 = sh._z(W1.W, U1.u, U1.X), sh._z(W2.W, 1, U2.X)
    abc1, abc2 = sh.multiply_vec_dev(z1), sh.multiply_vec_dev(z2)
    mark("spmv")
    raw = _evals_dev(S, W1.E, abc1, E, abc2)
    del z1, z2, abc1, abc2  # the read-back above synchronised
    mark("evals")
    e0, e2, e3, e4, e5 = (s * f % p for s, f in zip(raw, rho_factors(p, rho)))
    poly = UniPoly.from_evals(p, [e0, (T - e0) % p, e2, e3, e4, e5])
    for c in poly.coeffs:
        ro.absorb(c)
    r_b = ro.squeeze(NUM_CHALLENGE_BITS, False)
    T_out = _t_out(p, poly, rho, r_b)
    mark("host_ro")
    W = fold_witness(S, W1, W2, E, r_E, r_b)
    mark("folds")
    U = fold_instance(sh.curve, U1, U2, comm_E, r_b, T_out)
    mark("host_ro")
    return NIFS(comm_E, list(poly.coeffs)), (U, W)


def verify(curve, ro, pp_digest: int, nifs: NIFS, U1: FoldedInstance, U2) -> FoldedInstance:
    """NIFS::verify (nifs.rs:297-343): O(1) work on the instances.  Raises ValueError("InvalidSumcheckProof") when
    poly(0) + poly(1) != (1 - rho) U1.T."""
    p = fields.MODULUS[Curve(curve).scalar_field]
    ro.absorb(pp_digest)
    _absorb_instance(ro, U2)
    ro.squeeze(NUM_CHALLENGE_BITS, False)  # tau
    absorb_commitment(ro, nifs.comm_E)
    rho = ro.squeeze(NUM_CHALLENGE_BITS, False)
    T = (1 - rho) * U1.T % p
    poly = UniPoly(p, nifs.poly)
    if (poly.coeffs[0] + sum(poly.coeffs)) % p != T:
        raise ValueError("InvalidSumcheckProof")
    for c in poly.coeffs:
        ro.absorb(c)
    r_b = ro.squeeze(NUM_CHALLENGE_BITS, False)
    return fold_instance(curve, U1, U2, nifs.comm_E, r_b, _t_out(p, poly, rho, r_b))


def is_sat_sum(S: Structure, U: FoldedInstance, W: FoldedWitness) -> int:
    """sum_k E2[i] E1[j] (Az Bz - Cz)[k] of Structure::is_sat: the evals pass with both instances equal
    (every one of its five sums is this one)."""
    sh = S.S
    z = sh._z(W.W, U.u, U.X)
    abc = sh.multiply_vec_dev(z)
    return _evals_dev(S, W.E, abc, W.E, abc)[0]


def is_sat(ck, S: Structure, U: FoldedInstance, W: FoldedWitness) -> bool:
    """Structure::is_sat (relation.rs:71-116): the sum equals U.T and both commitments open."""
    sh = S.S
    if len(U.X) != sh.num_io:
        raise ValueError("InvalidInputLength")
    if is_sat_sum(S, U, W) != U.T:
        return False
    return (sh._commit(ck, W.W, sh.num_vars, W.r_W) == U.comm_W
            and sh._commit(ck, W.E, S.left + S.right, W.r_E) == U.comm_E)
