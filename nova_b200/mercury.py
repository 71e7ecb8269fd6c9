"""Host-side mirror of the Mercury evaluation engine (src/provider/mercury.rs), EvaluationEngine::prove
(:891-1268) with the BDFG20 batch opening generate_batch_evaluate_arg (:567-770), on BN254 with the HyperKZG
commitment key (Mercury reuses hyperkzg::setup, :884-888).

Every O(n) and O(b^2) step runs on the device and the polynomials never leave HBM:

  eq_row, eq_col = EqPolynomial(u_row / u_col).evals()       :937-938     b200_eq_table_dev
  h = compute_h_poly(f, eq_col)                               :966         b200_mat_vec_rows_dev
  (q, g) = divide_by_binomial(f, b_row, b, alpha)             :995         b200_div_binomial_dev
  s = make_s_polynomial((eq_col, eq_row), (g, h), gamma)      :1072-1077   b200_mercury_s_poly_dev
  d = rev(g)                                                  :1113-1120   b200_gather_dev
  g, h, s, d at zeta, 1/zeta, alpha                           :1136-1159   b200_poly_eval_many_dev (one launch)
  quot_f = (f - (zeta^b - alpha) q - g(zeta)) / (X - zeta)    :1163-1180   b200_rlc_dev + b200_poly_div_dev
  W, W' of the batch opening                                  :619-764     b200_rlc_dev + b200_poly_div_dev
  the eight commitments                                                    b200_commit_many_dev

W = m / Z_T is the unique polynomial with m = Z_T W, so it is computed term by term instead of through
multiply_by_linear_polynomial: with [P / D] the quotient of P by D (remainder dropped, which is linear in P),
    W = [([beta [h / (X - alpha)] + g + beta^2 s] / (X - 1/zeta)) + beta^3 d] / (X - zeta),
because g - g*, s - s* vanish at {zeta, 1/zeta}, h - h* at {zeta, 1/zeta, alpha} and d - d* at zeta, and the
interpolants g*, h*, s*, d* only ever change remainders.  For the same reason W' = [L / (X - z)] with
L = (z - alpha) g + beta h + beta^2 (z - alpha) s + beta^3 (z - alpha)(z - 1/zeta) d - Z_T(z) W: the constant
terms of m_z do not reach the quotient.  The host receives the eight commitments and the scalars it absorbs
and keeps only O(1) algebra on Python integers (zeta^b, the beta powers, Z_T(z)).
"""
from __future__ import annotations

import ctypes
from collections import namedtuple

from . import fields
from .native import c_size_t, check, lib
from .provider import CommitmentKey, Curve
from .spartan import DeviceVec, _commitment_bytes, commit_many_dev

EvaluationArgument = namedtuple("EvaluationArgument", [
    "comm_h", "comm_g", "comm_q", "comm_s", "comm_d", "comm_quot_f", "comm_w", "comm_w_prime",
    "g_zeta", "g_zeta_inv", "h_zeta", "h_zeta_inv", "s_zeta", "s_zeta_inv"])


def _resolve(ch, *msgs):
    return ch(*msgs) if callable(ch) else ch


def mercury_prove_resident(curve, ck: CommitmentKey, P, x: list, alpha, gamma, zeta, beta, z,
                           timings: dict | None = None, on_w_prime=None) -> EvaluationArgument:
    """EvaluationEngine::prove after the absorption of (comm_f, point, eval), on a polynomial in HBM
    (`P`: DeviceVec or Montgomery bytes of 2^ell coefficients).  The challenges are integers or callables that
    derive them from the messages sent so far, in the reference's transcript order:
        alpha(comm_h), gamma(comm_q, comm_g), zeta(comm_s, comm_d),
        beta(g_zeta, g_zeta_inv, h_zeta, h_zeta_inv, s_zeta, s_zeta_inv, comm_quot_f), z(comm_w);
    `on_w_prime(comm_w_prime)` sees the last message.  `timings` (optional) receives seconds per phase; the
    challenge callables (the host transcript) are timed as the phase "transcript".
    Raises ValueError for ell <= 1 (:914) or a polynomial that does not have 2^ell coefficients."""
    import time
    curve = Curve(curve)
    fid = curve.scalar_field
    p = fields.MODULUS[fid]
    ell = len(x)
    if ell <= 1:
        raise ValueError("Mercury needs at least two variables (mercury.rs:914)")
    n = 1 << ell
    if isinstance(P, (bytes, bytearray)):
        if len(P) != 32 * n:
            raise ValueError(f"polynomial has {len(P) // 32} coefficients, the point {ell} variables")
        P = DeviceVec.from_bytes(bytes(P))
    elif P.nbytes != 32 * n:
        raise ValueError(f"polynomial has {P.nbytes // 32} coefficients, the point {ell} variables")
    L = lib()
    t_last = [time.perf_counter()]

    def mark(name):
        if timings is not None:
            check(L.b200_sync())
            now = time.perf_counter()
            timings[name] = timings.get(name, 0.0) + now - t_last[0]
            t_last[0] = now

    def scalar(v):
        return DeviceVec.from_bytes(fields.to_mont_bytes(fid, v % p))

    keep = []  # device scalars / tables the queued launches read

    def rlc(polys, lens, coeffs, out_len):
        k = len(polys)
        cd = DeviceVec.from_bytes(fields.pack(fid, [c_ % p for c_ in coeffs]))
        keep.append(cd)
        out = DeviceVec(32 * out_len)
        check(L.b200_rlc_dev(fid, (ctypes.c_void_p * k)(*[v.ptr.value for v in polys]), (c_size_t * k)(*lens), k,
                             cd.ptr, out_len, out.ptr, None))
        return out

    def div(f, length, u):
        ud = scalar(u)
        keep.append(ud)
        out = DeviceVec(32 * (length - 1))
        check(L.b200_poly_div_dev(fid, f.ptr, length, ud.ptr, out.ptr, None))
        return out

    # the odd-ell padding (:911-933): the point gets a leading 0; f itself is not copied, only its first
    # b_row = n / b rows are non-zero
    point = [0] + list(x) if ell % 2 else list(x)
    log_b = len(point) // 2
    b = 1 << log_b
    b_row = n // b
    eq_row, eq_col = DeviceVec(32 * b), DeviceVec(32 * b)
    for u, out in ((point[:log_b], eq_row), (point[log_b:], eq_col)):
        ud = DeviceVec.from_bytes(fields.pack(fid, [v % p for v in u]))
        keep.append(ud)
        check(L.b200_eq_table_dev(fid, ud.ptr, log_b, out.ptr, None))
    h = DeviceVec(32 * b)
    if b_row < b:  # h padded to b (:967-970)
        check(L.b200_memset_dev(ctypes.c_void_p(h.ptr.value + 32 * b_row), 0, 32 * (b - b_row), None))
    check(L.b200_mat_vec_rows_dev(fid, P.ptr, b_row, b, eq_col.ptr, h.ptr, None))
    mark("h")
    comm_h, = commit_many_dev(curve, ck, [h], [b])
    mark("commit_h")
    alpha = _resolve(alpha, comm_h) % p
    mark("transcript")
    nq = (b_row - 1) * b
    q, g = DeviceVec(32 * max(nq, 1)), DeviceVec(32 * b)
    ad = scalar(alpha)
    check(L.b200_div_binomial_dev(fid, P.ptr, b_row, b, ad.ptr, q.ptr, g.ptr, None))
    mark("div_binomial")
    comm_q, comm_g = commit_many_dev(curve, ck, [q, g], [nq, b])
    mark("commit_q_g")
    gamma = _resolve(gamma, comm_q, comm_g) % p
    mark("transcript")
    s = DeviceVec(32 * (b - 1))
    gd = scalar(gamma)
    check(L.b200_mercury_s_poly_dev(fid, eq_col.ptr, g.ptr, eq_row.ptr, h.ptr, b, gd.ptr, s.ptr, None))
    d = DeviceVec(32 * b)
    rev = DeviceVec.from_bytes(bytes((ctypes.c_uint32 * b)(*range(b - 1, -1, -1))))
    check(L.b200_gather_dev(g.ptr, rev.ptr, b, d.ptr, None))
    mark("s_d")
    comm_s, comm_d = commit_many_dev(curve, ck, [s, d], [b - 1, b])
    mark("commit_s_d")
    zeta = _resolve(zeta, comm_s, comm_d) % p
    mark("transcript")
    zeta_inv = pow(zeta, -1, p)  # zeta.invert().unwrap() (:1134): zero with negligible probability
    us = DeviceVec.from_bytes(fields.pack(fid, [zeta, zeta_inv, alpha]))
    ev = DeviceVec(32 * 12)
    polys = [g, h, s, d]
    check(L.b200_poly_eval_many_dev(fid, (ctypes.c_void_p * 4)(*[v.ptr.value for v in polys]),
                                    (c_size_t * 4)(b, b, b - 1, b), 4, us.ptr, 3, ev.ptr, None))
    e = fields.unpack(fid, ev.to_bytes(32 * 12))
    g_zeta, g_zeta_inv = e[0], e[1]
    h_zeta, h_zeta_inv, h_alpha = e[3], e[4], e[5]
    s_zeta, s_zeta_inv = e[6], e[7]
    mark("evals")
    # quot_f = (f - (zeta^b - alpha) q - g(zeta)) / (X - zeta)  (:1163-1180): n - 1 coefficients
    gz = scalar(g_zeta)
    num = rlc([P, q, gz], [n, nq, 1], [1, -(pow(zeta, b, p) - alpha), -1], n)
    quot_f = div(num, n, zeta)
    del num
    mark("quot_f")
    comm_quot_f, = commit_many_dev(curve, ck, [quot_f], [n - 1])
    mark("commit_quot_f")
    del quot_f
    beta = _resolve(beta, g_zeta, g_zeta_inv, h_zeta, h_zeta_inv, s_zeta, s_zeta_inv, comm_quot_f) % p
    mark("transcript")
    beta2 = beta * beta % p
    beta3 = beta2 * beta % p
    t = rlc([div(h, b, alpha), g, s], [b - 1, b, b - 1], [beta, 1, beta2], b)
    w = div(rlc([div(t, b, zeta_inv), d], [b - 1, b], [1, beta3], b), b, zeta)
    mark("batch_w")
    comm_w, = commit_many_dev(curve, ck, [w], [b - 1])
    mark("commit_w")
    z = _resolve(z, comm_w) % p
    mark("transcript")
    t_s1 = (z - alpha) % p
    t_s4 = t_s1 * (z - zeta_inv) % p
    t_z = t_s4 * (z - zeta) % p
    w_prime = div(rlc([g, h, s, d, w], [b, b, b - 1, b, b - 1],
                      [t_s1, beta, beta2 * t_s1, beta3 * t_s4, -t_z], b), b, z)
    mark("batch_w_prime")
    comm_w_prime, = commit_many_dev(curve, ck, [w_prime], [b - 1])
    mark("commit_w_prime")
    if on_w_prime is not None:
        on_w_prime(comm_w_prime)
        mark("transcript")
    del keep, h_alpha
    return EvaluationArgument(comm_h, comm_g, comm_q, comm_s, comm_d, comm_quot_f, comm_w, comm_w_prime,
                              g_zeta, g_zeta_inv, h_zeta, h_zeta_inv, s_zeta, s_zeta_inv)


def mercury_prove(curve, ck: CommitmentKey, P, x: list, transcript, timings: dict | None = None,
                  comm=None, eval_: int | None = None) -> EvaluationArgument:
    """EvaluationEngine::prove (mercury.rs:891-1268) with the transcript: absorbs comm_f, the point and the
    evaluation, derives alpha, gamma, zeta, beta, z from the messages in the reference's order and squeezes
    `pd` after absorbing comm_w_prime, so the transcript ends in the verifier's final state.
    `comm` / `eval_`: the commitment to P and the claimed evaluation P(x) (the caller's instance, as the
    reference receives them); when omitted they are computed from P (a commitment without blinding)."""
    curve = Curve(curve)
    fid = curve.scalar_field
    p = fields.MODULUS[fid]
    ell = len(x)
    if ell <= 1:
        raise ValueError("Mercury needs at least two variables (mercury.rs:914)")
    n = 1 << ell
    if isinstance(P, (bytes, bytearray)):
        if len(P) != 32 * n:
            raise ValueError(f"polynomial has {len(P) // 32} coefficients, the point {ell} variables")
        P = DeviceVec.from_bytes(bytes(P))
    elif P.nbytes != 32 * n:
        raise ValueError(f"polynomial has {P.nbytes // 32} coefficients, the point {ell} variables")
    if comm is None:
        comm, = commit_many_dev(curve, ck, [P], [n])
    if eval_ is None:
        from .spartan import mle_eval_multi_dev
        xd = DeviceVec.from_bytes(fields.pack(fid, [v % p for v in x]))
        eval_, = mle_eval_multi_dev(fid, [P], ell, xd)
    tr = transcript
    rep = lambda vs: b"".join(int(v % p).to_bytes(32, "little") for v in vs)
    tr.absorb_bytes(b"f", _commitment_bytes(comm))
    tr.absorb_bytes(b"u", rep(x))
    tr.absorb_bytes(b"e", rep([eval_]))

    def alpha(comm_h):
        tr.absorb_bytes(b"h", _commitment_bytes(comm_h))
        return tr.squeeze(b"a")

    def gamma(comm_q, comm_g):
        tr.absorb_bytes(b"q", _commitment_bytes(comm_q))
        tr.absorb_bytes(b"g", _commitment_bytes(comm_g))
        return tr.squeeze(b"gm")

    def zeta(comm_s, comm_d):
        tr.absorb_bytes(b"s", _commitment_bytes(comm_s))
        tr.absorb_bytes(b"d", _commitment_bytes(comm_d))
        return tr.squeeze(b"zt")

    def beta(gz, gzi, hz, hzi, sz, szi, comm_quot_f):
        for label, v in ((b"gz", gz), (b"gzi", gzi), (b"hz", hz), (b"hzi", hzi), (b"sz", sz), (b"szi", szi)):
            tr.absorb_bytes(label, rep([v]))
        tr.absorb_bytes(b"t", _commitment_bytes(comm_quot_f))
        return tr.squeeze(b"b")

    def z(comm_w):
        tr.absorb_bytes(b"w", _commitment_bytes(comm_w))
        return tr.squeeze(b"z")

    def after(comm_w_prime):
        tr.absorb_bytes(b"wp", _commitment_bytes(comm_w_prime))
        tr.squeeze(b"pd")
    return mercury_prove_resident(curve, ck, P, x, alpha, gamma, zeta, beta, z, timings, after)
