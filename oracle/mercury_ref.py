"""CPU restatement of the Mercury evaluation argument (src/provider/mercury.rs) on top of the C oracle's
field passes and MSM.  TEST INFRASTRUCTURE ONLY.

prove  = EvaluationEngine::prove (mercury.rs:891-1268) incl. the BDFG20 batch opening
         generate_batch_evaluate_arg (:567-770), written in the reference's own order of operations:
         odd-ell padding, compute_h_poly, divide_by_binomial (per column, expand, transpose, trim),
         make_s_polynomial by forward NTT / pointwise combination / X^(b-1) twist / inverse NTT / trim /
         drop the low b coefficients, the evaluations, quot_f, and m(X) built with from_evals_with_xs,
         batch_add_with_polynomials, multiply_by_linear_polynomial and three divisions.
verify = EvaluationEngine::verify (:1270-1486) with extract_pairing_to_verify_batch_evaluation (:773-871);
         the final pairing check e(ll, [1]_2) = e(rl, [tau]_2) is replaced by the equivalent group
         equation  ll = [tau] rl,  which a TEST setup can evaluate because it knows tau (as in
         oracle/hyperkzg_ref.py).

A note on the root of unity.  s is a fixed polynomial: s[k] is the coefficient of X^(k+1), k < b-1, of the
Laurent polynomial  a1(X) b1(1/X) + a1(1/X) b1(X) + gamma (a2(X) b2(1/X) + a2(1/X) b2(X)).  The NTT of size 2b
only evaluates and re-interpolates the degree < 2b polynomial X^(b-1) * (that Laurent polynomial), so ANY
primitive 2b-th root of unity gives the same coefficients; the reference's choice of `ROOT_OF_UNITY` (a
constant of its field crate) changes no proof byte.  This module derives its own root from the field's
2-adicity, and `s_poly_direct` states the lag formula the device computes; the tests check that they agree.

The prover restatement is pinned by the verifier restatement: an honest proof must pass and a proof with
any of its 14 fields (or the claimed evaluation) altered must fail (tests/test_oracle_mercury.py).
"""
from . import coracle as co
from .pyref import CURVES, commitment_transcript_bytes, eq_evals, from_mont_bytes, mle_evaluate, mont_bytes, to_repr

FIELDS = ("comm_h", "comm_g", "comm_q", "comm_s", "comm_d", "comm_quot_f", "comm_w", "comm_w_prime",
          "g_zeta", "g_zeta_inv", "h_zeta", "h_zeta_inv", "s_zeta", "s_zeta_inv")


def _pack(p, xs):
    return b"".join(mont_bytes(p, x) for x in xs)


def _ints(p, b):
    return [from_mont_bytes(p, b[i:i + 32]) for i in range(0, len(b), 32)]


# ---- UniPoly helpers (mercury.rs:191-313) -------------------------------------------------------------
def evaluate(p, coeffs, r):
    acc = 0
    for c in reversed(coeffs):
        acc = (acc * r + c) % p
    return acc


def trim(coeffs):
    c = list(coeffs)
    while c and c[-1] == 0:
        c.pop()
    return c


def divide_by_linear_polynomial(p, coeffs, a):
    """f / (X - a) by Horner (:281-288) -> (quotient, remainder)."""
    c = list(coeffs)
    for i in range(len(c) - 2, -1, -1):
        c[i] = (c[i] + c[i + 1] * a) % p
    return c[1:], c[0]


def multiply_by_linear_polynomial(p, coeffs, a):
    """f(X) * (X + a) (:264-276)."""
    a_f = [x * a % p for x in coeffs]
    c = [0] + list(coeffs)
    for i in range(len(coeffs)):
        c[i] = (c[i] + a_f[i]) % p
    return c


def batch_add_with_polynomials(p, coeffs, polys, scalars):
    """coeffs += sum_k scalars[k] * polys[k] (:239-261)."""
    n = max(len(coeffs), max(len(q) for q in polys))
    c = list(coeffs) + [0] * (n - len(coeffs))
    for q, s in zip(polys, scalars):
        for i, x in enumerate(q):
            c[i] = (c[i] + s * x) % p
    return c


def gaussian_elimination(p, m):
    """Solve the n x (n+1) augmented system (spartan/polys/univariate.rs gaussian_elimination)."""
    n = len(m)
    m = [list(r) for r in m]
    for i in range(n):
        piv = next(k for k in range(i, n) if m[k][i] % p)
        m[i], m[piv] = m[piv], m[i]
        inv = pow(m[i][i], -1, p)
        m[i] = [x * inv % p for x in m[i]]
        for k in range(n):
            if k != i and m[k][i]:
                f = m[k][i]
                m[k] = [(x - f * y) % p for x, y in zip(m[k], m[i])]
    return [m[i][n] for i in range(n)]


def from_evals_with_xs(p, xs, evals):
    """The interpolant of degree < len(xs) (:205-230)."""
    if len(evals) == 1:
        return [evals[0] % p]
    rows = []
    for x, e in zip(xs, evals):
        row = [1, x % p]
        for _ in range(2, len(xs)):
            row.append(row[-1] * x % p)
        rows.append(row + [e % p])
    return gaussian_elimination(p, rows)


def eval_pu_poly(p, u, r):
    """eq(r) as a univariate polynomial evaluated at r: prod_i (u_i r^(2^i) + 1 - u_i), u reversed (:359-365)."""
    res = 1
    for i, ui in enumerate(reversed(u)):
        res = res * (ui * pow(r, 1 << i, p) + 1 - ui) % p
    return res


# ---- the pieces the device computes ----------------------------------------------------------------------
def compute_h_poly(p, f, eq_col, rows, cols):
    """:369-386"""
    return [sum(f[r * cols + c] * eq_col[c] for c in range(cols)) % p for r in range(rows)]


def divide_by_binomial(p, f, rows, cols, alpha):
    """f / (X^cols - alpha) (:319-356): each column divided by (Y - alpha), the per-column quotients expanded
    to `cols` entries, flattened column-major and transposed -> (quotient, remainder g)."""
    quotients, remainder = [], []
    for col in range(cols):
        column = f[col::cols]
        assert len(column) == rows
        q, r = divide_by_linear_polynomial(p, column, alpha)
        quotients.append(q + [0] * (cols - len(q)))
        remainder.append(r)
    flat = [x for q in quotients for x in q]
    flat += [0] * (cols * cols - len(flat))  # transpose (:291-312) expands to b * b first
    transposed = [flat[r * cols + c] for c in range(cols) for r in range(cols)]
    return transposed, remainder


def divide_columns(p, f, rows, cols, alpha):
    """The same division for any shape (the reference's transpose needs rows <= cols): -> (q, g) with
    q[r * cols + c], r < rows - 1, the quotient of column c and g[c] its remainder, column c at alpha."""
    q = [0] * ((rows - 1) * cols)
    g = []
    for col in range(cols):
        quot, rem = divide_by_linear_polynomial(p, f[col::cols], alpha)
        q[col::cols] = quot
        g.append(rem)
    return q, g


def root_of_unity(p, order):
    """A primitive `order`-th root of unity (order a power of two dividing p - 1)."""
    s = ((p - 1) & -(p - 1)).bit_length() - 1
    assert order & (order - 1) == 0 and order.bit_length() - 1 <= s
    g = 2
    while pow(g, (p - 1) // 2, p) == 1:  # a quadratic non-residue generates the whole 2-Sylow subgroup
        g += 1
    return pow(g, (p - 1) // order, p)


def ntt(p, a, w):
    """a_k -> sum_j a_j w^(jk), len(a) a power of two (halo2curves best_fft computes the same transform)."""
    n = len(a)
    if n == 1:
        return list(a)
    even, odd = ntt(p, a[0::2], w * w % p), ntt(p, a[1::2], w * w % p)
    out, t = [0] * n, 1
    for k in range(n // 2):
        x = odd[k] * t % p
        out[k], out[k + n // 2] = (even[k] + x) % p, (even[k] - x) % p
        t = t * w % p
    return out


def make_s_polynomial(p, a_polys, b_polys, log_b, gamma, omega=None):
    """:391-475, the reference's NTT route."""
    b = 1 << log_b
    b2 = 2 * b
    omega = root_of_unity(p, b2) if omega is None else omega
    (a1, a2), (b1, b2_) = a_polys, b_polys
    assert len(a1) == len(a2) == len(b1) == len(b2_) == b
    ae1, ae2, be1, be2 = (ntt(p, list(v) + [0] * b, omega) for v in (a1, a2, b1, b2_))
    ev = [0] * b2
    ev[0] = 2 * (ae1[0] * be1[0] + ae2[0] * be2[0] * gamma) % p
    for i in range(1, b2):
        s1 = ae1[i] * be1[b2 - i] + ae1[b2 - i] * be1[i]
        s2 = ae2[i] * be2[b2 - i] + ae2[b2 - i] * be2[i]
        ev[i] = (s1 + s2 * gamma) % p
    w_b1 = pow(omega, b - 1, p)
    pw = w_b1
    for i in range(1, b2):
        ev[i] = ev[i] * pw % p
        pw = pw * w_b1 % p
    res = trim(ntt(p, ev, pow(omega, -1, p)))
    inv = pow(b2, -1, p)
    res = [x * inv % p for x in res]
    assert len(res) < b2
    return res[b:]


def s_poly_direct(p, a1, b1, a2, b2, gamma):
    """s[k] = sum_j (a1[j+k+1] b1[j] + a1[j] b1[j+k+1]) + gamma * (the same over a2, b2), k < b - 1."""
    b = len(a1)
    out = []
    for m in range(1, b):
        s1 = sum(a1[j + m] * b1[j] + a1[j] * b1[j + m] for j in range(b - m))
        s2 = sum(a2[j + m] * b2[j] + a2[j] * b2[j + m] for j in range(b - m))
        out.append((s1 + gamma * s2) % p)
    return out


# ---- transcript ------------------------------------------------------------------------------------------
def _absorb_point(tr, label, P):
    tr.absorb_bytes(label, commitment_transcript_bytes(P))


def _absorb_scalars(tr, label, xs):
    tr.absorb_bytes(label, b"".join(to_repr(x) for x in xs))


def _split_point(x):
    """the odd-ell padding (:911-933): a 0 is prepended to the point -> (point, log_b)."""
    point = list(x)
    if len(point) % 2 == 1:
        point.insert(0, 0)
    return point, len(point) // 2


# ---- EvaluationEngine::prove -----------------------------------------------------------------------------
def prove(cid, ck: bytes, f: bytes, x: list, tr, comm=None, eval_=None, trace: dict | None = None):
    """mercury.rs:891-1268.  `f`: Montgomery bytes of the 2^ell coefficients; `comm` / `eval_`: the commitment
    to f and the claimed evaluation (computed here when not given).  -> the 14 fields of EvaluationArgument
    (FIELDS order).  `trace` (optional) receives the intermediate polynomials and challenges."""
    c = CURVES[cid]
    fid, p = c.scalar_field, c.q
    aff = c.affine_from_bytes

    def commit(v):
        return aff(co.msm(cid, _pack(p, v), ck[:64 * len(v)]))
    fv = _ints(p, f)
    original_size = len(fv)
    assert len(x) > 1 and original_size == 1 << len(x)  # :914
    if comm is None:
        comm = aff(co.msm(cid, f, ck[:2 * len(f)]))
    if eval_ is None:
        eval_ = mle_evaluate(p, fv, x)
    _absorb_point(tr, b"f", comm)
    _absorb_scalars(tr, b"u", x)
    _absorb_scalars(tr, b"e", [eval_])
    point, log_b = _split_point(x)
    b = 1 << log_b
    f_poly = fv + [0] * ((b * b) - original_size)
    b_row = original_size // b
    u_row, u_col = point[:log_b], point[log_b:]
    eq_row, eq_col = eq_evals(p, u_row), eq_evals(p, u_col)
    h = compute_h_poly(p, f_poly, eq_col, b_row, b)
    h += [0] * (b - len(h))
    comm_h = commit(h)
    _absorb_point(tr, b"h", comm_h)
    alpha = tr.squeeze(b"a")
    q, g = divide_by_binomial(p, fv, b_row, b, alpha)
    q = trim(q)
    assert len(g) == b
    comm_q, comm_g = commit(q), commit(g)
    _absorb_point(tr, b"q", comm_q)
    _absorb_point(tr, b"g", comm_g)
    gamma = tr.squeeze(b"gm")
    s = make_s_polynomial(p, (eq_col, eq_row), (g, h), log_b, gamma)
    d = g[::-1]
    comm_s, comm_d = commit(s), commit(d)
    _absorb_point(tr, b"s", comm_s)
    _absorb_point(tr, b"d", comm_d)
    zeta = tr.squeeze(b"zt")
    zeta_inv = pow(zeta, -1, p)
    ev = lambda v, pts: _ints(p, co.poly_eval(fid, _pack(p, v), _pack(p, pts))) if v else [0] * len(pts)
    g_zeta, g_zeta_inv = ev(g, [zeta, zeta_inv])
    h_zeta, h_zeta_inv, h_alpha = ev(h, [zeta, zeta_inv, alpha])
    s_zeta, s_zeta_inv = ev(s, [zeta, zeta_inv])
    d_zeta, = ev(d, [zeta])
    zeta_b_alpha = (pow(zeta, b, p) - alpha) % p
    quot_f = batch_add_with_polynomials(p, fv[:original_size], [q], [-zeta_b_alpha])
    quot_f[0] = (quot_f[0] - g_zeta) % p
    assert evaluate(p, quot_f, zeta) == 0  # :1177
    quot_f = _ints(p, co.poly_div(fid, _pack(p, quot_f), mont_bytes(p, zeta)))
    _absorb_scalars(tr, b"gz", [g_zeta])
    _absorb_scalars(tr, b"gzi", [g_zeta_inv])
    _absorb_scalars(tr, b"hz", [h_zeta])
    _absorb_scalars(tr, b"hzi", [h_zeta_inv])
    _absorb_scalars(tr, b"sz", [s_zeta])
    _absorb_scalars(tr, b"szi", [s_zeta_inv])
    comm_quot_f = commit(trim(quot_f[:original_size]))
    _absorb_point(tr, b"t", comm_quot_f)
    # generate_batch_evaluate_arg (:567-770)
    beta = tr.squeeze(b"b")
    beta2 = beta * beta % p
    beta3 = beta2 * beta % p
    g_star = from_evals_with_xs(p, [zeta, zeta_inv], [g_zeta, g_zeta_inv])
    h_star = from_evals_with_xs(p, [zeta, zeta_inv, alpha], [h_zeta, h_zeta_inv, h_alpha])
    s_star = from_evals_with_xs(p, [zeta, zeta_inv], [s_zeta, s_zeta_inv])
    d_star = from_evals_with_xs(p, [zeta], [d_zeta])
    polys = [batch_add_with_polynomials(p, v, [st], [-1]) for v, st in ((g, g_star), (h, h_star), (s, s_star), (d, d_star))]
    for i, pts in enumerate(([alpha], [], [alpha], [alpha, zeta_inv])):
        for pt in pts:
            polys[i] = multiply_by_linear_polynomial(p, polys[i], -pt)
    m = batch_add_with_polynomials(p, polys[0], polys[1:], [beta, beta2, beta3])
    quot_m = m
    for pt in (alpha, zeta, zeta_inv):
        quot_m, rem = divide_by_linear_polynomial(p, quot_m, pt)
        assert rem == 0  # :670-674
    comm_w = commit(quot_m)
    _absorb_point(tr, b"w", comm_w)
    z = tr.squeeze(b"z")
    t_s1 = (z - alpha) % p
    t_s4 = t_s1 * (z - zeta_inv) % p
    t_z = t_s4 * (z - zeta) % p
    stars_z = [evaluate(p, st, z) for st in (g_star, h_star, s_star, d_star)]
    shifted = []
    for v, sz in zip((g, h, s, d), stars_z):
        v = list(v) if v else [0]
        v[0] = (v[0] - sz) % p
        shifted.append(v)
    mz = [t_s1 * x % p for x in shifted[0]]
    mz = batch_add_with_polynomials(p, mz, shifted[1:], [beta, beta2 * t_s1 % p, beta3 * t_s4 % p])
    l_poly = batch_add_with_polynomials(p, mz, [quot_m], [-t_z])
    quot_l, rem = divide_by_linear_polynomial(p, l_poly, z)
    assert rem == 0  # :757-758
    comm_w_prime = commit(quot_l)
    _absorb_point(tr, b"wp", comm_w_prime)
    tr.squeeze(b"pd")
    if trace is not None:
        trace.update(b=b, b_row=b_row, u_row=u_row, u_col=u_col, eq_row=eq_row, eq_col=eq_col, h=h, q=q, g=g, s=s,
                     d=d, quot_f=quot_f, w=quot_m, w_prime=quot_l, alpha=alpha, gamma=gamma, zeta=zeta, beta=beta,
                     z=z, h_alpha=h_alpha, d_zeta=d_zeta, eval=eval_, f_padded=f_poly)
    return (comm_h, comm_g, comm_q, comm_s, comm_d, comm_quot_f, comm_w, comm_w_prime,
            g_zeta, g_zeta_inv, h_zeta, h_zeta_inv, s_zeta, s_zeta_inv)


# ---- EvaluationEngine::verify ----------------------------------------------------------------------------
def verify(cid, tau, C, x, y, proof, tr) -> bool:
    """mercury.rs:1270-1486 with e(ll, [1]_2) == e(rl, [tau]_2) replaced by ll == [tau] rl."""
    c = CURVES[cid]
    p = c.q
    (comm_h, comm_g, comm_q, comm_s, comm_d, comm_quot_f, comm_w, comm_w_prime,
     g_zeta, g_zeta_inv, h_zeta, h_zeta_inv, s_zeta, s_zeta_inv) = proof
    y %= p
    _absorb_point(tr, b"f", C)
    _absorb_scalars(tr, b"u", x)
    _absorb_scalars(tr, b"e", [y])
    _absorb_point(tr, b"h", comm_h)
    alpha = tr.squeeze(b"a")
    _absorb_point(tr, b"q", comm_q)
    _absorb_point(tr, b"g", comm_g)
    gamma = tr.squeeze(b"gm")
    _absorb_point(tr, b"s", comm_s)
    _absorb_point(tr, b"d", comm_d)
    zeta = tr.squeeze(b"zt")
    for label, v in ((b"gz", g_zeta), (b"gzi", g_zeta_inv), (b"hz", h_zeta), (b"hzi", h_zeta_inv),
                     (b"sz", s_zeta), (b"szi", s_zeta_inv)):
        _absorb_scalars(tr, label, [v])
    _absorb_point(tr, b"t", comm_quot_f)
    if zeta == 0:  # zeta.invert().unwrap() (:1345)
        return False
    point, _ = _split_point(x)
    log_n = len(point)
    u_row = point[:log_n // 2]
    u_col = point[log_n - len(u_row):]
    zeta_inv = pow(zeta, -1, p)
    zeta_b_one = pow(zeta, (1 << (log_n // 2)) - 1, p)
    pu_col_z, pu_col_zi = eval_pu_poly(p, u_col, zeta), eval_pu_poly(p, u_col, zeta_inv)
    pu_row_z, pu_row_zi = eval_pu_poly(p, u_row, zeta), eval_pu_poly(p, u_row, zeta_inv)
    d_zeta = zeta_b_one * g_zeta_inv % p  # implicit degree check (:1358)
    h_alpha = (g_zeta * pu_col_zi + g_zeta_inv * pu_col_z
               + gamma * (h_zeta * pu_row_zi + h_zeta_inv * pu_row_z - 2 * y)
               - zeta * s_zeta - zeta_inv * s_zeta_inv) * pow(2, -1, p) % p  # implicit IPA check (:1361-1369)
    g1 = c.gen
    zeta_b_alpha = (zeta_b_one * zeta - alpha) % p
    lhs_1_1 = c.add(C, c.msm_naive([-zeta_b_alpha % p, -g_zeta % p, zeta], [comm_q, g1, comm_quot_f]))
    lhs_2_1 = comm_quot_f
    # extract_pairing_to_verify_batch_evaluation (:773-871)
    beta = tr.squeeze(b"b")
    beta2, beta3 = pow(beta, 2, p), pow(beta, 3, p)
    _absorb_point(tr, b"w", comm_w)
    z = tr.squeeze(b"z")
    g_star = from_evals_with_xs(p, [zeta, zeta_inv], [g_zeta, g_zeta_inv])
    h_star = from_evals_with_xs(p, [zeta, zeta_inv, alpha], [h_zeta, h_zeta_inv, h_alpha])
    s_star = from_evals_with_xs(p, [zeta, zeta_inv], [s_zeta, s_zeta_inv])
    d_star = from_evals_with_xs(p, [zeta], [d_zeta])
    gs, hs, ss, ds = (evaluate(p, st, z) for st in (g_star, h_star, s_star, d_star))
    van_zeta, van_zeta_inv, van_alpha = (z - zeta) % p, (z - zeta_inv) % p, (z - alpha) % p
    t1, t2, t3, t4 = van_alpha, 1, van_alpha, van_zeta_inv * van_alpha % p
    t = t4 * van_zeta % p
    scalar = (t1 * gs + beta * t2 * hs + beta2 * t3 * ss + beta3 * t4 * ds) % p
    scalars = [t1, beta * t2 % p, beta2 * t3 % p, beta3 * t4 % p, -scalar % p, -t % p, z]
    lhs1 = c.msm_naive(scalars, [comm_g, comm_h, comm_s, comm_d, g1, comm_w, comm_w_prime])
    lhs2 = comm_w_prime
    _absorb_point(tr, b"wp", comm_w_prime)
    dd = tr.squeeze(b"pd")
    ll = c.add(lhs_1_1, c.mul(dd, lhs1))
    rl = c.add(lhs_2_1, c.mul(dd, lhs2))
    return ll == c.mul(tau, rl)
