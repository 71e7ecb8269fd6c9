"""The oracle's Mercury prover restatement (oracle/mercury_ref.py, mercury.rs:891-1268) must satisfy the
verifier restatement (:1270-1486, the pairing replaced by ll = [tau] rl for a test SRS whose tau is known),
and its pieces must satisfy the identities the reference checks in debug builds (:940-1109)."""
import pytest

from oracle import hyperkzg_ref as hk
from oracle import mercury_ref as mr
from oracle.pyref import CURVES, Keccak256Transcript, SplitMix64, mle_evaluate, mont_bytes

CID = 0


def pack(p, xs):
    return b"".join(mont_bytes(p, x) for x in xs)


_SRS = {}


def srs(n):
    """one test SRS per size, [tau^i] G for a fixed tau"""
    c = CURVES[CID]
    tau = SplitMix64(77).field(c.q)
    if n not in _SRS:
        _SRS[n] = hk.setup_srs(CID, n, tau)
    return tau, _SRS[n]


def instance(ell, seed):
    c = CURVES[CID]
    p = c.q
    rng = SplitMix64(seed)
    f = [rng.field(p) for _ in range(1 << ell)]
    x = [rng.field(p) for _ in range(ell)]
    return f, x


@pytest.mark.parametrize("ell", [2, 3, 4, 7, 10, 15, 16])
def test_honest_proofs_verify_and_tampered_ones_fail(oracle, ell):
    c = CURVES[CID]
    p = c.q
    n = 1 << ell
    tau, ck = srs(n)
    f, x = instance(ell, 500 + ell)
    y = mle_evaluate(p, f, x)
    C = c.affine_from_bytes(oracle.msm(CID, pack(p, f), ck))
    tp, tv = Keccak256Transcript(p, b"TestEval"), Keccak256Transcript(p, b"TestEval")
    proof = mr.prove(CID, ck, pack(p, f), x, tp)
    assert len(proof) == len(mr.FIELDS) == 14
    assert mr.verify(CID, tau, C, x, y, proof, tv)
    assert tp.squeeze(b"s") == tv.squeeze(b"s")  # both end in the same transcript state
    fresh = lambda: Keccak256Transcript(p, b"TestEval")
    assert not mr.verify(CID, tau, C, x, (y + 1) % p, proof, fresh())
    for i in range(14):
        bad = list(proof)
        bad[i] = c.add(bad[i], c.gen) if i < 8 else (bad[i] + 1) % p
        assert not mr.verify(CID, tau, C, x, y, tuple(bad), fresh()), mr.FIELDS[i]


def test_prove_rejects_ell_one(oracle):
    c = CURVES[CID]
    _, ck = srs(4)
    with pytest.raises(AssertionError):
        mr.prove(CID, ck, pack(c.q, [1, 2]), [5], Keccak256Transcript(c.q, b"TestEval"))


@pytest.mark.parametrize("ell", [2, 5, 8])
def test_divide_by_binomial(ell):
    """f(r) = (r^b - alpha) q(r) + g(r) (:1026-1042) and g[c] = column c at alpha (:1001-1024)."""
    p = CURVES[CID].q
    rng = SplitMix64(40 + ell)
    f, x = instance(ell, 41 + ell)
    _, log_b = mr._split_point(x)
    b = 1 << log_b
    rows = len(f) // b
    alpha, r = rng.field(p), rng.field(p)
    q, g = mr.divide_by_binomial(p, f, rows, b, alpha)
    assert len(g) == b and all(v == 0 for v in q[(rows - 1) * b:])
    assert mr.evaluate(p, f, r) == ((pow(r, b, p) - alpha) * mr.evaluate(p, q, r) + mr.evaluate(p, g, r)) % p
    for col in range(b):
        assert g[col] == mr.evaluate(p, f[col::b], alpha)


@pytest.mark.parametrize("log_b", [1, 2, 3, 6])
def test_ntt_s_polynomial_equals_the_lag_formula(log_b):
    """make_s_polynomial's NTT route (any primitive 2b-th root of unity) == the direct lag sums the device computes."""
    p = CURVES[CID].q
    rng = SplitMix64(60 + log_b)
    b = 1 << log_b
    a1, b1, a2, b2 = ([rng.field(p) for _ in range(b)] for _ in range(4))
    gamma = rng.field(p)
    direct = mr.s_poly_direct(p, a1, b1, a2, b2, gamma)
    assert len(direct) == b - 1
    w = mr.root_of_unity(p, 2 * b)
    assert pow(w, b, p) == p - 1
    for omega in (w, pow(w, 3, p), pow(w, -1, p)):  # other primitive 2b-th roots give the same s
        got = mr.make_s_polynomial(p, (a1, a2), (b1, b2), log_b, gamma, omega)
        assert got == mr.trim(direct)


@pytest.mark.parametrize("ell", [2, 3, 6, 7])
def test_debug_identities(oracle, ell):
    """The checks of mercury.rs:940-1109 on the oracle's intermediates, at a random r."""
    c = CURVES[CID]
    p = c.q
    _, ck = srs(1 << ell)
    f, x = instance(ell, 700 + ell)
    tr = {}
    proof = mr.prove(CID, ck, pack(p, f), x, Keccak256Transcript(p, b"TestEval"), trace=tr)
    r = SplitMix64(900 + ell).field(p)
    ri = pow(r, -1, p)
    ev = lambda v, t: mr.evaluate(p, v, t)
    # pu_row, pu_col (:940-962)
    assert mr.eval_pu_poly(p, tr["u_row"], r) == ev(tr["eq_row"], r)
    assert mr.eval_pu_poly(p, tr["u_col"], r) == ev(tr["eq_col"], r)
    # <eq_row, h> = eval (:972-984)
    assert sum(a * b for a, b in zip(tr["eq_row"], tr["h"])) % p == tr["eval"] == mle_evaluate(p, f, x)
    # g is f's columns at alpha, q and g divide f (:1001-1042)
    b, alpha = tr["b"], tr["alpha"]
    fp = tr["f_padded"]
    assert tr["g"] == [ev(fp[col::b], alpha) for col in range(b)]
    assert ev(fp, r) == ((pow(r, b, p) - alpha) * ev(tr["q"], r) + ev(tr["g"], r)) % p
    # <eq_col, g> = h(alpha) (:1053-1065)
    assert sum(a * b for a, b in zip(tr["eq_col"], tr["g"])) % p == ev(tr["h"], alpha) == tr["h_alpha"]
    # the s polynomial's inner-product identity (:1079-1109)
    gm = tr["gamma"]
    pc, pci = mr.eval_pu_poly(p, tr["u_col"], r), mr.eval_pu_poly(p, tr["u_col"], ri)
    pr_, pri = mr.eval_pu_poly(p, tr["u_row"], r), mr.eval_pu_poly(p, tr["u_row"], ri)
    g, h, s = tr["g"], tr["h"], tr["s"]
    lhs = (ev(g, r) * pci + ev(g, ri) * pc + gm * (ev(h, r) * pri + ev(h, ri) * pr_)) % p
    rhs = (2 * (tr["h_alpha"] + gm * tr["eval"]) + r * ev(s, r) + ri * ev(s, ri)) % p
    assert lhs == rhs
    # quot_f (:1182-1200)
    zeta = tr["zeta"]
    g_zeta = proof[8]
    assert ev(tr["quot_f"], r) * (r - zeta) % p == (ev(fp, r) - (pow(zeta, b, p) - alpha) * ev(tr["q"], r) - g_zeta) % p
