"""oracle/neutron_ref.py, the restatement of NeutronNova's folding scheme (src/neutron/), checked against equations
none of its parts is defined by: execute_sequence / test_tiny_r1cs_bellpepper (nifs.rs:366-503) on three shapes
over the BN254 and Pallas scalar fields (verify reproduces every prover instance, is_sat holds after every fold),
tampered folds are rejected, the power polynomial's split table is a tensor factorisation of its evaluations
(power.rs tests), from_evals interpolates, and the C-oracle composition of the prove_helper sums equals the literal
loop."""
import pytest

import neutron_parity as npar
from oracle import neutron_ref as nr
from oracle.pyref import CURVES, FIELD_MODULUS, SplitMix64


@pytest.mark.parametrize("cid", [0, 2])
@pytest.mark.parametrize("kind,log2n", [("cubic", None), ("squaring", None), ("boolean", 6)])
def test_execute_sequence(oracle, cid, kind, log2n):
    npar.run_sequence(None, oracle, cid, kind, log2n)


def _one_fold(oracle, cid):
    c = CURVES[cid]
    fid, p = c.scalar_field, c.q
    S, fresh = npar.fixture("squaring", fid)
    st = nr.Structure.new(S)
    _, ck = npar.keys(None, oracle, cid, max(S.num_vars, st.left + st.right))
    rng = SplitMix64(77)
    U1, W1 = nr.FoldedInstance.default(st), nr.FoldedWitness.default(st)
    for _ in range(2):  # fold twice so that U1.T is not zero
        Wv, X = fresh(rng)
        U2, W2 = nr.R1CSInstance(nr.commit(ck, fid, Wv, 5), X), nr.R1CSWitness(Wv, 5)
        nifs, (U, W) = nr.nifs_prove(ck, npar.oracle_ro(fid), 0, st, U1, W1, U2, W2, 9)
        prev = (U1, U2)
        U1, W1 = U, W
    return c, st, ck, nifs, prev, (U, W)


@pytest.mark.parametrize("cid", [0, 2])
def test_tampering_is_rejected(oracle, cid):
    c, st, ck, nifs, (U1, U2), (U, W) = _one_fold(oracle, cid)
    p = c.q
    assert U1.T != 0
    verify = lambda n: nr.nifs_verify(cid, p, n, npar.oracle_ro(c.scalar_field), 0, U1, U2)
    assert verify(nifs) == U and nr.is_sat(ck, st, U, W)
    for k in range(6):  # any coefficient: the sum-check identity or the fold breaks
        poly = list(nifs.poly)
        poly[k] = (poly[k] + 1) % p
        Ub = verify(nr.NIFS(nifs.comm_E, poly))
        assert Ub is None or not nr.is_sat(ck, st, Ub, W)
    Ub = verify(nr.NIFS(c.add(nifs.comm_E, c.gen), nifs.poly))  # another comm_E: other challenges
    assert Ub is None or (Ub != U and not nr.is_sat(ck, st, Ub, W))
    for T in ((U.T + 1) % p, 0):
        assert not nr.is_sat(ck, st, nr.FoldedInstance(U.comm_W, U.comm_E, T, U.u, U.X), W)
    Wb = nr.FoldedWitness(W.W, W.r_W, W.E, (W.r_E + 1) % p)
    assert not nr.is_sat(ck, st, U, Wb)


@pytest.mark.parametrize("fid", [0, 3])
def test_split_evals_is_a_tensor_factorisation(fid):
    p = FIELD_MODULUS[fid]
    tau = SplitMix64(fid).field(p)
    for ell in range(2, 10):
        left, right = 1 << ((ell + 1) // 2), 1 << (ell // 2)
        E = nr.split_evals(p, tau, left, right)
        assert len(E) == left + right
        assert [E[left + i] * E[j] % p for i in range(right) for j in range(left)] == nr.evals(p, tau, ell)


def test_split_evals_rejects_right_one():
    with pytest.raises(IndexError):
        nr.split_evals(FIELD_MODULUS[0], 5, 2, 1)


@pytest.mark.parametrize("n", [1, 2, 3, 6])
def test_from_evals_interpolates(n):
    from nova_b200.spartan import UniPoly
    p = FIELD_MODULUS[0]
    rng = SplitMix64(n)
    ev = [rng.field(p) for _ in range(n)]
    coeffs = nr.from_evals(p, ev)
    assert [nr.uni_eval(p, coeffs, x) for x in range(n)] == ev
    assert UniPoly.from_evals(p, ev).coeffs == coeffs  # the mirror's Lagrange route
    direct = [rng.field(p) for _ in range(n)]  # a known polynomial comes back
    assert nr.from_evals(p, [nr.uni_eval(p, direct, x) for x in range(n)]) == direct


@pytest.mark.parametrize("fid", [0, 1, 2, 3])
@pytest.mark.parametrize("left,right", [(2, 2), (4, 2), (8, 8), (16, 8)])
def test_c_composition_equals_the_literal_loop(oracle, fid, left, right):
    p = FIELD_MODULUS[fid]
    for kind in ("random", "zero", "last_row", "p_minus_1"):
        e1, abc1, e2, abc2 = npar._vectors(fid, left, right, kind, 11 + left)
        lit = nr.prove_helper_raw(p, left, right, e1, *(npar.ints(p, v) for v in abc1), e2,
                                  *(npar.ints(p, v) for v in abc2))
        assert nr.evals_raw(fid, left, right, e1, *abc1, e2, *abc2) == lit
    # one instance twice: every sum is the is_sat sum
    e, abc = e1, [npar.ints(p, v) for v in abc1]
    s = nr.prove_helper_raw(p, left, right, e, *abc, e, *abc)
    assert s == [s[0]] * 5


def test_pad_tiny_cubic():
    S, _ = npar.fixture("cubic", 0)
    assert (S.num_cons, S.num_vars, S.num_io) == (4, 4, 2)
    assert nr.is_regular_shape(S) and S.A[1] == [5, 0, 1, 5, 2, 4]  # u and X move up by the padded variable
    st = nr.Structure.new(S)
    assert (st.ell, st.left, st.right) == (2, 2, 2)
