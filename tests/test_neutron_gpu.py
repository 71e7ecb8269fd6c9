"""The NeutronNova entry points (b200_neutron_evals, b200_pow_split_evals, b200_lerp) bit-exact against the oracle in
all four fields, the device fold (nova_b200.neutron) field for field against oracle/neutron_ref.py, and a sequence of
three folds at 2^20 constraints checked by the restated verifier, the device is_sat and the C oracle."""
import pytest

import neutron_parity as npar

pytestmark = pytest.mark.gpu

ELLS = [2, 3, 4, 5, 10, 11, 16, 20, 21]


def _split(ell):
    return 1 << ((ell + 1) // 2), 1 << (ell // 2)


@pytest.fixture(scope="module")
def L(b200):
    from nova_b200.native import lib
    return lib()


@pytest.mark.parametrize("fid", [0, 1, 2, 3])
@pytest.mark.parametrize("ell", ELLS)
def test_evals(L, oracle, fid, ell):
    # every input kind at the sizes where the oracle is cheap; random and last-row inputs at the large ones
    kinds = ("random", "zero", "last_row", "p_minus_1") if ell <= 16 else ("random", "last_row")
    for kind in kinds:
        npar.check_evals(L, oracle, fid, *_split(ell), kind)


@pytest.mark.parametrize("left,right", [(3, 5), (257, 3), (1000, 7)])
def test_evals_left_not_a_power_of_two(L, left, right):
    """rows do not line up with blocks or tiles: the literal loop of the reference is the expectation"""
    from nova_b200.provider import _cbuf
    from oracle import neutron_ref as nr
    import ctypes
    fid = 0
    p = npar.FIELD_MODULUS[fid]
    rng = npar.SplitMix64(left)
    vs = [[rng.field(p) for _ in range(left + right if k % 4 == 0 else left * right)] for k in range(8)]
    out = ctypes.create_string_buffer(32 * 5)
    assert L.b200_neutron_evals(fid, *[_cbuf(npar.pack(p, v)) for v in vs], left, right, out) == 0
    assert npar.ints(p, out.raw) == nr.prove_helper_raw(p, left, right, *vs)


def test_evals_rejects_empty_split(L):
    import ctypes
    buf = ctypes.create_string_buffer(32 * 8)
    assert L.b200_neutron_evals(0, *[buf] * 8, 0, 4, buf) == 1
    assert L.b200_neutron_evals(0, *[buf] * 8, 4, 0, buf) == 1


@pytest.mark.parametrize("fid", [0, 1, 2, 3])
def test_pow_split_evals(L, fid):
    for ell in ELLS:
        npar.check_pow_split(L, fid, *_split(ell))
    npar.check_pow_split(L, fid, 3, 5)
    import ctypes
    buf = ctypes.create_string_buffer(32 * 8)
    assert L.b200_pow_split_evals(fid, buf, 2, 1, buf) == 1  # right = 1: the reference panics
    assert L.b200_pow_split_evals(fid, buf, 0, 4, buf) == 1


@pytest.mark.parametrize("fid", [0, 1, 2, 3])
@pytest.mark.parametrize("n", [1, 255, 257, (1 << 20) + 1, 3 * (1 << 20) + 7])
def test_lerp(L, fid, n):
    """(1 << 20) + 1 and 3 * 2^20 + 7 need several grid-stride passes of the capped grid"""
    for aliased in (False, True):
        npar.check_lerp(L, fid, n, aliased)


def _device_ro(fid):
    from nova_b200.poseidon import PoseidonRO
    return PoseidonRO(fid)


@pytest.mark.parametrize("cid", [0, 2])
@pytest.mark.parametrize("kind,log2n", [("cubic", None), ("squaring", None), ("boolean", 10), ("boolean", 16)])
def test_nifs_prove_matches_oracle(b200, oracle, cid, kind, log2n):
    npar.run_sequence(b200, oracle, cid, kind, log2n, mirror_ro=_device_ro)


def test_three_folds_at_2_20(b200, oracle):
    """ell = 20 on BN254: every U is reproduced by the restated verify, the device is_sat holds after every fold and
    its sum equals the C oracle's, and a tampered T is rejected"""
    import numpy as np
    from nova_b200 import fields, neutron as ne, r1cs
    from nova_b200.ppsnark import dev_from_u64
    from oracle import neutron_ref as nr
    cid, log2n = 0, 20
    n = 1 << log2n
    fid = 0
    p = npar.FIELD_MODULUS[fid]
    M = ([1] * n, list(range(n)), list(range(n + 1)))
    S = nr.Shape(fid, n, n, 1, M, M, M)
    st_dev = ne.Structure(npar.device_shape(b200, cid, S))
    ck, _ = npar.keys(b200, oracle, cid, n)
    rng = npar.SplitMix64(20)
    U, W = ne.FoldedInstance.default(st_dev), ne.FoldedWitness.default(st_dev)
    Uo = nr.FoldedInstance(None, None, 0, 0, [0])
    for step in range(3):
        w = np.frombuffer(rng.bytes(n), dtype=np.uint8) & 1
        W2 = r1cs.R1CSWitness(dev_from_u64(fid, w), rng.field(p))
        U2 = r1cs.R1CSInstance(st_dev.S._commit(ck, W2.W, n, W2.r_W), [0])
        nifs, (U_new, W_new) = ne.nifs_prove(ck, _device_ro(fid), 7, st_dev, U, W, U2, W2, rng.field(p))
        Uv = nr.nifs_verify(cid, p, nr.NIFS(nifs.comm_E, list(nifs.poly)), npar.oracle_ro(fid), 7, Uo,
                            nr.R1CSInstance(U2.comm_W, U2.X))
        assert Uv is not None and (Uv.comm_W, Uv.comm_E, Uv.T, Uv.u, Uv.X) == (U_new.comm_W, U_new.comm_E, U_new.T,
                                                                               U_new.u, U_new.X), step
        assert ne.is_sat(ck, st_dev, U_new, W_new), step
        Wb = W_new.W.to_bytes(32 * n)
        E = fields.unpack(fid, W_new.E.to_bytes(32 * (st_dev.left + st_dev.right)))
        # this shape has Az = Bz = Cz = W
        assert nr.evals_raw(fid, st_dev.left, st_dev.right, E, Wb, Wb, Wb, E, Wb, Wb, Wb)[0] == U_new.T, step
        assert not ne.is_sat(ck, st_dev, ne.FoldedInstance(U_new.comm_W, U_new.comm_E, (U_new.T + 1) % p, U_new.u,
                                                           U_new.X), W_new), step
        U, W, Uo = U_new, W_new, Uv
    ck.release()
