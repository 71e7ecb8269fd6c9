"""Host logic of nova_b200/neutron.py (the mirror of NeutronNova's NIFS::prove / verify and Structure::is_sat) on the
CPU: the library is replaced by tests/emulated_device.py, extended with the three NeutronNova entries by
tests/emulated_neutron.py, so the mirror's glue -- buffer sizes, z layout, the RO2 absorption order, the rho factors,
the interpolation, the folds -- is compared field for field with oracle/neutron_ref.py.  The CUDA kernels themselves
are covered by tests/test_neutron_gpu.py, whose bodies (tests/neutron_parity.py) run here at small sizes."""
import gc

import pytest

import emulated_neutron
import neutron_parity as npar


@pytest.fixture()
def emulated():
    import nova_b200
    dev = emulated_neutron.install()
    yield nova_b200, dev
    gc.collect()
    emulated_neutron.uninstall()


@pytest.mark.parametrize("cid", [0, 2])
@pytest.mark.parametrize("kind,log2n", [("cubic", None), ("squaring", None), ("boolean", 5)])
def test_sequence_matches_oracle(emulated, oracle, cid, kind, log2n):
    nb, _ = emulated
    npar.run_sequence(nb, oracle, cid, kind, log2n, mirror_ro=npar.oracle_ro)


def test_entry_points_host_logic(emulated, oracle):
    _, dev = emulated
    for fid in (0, 3):
        for left, right in ((2, 2), (4, 2), (8, 4)):
            for kind in ("random", "last_row"):
                npar.check_evals(dev, oracle, fid, left, right, kind)
            npar.check_pow_split(dev, fid, left, right)
        for aliased in (False, True):
            npar.check_lerp(dev, fid, 9, aliased)


def test_structure_rejections(emulated, oracle):
    nb, _ = emulated
    from nova_b200 import neutron as ne
    from oracle import neutron_ref as nr
    S, _ = npar.fixture("cubic", 0)
    raw = nr.Shape(0, 4, 3, 2, S.A, S.B, S.C)  # three variables: not padded
    with pytest.raises(ValueError):
        ne.Structure(npar.device_shape(nb, 0, raw))
    I2 = ([1, 1], [0, 1], [0, 1, 2])
    with pytest.raises(ValueError):  # ell = 1: right = 1
        ne.Structure(npar.device_shape(nb, 0, nr.Shape(0, 2, 2, 1, I2, I2, I2)))
    st = ne.Structure(npar.device_shape(nb, 0, S))
    assert (st.ell, st.left, st.right) == (2, 2, 2)


def test_prove_rejects_bad_lengths(emulated, oracle):
    nb, _ = emulated
    from nova_b200 import neutron as ne, r1cs, spartan as sp
    S, fresh = npar.fixture("cubic", 0)
    st = ne.Structure(npar.device_shape(nb, 0, S))
    ck, _ = npar.keys(nb, oracle, 0, 4)
    U, W = ne.FoldedInstance.default(st), ne.FoldedWitness.default(st)
    good = r1cs.R1CSWitness(sp.DeviceVec.from_bytes(bytes(32 * 4)), 0)
    with pytest.raises(ValueError):  # X of the wrong length
        ne.nifs_prove(ck, npar.oracle_ro(0), 0, st, U, W, r1cs.R1CSInstance(None, [0]), good, 1)
    with pytest.raises(ValueError):  # W of the wrong length
        ne.nifs_prove(ck, npar.oracle_ro(0), 0, st, U, W, r1cs.R1CSInstance(None, [0, 0]),
                      r1cs.R1CSWitness(sp.DeviceVec.from_bytes(bytes(32 * 3)), 0), 1)
    ck.release()


def test_zero_denominator_raises():
    from nova_b200 import neutron as ne
    from nova_b200.spartan import UniPoly
    p = npar.FIELD_MODULUS[0]
    # (1 - rho)(1 - r_b) + rho r_b = 3 r_b - 1 for rho = 2: zero at r_b = 1/3
    with pytest.raises(ValueError):
        ne._t_out(p, UniPoly(p, [1, 2, 3, 4, 5, 6]), 2, pow(3, -1, p))
