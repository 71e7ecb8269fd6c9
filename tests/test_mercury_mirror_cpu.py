"""Host logic of nova_b200/mercury.py (the mirror of provider/mercury.rs EvaluationEngine::prove) and of
snark / ppsnark with ee="mercury" on the CPU: the library is replaced by tests/emulated_device.py, extended with the three Mercury
entries by tests/emulated_mercury.py, which answers every `*_dev` call with the oracle on host memory, so the mirror's glue --
buffer sizes, the odd-ell padding, the term-by-term batch opening, transcript order -- is compared field for
field with oracle/mercury_ref.py.  The CUDA kernels themselves are covered by tests/test_mercury_gpu.py, whose
bodies (tests/mercury_parity.py) run here unchanged at small sizes."""
import gc

import pytest

import emulated_mercury
import mercury_parity as mp


@pytest.fixture()
def emulated():
    import nova_b200
    emulated_mercury.install()
    yield nova_b200
    gc.collect()
    emulated_mercury.uninstall()


@pytest.mark.parametrize("rows,cols", [(1, 1), (1, 4), (2, 2), (3, 8), (65, 2), (8, 64), (130, 3)])
def test_div_binomial_host_logic(emulated, oracle, rows, cols):
    from nova_b200 import spartan as sp
    for kind in ("random", "zero", "last_row"):
        mp.check_div_binomial(sp, oracle, rows, cols, kind)


@pytest.mark.parametrize("rows,cols", [(1, 1), (4, 4), (3, 17), (8, 600)])
def test_mat_vec_rows_host_logic(emulated, oracle, rows, cols):
    from nova_b200 import spartan as sp
    mp.check_mat_vec_rows(sp, oracle, rows, cols)


@pytest.mark.parametrize("b", [2, 4, 16])
def test_s_poly_host_logic(emulated, oracle, b):
    from nova_b200 import spartan as sp
    mp.check_s_poly(sp, oracle, b)


@pytest.mark.parametrize("ell", [2, 3, 4, 7, 10])
def test_mercury_prove_host_logic(emulated, oracle, ell):
    mp.run_prove(emulated, oracle, ell)


def test_mercury_prove_rejections(emulated, oracle):
    from nova_b200 import mercury as dm
    from oracle.pyref import Keccak256Transcript
    _, srs = mp.srs_for(8)
    ck = emulated.CommitmentKey(emulated.Curve(0), srs)
    p = emulated.fields.MODULUS[0]
    with pytest.raises(ValueError):  # ell <= 1 (mercury.rs:914)
        dm.mercury_prove(emulated.Curve(0), ck, bytes(64), [3], Keccak256Transcript(p, b"T"))
    with pytest.raises(ValueError):  # len(P) != 2^ell
        dm.mercury_prove(emulated.Curve(0), ck, bytes(32 * 4), [3, 4, 5], Keccak256Transcript(p, b"T"))
    ck.release()


def test_verify_only_at_small_size(emulated, oracle):
    mp.run_verify_only(emulated, oracle, 5)


@pytest.mark.parametrize("device_transcript", [False, True])
def test_snark_with_mercury_host_logic(emulated, oracle, device_transcript):
    mp.run_snark(emulated, oracle, device_transcript=device_transcript)


def test_ppsnark_with_mercury_host_logic(emulated, oracle):
    mp.run_ppsnark(emulated, oracle)


def test_unknown_engine_is_refused(emulated):
    from nova_b200 import ppsnark as dp
    with pytest.raises(ValueError):
        dp.prove(0, None, {}, None, {}, {}, 0, None, ee="ipa")
    with pytest.raises(ValueError):
        dp.prove(0, None, {}, None, {}, {}, 0, None, ee="mercury")  # needs S_comm
