"""Host logic of ppsnark's device setup (SparkRepr.from_shape, setup) and of prove(ee="ipa") on the CPU: the library
is replaced by tests/emulated_device.py, extended with b200_spark_repr_dev by tests/emulated_spark.py, so the mirror's
glue -- N, the vector order of the entry, the seven commitments, the batched commitment, b_vec and the IPA's
transcript -- is compared field for field with the oracle (oracle/ppsnark_ref.py,
composed with the IPA in tests/ppsnark_ipa_ref.py).  The CUDA kernel itself is covered by
tests/test_spark_ipa_gpu.py, which runs the same bodies (tests/spark_ipa_parity.py)."""
import gc

import pytest

import emulated_spark
import spark_ipa_parity as sip


@pytest.fixture()
def emulated():
    import nova_b200
    emulated_spark.install()
    yield nova_b200
    gc.collect()
    emulated_spark.uninstall()


@pytest.mark.parametrize("kind", sip.SHAPES)
def test_from_shape_equals_oracle(emulated, kind):
    sip.check_from_shape(emulated, 0, kind)


@pytest.mark.parametrize("cid", [0, 1, 2, 3])
def test_setup_commitments_equal_oracle(emulated, oracle, cid):
    sip.check_setup_commitments(emulated, oracle, cid)


@pytest.mark.parametrize("device_transcript", [False, True])
@pytest.mark.parametrize("cid", [0, 1, 2, 3])
def test_prove_ipa_equals_oracle(emulated, oracle, cid, device_transcript):
    sip.run_prove(emulated, cid, device_transcript)


def test_ipa_needs_shape_commitments_and_a_blinding_generator(emulated, oracle):
    from nova_b200 import ppsnark as dp
    with pytest.raises(ValueError):
        dp.prove(0, None, {}, None, {}, {}, 0, None, ee="ipa")  # no S_comm: refused before any device work
    ck = emulated.CommitmentKey(emulated.Curve(1), oracle.gen_bases(1, 8))  # no ck_c
    spark = type("Spark", (), {"N": 8})()
    with pytest.raises(ValueError):
        dp.prove(1, ck, {}, spark, {}, {}, 0, None, ee="ipa", S_comm={})
    ck_h = emulated.CommitmentKey(emulated.Curve(1), oracle.gen_bases(1, 4), oracle.gen_bases(1, 1, 99))  # N > len(ck)
    with pytest.raises(ValueError):
        dp.prove(1, ck_h, {}, spark, {}, {}, 0, None, ee="ipa", S_comm={})
