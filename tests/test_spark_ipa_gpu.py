"""ppsnark's setup on the device (b200_spark_repr_dev behind SparkRepr.from_shape, the seven shape commitments of
ppsnark.setup) and ppsnark + IPA (ppsnark.prove(ee="ipa")) on an H100: byte parity of the spark vectors with the
oracle in all four fields and with SparkRepr.from_numpy at N = 2^20, the argument checks of the entry, S_comm against
the C oracle, and whole proofs against tests/ppsnark_ipa_ref.prove_ipa / verify_ipa, once at N = 2^18."""
import ctypes
import os
import sys

import pytest

import spark_ipa_parity as sip

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("kind", sip.SHAPES)
@pytest.mark.parametrize("cid", [0, 1, 2, 3])
def test_from_shape_equals_oracle(b200, cid, kind):
    sip.check_from_shape(b200, cid, kind)


def _replay():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import spark_ipa_replay
    return spark_ipa_replay


def test_from_shape_at_scale_equals_from_numpy(b200):
    """N = 2^20 slots (about four grid-strides of the kernel): every vector equals SparkRepr.from_numpy's, whose
    timestamps are np.bincount over the host arrays"""
    from nova_b200 import ppsnark as dp
    inst = _replay().build(1, 18)
    fid, S = inst["fid"], inst["S"]
    rows, cols, vals = inst["host"]
    got = dp.SparkRepr.from_shape(fid, S)
    exp = dp.SparkRepr.from_numpy(fid, rows, cols, vals, S["num_cons"], S["num_vars"])
    assert got.N == exp.N == 1 << 20 and len(rows) < got.N
    for name in sip.SPARK_NAMES + ("row_idx", "col_idx"):
        assert getattr(got, name).to_bytes() == getattr(exp, name).to_bytes(), name


def _sentinel(n_bytes):
    from nova_b200 import spartan as sp
    from nova_b200.native import check, lib
    v = sp.DeviceVec(n_bytes)
    check(lib().b200_memset_dev(v.ptr, 0xAB, n_bytes, None))
    return v


def test_bad_arguments_are_refused_without_writes(b200):
    from nova_b200 import spartan as sp
    from nova_b200.native import lib
    from oracle.pyref import FIELD_MODULUS
    p = FIELD_MODULUS[0]
    A, B, C, nc, nv, ncols = sip.shape(p, "by_nnz")  # nnz 56, N = 64
    m = sip.register(sp, 0, p, A, B, C, nc, ncols)
    other_rows = sip.register(sp, 0, p, A, B, C, nc + 1, ncols)["A"]
    other_cols = sip.register(sp, 0, p, A, B, C, nc, ncols + 1)["A"]
    other_field = sip.register(sp, 2, FIELD_MODULUS[2], A, B, C, nc, ncols)["A"]
    n_max = 128
    vecs = [_sentinel(32 * n_max) for _ in range(7)]
    ri, ci = _sentinel(4 * n_max), _sentinel(4 * n_max)
    ptrs = (ctypes.c_void_p * 7)(*[v.ptr.value for v in vecs])
    ha, hb, hc = m["A"].handle, m["B"].handle, m["C"].handle
    cases = [((ha, hb, 987654321), 64, 3),                  # unknown handle
             ((ha, other_rows.handle, hc), 64, 1),          # rows differ
             ((ha, hb, other_cols.handle), 64, 1),          # cols differ
             ((other_field.handle, hb, hc), 64, 1),         # field differs
             ((ha, hb, hc), 96, 1), ((ha, hb, hc), 0, 1),   # not a power of two
             ((ha, hb, hc), 1 << 32, 1),                    # not below 2^32
             ((ha, hb, hc), 32, 5)]                         # below nnz = 56
    before = [v.to_bytes() for v in vecs + [ri, ci]]
    for (h1, h2, h3), N, code in cases:
        assert lib().b200_spark_repr_dev(h1, h2, h3, N, ptrs, ri.ptr, ci.ptr, None) == code, (N, code)
    assert lib().b200_spark_repr_dev(ha, hb, hc, 64, ptrs, None, ci.ptr, None) == 1  # null index output
    nulls = (ctypes.c_void_p * 7)(*([v.ptr.value for v in vecs[:6]] + [None]))
    assert lib().b200_spark_repr_dev(ha, hb, hc, 64, nulls, ri.ptr, ci.ptr, None) == 1  # null ts_col
    wide = sip.register(sp, 0, p, [], [], [(0, 100, 1)], nc, 101)  # cols 101 > N = 64 >= nnz
    assert lib().b200_spark_repr_dev(wide["A"].handle, wide["B"].handle, wide["C"].handle, 64, ptrs, ri.ptr, ci.ptr,
                                     None) == 5
    tall = sip.register(sp, 0, p, [], [], [(99, 0, 1)], 100, ncols)  # rows 100 > N = 64
    assert lib().b200_spark_repr_dev(tall["A"].handle, tall["B"].handle, tall["C"].handle, 64, ptrs, ri.ptr, ci.ptr,
                                     None) == 5
    assert [v.to_bytes() for v in vecs + [ri, ci]] == before  # nothing was written
    assert lib().b200_spark_repr_dev(ha, hb, hc, 64, ptrs, ri.ptr, ci.ptr, None) == 0
    after = [v.to_bytes() for v in vecs]
    assert all(a[32 * 64:] == b[32 * 64:] for a, b in zip(after, before))  # N = 64 of the 128 elements written


@pytest.mark.parametrize("cid", [0, 1, 2, 3])
def test_setup_commitments_equal_c_oracle(b200, oracle, cid):
    sip.check_setup_commitments(b200, oracle, cid)


@pytest.mark.parametrize("device_transcript", [False, True])
@pytest.mark.parametrize("cid", [0, 1, 2, 3])
def test_prove_ipa_equals_oracle(b200, oracle, cid, device_transcript):
    sip.run_prove(b200, cid, device_transcript)


@pytest.mark.parametrize("cid", [1, 3])
def test_prove_ipa_at_scale_verifies(b200, oracle, cid):
    """Grumpkin and Vesta, N = 2^18: setup, prove(ee="ipa") and the restated verifier with S_comm, U and its N-point
    MSM from the C oracle"""
    from nova_b200 import ppsnark as dp
    from nova_b200.transcript import Keccak256Transcript
    rp = _replay()
    inst = rp.build(cid, 16)
    curve, S = inst["curve"], inst["S"]
    spark0 = dp.SparkRepr.from_shape(inst["fid"], S)
    assert spark0.N == 1 << 18
    ck = rp.key_for(curve, spark0.N)
    spark, S_comm = dp.setup(curve, ck, S)
    U = dict(comm_W=dp.commit_dev(curve, ck, inst["W"], S["num_vars"]),
             comm_E=dp.commit_dev(curve, ck, inst["E"], S["num_cons"]), u=inst["u"], X=inst["X"])
    proof = dp.prove(curve, ck, S, spark, U, dict(W=inst["W"], E=inst["E"]), rp.VK_DIGEST,
                     Keccak256Transcript(inst["p"], b"RelaxedR1CSSNARK"), ee="ipa", S_comm=S_comm)
    assert rp.oracle_check(inst, ck, spark, S_comm, U, proof) == {"S_comm_equal": True, "U_equal": True,
                                                                  "verified": True}
    ck.release()
