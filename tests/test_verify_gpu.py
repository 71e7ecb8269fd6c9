"""The verifier's device pieces on an H100: b200_r1cs_eval(_dev) byte-equal to the C restatement of multi_evaluate
(tests/verify_oracle.c) in all four fields -- skewed and empty rows, an empty matrix, cols == len(T_y), and 2^20 rows
with more than 3 * 2^20 entries, where it also equals the SpMV + dot composition -- and its errors; b200_ipa_s_dev
against the reference's s and the prover's final weights; and whole verifications: snark.verify(ee="ipa") on proofs
of snark.prove(ee="ipa"), equal to the oracle's verdicts at small sizes and at 2^16 constraints on Grumpkin and
Vesta, and verify_core + the oracle's HyperKZG check on BN254."""
import ctypes
import os
import sys

import pytest

import verify_ref
from oracle.pyref import CURVES, FIELD_MODULUS, Keccak256Transcript, SplitMix64, eq_evals, mont_bytes
from test_verify_kernels_host import matrix, pack, shapes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def register(sp, fid, p, data, indices, indptr, cols):
    return sp.SparseMatrix(fid, pack(p, data), indices, indptr, cols)


def dev_eval(sp, mats, Tx: bytes, Ty: bytes, k=None):
    from nova_b200.native import check, lib
    k = len(mats) if k is None else k
    hs = (ctypes.c_uint64 * 3)(*([m.handle for m in mats] + [0] * (3 - len(mats))))
    tx, ty = sp.DeviceVec.from_bytes(Tx), sp.DeviceVec.from_bytes(Ty)
    out = sp.DeviceVec(96)
    check(lib().b200_r1cs_eval_dev(hs, k, tx.ptr, len(Tx) // 32, ty.ptr, len(Ty) // 32, out.ptr, None))
    return out.to_bytes(32 * k)


@pytest.mark.parametrize("fid", [0, 1, 2, 3])
def test_r1cs_eval_equals_c_restatement(b200, fid):
    from nova_b200 import spartan as sp
    p = FIELD_MODULUS[fid]
    rng = SplitMix64(9500 + fid)
    for name, rows, cols, lens in shapes(rng):
        ell_x, ell_y = (rows - 1).bit_length(), (cols - 1).bit_length()
        rx, ry = [rng.field(p) for _ in range(ell_x)], [rng.field(p) for _ in range(ell_y)]
        Tx, Ty = pack(p, eq_evals(p, rx)), pack(p, eq_evals(p, ry))
        mats = [matrix(p, rng, lens, cols) for _ in range(3)]
        want = b"".join(verify_ref.r1cs_eval(fid, pack(p, d), i, ip, Tx, Ty) for (d, i, ip) in mats)
        dm = [register(sp, fid, p, d, i, ip, cols) for (d, i, ip) in mats]
        assert dev_eval(sp, dm, Tx, Ty) == want, name
        assert dev_eval(sp, dm[2:], Tx, Ty) == want[64:], name
        got = sp.R1CSShape(*dm).multi_evaluate(rx, ry)  # the host form builds both eq tables itself
        assert pack(p, got) == want, name


def big_matrix(rng, p, rows, cols, heavy_at):
    """2^20 rows: one row of 2^20 entries, 2^16 empty rows in a run, the rest 1..4 entries (every class)"""
    import numpy as np
    g = np.random.default_rng(rng.next())
    lens = g.integers(1, 5, size=rows)
    lens[heavy_at] = 1 << 20
    lens[rows // 2:rows // 2 + (1 << 16)] = 0
    indptr = np.concatenate([[0], np.cumsum(lens)])
    nnz = int(indptr[-1])
    indices = g.integers(0, cols, size=nnz)
    indices[:cols] = np.arange(cols)  # the last column of T_y is used
    classes = g.integers(0, 4, size=nnz)
    small = np.array([1, 2, 3, 7], dtype=np.int64)
    data = []
    for c, v in zip(classes, g.integers(0, 1 << 62, size=nnz)):
        if c < 3:
            k = int(small[v % 4])
            data.append(k if v & 1 else p - k)
        else:
            data.append(int(v))
    return data, indices.tolist(), indptr.tolist()


@pytest.mark.parametrize("fid", [0, 1, 2, 3])
def test_r1cs_eval_at_scale(b200, fid):
    """2^20 rows and more than 3 * 2^20 entries per matrix: equal to the C restatement and to the composition it
    replaces (b200_spmv_dev with z = T_y, then the dot with T_x)"""
    from nova_b200 import fields, spartan as sp
    from nova_b200.native import check, lib
    p = FIELD_MODULUS[fid]
    rng = SplitMix64(9600 + fid)
    rows, cols = 1 << 20, 1 << 12
    d, i, ip = big_matrix(rng, p, rows, cols, heavy_at=12345)
    assert len(i) > 3 << 20
    rx, ry = [rng.field(p) for _ in range(20)], [rng.field(p) for _ in range(12)]
    Tx = sp.DeviceVec(32 << 20)
    Ty = sp.DeviceVec(32 << 12)
    rxd, ryd = sp.DeviceVec.from_bytes(fields.pack(fid, rx)), sp.DeviceVec.from_bytes(fields.pack(fid, ry))
    check(lib().b200_eq_table_dev(fid, rxd.ptr, 20, Tx.ptr, None))
    check(lib().b200_eq_table_dev(fid, ryd.ptr, 12, Ty.ptr, None))
    txb, tyb = Tx.to_bytes(), Ty.to_bytes()
    M = register(sp, fid, p, d, i, ip, cols)
    want = verify_ref.r1cs_eval(fid, pack(p, d), i, ip, txb, tyb, nthreads=os.cpu_count() or 1)
    hs = (ctypes.c_uint64 * 1)(M.handle)
    out = sp.DeviceVec(32)
    check(lib().b200_r1cs_eval_dev(hs, 1, Tx.ptr, 1 << 20, Ty.ptr, 1 << 12, out.ptr, None))
    assert out.to_bytes() == want
    Mz, dot = sp.DeviceVec(32 << 20), sp.DeviceVec(32)
    check(lib().b200_spmv_dev(M.handle, Ty.ptr, None, Mz.ptr, None, None))
    check(lib().b200_sc_eval_dev(fid, 11, Mz.ptr, Tx.ptr, None, 1 << 20, None, None, 0, dot.ptr, None))
    assert dot.to_bytes() == want


def test_r1cs_eval_errors_write_nothing(b200):
    from nova_b200 import spartan as sp
    from nova_b200.native import B200_E_ARG, B200_E_HANDLE, B200_E_RANGE, check, lib
    p0, p2 = FIELD_MODULUS[0], FIELD_MODULUS[2]
    rng = SplitMix64(9700)
    d, i, ip = matrix(p0, rng, [2] * 8, 16)
    A = register(sp, 0, p0, d, i, ip, 16)
    B = register(sp, 0, p0, d, i, ip, 16)
    other = register(sp, 2, p2, d, i, ip, 16)
    empty = sp.SparseMatrix(0, b"", [], [0] * 9, 16)
    tx, ty = sp.DeviceVec.from_bytes(bytes(32 * 8)), sp.DeviceVec.from_bytes(bytes(32 * 16))
    out = sp.DeviceVec(96)
    sentinel = b"\xab" * 96
    hs = lambda *h: (ctypes.c_uint64 * 4)(*h)
    cases = [(hs(A.handle, 987654, B.handle), 3, 8, 16, B200_E_HANDLE), (hs(A.handle), 0, 8, 16, B200_E_ARG),
             (hs(A.handle, B.handle, A.handle, B.handle), 4, 8, 16, B200_E_ARG),
             (hs(A.handle, other.handle), 2, 8, 16, B200_E_ARG), (hs(A.handle), 1, 7, 16, B200_E_RANGE),
             (hs(A.handle, B.handle), 2, 8, 15, B200_E_RANGE)]
    for h, k, txl, tyl, code in cases:
        check(lib().b200_memcpy_h2d(out.ptr, ctypes.create_string_buffer(sentinel, 96), 96))
        assert lib().b200_r1cs_eval_dev(h, k, tx.ptr, txl, ty.ptr, tyl, out.ptr, None) == code, (k, txl, tyl)
        check(lib().b200_sync())
        assert out.to_bytes() == sentinel
    r = ctypes.create_string_buffer(32 * 4)
    host_out = ctypes.create_string_buffer(sentinel, 96)
    assert lib().b200_r1cs_eval(hs(A.handle, 987654), 2, r, 3, r, 4, host_out) == B200_E_HANDLE
    assert lib().b200_r1cs_eval(hs(A.handle), 1, r, 2, r, 4, host_out) == B200_E_RANGE
    assert host_out.raw == sentinel
    check(lib().b200_memcpy_h2d(out.ptr, ctypes.create_string_buffer(sentinel, 96), 96))
    check(lib().b200_r1cs_eval_dev(hs(empty.handle), 1, tx.ptr, 8, ty.ptr, 16, out.ptr, None))
    assert out.to_bytes(32) == bytes(32)  # an empty matrix gives 0


def ipa_s_against_weights(fid, L, rng):
    """b200_ipa_s_dev with and without scale against the reference's recurrence (C), and unscaled against the
    prover's weights after all L rounds of b200_ipa_weights_dev"""
    from nova_b200 import fields, spartan as sp
    from nova_b200.native import check, lib
    p = FIELD_MODULUS[fid]
    r = [rng.field(p) for _ in range(L)]
    ri = [pow(x, -1, p) for x in r]
    rd, rid = sp.DeviceVec.from_bytes(fields.pack(fid, r)), sp.DeviceVec.from_bytes(fields.pack(fid, ri))
    n = 1 << L
    w = sp.DeviceVec(32 * n)
    check(lib().b200_ipa_weights_dev(fid, w.ptr, n, 0, None, None, None))
    for k in range(L):
        check(lib().b200_ipa_weights_dev(fid, w.ptr, n, n >> k, ctypes.c_void_p(rd.ptr.value + 32 * k),
                                         ctypes.c_void_p(rid.ptr.value + 32 * k), None))
    for scale in (None, rng.field(p)):
        s = sp.DeviceVec(32 * n)
        sc = sp.DeviceVec.from_bytes(mont_bytes(p, scale)) if scale is not None else None
        check(lib().b200_ipa_s_dev(fid, rd.ptr, rid.ptr, L, sc.ptr if sc else None, s.ptr, None))
        got = s.to_bytes()
        assert got == verify_ref.ipa_s(fid, r, scale), (fid, L, scale is None)
        if scale is None:
            assert got == w.to_bytes(), (fid, L)


def test_ipa_s_equals_reference_and_prover_weights(b200):
    """L = 1 .. 20 in one field; in the other three a size of the direct pass and one past it"""
    from nova_b200 import spartan as sp
    from nova_b200.native import B200_E_ARG, lib
    rng = SplitMix64(9800)
    for L in range(1, 21):
        ipa_s_against_weights(3, L, rng)
    for fid in (0, 1, 2):
        for L in (4, 13):
            ipa_s_against_weights(fid, L, rng)
    s, r = sp.DeviceVec(32), sp.DeviceVec(32 * 32)
    assert lib().b200_ipa_s_dev(0, r.ptr, r.ptr, 32, None, s.ptr, None) == B200_E_ARG
    assert lib().b200_ipa_s_dev(0, r.ptr, r.ptr, -1, None, s.ptr, None) == B200_E_ARG


def test_r1cs_eval_skips_entries_before_indptr0(b200):
    """a registered matrix whose indptr starts above 0: the entries before indptr[0] count for nothing, as in the
    reference's loop over indptr windows (and in b200_spmv_dev); no rows at all gives 0"""
    from nova_b200 import spartan as sp
    from test_verify_kernels_host import offset_matrix
    for fid in (0, 3):
        p = FIELD_MODULUS[fid]
        rng = SplitMix64(9750 + fid)
        d, i, ip = offset_matrix(p, rng, [3, 0, 1, 700, 0, 0, 2, 4], 8, skipped=300)
        Tx, Ty = (pack(p, eq_evals(p, [rng.field(p) for _ in range(3)])) for _ in range(2))
        want = verify_ref.r1cs_eval(fid, pack(p, d), i, ip, Tx, Ty)
        assert dev_eval(sp, [register(sp, fid, p, d, i, ip, 8)], Tx, Ty) == want
        assert dev_eval(sp, [register(sp, fid, p, d[:300], i[:300], [300], 8)], Tx, Ty) == bytes(32)


def test_cpp_mirror_verifier_wrappers(b200):
    """R1CSShape::multi_evaluate (from the points), R1CSShapeDev::multi_evaluate (resident eq tables) and ipa_s with
    and without scale (include/nova_b200.hpp), run from C++, against the C restatement"""
    import struct
    import subprocess
    import tempfile
    fid = 2
    p = FIELD_MODULUS[fid]
    rng = SplitMix64(9990)
    d, i, ip = matrix(p, rng, [1 + rng.next() % 5 for _ in range(16)], 32)
    rx, ry = [rng.field(p) for _ in range(4)], [rng.field(p) for _ in range(5)]
    r = [rng.field(p) for _ in range(11)]
    scale = rng.field(p)
    blob = lambda raw, k: struct.pack("<Q", k) + raw
    u64 = lambda xs: b"".join(struct.pack("<Q", x) for x in xs)
    with tempfile.TemporaryDirectory() as tmp:
        case = os.path.join(tmp, "case")
        with open(case, "wb") as f:
            f.write(blob(pack(p, d), len(d)) + blob(u64(i), len(i)) + blob(u64(ip), len(ip)) + blob(u64([32]), 1)
                    + blob(pack(p, rx), 4) + blob(pack(p, ry), 5) + blob(pack(p, r), 11)
                    + blob(pack(p, [pow(x, -1, p) for x in r]), 11) + blob(pack(p, [scale]), 1))
        subprocess.check_call([verify_ref.cpp_mirror(), case])
        out = open(case + ".out", "rb").read()
    one = verify_ref.r1cs_eval(fid, pack(p, d), i, ip, pack(p, eq_evals(p, rx)), pack(p, eq_evals(p, ry)))
    assert out[:96] == one * 3 and out[96:192] == one * 3
    n = 32 << 11
    assert out[192:192 + n] == verify_ref.ipa_s(fid, r) and out[192 + n:] == verify_ref.ipa_s(fid, r, scale)


@pytest.mark.parametrize("cid", [0, 1, 2, 3])
def test_snark_verify_small_equals_oracle(b200, oracle, cid):
    """device proofs (snark.prove(ee="ipa")) accepted; every tampered field rejected; verdicts equal the oracle's"""
    import test_verify_mirror_cpu as vm
    from nova_b200 import snark
    from oracle import snark_ref as sr
    from oracle.ppsnark_ref import random_instance
    from snark_parity import csr
    c = CURVES[cid]
    p = c.q
    rng = SplitMix64(9900 + cid)
    S, W, u, X = random_instance(p, rng, 16, 8, 2)
    pts = c.bases_arith(17, k0=99)
    ck_pts, ck_c = pts[:16], pts[16]
    U = dict(comm_W=c.msm_naive(W["W"], ck_pts[:8]), comm_E=c.msm_naive(W["E"], ck_pts[:16]), u=u, X=X)
    ck = vm.key(b200, cid, ck_pts, ck_c)
    shape = vm.device_shape(b200, cid, S, 2)
    proof = snark.prove(b200.Curve(cid), ck, shape, U, dict(W=pack(p, W["W"]), E=pack(p, W["E"])), 321,
                        Keccak256Transcript(p, b"RelaxedR1CSSNARK"), ee="ipa")
    proof.pop("batched_poly")
    assert vm.mirror(b200, cid, S, 2, U, proof, ck) is None
    assert vm.oracle_verdict(cid, S, U, proof, ck_pts, ck_c)
    C, x, e = snark.verify_core(b200.Curve(cid), shape, U, 321, proof, Keccak256Transcript(p, b"RelaxedR1CSSNARK"))
    assert (C, x, e) == sr.verify_core(p, c, S, U, 321, proof)
    for field in ("sc_outer", "claims_outer", "eval_E", "eval_W", "evals_batch", "L_vec", "R_vec", "a_hat"):
        bad = vm.tampered(proof, field, p)
        assert vm.mirror(b200, cid, S, 2, U, bad, ck) is not None, field
        assert not vm.oracle_verdict(cid, S, U, bad, ck_pts, ck_c), field


def _replay():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import verify_replay
    return verify_replay


@pytest.mark.parametrize("cid", [1, 3])
def test_snark_verify_at_2_16(b200, cid):
    """2^16 constraints, 2^17 witness variables, a setup_synthetic key: the device proof is accepted, a_hat + 1 and an
    altered eval_W are rejected"""
    vr = _replay()
    inst = vr.build(cid, 16)
    ck = vr.key_for(inst["curve"], inst["S"]["num_vars"])
    U, proof = vr.prove(inst, ck)
    vr.verify(inst, ck, U, proof)
    L_vec, R_vec, a_hat = proof["eval_arg"]
    with pytest.raises(ValueError, match="InvalidPCS"):
        vr.verify(inst, ck, U, dict(proof, eval_arg=(L_vec, R_vec, (a_hat + 1) % inst["p"])))
    with pytest.raises(ValueError, match="InvalidSumcheckProof"):
        vr.verify(inst, ck, U, dict(proof, eval_W=(proof["eval_W"] + 1) % inst["p"]))
    ck.release()


def test_verify_core_with_oracle_hyperkzg(b200, oracle):
    """BN254 + HyperKZG: the device verify_core's claim and transcript, finished by the oracle's HyperKZG check with
    the known tau of the test SRS"""
    from nova_b200 import snark
    from oracle import hyperkzg_ref as hk
    from oracle.ppsnark_ref import random_instance
    import test_verify_mirror_cpu as vm
    cid = 0
    c = CURVES[cid]
    p = c.q
    rng = SplitMix64(9950)
    S, W, u, X = random_instance(p, rng, 16, 16, 2)
    tau = rng.field(p)
    srs = hk.setup_srs(cid, 16, tau)
    commit = lambda v: c.affine_from_bytes(oracle.msm(cid, pack(p, v), srs[:64 * len(v)]))
    U = dict(comm_W=commit(W["W"]), comm_E=commit(W["E"]), u=u, X=X)
    ck = b200.CommitmentKey(b200.Curve(cid), srs)
    shape = vm.device_shape(b200, cid, S, 2)
    proof = snark.prove(b200.Curve(cid), ck, shape, U, dict(W=pack(p, W["W"]), E=pack(p, W["E"])), 77,
                        Keccak256Transcript(p, b"RelaxedR1CSSNARK"))
    tr = Keccak256Transcript(p, b"RelaxedR1CSSNARK")
    C, x, e = snark.verify_core(b200.Curve(cid), shape, U, 77, proof, tr)
    assert hk.verify(cid, tau, C, x, e, proof["eval_arg"], tr)
    with pytest.raises(ValueError):
        snark.verify(b200.Curve(cid), shape, U, 77, proof, Keccak256Transcript(p, b"RelaxedR1CSSNARK"), ee="hyperkzg",
                     ck=ck)


@pytest.mark.parametrize("cid", [1, 3])
def test_ipa_verify_at_point_opens_ppsnark_at_2_18(b200, cid):
    """The IPA half of ppsnark + IPA at N = 2^18 (Grumpkin, Vesta): the device proof of ppsnark.prove(ee="ipa"), its
    batched instance (C, r_inner_batched, e) re-derived by the restated verifier core of tests/ppsnark_ipa_ref.py
    (oracle/ppsnark_ref.verify_core, then the batched commitment over the 15 commitments), opened by
    ipa.verify_at_point on the device; a_hat + 1 is rejected with InvalidPCS"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import spark_ipa_replay as sir
    from nova_b200 import ipa, ppsnark as dp
    from nova_b200.transcript import Keccak256Transcript
    from oracle import ppsnark_ref as pr
    inst = sir.build(cid, 16)
    curve, fid, p, S = inst["curve"], inst["fid"], inst["p"], inst["S"]
    N = dp.SparkRepr.from_shape(fid, S).N
    assert N == 1 << 18
    ck = sir.key_for(curve, N)
    spark, S_comm = dp.setup(curve, ck, S)
    U = dict(comm_W=dp.commit_dev(curve, ck, inst["W"], S["num_vars"]),
             comm_E=dp.commit_dev(curve, ck, inst["E"], S["num_cons"]), u=inst["u"], X=inst["X"])
    proof = dp.prove(curve, ck, S, spark, U, dict(W=inst["W"], E=inst["E"]), sir.VK_DIGEST,
                     Keccak256Transcript(p, b"RelaxedR1CSSNARK"), ee="ipa", S_comm=S_comm)

    def batched_instance():  # the verifier of tests/ppsnark_ipa_ref.verify_ipa up to its ipa_verify call
        holder = {}
        assert pr.verify_core(p, S["num_cons"], S["num_vars"], N, U, sir.VK_DIGEST, proof, holder)
        tr = holder["tr"]
        eval_vec = [proof[k] for k in pr.EVAL_ORDER]
        tr.absorb_bytes(b"e", pr.scalars_bytes(eval_vec))
        c = tr.squeeze(b"c")
        C = pr.batch_commitment(p, CURVES[cid], pr.comm_vec_of(U, S_comm, proof), c)
        return C, proof["r_inner_batched"], sum(pow(c, i, p) * v for i, v in enumerate(eval_vec)) % p, tr

    C, x, e, tr = batched_instance()
    assert len(x) == 18
    assert ipa.verify_at_point(curve, ck, C, x, e, proof["eval_arg"], tr) is None
    L_vec, R_vec, a_hat = proof["eval_arg"]
    C, x, e, tr = batched_instance()
    with pytest.raises(ValueError, match="InvalidPCS"):
        ipa.verify_at_point(curve, ck, C, x, e, (L_vec, R_vec, (a_hat + 1) % p), tr)
    ck.release()
