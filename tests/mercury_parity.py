"""Shared bodies of the Mercury checks (GPU: tests/test_mercury_gpu.py; CPU with the emulated device:
tests/test_mercury_mirror_cpu.py): the three Mercury entry points against the oracle, nova_b200.mercury's
proof field for field against oracle/mercury_ref.py (pinned by the restated verifier,
tests/test_oracle_mercury.py), and the two SNARKs with ee="mercury" against the oracle composition."""
import numpy as np

from oracle import hyperkzg_ref as hk
from oracle import mercury_ref as mr
from oracle import ppsnark_ref as pr
from oracle import snark_ref as sr
from oracle.ppsnark_ref import random_instance
from oracle.pyref import CURVES, Keccak256Transcript, SplitMix64, from_mont_bytes, mle_evaluate, mont_bytes
from snark_parity import csr

CID = 0


def pack(p, xs):
    return b"".join(mont_bytes(p, x) for x in xs)


def ints(p, b: bytes):
    return [from_mont_bytes(p, b[i:i + 32]) for i in range(0, len(b), 32)]


def _dev(sp, b: bytes):
    return sp.DeviceVec.from_bytes(b)


# ---- the kernels ------------------------------------------------------------------------------------------
def div_binomial_oracle(oracle, fid, f: bytes, rows, cols, alpha: bytes):
    """per column: the C oracle's quotient by (Y - alpha) and its value at alpha -> (q row-major, g) bytes"""
    m = np.frombuffer(f, dtype=np.uint8).reshape(rows, cols, 32)
    q = np.zeros((max(rows - 1, 0), cols, 32), dtype=np.uint8)
    g = []
    for c in range(cols):
        col = m[:, c, :].tobytes()
        if rows > 1:
            q[:, c, :] = np.frombuffer(oracle.poly_div(fid, col, alpha), dtype=np.uint8).reshape(rows - 1, 32)
        g.append(oracle.poly_eval(fid, col, alpha))
    return q.tobytes(), b"".join(g)


def div_binomial_device(sp, fid, f: bytes, rows, cols, alpha: bytes):
    from nova_b200.native import check, lib
    df, da = _dev(sp, f), _dev(sp, alpha)
    q, g = sp.DeviceVec(32 * max((rows - 1) * cols, 1)), sp.DeviceVec(32 * cols)
    check(lib().b200_div_binomial_dev(fid, df.ptr, rows, cols, da.ptr, q.ptr, g.ptr, None))
    check(lib().b200_sync())
    return q.to_bytes(32 * (rows - 1) * cols), g.to_bytes(32 * cols)


def check_div_binomial(sp, oracle, rows, cols, kind="random", seed=0):
    c = CURVES[CID]
    fid, p = c.scalar_field, c.q
    n = rows * cols
    if kind == "random":
        f = oracle.gen_scalars(fid, 9000 + seed + rows + 7 * cols, n)
    elif kind == "zero":
        f = bytes(32 * n)
    else:  # only the last row non-zero: its carry has to cross every chunk of every column
        f = bytes(32 * (n - cols)) + oracle.gen_scalars(fid, 9100 + rows + cols, cols)
    alpha = mont_bytes(p, SplitMix64(9200 + rows + cols + seed).field(p))
    assert div_binomial_device(sp, fid, f, rows, cols, alpha) == div_binomial_oracle(oracle, fid, f, rows, cols, alpha), \
        (rows, cols, kind)


def check_mat_vec_rows(sp, oracle, rows, cols):
    from nova_b200.native import check, lib
    c = CURVES[CID]
    fid, p = c.scalar_field, c.q
    f, v = oracle.gen_scalars(fid, 9300 + rows, rows * cols), oracle.gen_scalars(fid, 9400 + cols, cols)
    if rows * cols <= 4096:
        exp = pack(p, mr.compute_h_poly(p, ints(p, f), ints(p, v), rows, cols))
    else:  # the same sums by the C oracle: the columns of f combined with the entries of v as coefficients
        m = np.frombuffer(f, dtype=np.uint8).reshape(rows, cols, 32)
        exp = oracle.rlc(fid, [m[:, c, :].tobytes() for c in range(cols)], v, rows)
    df, dv, out = _dev(sp, f), _dev(sp, v), sp.DeviceVec(32 * rows)  # held until the launch is done
    check(lib().b200_mat_vec_rows_dev(fid, df.ptr, rows, cols, dv.ptr, out.ptr, None))
    assert out.to_bytes(32 * rows) == exp, (rows, cols)


def check_s_poly(sp, oracle, b):
    from nova_b200.native import check, lib
    c = CURVES[CID]
    fid, p = c.scalar_field, c.q
    rng = SplitMix64(9500 + b)
    vs = [[rng.field(p) for _ in range(b)] for _ in range(4)]
    gamma = rng.field(p)
    exp = pack(p, mr.s_poly_direct(p, *vs, gamma))
    ds = [_dev(sp, pack(p, v)) for v in vs]
    dg, out = _dev(sp, mont_bytes(p, gamma)), sp.DeviceVec(32 * (b - 1))
    check(lib().b200_mercury_s_poly_dev(fid, ds[0].ptr, ds[1].ptr, ds[2].ptr, ds[3].ptr, b, dg.ptr, out.ptr, None))
    assert out.to_bytes(32 * (b - 1)) == exp, b
    if b <= 64:  # and the reference's NTT route agrees (any root of unity)
        assert mr.trim(mr.s_poly_direct(p, *vs, gamma)) == mr.make_s_polynomial(p, (vs[0], vs[2]), (vs[1], vs[3]),
                                                                                 b.bit_length() - 1, gamma)


# ---- the whole evaluation argument ------------------------------------------------------------------------
_SRS = {}


def srs_for(n):
    c = CURVES[CID]
    if n not in _SRS:
        tau = SplitMix64(4242).field(c.q)
        _SRS[n] = (tau, hk.setup_srs(CID, n, tau))
    return _SRS[n]


def run_prove(nb, oracle, ell, verify=True):
    """mercury_prove == mercury_ref.prove field for field, same final transcript state, and the restated
    verifier accepts (C from the C oracle)."""
    from nova_b200 import mercury as dm
    c = CURVES[CID]
    fid, p = c.scalar_field, c.q
    n = 1 << ell
    tau, srs = srs_for(n)
    f = oracle.gen_scalars(fid, 7000 + ell, n)
    rng = SplitMix64(7100 + ell)
    x = [rng.field(p) for _ in range(ell)]
    C = c.affine_from_bytes(oracle.msm(CID, f, srs))
    y = mle_evaluate(p, ints(p, f), x)
    ck = nb.CommitmentKey(nb.Curve(CID), srs)
    tg, tr_ = Keccak256Transcript(p, b"TestEval"), Keccak256Transcript(p, b"TestEval")
    got = dm.mercury_prove(nb.Curve(CID), ck, f, x, tg, comm=C, eval_=y)
    ref = mr.prove(CID, srs, f, x, tr_, comm=C, eval_=y)
    for name, a, b in zip(mr.FIELDS, got, ref):
        assert a == b, (ell, name)
    assert tg.squeeze(b"s") == tr_.squeeze(b"s")
    if verify:
        assert mr.verify(CID, tau, C, x, y, tuple(got), Keccak256Transcript(p, b"TestEval"))
    ck.release()


def run_verify_only(nb, oracle, ell):
    """The device proof at benchmark-like size is accepted by the restated verifier (C by the C oracle's MSM);
    the claimed evaluation comes from the device (the verifier then pins it)."""
    from nova_b200 import mercury as dm
    c = CURVES[CID]
    fid, p = c.scalar_field, c.q
    n = 1 << ell
    ck = nb.CommitmentKey.setup_tau(nb.Curve(CID), n, 0x1234567890ABCDEF)
    srs = ck.export_bases(0, n)
    f = oracle.gen_scalars(fid, 7200 + ell, n)
    rng = SplitMix64(7300 + ell)
    x = [rng.field(p) for _ in range(ell)]
    C = c.affine_from_bytes(oracle.msm(CID, f, srs))
    proof = dm.mercury_prove(nb.Curve(CID), ck, f, x, Keccak256Transcript(p, b"TestEval"), comm=C)
    from nova_b200 import spartan as sp
    df, dx = sp.DeviceVec.from_bytes(f), sp.DeviceVec.from_bytes(pack(p, x))
    y, = sp.mle_eval_multi_dev(fid, [df], ell, dx)
    assert mr.verify(CID, 0x1234567890ABCDEF, C, x, y, tuple(proof), Keccak256Transcript(p, b"TestEval"))
    assert not mr.verify(CID, 0x1234567890ABCDEF, C, x, (y + 1) % p, tuple(proof), Keccak256Transcript(p, b"TestEval"))
    ck.release()


# ---- the SNARKs with ee="mercury" -------------------------------------------------------------------------
def _compare(got, ref):
    for name, a, b in zip(mr.FIELDS, got, ref):
        assert a == b, name


def run_snark(nb, oracle, num_cons=8, num_vars=8, num_io=2, device_transcript=True):
    from nova_b200 import snark as ds
    from nova_b200 import spartan as sp
    c = CURVES[CID]
    fid, p = c.scalar_field, c.q
    rng = SplitMix64(2500 + num_cons + num_vars)
    S, W, u, X = random_instance(p, rng, num_cons, num_vars, num_io)
    tau = rng.field(p)
    srs = hk.setup_srs(CID, max(num_cons, num_vars), tau)

    def commit_ref(v):
        return c.affine_from_bytes(oracle.msm(CID, pack(p, v), srs[:64 * len(v)]))
    U = dict(comm_W=commit_ref(W["W"]), comm_E=commit_ref(W["E"]), u=u, X=X)
    ref = sr.prove_core(p, c, S, U, W, 555)
    ref["eval_arg"] = mr.prove(CID, srs, pack(p, ref["batched_poly"]), ref["batched_x"], ref["transcript"],
                               comm=ref["batched_c"], eval_=ref["batched_e"])
    mats = {}
    for name in "ABC":
        d, idx, ptr = csr(S[name], num_cons)
        mats[name] = sp.SparseMatrix(fid, pack(p, d), idx, ptr, num_vars + 1 + num_io)
    ck = nb.CommitmentKey(nb.Curve(CID), srs)
    tr = Keccak256Transcript(p, b"RelaxedR1CSSNARK")
    got = ds.prove(nb.Curve(CID), ck, dict(num_cons=num_cons, num_vars=num_vars, **mats), U,
                   dict(W=pack(p, W["W"]), E=pack(p, W["E"])), 555, tr, device_transcript=device_transcript,
                   ee="mercury")
    _compare(got["eval_arg"], ref["eval_arg"])
    assert tr.squeeze(b"x") == ref["transcript"].squeeze(b"x")
    holder = {}
    C, x, e = sr._verify_core_with_transcript(p, c, S, U, 555, got, holder)
    assert mr.verify(CID, tau, C, x, e, tuple(got["eval_arg"]), holder["tr"])
    holder = {}
    C, x, e = sr._verify_core_with_transcript(p, c, S, U, 555, got, holder)
    assert not mr.verify(CID, tau, C, x, (e + 1) % p, tuple(got["eval_arg"]), holder["tr"])
    ck.release()


def run_ppsnark(nb, oracle, num_cons=8, num_vars=8, device_transcript=False):
    from nova_b200 import ppsnark as dp
    from nova_b200 import spartan as sp
    c = CURVES[CID]
    fid, p = c.scalar_field, c.q
    rng = SplitMix64(3500 + num_cons)
    S, W, u, X = pr.random_instance(p, rng, num_cons, num_vars, num_io=2)
    spark_ref = pr.SparkRepr(p, S["A"], S["B"], S["C"], num_cons, num_vars)
    N = spark_ref.N
    tau = rng.field(p)
    srs = hk.setup_srs(CID, N, tau)

    def commit_ref(v):
        return c.affine_from_bytes(oracle.msm(CID, pack(p, v), srs[:64 * len(v)]))
    U = dict(comm_W=commit_ref(W["W"]), comm_E=commit_ref(W["E"]), u=u, X=X)
    S_comm = pr.shape_commitments(commit_ref, spark_ref)
    ref = pr.prove_core(p, commit_ref, S, spark_ref, U, W, 4711)
    C_ref = pr.batch_commitment(p, c, pr.comm_vec_of(U, S_comm, ref), ref["batch_challenge"])
    ref["eval_arg"] = mr.prove(CID, srs, pack(p, ref["batched_poly"]), ref["r_inner_batched"], ref["transcript"],
                               comm=C_ref, eval_=ref["batched_eval"])
    ck = nb.CommitmentKey(nb.Curve(CID), srs)
    mats = {}
    for name in "ABC":
        d, idx, ptr = csr(S[name], num_cons)
        mats[name] = sp.SparseMatrix(fid, pack(p, d), idx, ptr, num_vars + 1 + len(X))
    spark = dp.SparkRepr(fid, S["A"], S["B"], S["C"], num_cons, num_vars)
    tr = Keccak256Transcript(p, b"RelaxedR1CSSNARK")
    got = dp.prove(nb.Curve(CID), ck, dict(num_cons=num_cons, num_vars=num_vars, **mats), spark, U,
                   dict(W=pack(p, W["W"]), E=pack(p, W["E"])), 4711, tr, device_transcript=device_transcript,
                   ee="mercury", S_comm=S_comm)
    _compare(got["eval_arg"], ref["eval_arg"])
    assert tr.squeeze(b"x") == ref["transcript"].squeeze(b"x")
    for y_off, ok in ((0, True), (1, False)):  # the restated ppsnark verifier, then Mercury's on its claim
        holder = {}
        pr.verify_core(p, num_cons, num_vars, N, U, 4711, got, holder)
        vt = holder["tr"]
        eval_vec = [got[k] for k in pr.EVAL_ORDER]
        vt.absorb_bytes(b"e", pr.scalars_bytes(eval_vec))
        cc = vt.squeeze(b"c")
        C = pr.batch_commitment(p, c, pr.comm_vec_of(U, S_comm, got), cc)
        e = (sum(pow(cc, i, p) * v for i, v in enumerate(eval_vec)) + y_off) % p
        assert mr.verify(CID, tau, C, got["r_inner_batched"], e, tuple(got["eval_arg"]), vt) == ok
    ck.release()
