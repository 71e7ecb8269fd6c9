"""Shared bodies of the ppsnark setup + IPA checks (GPU: tests/test_spark_ipa_gpu.py; CPU with the emulated device:
tests/test_spark_ipa_mirror_cpu.py): SparkRepr.from_shape against oracle/ppsnark_ref.SparkRepr, setup's S_comm
against the oracle's commitments, and ppsnark.prove(ee="ipa") field for field against ppsnark_ipa_ref.prove_ipa,
pinned by the restated verifier ppsnark_ipa_ref.verify_ipa (tests/test_oracle_ppsnark_ipa.py)."""
import copy

import ppsnark_ipa_ref as ipr
from oracle import ppsnark_ref as pr
from oracle.pyref import CURVES, Keccak256Transcript, SplitMix64, mont_bytes
from snark_parity import csr

SPARK_NAMES = ("row", "col", "val_A", "val_B", "val_C", "ts_row", "ts_col")


def pack(p, xs):
    return b"".join(mont_bytes(p, x) for x in xs)


def u32(xs):
    return b"".join(int(x).to_bytes(4, "little") for x in xs)


# ---- shapes for the setup checks: (num_cons, num_vars, ncols, rows holding entries of A / B / C, entries per row) --
def shape(p, kind: str, seed: int = 0):
    """-> (A, B, C triplet lists in CSR order, num_cons, num_vars, ncols) for one of SHAPES; N = next_pow2(max(nnz,
    2 num_vars, num_cons)) is set by the named quantity or has the named property."""
    rng = SplitMix64(4400 + seed + 17 * SHAPES.index(kind))
    nc, nv, ncols, rows, per = {
        "by_nnz": (8, 4, 7, [range(8)] * 3, (3, 3, 1)),                       # 56 entries -> N = 64
        "by_num_vars": (4, 32, 35, [range(4)] * 3, (1, 1, 1)),                # N = 2 num_vars = 64
        "by_num_cons": (64, 4, 7, [range(1, 64, 4)] * 3, (1, 1, 1)),          # empty rows (row 0 and the last too)
        "no_padding": (8, 4, 7, [range(8), range(0, 8, 2), range(1, 8, 2)], (1, 1, 1)),  # nnz == N == 16
        "cols_eq_N": (8, 8, 16, [range(8), range(0, 8, 2), range(1, 8, 4)], (1, 1, 1)),  # ncols == N == 16, col N - 1
        "empty_B": (8, 8, 10, [range(8), range(0), range(8)], (1, 0, 2)),     # nnz_B == 0
    }[kind]

    def mat(rs, k):
        out = []
        for r in rs:
            cols = set()
            while len(cols) < k:
                cols.add(ncols - 1 if not cols and r % 3 == 0 else rng.next() % ncols)  # the last column often
            for c in sorted(cols):
                out.append((r, c, [1, p - 1, 2, rng.field(p)][rng.next() % 4]))
        return out
    A, B, C = (mat(rs, k) for rs, k in zip(rows, per))
    return A, B, C, nc, nv, ncols


SHAPES = ["by_nnz", "by_num_vars", "by_num_cons", "no_padding", "cols_eq_N", "empty_B"]


def register(sp, fid, p, A, B, C, nc, ncols) -> dict:
    mats = {}
    for name, M in zip("ABC", (A, B, C)):
        d, idx, ptr = csr(M, nc)
        mats[name] = sp.SparseMatrix(fid, pack(p, d), idx, ptr, ncols)
    return mats


def check_from_shape(nb, cid, kind):
    """the nine device vectors of SparkRepr.from_shape are byte-equal to the oracle's SparkRepr"""
    from nova_b200 import ppsnark as dp
    from nova_b200 import spartan as sp
    c = CURVES[cid]
    fid, p = c.scalar_field, c.q
    A, B, C, nc, nv, ncols = shape(p, kind, cid)
    ref = pr.SparkRepr(p, A, B, C, nc, nv)
    mats = register(sp, fid, p, A, B, C, nc, ncols)
    got = dp.SparkRepr.from_shape(fid, dict(num_cons=nc, num_vars=nv, **mats))
    N = ref.N
    assert got.N == N, kind
    if kind == "no_padding":
        assert ref.nnz == N
    if kind == "cols_eq_N":
        assert ncols == N and (N - 1) in ref.col[:ref.nnz]
    for name in SPARK_NAMES:
        assert getattr(got, name).to_bytes(32 * N) == pack(p, getattr(ref, name)), (kind, name)
    assert got.row_idx.to_bytes(4 * N) == u32(ref.row_idx), kind
    assert got.col_idx.to_bytes(4 * N) == u32(ref.col_idx), kind


def check_setup_commitments(nb, oracle, cid, kind="by_nnz"):
    """setup's S_comm equals the oracle's shape_commitments, each an MSM of the C oracle over the exported key"""
    from nova_b200 import ppsnark as dp
    from nova_b200 import spartan as sp
    c = CURVES[cid]
    fid, p = c.scalar_field, c.q
    A, B, C, nc, nv, ncols = shape(p, kind, cid)
    ref = pr.SparkRepr(p, A, B, C, nc, nv)
    mats = register(sp, fid, p, A, B, C, nc, ncols)
    ck = nb.CommitmentKey(nb.Curve(cid), oracle.gen_bases(cid, ref.N))
    bases = ck.export_bases(0, ref.N)
    spark, S_comm = dp.setup(nb.Curve(cid), ck, dict(num_cons=nc, num_vars=nv, **mats))
    assert set(S_comm) == set(dp.SHAPE_COMMITMENTS)
    exp = pr.shape_commitments(lambda v: c.affine_from_bytes(oracle.msm(cid, pack(p, v), bases[:64 * len(v)])), ref)
    assert S_comm == exp, kind
    ck.release()


# ---- the whole proof ---------------------------------------------------------------------------------------------
_REF = {}


def instance(cid, num_cons=8, num_vars=8, num_io=2):
    """a random satisfying instance, its Pedersen key (pyref's bases_arith, ck_c the last point) and the oracle's
    prove_ipa proof (cached per curve)"""
    key = (cid, num_cons, num_vars, num_io)
    if key not in _REF:
        c = CURVES[cid]
        p = c.q
        rng = SplitMix64(5100 + cid + num_cons)
        S, W, u, X = pr.random_instance(p, rng, num_cons, num_vars, num_io)
        spark_ref = pr.SparkRepr(p, S["A"], S["B"], S["C"], num_cons, num_vars)
        N = spark_ref.N
        pts = c.bases_arith(N + 1, k0=5151 + cid)
        ck_pts, ck_c = pts[:N], pts[N]
        commit = lambda v: c.msm_naive(v, ck_pts[:len(v)])
        U = dict(comm_W=commit(W["W"]), comm_E=commit(W["E"]), u=u, X=X)
        S_comm = pr.shape_commitments(commit, spark_ref)
        ref = ipr.prove_ipa(p, c, ck_pts, ck_c, S, spark_ref, U, W, 909, S_comm)
        _REF[key] = dict(S=S, W=W, U=U, N=N, ck_pts=ck_pts, ck_c=ck_c, S_comm=S_comm, ref=ref, ncols=num_vars + 1 + num_io)
    return _REF[key]


PROOF_FIELDS = ["comm_L_row", "comm_L_col", "comm_mem", "sc_outer", "r_outer", "eval_Az_at_r_outer",
                "eval_Bz_at_r_outer", "eval_Cz_at_r_outer", "eval_E_at_r_outer", "sc_inner_batched",
                "r_inner_batched", "batched_eval", "batch_challenge"] + pr.EVAL_ORDER


def run_prove(nb, cid, device_transcript):
    """setup + prove(ee="ipa") on the device equals prove_ipa field for field, leaves the transcript in the same
    state, and passes verify_ipa; an altered eval_W, L_vec[0] or a_hat is rejected"""
    from nova_b200 import ppsnark as dp
    from nova_b200 import spartan as sp
    c = CURVES[cid]
    fid, p = c.scalar_field, c.q
    inst = instance(cid)
    S, W, U, N, ref = inst["S"], inst["W"], inst["U"], inst["N"], inst["ref"]
    nc, nv = S["num_cons"], S["num_vars"]
    mats = register(sp, fid, p, S["A"], S["B"], S["C"], nc, inst["ncols"])
    ck = nb.CommitmentKey(nb.Curve(cid), b"".join(c.affine_bytes(P) for P in inst["ck_pts"]), c.affine_bytes(inst["ck_c"]))
    spark, S_comm = dp.setup(nb.Curve(cid), ck, dict(num_cons=nc, num_vars=nv, **mats))
    assert S_comm == inst["S_comm"]
    tr = Keccak256Transcript(p, b"RelaxedR1CSSNARK")
    got = dp.prove(nb.Curve(cid), ck, dict(num_cons=nc, num_vars=nv, **mats), spark, U,
                   dict(W=pack(p, W["W"]), E=pack(p, W["E"])), 909, tr, device_transcript=device_transcript, ee="ipa",
                   S_comm=S_comm)
    for k in PROOF_FIELDS:
        assert got[k] == ref[k], k
    assert tuple(got["eval_arg"]) == tuple(ref["eval_arg"])
    assert tr.squeeze(b"x") == copy.deepcopy(ref["transcript"]).squeeze(b"x")  # the cached proof stays as it is
    verify = lambda proof: ipr.verify_ipa(p, c, inst["ck_pts"], inst["ck_c"], nc, nv, N, U, S_comm, 909, proof)
    assert verify(got)
    L_vec, R_vec, a_hat = got["eval_arg"]
    assert not verify(dict(got, eval_W=(got["eval_W"] + 1) % p))
    assert not verify(dict(got, eval_arg=([R_vec[0]] + list(L_vec[1:]), R_vec, a_hat)))
    assert not verify(dict(got, eval_arg=(L_vec, R_vec, (a_hat + 1) % p)))
    ck.release()
