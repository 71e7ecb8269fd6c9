"""Host-pointer forms of the field / polynomial entries against their `_dev` twins.

Every host form stages its arguments through the device and calls its `_dev` twin.  Here each one runs on seeded
inputs next to a direct call of the twin on `DeviceVec` copies of the same inputs, in all four fields and at edge
sizes (empty or minimal, 1, odd, past 2^16); status and output bytes must agree.  Output buffers start as a fill
pattern, so bytes a form must not write are checked as well.  A table of argument errors pins the status codes.
"""
import ctypes
import random

import pytest

from nova_b200.native import lib
from nova_b200.spartan import DeviceVec, SparseMatrix

pytestmark = pytest.mark.gpu

FIDS = [0, 1, 2, 3]
OK, E_ARG, E_HANDLE, E_RANGE, E_ZERO = 0, 1, 3, 5, 6
FILL = b"\xa5"
P, U64, SZ = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_size_t


def hbuf(b: bytes):
    """A writable host copy of b (never a null pointer, even when empty)."""
    return (ctypes.c_char * max(len(b), 1)).from_buffer_copy(b or b"\0")


def vec(oracle, fid, seed, n):
    return oracle.gen_scalars(fid, seed, n) if n else b""


def parity(host, dev, ins, outs):
    """host(in_ptrs, out_ptrs) and dev(in_ptrs, out_ptrs) on copies of `ins` (bytes or None).  `outs` holds the byte
    count of each output, or (host bytes, device bytes) where the device form writes more than the host form returns.
    Both calls must return the same status and the same visible bytes; the host buffer past its bytes stays untouched."""
    sizes = [o if isinstance(o, tuple) else (o, o) for o in outs]
    hi = [None if b is None else hbuf(b) for b in ins]
    ho = [hbuf(FILL * d) for _, d in sizes]
    di = [None if b is None else DeviceVec.from_bytes(b) for b in ins]
    do = [DeviceVec.from_bytes(FILL * d) for _, d in sizes]
    rh = host(hi, ho)
    rd = dev([None if v is None else v.ptr for v in di], [v.ptr for v in do])
    assert rh == rd
    for (h, d), hb, dv in zip(sizes, ho, do):
        assert hb.raw[:h] == dv.to_bytes(h)
        assert hb.raw[h:d] == FILL * (d - h)
    return rh


def ptrs(vs):
    """A C array of pointers to the buffers `vs`; it keeps them alive."""
    arr = (P * max(len(vs), 1))(*[ctypes.cast(v, P) if v is not None else None for v in vs])
    arr.keep = list(vs)
    return arr


# ---- elementwise vector forms ---------------------------------------------------------------------------------
SIZES = [0, 1, 33, 65537]


@pytest.mark.parametrize("fid", FIDS)
@pytest.mark.parametrize("n", SIZES)
def test_vector_forms(b200, oracle, fid, n):
    L = lib()
    v = [vec(oracle, fid, 10 * k + n, n) for k in range(5)]
    r = vec(oracle, fid, 7, 1)
    for e2 in (None, v[4]):
        assert parity(lambda i, o: L.b200_cross_term(fid, *i, n, o[0]),
                      lambda i, o: L.b200_cross_term_dev(fid, *i, n, o[0], None),
                      [v[0], v[1], v[2], v[3], e2, r], [32 * n]) == OK
    assert parity(lambda i, o: L.b200_axpy(fid, *i, n, o[0]), lambda i, o: L.b200_axpy_dev(fid, *i, n, o[0], None),
                  [v[0], v[1], r], [32 * n]) == OK
    assert parity(lambda i, o: L.b200_vec_add(fid, *i, n, o[0]),
                  lambda i, o: L.b200_vec_add_dev(fid, *i, n, o[0], None), [v[0], v[1]], [32 * n]) == OK
    assert parity(lambda i, o: L.b200_lerp(fid, *i, n, o[0]), lambda i, o: L.b200_lerp_dev(fid, *i, n, o[0], None),
                  [v[0], v[1], r], [32 * n]) == OK


@pytest.mark.parametrize("fid", FIDS)
@pytest.mark.parametrize("n", [0, 2, 34, 65538])
def test_bind_top_in_place(b200, oracle, fid, n):
    z, r = vec(oracle, fid, 3 + n, n), vec(oracle, fid, 4, 1)
    hz = hbuf(z)
    assert lib().b200_bind_top(fid, hz, n, hbuf(r)) == OK
    dz, dr = DeviceVec.from_bytes(z), DeviceVec.from_bytes(r)
    assert lib().b200_bind_top_dev(fid, dz.ptr, n, dr.ptr, None) == OK
    half = 16 * n if n >= 2 else 0
    assert hz.raw[:half] == dz.to_bytes(half)
    assert hz.raw[half:32 * n] == z[half:]  # the upper half of the host buffer is left as it was


@pytest.mark.parametrize("fid", FIDS)
@pytest.mark.parametrize("n", [0, 1, 33, 65537])
def test_poseidon_ro(b200, oracle, fid, n):
    from nova_b200.poseidon import PoseidonConstants
    h = PoseidonConstants.get(fid).handle
    L = lib()
    for num_bits, one in ((128, 0), (250, 1)):
        assert parity(lambda i, o: L.b200_poseidon_ro(h, i[0], n, num_bits, one, o[0]),
                      lambda i, o: L.b200_poseidon_ro_dev(h, i[0], n, num_bits, one, o[0], None),
                      [vec(oracle, fid, 5 + n, n)], [96]) == OK


# ---- sum-check, eq, MLE, inversion ------------------------------------------------------------------------------
@pytest.mark.parametrize("fid", FIDS)
def test_sc_eval(b200, oracle, fid):
    L = lib()
    nout = {0: 2, 3: 3, 10: 1, 11: 1}
    cases = [(form, ln) for form in (0, 3) for ln in (0, 2, 34, (1 << 17) + 2)]
    cases += [(11, ln) for ln in (0, 1, 33, 65537)] + [(10, 1 << ell) for ell in (0, 1, 17)]
    for form, ln in cases:
        A, B, C = (vec(oracle, fid, 20 + k + ln, ln) for k in range(3))
        B = None if form == 10 else B
        C = C if form == 3 else None
        shift = (ln.bit_length() - 1) // 2 if form == 10 else 0
        el = vec(oracle, fid, 30, ln >> shift) if form == 10 else None
        er = vec(oracle, fid, 31, 1 << shift) if form == 10 else None
        nl, nr = (ln >> shift, 1 << shift) if form == 10 else (0, 0)
        assert parity(lambda i, o: L.b200_sc_eval(fid, form, i[0], i[1], i[2], ln, i[3], nl, i[4], nr, shift, o[0]),
                      lambda i, o: L.b200_sc_eval_dev(fid, form, *i[:3], ln, i[3], i[4], shift, o[0], None),
                      [A, B, C, el, er], [(32 * nout[form], 96)]) == OK


@pytest.mark.parametrize("fid", FIDS)
@pytest.mark.parametrize("ell", [0, 1, 11, 17])
def test_eq_table_and_mle_eval(b200, oracle, fid, ell):
    L = lib()
    r, Z = vec(oracle, fid, 40 + ell, ell), vec(oracle, fid, 41 + ell, 1 << ell)
    assert parity(lambda i, o: L.b200_eq_table(fid, i[0], ell, o[0]),
                  lambda i, o: L.b200_eq_table_dev(fid, i[0], ell, o[0], None), [r], [32 << ell]) == OK
    assert parity(lambda i, o: L.b200_mle_eval(fid, i[0], ell, i[1], o[0]),
                  lambda i, o: L.b200_mle_eval_dev(fid, i[0], ell, i[1], o[0], None), [Z, r], [32]) == OK


@pytest.mark.parametrize("fid", FIDS)
@pytest.mark.parametrize("n", SIZES)
def test_batch_invert(b200, oracle, fid, n):
    L = lib()
    x = vec(oracle, fid, 50 + n, n)
    flag = DeviceVec(4)

    def dev(i, o):
        rc = L.b200_batch_invert_dev(fid, i[0], n, o[0], flag.ptr, None)
        return E_ZERO if rc == OK and n and flag.to_bytes(4) != b"\0" * 4 else rc

    assert parity(lambda i, o: L.b200_batch_invert(fid, i[0], n, o[0]), dev, [x], [32 * n]) == OK
    if n:  # a zero element: B200_E_ZERO, with the output written all the same
        xz = x[:32 * (n // 2)] + b"\0" * 32 + x[32 * (n // 2 + 1):]
        assert parity(lambda i, o: L.b200_batch_invert(fid, i[0], n, o[0]), dev, [xz], [32 * n]) == E_ZERO


# ---- polynomial forms -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fid", FIDS)
@pytest.mark.parametrize("n", SIZES)
def test_rlc(b200, oracle, fid, n):
    L = lib()
    for lens in ([], [n], [n, n // 2, 0, 1 if n else 0]):
        k = len(lens)
        polys = [vec(oracle, fid, 60 + j + n, m) for j, m in enumerate(lens)]
        coeffs = vec(oracle, fid, 70, k)
        c_lens = (SZ * max(k, 1))(*lens)
        assert parity(lambda i, o: L.b200_rlc(fid, ptrs(i[1:]), c_lens, k, i[0], n, o[0]),
                      lambda i, o: L.b200_rlc_dev(fid, ptrs(i[1:]), c_lens, k, i[0], n, o[0], None),
                      [coeffs] + polys, [32 * n]) == OK


@pytest.mark.parametrize("fid", FIDS)
@pytest.mark.parametrize("n", [0, 2, 34, 65538])
def test_kzg_fold(b200, oracle, fid, n):
    L = lib()
    assert parity(lambda i, o: L.b200_kzg_fold(fid, i[0], n, i[1], o[0]),
                  lambda i, o: L.b200_kzg_fold_dev(fid, i[0], n, i[1], o[0], None),
                  [vec(oracle, fid, 80 + n, n), vec(oracle, fid, 81, 1)], [16 * n]) == OK


@pytest.mark.parametrize("fid", FIDS)
@pytest.mark.parametrize("n", SIZES)
def test_poly_eval_and_div(b200, oracle, fid, n):
    L = lib()
    f = vec(oracle, fid, 90 + n, n)
    for nu in (0, 1, 3, 8):
        assert parity(lambda i, o: L.b200_poly_eval(fid, i[0], n, i[1], nu, o[0]),
                      lambda i, o: L.b200_poly_eval_dev(fid, i[0], n, i[1], nu, o[0], None),
                      [f, vec(oracle, fid, 91 + nu, nu)], [32 * nu]) == OK
    if n:
        assert parity(lambda i, o: L.b200_poly_div(fid, i[0], n, i[1], o[0]),
                      lambda i, o: L.b200_poly_div_dev(fid, i[0], n, i[1], o[0], None),
                      [f, vec(oracle, fid, 92, 1)], [(32 * (n - 1), 32 * n)]) == OK


@pytest.mark.parametrize("fid", FIDS)
def test_mercury_forms(b200, oracle, fid):
    L = lib()
    for rows, cols in ((0, 3), (1, 1), (3, 0), (5, 7), (257, 300)):
        assert parity(lambda i, o: L.b200_mat_vec_rows(fid, i[0], rows, cols, i[1], o[0]),
                      lambda i, o: L.b200_mat_vec_rows_dev(fid, i[0], rows, cols, i[1], o[0], None),
                      [vec(oracle, fid, 100 + rows, rows * cols), vec(oracle, fid, 101, cols)], [32 * rows]) == OK
    for rows, cols in ((1, 1), (1, 4), (2, 3), (33, 5), (300, 257)):
        assert parity(lambda i, o: L.b200_div_binomial(fid, i[0], rows, cols, i[1], o[0], o[1]),
                      lambda i, o: L.b200_div_binomial_dev(fid, i[0], rows, cols, i[1], o[0], o[1], None),
                      [vec(oracle, fid, 102 + rows, rows * cols), vec(oracle, fid, 103, 1)],
                      [32 * (rows - 1) * cols, 32 * cols]) == OK
    for b in (1, 2, 33, 65537):
        assert parity(lambda i, o: L.b200_mercury_s_poly(fid, *i[:4], b, i[4], o[0]),
                      lambda i, o: L.b200_mercury_s_poly_dev(fid, *i[:4], b, i[4], o[0], None),
                      [vec(oracle, fid, 104 + k + b, b) for k in range(4)] + [vec(oracle, fid, 108, 1)],
                      [(32 * (b - 1), 32 * b) if b >= 2 else 0]) == OK


@pytest.mark.parametrize("fid", FIDS)
def test_neutron_forms(b200, oracle, fid):
    L = lib()
    for left, right in ((1, 2), (2, 2), (3, 5), (256, 257)):
        n, ne = left * right, left + right
        ins = [vec(oracle, fid, 110 + k, ne if k % 4 == 0 else n) for k in range(8)]
        assert parity(lambda i, o: L.b200_neutron_evals(fid, *i, left, right, o[0]),
                      lambda i, o: L.b200_neutron_evals_dev(fid, *i, left, right, o[0], None), ins, [160]) == OK
        if right >= 2:
            assert parity(lambda i, o: L.b200_pow_split_evals(fid, i[0], left, right, o[0]),
                          lambda i, o: L.b200_pow_split_evals_dev(fid, i[0], left, right, o[0], None),
                          [vec(oracle, fid, 120, 1)], [32 * ne]) == OK


# ---- sparse matrices and gather ---------------------------------------------------------------------------------
def random_csr(oracle, fid, rows, cols, seed):
    rng = random.Random(seed)
    indptr, indices = [0], []
    for _ in range(rows):
        indices += sorted(rng.sample(range(cols), min(cols, rng.randint(0, 3))))
        indptr.append(len(indices))
    return SparseMatrix(fid, vec(oracle, fid, seed, len(indices)), indices, indptr, cols)


@pytest.mark.parametrize("fid", FIDS)
@pytest.mark.parametrize("rows,cols", [(0, 4), (1, 1), (33, 17), (65537, 65539)])
def test_spmv_forms(b200, oracle, fid, rows, cols):
    L = lib()
    ms = [random_csr(oracle, fid, rows, cols, 130 + k) for k in range(2)]
    hs = (U64 * 2)(*[m.handle for m in ms])
    z1, z2 = vec(oracle, fid, 140, cols), vec(oracle, fid, 141, cols)
    for out_len in (cols, cols + 3):
        assert parity(lambda i, o: L.b200_spmv_t(ms[0].handle, i[0], out_len, o[0]),
                      lambda i, o: L.b200_spmv_t_dev(ms[0].handle, i[0], out_len, o[0], None),
                      [vec(oracle, fid, 142, rows)], [32 * out_len]) == OK
    for zb in (None, z2):
        outs = [32 * rows] * (4 if zb is not None else 2)

        def dev(i, o):
            for j, m in enumerate(ms):
                o2 = o[2 + j] if zb is not None else None
                rc = L.b200_spmv_dev(m.handle, i[0], i[1], o[j], o2, None)
                if rc:
                    return rc
            return OK

        assert parity(lambda i, o: L.b200_spmv_multi(hs, 2, i[0], i[1], cols, ptrs(o[:2]),
                                                     ptrs(o[2:]) if zb is not None else None),
                      dev, [z1, zb], outs) == OK


@pytest.mark.parametrize("table_len,n", [(1, 0), (1, 1), (33, 33), (65537, 65539)])
def test_gather(b200, oracle, table_len, n):
    L = lib()
    rng = random.Random(n)
    idx = [rng.randrange(table_len) for _ in range(n)]
    i64 = (U64 * max(n, 1))(*idx)
    i32 = b"".join(i.to_bytes(4, "little") for i in idx)
    assert parity(lambda i, o: L.b200_gather(i[0], table_len, i64, n, o[0]),
                  lambda i, o: L.b200_gather_dev(i[0], i[1], n, o[0], None),
                  [vec(oracle, 0, 150, table_len), i32], [32 * n]) == OK


# ---- argument errors --------------------------------------------------------------------------------------------
N = 4


def _calls(oracle, m):
    """Each host form with valid arguments of length N over field 0 (`m`: an N x N matrix): name -> (args, indices
    of pointer arguments that must not be null)."""
    def v(n=N):
        return hbuf(vec(oracle, 0, 160 + n, n))

    def o(n=N):
        return hbuf(FILL * 32 * n)

    from nova_b200.poseidon import PoseidonConstants
    lens = (SZ * 2)(N, N)
    return {
        "b200_cross_term": ([0, v(), v(), v(), v(), v(), v(1), N, o()], [1, 2, 3, 4, 6, 8]),
        "b200_axpy": ([0, v(), v(), v(1), N, o()], [1, 2, 3, 5]),
        "b200_vec_add": ([0, v(), v(), N, o()], [1, 2, 4]),
        "b200_bind_top": ([0, v(), N, v(1)], [1, 3]),
        "b200_poseidon_ro": ([PoseidonConstants.get(0).handle, v(), N, 128, 0, o(3)], [1, 5]),
        "b200_sc_eval": ([0, 3, v(), v(), v(), N, None, 0, None, 0, 0, o(3)], [2, 11]),
        "b200_eq_table": ([0, v(2), 2, o()], [1, 3]),
        "b200_mle_eval": ([0, v(), 2, v(2), o(1)], [1, 3, 4]),
        "b200_batch_invert": ([0, v(), N, o()], [1, 3]),
        "b200_rlc": ([0, ptrs([v(), v()]), lens, 2, v(2), N, o()], [1, 2, 4, 6]),
        "b200_kzg_fold": ([0, v(), N, v(1), o(N // 2)], [1, 3, 4]),
        "b200_poly_eval": ([0, v(), N, v(2), 2, o(2)], [1, 3, 5]),
        "b200_poly_div": ([0, v(), N, v(1), o()], [1, 3, 4]),
        "b200_mat_vec_rows": ([0, v(), 2, 2, v(2), o(2)], [1, 4, 5]),
        "b200_div_binomial": ([0, v(), 2, 2, v(1), o(2), o(2)], [1, 4, 5, 6]),
        "b200_mercury_s_poly": ([0, v(), v(), v(), v(), N, v(1), o()], [1, 2, 3, 4, 6, 7]),
        "b200_spmv_t": ([m.handle, v(), N, o()], [1, 3]),
        "b200_gather": ([v(), N, (U64 * N)(0, 1, 2, 3), N, o()], [0, 2, 4]),
        "b200_spmv_multi": ([(U64 * 1)(m.handle), 1, v(), None, N, ptrs([o()]), None], [0, 2, 5]),
        "b200_neutron_evals": ([0] + [v(4) if k % 4 == 0 else v() for k in range(8)] + [2, 2, o(5)],
                               [1, 2, 3, 4, 5, 6, 7, 8, 11]),
        "b200_pow_split_evals": ([0, v(1), 2, 2, o()], [1, 4]),
        "b200_lerp": ([0, v(), v(), v(1), N, o()], [1, 2, 3, 5]),
    }


def _with(args, **at):
    args = list(args)
    for i, val in at.items():
        args[int(i[1:])] = val
    return args


def error_table(oracle, m):
    """(case id, entry, arguments, expected status)"""
    calls = _calls(oracle, m)
    rows = []
    for name, (args, nonnull) in calls.items():
        if isinstance(args[0], int) and name not in ("b200_poseidon_ro", "b200_spmv_t"):
            rows.append((f"{name}:field", name, _with(args, a0=7), E_ARG))
        for i in nonnull:
            rows.append((f"{name}:null{i}", name, _with(args, **{f"a{i}": None}), E_ARG))
    bad = 1 << 60
    rows += [
        ("b200_bind_top:odd", "b200_bind_top", _with(calls["b200_bind_top"][0], a2=3), E_ARG),
        ("b200_kzg_fold:odd", "b200_kzg_fold", _with(calls["b200_kzg_fold"][0], a2=3), E_ARG),
        ("b200_sc_eval:odd", "b200_sc_eval", _with(calls["b200_sc_eval"][0], a5=3), E_ARG),
        ("b200_sc_eval:form", "b200_sc_eval", _with(calls["b200_sc_eval"][0], a1=12), E_ARG),
        ("b200_eq_table:ell35", "b200_eq_table", _with(calls["b200_eq_table"][0], a2=35), E_ARG),
        ("b200_mle_eval:ell35", "b200_mle_eval", _with(calls["b200_mle_eval"][0], a2=35), E_ARG),
        ("b200_rlc:k33", "b200_rlc", _with(calls["b200_rlc"][0], a3=33), E_ARG),
        ("b200_rlc:null_poly", "b200_rlc", _with(calls["b200_rlc"][0], a1=ptrs([None, hbuf(FILL * 32 * N)])), E_ARG),
        ("b200_gather:range", "b200_gather", _with(calls["b200_gather"][0], a2=(U64 * N)(0, 1, N, 3)), E_RANGE),
        ("b200_spmv_t:handle", "b200_spmv_t", _with(calls["b200_spmv_t"][0], a0=bad), E_HANDLE),
        ("b200_spmv_multi:handle", "b200_spmv_multi", _with(calls["b200_spmv_multi"][0], a0=(U64 * 1)(bad)), E_HANDLE),
        ("b200_spmv_multi:cols", "b200_spmv_multi", _with(calls["b200_spmv_multi"][0], a4=N + 1), E_ARG),
        ("b200_poseidon_ro:handle", "b200_poseidon_ro", _with(calls["b200_poseidon_ro"][0], a0=bad), E_HANDLE),
        ("b200_poseidon_ro:bits", "b200_poseidon_ro", _with(calls["b200_poseidon_ro"][0], a3=251), E_ARG),
        ("b200_div_binomial:empty", "b200_div_binomial", _with(calls["b200_div_binomial"][0], a2=0, a3=0), E_ARG),
        ("b200_poly_div:empty", "b200_poly_div", _with(calls["b200_poly_div"][0], a2=0), E_ARG),
        ("b200_pow_split_evals:right1", "b200_pow_split_evals", _with(calls["b200_pow_split_evals"][0], a3=1), E_ARG),
        ("b200_neutron_evals:empty", "b200_neutron_evals", _with(calls["b200_neutron_evals"][0], a9=0), E_ARG),
        ("b200_batch_invert:zero", "b200_batch_invert", _with(calls["b200_batch_invert"][0], a1=hbuf(b"\0" * 32 * N)),
         E_ZERO),
    ]
    return rows


def test_argument_errors(b200, oracle):
    m, got = random_csr(oracle, 0, N, N, 170), {}
    for case, name, args, want in error_table(oracle, m):
        got[case] = (getattr(lib(), name)(*args), want)
    assert {c: g for c, (g, w) in got.items() if g != w} == {}


def test_valid_calls_succeed(b200, oracle):
    """The table's base arguments are valid: every failure above comes from the one argument it changes."""
    m = random_csr(oracle, 0, N, N, 170)
    for name, (args, _) in _calls(oracle, m).items():
        assert getattr(lib(), name)(*args) == OK, name
