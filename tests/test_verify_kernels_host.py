"""The verifier kernels on the CPU: the real k_r1cs_eval / k_r1cs_final and k_ipa_s_half / k_eq_outer
(nova_b200/csrc/poly_kernels.cuh) run as blocks of host threads through tests/hostcheck/simt_host.h and are compared
with the C restatement of the reference's loops (tests/verify_oracle.c) and with Python integers."""
import pytest

import verify_ref
from oracle.pyref import FIELD_MODULUS, SplitMix64, eq_evals, from_mont_bytes, mont_bytes

SMALL = [1, 2, 3, 4, 5, 6, 7]


def pack(p, xs):
    return b"".join(mont_bytes(p, x) for x in xs)


def coeff(p, rng, cls):
    """one coefficient of a class: +-1, +-2..7 (small_mul) or general (a full product)"""
    if cls == "one":
        return 1 if rng.next() & 1 else p - 1
    if cls == "small":
        k = SMALL[1 + rng.next() % 6]
        return k if rng.next() & 1 else p - k
    return rng.field(p)


def matrix(p, rng, row_lens, cols, classes=("one", "small", "general")):
    data, indices, indptr = [], [], [0]
    for n in row_lens:
        for _ in range(n):
            data.append(coeff(p, rng, classes[rng.next() % len(classes)]))
            indices.append(rng.next() % cols)
        indptr.append(len(indices))
    return data, indices, indptr


def python_eval(p, data, indices, indptr, Tx, Ty):
    acc = 0
    for r in range(len(indptr) - 1):
        for e in range(indptr[r], indptr[r + 1]):
            acc += Tx[r] * Ty[indices[e]] * data[e]
    return acc % p


def shapes(rng):
    """(name, rows, cols, row lengths): one row holding most entries, runs of empty rows, an empty matrix, a row that
    spans many threads' slices, a matrix whose first and last rows are empty"""
    heavy = [0] * 64
    heavy[5] = 900
    for i in range(10, 64, 3):
        heavy[i] = 1 + rng.next() % 4
    sparse = [0] * 128
    for i in (0, 1, 77, 127):
        sparse[i] = 3
    edges = [0, 0] + [2] * 28 + [0, 0]
    return [("heavy_row", 64, 64, heavy), ("empty_runs", 128, 32, sparse), ("empty", 16, 16, [0] * 16),
            ("edges", 32, 64, edges), ("uniform", 64, 128, [1 + rng.next() % 6 for _ in range(64)])]


@pytest.mark.parametrize("fid", [0, 1, 2, 3])
def test_r1cs_eval_kernel_on_host_threads(fid):
    p = FIELD_MODULUS[fid]
    rng = SplitMix64(9100 + fid)
    for name, rows, cols, lens in shapes(rng):
        ell_x, ell_y = (rows - 1).bit_length(), (cols - 1).bit_length()
        rx, ry = [rng.field(p) for _ in range(ell_x)], [rng.field(p) for _ in range(ell_y)]
        Tx, Ty = eq_evals(p, rx), eq_evals(p, ry)  # cols == ty_len: the last column of T_y is reachable
        mats = [matrix(p, rng, lens, cols) for _ in range(3)]
        packed = [(pack(p, d), i, ip) for (d, i, ip) in mats]
        want = [python_eval(p, d, i, ip, Tx, Ty) for (d, i, ip) in mats]
        assert [from_mont_bytes(p, verify_ref.r1cs_eval(fid, *m, pack(p, Tx), pack(p, Ty))) for m in packed] == want
        exp = pack(p, want)
        # slices of 3 entries: the heavy row spans hundreds of threads' slices over both blocks
        # (3, 1): fewer threads than entries, so the slices wrap around the grid
        for grid, chunk in ((2, 3), (3, 1)) if name == "heavy_row" else ((1, 0),):
            assert verify_ref.simt_r1cs_eval(fid, packed, pack(p, Tx), pack(p, Ty), grid, chunk) == exp, (name, grid)
        if name == "heavy_row":  # k = 1 and k = 2 launch only grid.y rows of blocks
            assert verify_ref.simt_r1cs_eval(fid, packed[:1], pack(p, Tx), pack(p, Ty), 2, 5) == exp[:32]
            assert verify_ref.simt_r1cs_eval(fid, packed[1:], pack(p, Tx), pack(p, Ty), 1, 7) == exp[32:]


def offset_matrix(p, rng, lens, cols, skipped=5):
    """a CSR matrix whose indptr starts at `skipped`: the entries before indptr[0] belong to no row"""
    d, i, ip = matrix(p, rng, lens, cols)
    junk = [rng.field(p) for _ in range(skipped)]
    return junk + d, [rng.next() % cols for _ in range(skipped)] + i, [x + skipped for x in ip]


def test_r1cs_eval_skips_entries_before_indptr0():
    """indptr[0] > 0 (which registration accepts): the entries before it are in no row and count for nothing, as in
    the reference's loop over indptr windows; rows = 0 with such entries gives 0"""
    fid = 0
    p = FIELD_MODULUS[fid]
    rng = SplitMix64(9250)
    lens = [3, 0, 1, 5, 0, 0, 2, 4]
    d, i, ip = offset_matrix(p, rng, lens, 8)
    Tx = eq_evals(p, [rng.field(p) for _ in range(3)])
    Ty = eq_evals(p, [rng.field(p) for _ in range(3)])
    want = python_eval(p, d, i, ip, Tx, Ty)
    assert from_mont_bytes(p, verify_ref.r1cs_eval(fid, pack(p, d), i, ip, pack(p, Tx), pack(p, Ty))) == want
    for grid, chunk in ((1, 1), (2, 3), (1, 0)):
        got = verify_ref.simt_r1cs_eval(fid, [(pack(p, d), i, ip)], pack(p, Tx), pack(p, Ty), grid, chunk)
        assert from_mont_bytes(p, got) == want, (grid, chunk)
    got = verify_ref.simt_r1cs_eval(fid, [(pack(p, d[:3]), i[:3], [3])], pack(p, Tx), pack(p, Ty), 1, 1)
    assert got == bytes(32)


@pytest.mark.parametrize("cls", ["one", "small", "general"])
def test_r1cs_eval_every_coefficient_class(cls):
    """each class on its own, every value of +-1..7 included, over fields 0 and 3"""
    for fid in (0, 3):
        p = FIELD_MODULUS[fid]
        rng = SplitMix64(9200 + fid)
        lens = [1 + rng.next() % 9 for _ in range(32)]
        d, i, ip = matrix(p, rng, lens, 32, classes=(cls,))
        if cls == "small":
            d[:14] = SMALL + [p - k for k in SMALL]
        Tx = eq_evals(p, [rng.field(p) for _ in range(5)])
        Ty = eq_evals(p, [rng.field(p) for _ in range(5)])
        got = verify_ref.simt_r1cs_eval(fid, [(pack(p, d), i, ip)], pack(p, Tx), pack(p, Ty), 2, 2)
        assert from_mont_bytes(p, got) == python_eval(p, d, i, ip, Tx, Ty)


def ipa_s_python(p, r, scale=1):
    L = len(r)
    out = []
    for i in range(1 << L):
        v = scale
        for j in range(L):
            v = v * (r[j] if (i >> (L - 1 - j)) & 1 else pow(r[j], -1, p)) % p
        out.append(v)
    return out


@pytest.mark.parametrize("fid", [0, 1, 2, 3])
def test_ipa_s_kernel_on_host_threads(fid):
    """direct pass and half tables + outer product, with and without scale, against the reference's recurrence
    (C) and the per-bit product (Python)"""
    p = FIELD_MODULUS[fid]
    rng = SplitMix64(9300 + fid)
    for L, direct in ((0, 10), (1, 10), (5, 10), (7, 3), (9, 4)):
        r = [rng.field(p) for _ in range(L)]
        rb, rib = pack(p, r), pack(p, [pow(x, -1, p) for x in r])
        for scale in (None, rng.field(p)):
            want = verify_ref.ipa_s(fid, r, scale)
            assert [from_mont_bytes(p, want[k:k + 32]) for k in range(0, len(want), 32)] == \
                ipa_s_python(p, r, 1 if scale is None else scale)
            got = verify_ref.simt_ipa_s(fid, rb, rib, L, mont_bytes(p, scale) if scale is not None else None, direct)
            assert got == want, (L, direct, scale is None)
