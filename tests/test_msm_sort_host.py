"""The bucket sort of the MSM on the CPU: k_digits_small, every k_sort_pass and k_sort_starts
(nova_b200/csrc/msm_sort.cuh) run as written through tests/hostcheck/simt_host.h and simt_host_sort.h -- block
histograms, ballot ranking, decoupled look-back over the tiles, the bucket-start search -- and their output is compared
EXACTLY with a stable sort by key of the (window, index)-ordered non-zero digits: the sort is stable, so there is one
right answer."""
import ctypes
import os
import random
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
TILE = 4096


@pytest.fixture(scope="module")
def hc_sort():
    src = os.path.join(HERE, "hostcheck", "sort_check.cpp")
    so = os.path.join(HERE, "hostcheck", "libhostcheck_sort.so")
    deps = [src, os.path.join(HERE, "hostcheck", "simt_host.h"), os.path.join(HERE, "hostcheck", "simt_host_sort.h"),
            os.path.join(HERE, "..", "nova_b200", "csrc", "msm_sort.cuh"),
            os.path.join(HERE, "..", "nova_b200", "csrc", "field.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", "-shared", "-fPIC", "-x", "c++", src, "-o", so])
    return ctypes.CDLL(so)


def signed_digits(v, c, W):
    """the signed c-bit digits of k_digits_small: digits in [-(2^(c-1) - 1), 2^(c-1)], carry into the next window"""
    half, out, carry = 1 << (c - 1), [], 0
    for w in range(W):
        d = ((v >> (w * c)) & ((1 << c) - 1) if w * c < 64 else 0) + carry
        carry = 1 if d > half else 0
        out.append(d - (1 << c) if d > half else d)
    return out


def expected_sort(digits, n, c, W, G, n_ck, base_offset, blind_i, h_index):
    B = 1 << (c - 1)
    ents = []
    for w in range(W):
        for i in range(n):
            d = digits[w * n + i]
            if d == 0:
                continue
            key = (w % G) * B + abs(d) - 1
            bi = h_index if i == blind_i else base_offset + i
            ents.append((key << 32) | ((d < 0) << 31) | ((w // G) * n_ck + bi))
    ents.sort(key=lambda e: e >> 32)  # stable
    K = G * B
    start, k = [], 0
    for key in range(K + 1):
        while k < len(ents) and (ents[k] >> 32) < key:
            k += 1
        start.append(k)
    return ents, start


def run_sort(hc, n, c, W, G, digits=None, small=None, blinded=False, heavy_min=64, digit_blocks=3):
    B, K = 1 << (c - 1), G * (1 << (c - 1))
    n_ck, base_offset = n + 5, 3
    blind_i, h_index = (n - 1, n + 4) if blinded else (0xFFFFFFFF, 0)
    cnt = n * W
    dig = (ctypes.c_int32 * cnt)(*(digits or [0] * cnt))
    sm = (ctypes.c_uint64 * n)(*small) if small is not None else None
    heavy_cap = cnt // max(heavy_min, 1) + 2
    ent = (ctypes.c_uint64 * cnt)()
    start = (ctypes.c_uint32 * (K + 1))()
    heavy = (ctypes.c_uint32 * (1 + heavy_cap))()
    passes = ctypes.c_int()
    rc = hc.hc_sort_run(dig, sm, digit_blocks, n, c, W, G, n_ck, base_offset, blind_i, h_index, heavy_min, heavy_cap,
                        ent, start, heavy, ctypes.byref(passes))
    assert rc == 0, "two sorts on the same look-back words disagree" if rc == 2 else rc
    if small is not None:  # the digit kernel's own output
        want = [0] * cnt
        for i, v in enumerate(small):
            for w, d in enumerate(signed_digits(v, c, W)):
                want[w * n + i] = d
        assert list(dig) == want
    exp_ent, exp_start = expected_sort(list(dig), n, c, W, G, n_ck, base_offset,
                                       n - 1 if blinded else -1, h_index)
    M = len(exp_ent)
    assert list(ent[:M]) == exp_ent
    assert list(start) == exp_start
    exp_heavy = sorted(k for k in range(K) if exp_start[k + 1] - exp_start[k] > heavy_min)
    assert heavy[0] == len(exp_heavy)
    assert sorted(heavy[1:1 + min(heavy[0], heavy_cap)]) == exp_heavy[:heavy_cap]
    return passes.value, M


def uniform_digits(rng, n, c, W, density=1.0):
    half = 1 << (c - 1)
    return [rng.randint(-(half - 1), half) if rng.random() < density else 0 for _ in range(n * W)]


@pytest.mark.parametrize("c,W,G,n,passes", [
    (17, 15, 1, 700, 2),   # the 2^20 headline shape: 16 key bits, two 8-bit passes, several tiles
    (10, 26, 2, 400, 2),   # an un-expanded key (two bucket groups): table index = (w / G) * n_ck + base
    (13, 20, 4, 300, 2),   # four groups, 14 key bits
    (4, 64, 1, 90, 1),     # 3 key bits: one pass
    (2, 127, 1, 40, 1),    # the narrowest window
])
def test_uniform_digits_sort_exactly(hc_sort, c, W, G, n, passes):
    rng = random.Random(c * 1000 + W)
    digits = uniform_digits(rng, n, c, W)
    got_passes, M = run_sort(hc_sort, n, c, W, G, digits=digits)
    assert got_passes == passes
    assert M > TILE or n * W < 2 * TILE


def test_wide_window_three_passes(hc_sort):
    """c = 20 (the 2^22 and 2^24 sizes): 19 key bits in three 7-bit passes, sparse digits, blinded"""
    rng = random.Random(20)
    got, _ = run_sort(hc_sort, 400, 20, 13, 1, digits=uniform_digits(rng, 400, 20, 13, 0.6), blinded=True)
    assert got == 3


@pytest.mark.parametrize("kind", ["zero", "bits", "repeated", "small", "padding"])
@pytest.mark.parametrize("blinded", [False, True])
def test_structured_scalars_through_the_digit_kernel(hc_sort, kind, blinded):
    """skewed inputs: every tile holds one key (or none), heavy buckets, the block histograms of k_digits_small
    over a grid-stride loop of several blocks"""
    rng = random.Random(sum(map(ord, kind)))
    n, c, W = 1500, 17, 15
    small = {
        "zero": [0] * n,
        "bits": [rng.randint(0, 1) for _ in range(n)],
        "repeated": [0xDEADBEEFCAFE1234] * n,
        "small": [rng.randint(0, 1 << 20) for _ in range(n)],
        "padding": [rng.getrandbits(64) if i < n // 3 else 1 for i in range(n)],
    }[kind]
    run_sort(hc_sort, n, c, W, 1, small=small, blinded=blinded, heavy_min=100)


def test_one_digit_per_window_group_key(hc_sort):
    """G > 1 with repeated values: one key per window group, every pass ranks single-key tiles"""
    n, c, W, G = 600, 12, 22, 2
    run_sort(hc_sort, n, c, W, G, small=[0x0123456789ABCDEF] * n, heavy_min=50, digit_blocks=1)
