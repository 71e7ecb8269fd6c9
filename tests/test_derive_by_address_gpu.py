"""ck_derive_by_address on the H100 (b200_ck_derive_by_address / _dev): the derived bases, read back with
b200_ck_export_bases, equal the C oracle's restatement of the reference loop byte for byte (affine coordinates are
unique, whatever order the device sums in); the derived key commits like the source key over the gathered vector;
errors, user streams, a concurrent commit on the source and the release of the source."""
import ctypes
import struct
import subprocess
import threading

import numpy as np
import pytest

import derive_ref
from test_derive_by_address_cpu import build_cpp, edge_bases

pytestmark = pytest.mark.gpu

SIZE_NONE = ctypes.c_size_t(-1).value


def _engine(cid):
    import nova_b200 as nb
    return nb.CommitmentEngine(cid)


def _host_key(cid, bases, h=None):
    import nova_b200 as nb
    return nb.CommitmentKey(nb.Curve(cid), bases, h)


def _jac(cid, raw):
    from nova_b200.provider import Curve, _jac_to_affine
    return _jac_to_affine(Curve(cid), raw)


def _aff(cid, b64):
    from oracle.pyref import CURVES
    return CURVES[cid].affine_from_bytes(b64)


def _u32(addrs) -> bytes:
    return np.asarray(addrs, dtype=np.uint32).tobytes()


def _commit_dev(ck, d_scalars, n, d_blind=None):
    """commit_dev on the library stream -> affine"""
    from nova_b200.native import check, lib
    from nova_b200.spartan import DeviceVec
    out = DeviceVec(96)
    check(lib().b200_commit_dev(ck.handle, d_scalars.ptr, n, d_blind.ptr if d_blind else None, out.ptr, None))
    return _jac(int(ck.curve), out.to_bytes())


def _commit_gathered(ck, T: bytes, addrs):
    """commit(ck, T[addresses]) through b200_gather_dev and the ordinary commit: a device path independent of the
    derivation"""
    from nova_b200.native import check, lib
    from nova_b200.spartan import DeviceVec
    m = len(addrs)
    dT, dA, dG = DeviceVec.from_bytes(T), DeviceVec.from_bytes(_u32(addrs)), DeviceVec(32 * m)
    check(lib().b200_gather_dev(dT.ptr, dA.ptr, m, dG.ptr, None))
    return _commit_dev(ck, dG, m)


@pytest.mark.parametrize("cid", [0, 1, 2, 3])
@pytest.mark.parametrize("with_h", [False, True])
@pytest.mark.parametrize("n,m,table_size", [(64, 50, 37), (1 << 16, 1 << 16, 1 << 12), (1 << 16, 40000, 1 << 16)])
def test_parity_with_oracle(b200, oracle, cid, with_h, n, m, table_size):
    from oracle.pyref import CURVES
    c = CURVES[cid]
    bases = oracle.gen_bases(cid, n + 1)
    h = bases[64 * n:] if with_h else None
    ck = _host_key(cid, bases[:64 * n], h)
    rng = np.random.default_rng(1000 * cid + n + m)
    addrs = rng.integers(0, table_size, m).tolist()
    d = _engine(cid).ck_derive_by_address(ck, addrs, table_size)
    exp = derive_ref.derive(cid, bases[:64 * n], addrs, table_size)
    assert d.export_bases() == exp
    assert d.h == h and d.has_h == with_h
    T = oracle.gen_scalars(c.scalar_field, 5 + cid, table_size)
    r = oracle.gen_scalars(c.scalar_field, 6 + cid, 1) if with_h else None
    got = _engine(cid).commit(d, T, r)
    assert got == _aff(cid, oracle.msm(cid, T + (r or b""), exp + (h or b"")))


@pytest.mark.parametrize("cid", [0, 1, 2, 3])
def test_edge_cases(b200, oracle, cid):
    """ck[1] = -ck[0] on one slot (identity), ck[3] = ck[2] on one slot (doubling), unaddressed slots, a table size
    that is not a power of two and exceeds m"""
    from oracle.pyref import CURVES
    c = CURVES[cid]
    bases = edge_bases(cid, 24)
    ck = _host_key(cid, bases)
    addrs = [6, 6, 2, 2, 0, 9, 9, 9, 30, 17]  # m = 10 < n = 24 < table_size = 45
    d = _engine(cid).ck_derive_by_address(ck, addrs, 45)
    got = d.export_bases()
    assert got == derive_ref.derive(cid, bases, addrs, 45)
    assert got[64 * 6:64 * 7] == bytes(64)
    P2 = c.affine_from_bytes(bases[128:192])
    assert got[128:192] == c.affine_bytes(c.add(P2, P2))
    assert got[64 * 31:] == bytes(64 * 14)


# ---- a 2^20-base synthetic key, m = 2^20, skewed address patterns ------------------------------------------------
N_BIG = 1 << 20


@pytest.fixture(scope="module")
def big_key(b200):
    import nova_b200 as nb
    ck = nb.CommitmentKey.setup_synthetic(nb.Curve(0), N_BIG)
    return ck, ck.export_bases()


def _pattern(name):
    rng = np.random.default_rng(77)
    if name == "uniform_2^16":
        return rng.integers(0, 1 << 16, N_BIG), 1 << 16
    if name == "permutation_2^20":
        return rng.permutation(N_BIG), N_BIG
    if name == "all_equal":  # one slot receives every base: the heavy-bucket path
        return np.full(N_BIG, 12345), 1 << 16
    if name == "half_on_one_slot":
        a = rng.integers(0, 1 << 16, N_BIG)
        a[rng.permutation(N_BIG)[:N_BIG // 2]] = 777
        return a, 1 << 16
    if name == "even_slots":
        return 2 * rng.integers(0, N_BIG // 2, N_BIG), N_BIG
    raise ValueError(name)


@pytest.mark.parametrize("pattern", ["uniform_2^16", "permutation_2^20", "all_equal", "half_on_one_slot", "even_slots"])
def test_scale_and_skew(b200, oracle, big_key, pattern):
    from oracle.pyref import CURVES
    ck, bases = big_key
    addrs_np, table_size = _pattern(pattern)
    addrs = addrs_np.tolist()
    d = _engine(0).ck_derive_by_address(ck, addrs, table_size)
    assert d.export_bases() == derive_ref.derive(0, bases, addrs, table_size)
    T = oracle.gen_scalars(CURVES[0].scalar_field, 31, table_size)
    from nova_b200.spartan import DeviceVec
    assert _commit_dev(d, DeviceVec.from_bytes(T), table_size) == _commit_gathered(ck, T, addrs)


# ---- using the derived key -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("cid", [0, 2])
def test_derived_key_commits_after_source_release(b200, oracle, cid):
    """blinded commit_dev and commit_small on the derived key, with the source released first"""
    from nova_b200.spartan import DeviceVec
    from oracle.pyref import CURVES
    c = CURVES[cid]
    n, table_size = 5000, 1500
    bases = oracle.gen_bases(cid, n + 1)
    h = bases[64 * n:]
    ck = _host_key(cid, bases[:64 * n], h)
    addrs = [(7 * i) % table_size for i in range(n)]
    d = _engine(cid).ck_derive_by_address(ck, addrs, table_size)
    ck.release()
    derived = derive_ref.derive(cid, bases[:64 * n], addrs, table_size)
    T = oracle.gen_scalars(c.scalar_field, 41, table_size)
    r = oracle.gen_scalars(c.scalar_field, 42, 1)
    got = _commit_dev(d, DeviceVec.from_bytes(T), table_size, DeviceVec.from_bytes(r))
    assert got == _aff(cid, oracle.msm(cid, T + r, derived + h))
    small = [(3 * j + 1) % 1000 for j in range(table_size)]
    got_small = _engine(cid).commit_small(d, small, 8, r)
    from oracle.pyref import from_mont_bytes
    exp_small = c.add(_aff(cid, oracle.msm_small(cid, small, derived)), c.mul(from_mont_bytes(c.q, r), _aff(cid, h)))
    assert got_small == exp_small


def test_table_2_22_routes_both_table_sets(b200, oracle, big_key):
    """a 2^22-slot derived key carries the 17-bit table set: commits of <= 2^21 scalars use it, longer ones the wide set"""
    from nova_b200.native import check, lib
    from nova_b200.spartan import DeviceVec
    from oracle.pyref import CURVES
    ck, _ = big_key
    table_size = 1 << 22
    addrs = np.random.default_rng(5).integers(0, table_size, N_BIG).tolist()
    d = _engine(0).ck_derive_by_address(ck, addrs, table_size)
    nb_, wb, nt = ctypes.c_size_t(), ctypes.c_int(), ctypes.c_int()
    check(lib().b200_ck_len(d.handle, ctypes.byref(nb_), ctypes.byref(wb), ctypes.byref(nt)))
    assert (nb_.value, wb.value) == (table_size, 20)
    T = oracle.gen_scalars(CURVES[0].scalar_field, 51, table_size)
    half = table_size // 2
    assert _commit_dev(d, DeviceVec.from_bytes(T), table_size) == _commit_gathered(ck, T, addrs)
    T_low = T[:32 * half] + bytes(32 * half)  # the prefix commit sees only the slots below 2^21
    assert _commit_dev(d, DeviceVec.from_bytes(T[:32 * half]), half) == _commit_gathered(ck, T_low, addrs)


# ---- errors, user streams, concurrency -----------------------------------------------------------------------------
def _call_dev(handle, d_addr, m, table_size, stream, window_bits=0):
    from nova_b200.native import lib
    out, bad = ctypes.c_uint64(777), ctypes.c_size_t(0)
    rc = lib().b200_ck_derive_by_address_dev(handle, d_addr, m, table_size, window_bits, ctypes.byref(out),
                                             ctypes.byref(bad), stream)
    return rc, out.value, (None if bad.value == SIZE_NONE else bad.value)


def test_errors_on_user_stream(b200, oracle):
    import torch
    from nova_b200.native import (B200_E_ARG, B200_E_HANDLE, B200_E_INDEX, B200_E_POINT, B200_E_RANGE, lib)
    from nova_b200.spartan import DeviceVec
    stream = torch.cuda.Stream()
    s = ctypes.c_void_p(stream.cuda_stream)
    n = 1000
    bases = oracle.gen_bases(1, n)
    ck = _host_key(1, bases)
    holed = _host_key(1, bases[:64 * 700] + bytes(64) + bases[64 * 701:])
    ok = DeviceVec.from_bytes(_u32([i % 10 for i in range(n)]))
    bad3 = DeviceVec.from_bytes(_u32([1, 2, 3, 50, 4, 60] + [0] * (n - 6)))
    assert _call_dev(999999, ok.ptr, n, 10, s) == (B200_E_HANDLE, 777, None)
    assert _call_dev(holed.handle, bad3.ptr, n, 10, s) == (B200_E_POINT, 777, 700)  # before the index check
    longer = DeviceVec.from_bytes(_u32([0] * (n + 1)))
    assert _call_dev(ck.handle, longer.ptr, n + 1, 10, s) == (B200_E_RANGE, 777, None)
    assert _call_dev(ck.handle, bad3.ptr, n, 10, s) == (B200_E_INDEX, 777, 3)
    assert _call_dev(ck.handle, ok.ptr, n, 0, s) == (B200_E_INDEX, 777, 0)  # table_size = 0 with addresses
    assert _call_dev(ck.handle, None, 0, 0, s) == (B200_E_ARG, 777, None)  # table_size = 0, m = 0
    assert _call_dev(ck.handle, ok.ptr, n, 1 << 31, s) == (B200_E_RANGE, 777, None)
    assert _call_dev(ck.handle, ok.ptr, n, 1 << 28, s)[0] == B200_E_RANGE  # 13 tables of 2^28 rows
    assert _call_dev(ck.handle, None, 5, 10, s)[0] == B200_E_ARG
    assert _call_dev(ck.handle, ok.ptr, n, 10, s, window_bits=1)[0] == B200_E_ARG
    rc, h, bad = _call_dev(ck.handle, ok.ptr, n, 10, s)
    assert rc == 0 and bad is None and h != 777
    stream.synchronize()
    check_bases = ctypes.create_string_buffer(640)
    assert lib().b200_ck_export_bases(h, 0, 10, check_bases) == 0
    assert check_bases.raw == derive_ref.derive(1, bases, [i % 10 for i in range(n)], 10)
    assert lib().b200_ck_release(h) == 0
    # the host entry checks 64-bit addresses before narrowing them: 2^32 + 3 does not become slot 3
    arr = (ctypes.c_uint64 * 3)(1, (1 << 32) + 3, 2)
    out, first = ctypes.c_uint64(777), ctypes.c_size_t(0)
    assert lib().b200_ck_derive_by_address(ck.handle, arr, 3, 8, 0, ctypes.byref(out), ctypes.byref(first)) == B200_E_INDEX
    assert (out.value, first.value) == (777, 1)


def test_derive_while_committing_on_source(b200, oracle):
    """one thread derives from the key while another commits on it; both results are checked"""
    from oracle.pyref import CURVES
    cid, n = 3, 1 << 16
    c = CURVES[cid]
    bases = oracle.gen_bases(cid, n)
    ck = _host_key(cid, bases)
    v = oracle.gen_scalars(c.scalar_field, 61, n)
    exp_commit = _aff(cid, oracle.msm(cid, v, bases))
    addrs = np.random.default_rng(3).integers(0, 4096, n).tolist()
    commits, errors = [], []

    def committer():
        try:
            for _ in range(8):
                commits.append(_engine(cid).commit(ck, v))
        except Exception as e:  # surfaced below
            errors.append(e)
    t = threading.Thread(target=committer)
    t.start()
    d = _engine(cid).ck_derive_by_address(ck, addrs, 4096)
    t.join()
    assert not errors and commits == [exp_commit] * 8
    assert d.export_bases() == derive_ref.derive(cid, bases, addrs, 4096)


def test_cpp_mirror_derive(b200, oracle, tmp_path):
    """CommitmentEngine<BN254>::ck_derive_by_address: the derived key commits after the source is gone, and the named
    exceptions carry the reference's errors"""
    from oracle.pyref import CURVES
    c = CURVES[0]
    n, table_size = 3000, 700
    bases = oracle.gen_bases(0, n + 1)
    addrs = [(11 * i) % table_size for i in range(2000)]
    T = oracle.gen_scalars(c.scalar_field, 71, table_size)
    r = oracle.gen_scalars(c.scalar_field, 72, 1)
    case = tmp_path / "derive.bin"
    with open(case, "wb") as f:
        for blob, k in ((bases[:64 * n], n), (bases[64 * n:], 1), (struct.pack(f"<{len(addrs)}Q", *addrs), len(addrs)),
                        (struct.pack("<Q", table_size), 1), (T, table_size), (r, 1)):
            f.write(struct.pack("<Q", k) + blob)
    out = subprocess.run([build_cpp(), str(case)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    raw = open(str(case) + ".out", "rb").read()
    derived = derive_ref.derive(0, bases[:64 * n], addrs, table_size)
    assert _jac(0, raw[:96]) == _aff(0, oracle.msm(0, T + r, derived + bases[64 * n:]))
    assert _jac(0, raw[96:192]) == _aff(0, oracle.msm(0, T, derived))
    assert struct.unpack("<QQ", raw[192:208]) == (len(addrs) - 1, 1)
