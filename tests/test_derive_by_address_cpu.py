"""ck_derive_by_address (traits/commitment.rs:177-194) without a GPU: the C oracle's restatement against the naive
Python group law, the trait's identity Comm(T[addresses], ck[..m]) = Comm(T, derived) on the oracle, the Python mirror's
host logic on the emulated device (tests/emulated_derive.py), and the C++ mirror's compile and link."""
import os
import subprocess

import pytest

import derive_ref
import emulated_derive
from nova_b200.native import B200_E_ARG, B200_E_HANDLE, B200_E_INDEX, B200_E_POINT, B200_E_RANGE, B200Error
from oracle import coracle as co
from oracle.pyref import CURVES, SplitMix64

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def edge_bases(cid: int, n: int) -> bytes:
    """n generated bases with ck[1] = -ck[0] and ck[3] = ck[2]: a sum that cancels and one that doubles"""
    c = CURVES[cid]
    b = bytearray(co.gen_bases(cid, n))
    b[64:128] = c.affine_bytes(c.neg(c.affine_from_bytes(bytes(b[0:64]))))
    b[192:256] = b[128:192]
    return bytes(b)


@pytest.mark.parametrize("cid", [0, 1, 2, 3])
def test_c_restatement_equals_naive_group_law(cid):
    n, table_size = 40, 13
    bases = edge_bases(cid, n)
    rng = SplitMix64(100 + cid)
    rest = [1 + rng.next() % 9 for _ in range(n - 8)]  # slots 1..9 except 5; 10..12 are never addressed
    addrs = [0, 0, 5, 5] + [6 if a == 5 else a for a in rest]  # m = n - 4 < n
    got = derive_ref.derive(cid, bases, addrs, table_size)
    assert got == derive_ref.derive_naive(cid, bases, addrs, table_size)
    c = CURVES[cid]
    P2 = c.affine_from_bytes(bases[128:192])
    assert got[0:64] == bytes(64)  # ck[0] + ck[1] = identity
    assert got[320:384] == c.affine_bytes(c.add(P2, P2))  # ck[2] + ck[3] = 2 ck[2]
    assert got[64 * 10:] == bytes(64 * 3)


@pytest.mark.parametrize("cid", [0, 3])
def test_trait_identity_on_oracle(cid):
    """msm(T[addresses], ck[..m]) == msm(T, derived) with the C MSM (the purpose of the derivation: a lookup commitment
    over the table)"""
    c = CURVES[cid]
    n, m, table_size = 300, 257, 64
    bases = co.gen_bases(cid, n)
    rng = SplitMix64(7 + cid)
    addrs = [rng.next() % table_size for _ in range(m)]
    T = co.gen_scalars(c.scalar_field, 9, table_size)
    lookup = b"".join(T[32 * a:32 * a + 32] for a in addrs)
    derived = derive_ref.derive(cid, bases, addrs, table_size)
    assert co.msm(cid, T, derived) == co.msm(cid, lookup, bases[:64 * m])


def test_c_restatement_errors():
    bases = co.gen_bases(2, 6)
    with pytest.raises(derive_ref.DeriveError) as e:
        derive_ref.derive(2, bases, [0] * 7, 4)
    assert e.value.code == derive_ref.KEY_LENGTH
    with pytest.raises(derive_ref.DeriveError) as e:
        derive_ref.derive(2, bases, [0, 3, 4, 9], 4)
    assert (e.value.code, e.value.first_bad) == (derive_ref.INVALID_INDEX, 2)
    holed = bases[:128] + bytes(64) + bases[192:]
    with pytest.raises(derive_ref.DeriveError) as e:  # the identity check runs first and covers the whole key
        derive_ref.derive(2, holed, [9] * 7, 4)
    assert (e.value.code, e.value.first_bad) == (derive_ref.IDENTITY_GENERATOR, 2)
    assert derive_ref.derive(2, bases, [], 0) == b""


# ---- the Python mirror on the emulated device ------------------------------------------------------------------
@pytest.fixture
def emu():
    dev = emulated_derive.install()
    yield dev
    emulated_derive.uninstall()


def _key(cid, n, with_h=True, hole=None):
    import nova_b200 as nb
    bases = bytearray(co.gen_bases(cid, n + 1))
    if hole is not None:
        bases[64 * hole:64 * hole + 64] = bytes(64)
    return nb.CommitmentKey(nb.Curve(cid), bytes(bases[:64 * n]), bytes(bases[64 * n:]) if with_h else None)


@pytest.mark.parametrize("cid", [0, 1, 2, 3])
def test_mirror_derives_and_carries_h(emu, cid):
    import nova_b200 as nb
    ck = _key(cid, 50)
    ce = nb.CommitmentEngine(cid)
    addrs = [i * 7 % 11 for i in range(30)]  # m < n
    d = ce.ck_derive_by_address(ck, addrs, 11)
    assert (d.n, d.bases, d.h, d.has_h) == (11, None, ck.h, True)
    assert emu.keys[d.handle][1] == derive_ref.derive(cid, ck.bases, addrs, 11)
    T = co.gen_scalars(CURVES[cid].scalar_field, 3, 11)
    r = co.gen_scalars(CURVES[cid].scalar_field, 4, 1)
    lookup = b"".join(T[32 * a:32 * a + 32] for a in addrs)
    assert ce.commit(d, T, r) == ce.commit(ck, lookup + bytes(32 * 20), r)


def test_mirror_edge_sizes(emu):
    import nova_b200 as nb
    ck = _key(1, 20, with_h=False)
    ce = nb.CommitmentEngine(1)
    d0 = ce.ck_derive_by_address(ck, [], 5)  # m = 0: every slot is the identity
    assert emu.keys[d0.handle][1] == bytes(64 * 5) and d0.h is None and not d0.has_h
    d1 = ce.ck_derive_by_address(ck, [0] * 20, 1)  # table_size = 1: the sum of the whole key
    assert emu.keys[d1.handle][1] == derive_ref.derive_naive(1, ck.bases, [0] * 20, 1)
    dev_addr = (__import__("ctypes").c_uint32 * 3)(2, 0, 2)
    d2 = ce.ck_derive_by_address_dev(ck, dev_addr, 3, 4)
    assert emu.keys[d2.handle][1] == derive_ref.derive(1, ck.bases, [2, 0, 2], 4)


def _err(fn):
    with pytest.raises(B200Error) as e:
        fn()
    return e.value.code, e.value.first_bad


def test_mirror_errors_and_precedence(emu):
    import nova_b200 as nb
    ce = nb.CommitmentEngine(0)
    ck = _key(0, 8)
    holed = _key(0, 8, hole=5)
    before = set(emu.keys)
    # an identity generator anywhere in the key comes first, with its index, whatever else is wrong
    assert _err(lambda: ce.ck_derive_by_address(holed, [99] * 9, 0)) == (B200_E_POINT, 5)
    assert _err(lambda: ce.ck_derive_by_address(ck, [0] * 9, 4)) == (B200_E_RANGE, None)  # m > n, before the index
    assert _err(lambda: ce.ck_derive_by_address(ck, [1, 2, 7, 4, 9], 4)) == (B200_E_INDEX, 2)  # the smallest position
    assert _err(lambda: ce.ck_derive_by_address(ck, [0], 0)) == (B200_E_INDEX, 0)  # table_size = 0 with an address
    assert _err(lambda: ce.ck_derive_by_address(ck, [], 0)) == (B200_E_ARG, None)  # table_size = 0, m = 0
    assert _err(lambda: ce.ck_derive_by_address(ck, [0], 1 << 31)) == (B200_E_RANGE, None)  # 31-bit table indices
    assert _err(lambda: ce.ck_derive_by_address(ck, [0], 4, window_bits=30)) == (B200_E_ARG, None)
    # a 64-bit address that would wrap to slot 3 in 32 bits is out of range at its own position
    assert _err(lambda: ce.ck_derive_by_address(ck, [0, (1 << 32) + 3], 8)) == (B200_E_INDEX, 1)
    unknown = nb.CommitmentKey.from_handle(nb.Curve(0), 987654, None, None, 8)
    assert _err(lambda: ce.ck_derive_by_address(unknown, [0], 1)) == (B200_E_HANDLE, None)
    unknown.handle = 0
    assert set(emu.keys) == before  # nothing registered on an error


# ---- the C++ mirror ------------------------------------------------------------------------------------------------
def build_cpp():
    exe = os.path.join(ROOT, "tests", "cpp", "derive_mirror_test")
    src = exe + ".cpp"
    hdrs = [os.path.join(ROOT, "include", f) for f in ("nova_b200.hpp", "nova_b200.h")]
    lib = os.path.join(ROOT, "nova_b200", "libnova_b200.so")
    if not os.path.exists(exe) or any(os.path.getmtime(p) > os.path.getmtime(exe) for p in [src, lib] + hdrs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", src, "-o", exe, "-L" + os.path.dirname(lib),
                               "-lnova_b200", "-Wl,-rpath," + os.path.dirname(lib)])
    return exe


def test_cpp_mirror_derive_compiles_and_links():
    out = subprocess.check_output([build_cpp(), "--compile-check"], text=True)
    assert "derive_mirror_test" in out
