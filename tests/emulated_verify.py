"""The verifier entries (b200_r1cs_eval, b200_r1cs_eval_dev, b200_ipa_s_dev) for the CPU stand-in of the library,
tests/emulated_device.py.  TEST INFRASTRUCTURE ONLY.

`install()` installs the emulated device as `emulated_device.install()` does and adds the three entries, answered by
the C restatement of the reference's loops (tests/verify_ref.py) with the library's status codes and order of checks
(include/nova_b200.h); `uninstall()` is `emulated_device.uninstall()`.  This checks the host logic of the mirror, not
the CUDA kernels (tests/test_verify_kernels_host.py and tests/test_verify_gpu.py do that)."""
import ctypes
import types

import emulated_device
import verify_ref
from emulated_device import _addr, _rd, _wr
from oracle import coracle as co
from oracle.pyref import FIELD_MODULUS, from_mont_bytes

E_ARG, E_HANDLE, E_RANGE = 1, 3, 5


def _lookup(self, handles, k, tx_len, ty_len):
    if not _addr(handles):
        self.err = b"null pointer"
        return E_ARG, None
    if k == 0 or k > 3:
        self.err = b"r1cs_eval: k matrices (1 .. 3)"
        return E_ARG, None
    mats = []
    for y in range(k):
        if handles[y] not in self.mats:
            self.err = b"unknown matrix handle"
            return E_HANDLE, None
        mats.append(self.mats[handles[y]])
    if any(m[0] != mats[0][0] for m in mats):
        self.err = b"r1cs_eval: matrices of different fields"
        return E_ARG, None
    if any(m[4] > tx_len or m[5] > ty_len for m in mats):
        self.err = b"r1cs_eval: T_x or T_y too short"
        return E_RANGE, None
    return 0, mats


def b200_r1cs_eval_dev(self, handles, k, tx, tx_len, ty, ty_len, out, stream):
    rc, mats = _lookup(self, handles, k, tx_len, ty_len)
    if rc:
        return rc
    if not (_addr(tx) and _addr(ty) and _addr(out)):
        self.err = b"null pointer"
        return E_ARG
    Tx, Ty = _rd(tx, 32 * tx_len), _rd(ty, 32 * ty_len)
    _wr(out, b"".join(verify_ref.r1cs_eval(fid, data, idx, ip, Tx, Ty) for (fid, data, idx, ip, rows, cols) in mats))
    return 0


def b200_r1cs_eval(self, handles, k, r_x, ell_x, r_y, ell_y, out):
    if not (0 <= ell_x <= 34 and 0 <= ell_y <= 34):
        self.err = b"ell out of range"
        return E_ARG
    rc, mats = _lookup(self, handles, k, 1 << ell_x, 1 << ell_y)
    if rc:
        return rc
    fid = mats[0][0]
    Tx, Ty = (ctypes.create_string_buffer(co.eq_table(fid, _rd(r, 32 * ell))) for r, ell in ((r_x, ell_x), (r_y, ell_y)))
    return b200_r1cs_eval_dev(self, handles, k, Tx, 1 << ell_x, Ty, 1 << ell_y, out, None)


def b200_ipa_s_dev(self, fid, r, r_inv, L, scale, out, stream):
    if fid not in FIELD_MODULUS or not 0 <= L <= 31:
        self.err = b"ipa_s: bad field or L"
        return E_ARG
    if not _addr(out) or (L and not (_addr(r) and _addr(r_inv))):
        self.err = b"null pointer"
        return E_ARG
    p = FIELD_MODULUS[fid]
    rs = [from_mont_bytes(p, _rd(_addr(r) + 32 * j, 32)) for j in range(L)]
    sc = from_mont_bytes(p, _rd(scale, 32)) if _addr(scale) else None
    _wr(out, verify_ref.ipa_s(fid, rs, sc))
    return 0


def install() -> "emulated_device.EmulatedDevice":
    dev = emulated_device.install()
    dev.b200_r1cs_eval_dev = types.MethodType(b200_r1cs_eval_dev, dev)
    dev.b200_r1cs_eval = types.MethodType(b200_r1cs_eval, dev)
    dev.b200_ipa_s_dev = types.MethodType(b200_ipa_s_dev, dev)
    return dev


def uninstall():
    emulated_device.uninstall()
