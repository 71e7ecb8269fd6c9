"""The ck_derive_by_address entries (b200_ck_derive_by_address and its _dev twin) for the CPU stand-in of the library,
tests/emulated_device.py.  TEST INFRASTRUCTURE ONLY.

`install()` installs the emulated device as `emulated_device.install()` does and adds both entries, answered by the C
oracle's restatement (tests/derive_ref.py) with the library's status codes and order of checks
(include/nova_b200.h); `uninstall()` is `emulated_device.uninstall()`.  This checks the host logic of the mirror, not
the CUDA kernels (tests/test_derive_by_address_gpu.py does that)."""
import ctypes
import types

import derive_ref
import emulated_device
from emulated_device import _addr, _rd

E_ARG, E_HANDLE, E_RANGE, E_POINT, E_INDEX = 1, 3, 5, 7, 9
FIELD_BITS = {0: 254, 1: 254, 2: 255, 3: 255}  # scalar field bits per curve id


def _window(n: int) -> int:  # choose_window of csrc/capi.cu
    lg = max(n - 1, 0).bit_length()
    c = min(max(lg, 8), 16)
    return 20 if lg >= 22 else (17 if lg >= 19 else c)


def _derive(self, handle, addresses, table_size, window_bits, out_handle, first_bad):
    if first_bad is not None:
        first_bad._obj.value = ctypes.c_size_t(-1).value
    if window_bits != 0 and not 2 <= window_bits <= 24:
        self.err = b"window_bits out of range"
        return E_ARG
    if handle not in self.keys:
        self.err = b"unknown key handle"
        return E_HANDLE
    curve_id, bases, h = self.keys[handle]
    n = len(bases) // 64
    bad = next((i for i in range(n) if bases[64 * i:64 * i + 64] == bytes(64)), None)
    if bad is not None:  # the reference's panic in ck_to_group_elements
        return self._derive_fail(E_POINT, b"identity generator", first_bad, bad)
    if len(addresses) > n:
        return self._derive_fail(E_RANGE, b"InvalidCommitmentKeyLength", first_bad, None)
    bad = next((i for i, a in enumerate(addresses) if a >= table_size), None)
    if bad is not None:
        return self._derive_fail(E_INDEX, b"InvalidIndex", first_bad, bad)
    if table_size == 0:
        return self._derive_fail(E_ARG, b"table_size = 0", first_bad, None)
    c = window_bits or _window(table_size)
    if table_size >= 1 << 31 or -(-FIELD_BITS[curve_id] // c) * (table_size + (h is not None)) >= 1 << 31:
        return self._derive_fail(E_RANGE, b"table too large for 31-bit table indices", first_bad, None)
    derived = derive_ref.derive(curve_id, bases, addresses, table_size)
    self.keys[self.next_handle] = (curve_id, derived, h)
    out_handle._obj.value = self.next_handle
    self.next_handle += 1
    return 0


def _derive_fail(self, code, msg, first_bad, index):
    if index is not None and first_bad is not None:
        first_bad._obj.value = index
    self.err = msg
    return code


def b200_ck_derive_by_address(self, handle, addresses, m, table_size, window_bits, out_handle, first_bad):
    if m and not _addr(addresses):
        self.err = b"null pointer"
        return E_ARG
    return _derive(self, handle, [int(addresses[i]) for i in range(m)], table_size, window_bits, out_handle, first_bad)


def b200_ck_derive_by_address_dev(self, handle, d_addresses, m, table_size, window_bits, out_handle, first_bad,
                                  stream):
    if m and not _addr(d_addresses):
        self.err = b"null pointer"
        return E_ARG
    addrs = list((ctypes.c_uint32 * m).from_buffer_copy(_rd(d_addresses, 4 * m))) if m else []
    return _derive(self, handle, addrs, table_size, window_bits, out_handle, first_bad)


def install() -> "emulated_device.EmulatedDevice":
    dev = emulated_device.install()
    dev._derive_fail = types.MethodType(_derive_fail, dev)
    dev.b200_ck_derive_by_address = types.MethodType(b200_ck_derive_by_address, dev)
    dev.b200_ck_derive_by_address_dev = types.MethodType(b200_ck_derive_by_address_dev, dev)
    return dev


def uninstall():
    emulated_device.uninstall()
