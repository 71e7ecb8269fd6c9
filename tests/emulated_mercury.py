"""The Mercury entry points (b200_mat_vec_rows, b200_div_binomial, b200_mercury_s_poly) for the CPU stand-in of
the library, tests/emulated_device.py.  TEST INFRASTRUCTURE ONLY.

`install()` installs the emulated device as `emulated_device.install()` does and adds the three entries (and their
host-pointer forms) to it, answered by oracle/mercury_ref.py on the bytes behind the pointers; `uninstall()` is
`emulated_device.uninstall()`.  Like the rest of the emulation this checks the host logic of the mirror, not the
CUDA kernels (tests/test_mercury_gpu.py does that)."""
import types

import emulated_device
from emulated_device import FIELD_MODULUS


def b200_mat_vec_rows_dev(self, fid, f, rows, cols, v, out, stream):
    from oracle import mercury_ref as mr
    self._put(fid, out, mr.compute_h_poly(FIELD_MODULUS[fid], self._ints(fid, f, rows * cols),
                                          self._ints(fid, v, cols), rows, cols))
    return 0


def b200_div_binomial_dev(self, fid, f, rows, cols, alpha, q, g, stream):
    from oracle import mercury_ref as mr
    if rows == 0 or cols == 0:
        self.err = b"empty matrix"
        return 1
    quot, rem = mr.divide_columns(FIELD_MODULUS[fid], self._ints(fid, f, rows * cols), rows, cols,
                                  self._ints(fid, alpha, 1)[0])
    if rows > 1:
        self._put(fid, q, quot)
    self._put(fid, g, rem)
    return 0


def b200_mercury_s_poly_dev(self, fid, a1, b1, a2, b2, b, gamma, out, stream):
    from oracle import mercury_ref as mr
    vs = [self._ints(fid, v, b) for v in (a1, b1, a2, b2)]
    self._put(fid, out, mr.s_poly_direct(FIELD_MODULUS[fid], *vs, self._ints(fid, gamma, 1)[0]))
    return 0


def b200_mat_vec_rows(self, fid, f, rows, cols, v, out):
    return self.b200_mat_vec_rows_dev(fid, f, rows, cols, v, out, None)


def b200_div_binomial(self, fid, f, rows, cols, alpha, q, g):
    return self.b200_div_binomial_dev(fid, f, rows, cols, alpha, q, g, None)


def b200_mercury_s_poly(self, fid, a1, b1, a2, b2, b, gamma, out):
    return self.b200_mercury_s_poly_dev(fid, a1, b1, a2, b2, b, gamma, out, None)


_ENTRIES = (b200_mat_vec_rows_dev, b200_div_binomial_dev, b200_mercury_s_poly_dev,
            b200_mat_vec_rows, b200_div_binomial, b200_mercury_s_poly)


def install() -> "emulated_device.EmulatedDevice":
    dev = emulated_device.install()
    for fn in _ENTRIES:
        setattr(dev, fn.__name__, types.MethodType(fn, dev))
    return dev


def uninstall():
    emulated_device.uninstall()
