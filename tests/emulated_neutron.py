"""The NeutronNova entry points (b200_neutron_evals, b200_pow_split_evals, b200_lerp) for the CPU stand-in of the
library, tests/emulated_device.py.  TEST INFRASTRUCTURE ONLY.

`install()` installs the emulated device as `emulated_device.install()` does and adds the three entries (and their
host-pointer forms) to it, answered by oracle/neutron_ref.py on the bytes behind the pointers; `uninstall()` is
`emulated_device.uninstall()`.  Like the rest of the emulation this checks the host logic of the mirror, not the
CUDA kernels (tests/test_neutron_gpu.py does that)."""
import types

import emulated_device
from emulated_device import FIELD_MODULUS


def b200_neutron_evals_dev(self, fid, e1, az1, bz1, cz1, e2, az2, bz2, cz2, left, right, out, stream):
    from oracle import neutron_ref as nr
    if left == 0 or right == 0:
        self.err = b"empty split"
        return 1
    n = left * right
    vs = [self._ints(fid, v, left + right if k % 4 == 0 else n)
          for k, v in enumerate((e1, az1, bz1, cz1, e2, az2, bz2, cz2))]
    self._put(fid, out, nr.prove_helper_raw(FIELD_MODULUS[fid], left, right, *vs))
    return 0


def b200_pow_split_evals_dev(self, fid, tau, left, right, out, stream):
    from oracle import neutron_ref as nr
    if left == 0 or right < 2:
        self.err = b"split_evals needs left >= 1 and right >= 2"
        return 1
    self._put(fid, out, nr.split_evals(FIELD_MODULUS[fid], self._ints(fid, tau, 1)[0], left, right))
    return 0


def b200_lerp_dev(self, fid, a, b, r, n, out, stream):
    p = FIELD_MODULUS[fid]
    rv = self._ints(fid, r, 1)[0]
    self._put(fid, out, [(x + rv * (y - x)) % p for x, y in zip(self._ints(fid, a, n), self._ints(fid, b, n))])
    return 0


def b200_neutron_evals(self, fid, e1, az1, bz1, cz1, e2, az2, bz2, cz2, left, right, out):
    return self.b200_neutron_evals_dev(fid, e1, az1, bz1, cz1, e2, az2, bz2, cz2, left, right, out, None)


def b200_pow_split_evals(self, fid, tau, left, right, out):
    return self.b200_pow_split_evals_dev(fid, tau, left, right, out, None)


def b200_lerp(self, fid, a, b, r, n, out):
    return self.b200_lerp_dev(fid, a, b, r, n, out, None)


_ENTRIES = (b200_neutron_evals_dev, b200_pow_split_evals_dev, b200_lerp_dev,
            b200_neutron_evals, b200_pow_split_evals, b200_lerp)


def install() -> "emulated_device.EmulatedDevice":
    dev = emulated_device.install()
    for fn in _ENTRIES:
        setattr(dev, fn.__name__, types.MethodType(fn, dev))
    return dev


def uninstall():
    emulated_device.uninstall()
