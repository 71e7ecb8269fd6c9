"""The spark entry point (b200_spark_repr_dev) for the CPU stand-in of the library, tests/emulated_device.py.
TEST INFRASTRUCTURE ONLY.

`install()` installs the emulated device as `emulated_device.install()` does and adds the entry, answered by
oracle/ppsnark_ref.py's SparkRepr on the CSR the emulated spmv registry holds; `uninstall()` is
`emulated_device.uninstall()`.  Like the rest of the emulation this checks the host logic of the mirror, not the
CUDA kernel (tests/test_spark_ipa_gpu.py does that)."""
import ctypes
import types

import emulated_device
from emulated_device import FIELD_MODULUS, _wr
from oracle.pyref import from_mont_bytes, mont_bytes


def b200_spark_repr_dev(self, hA, hB, hC, N, vecs, row_idx, col_idx, stream):
    from oracle import ppsnark_ref as pr
    if any(h not in self.mats for h in (hA, hB, hC)):
        self.err = b"unknown matrix handle"
        return 3
    mats = [self.mats[h] for h in (hA, hB, hC)]
    if len({(m[0], m[4], m[5]) for m in mats}) != 1:
        self.err = b"spark_repr: matrices differ in field or shape"
        return 1
    fid, _, _, _, rows, cols = mats[0]
    P = FIELD_MODULUS[fid]
    triplets = []
    for _, data, idx, ip, _, _ in mats:
        triplets.append([(r, idx[e], from_mont_bytes(P, data[32 * e:32 * e + 32]))
                         for r in range(rows) for e in range(ip[r], ip[r + 1])])
    total = sum(len(t) for t in triplets)
    if N == 0 or N & (N - 1) or N >= 1 << 32:
        self.err = b"spark_repr: N is not a power of two below 2^32"
        return 1
    if N < max(total, rows, cols):
        self.err = b"spark_repr: N is below nnz, rows or cols"
        return 5
    spark = pr.SparkRepr(P, *triplets, N, 0)  # num_cons = N, num_vars = 0: the size is the caller's N
    assert spark.N == N
    for j, name in enumerate(("row", "col", "val_A", "val_B", "val_C", "ts_row", "ts_col")):
        _wr(vecs[j], b"".join(mont_bytes(P, x) for x in getattr(spark, name)))
    _wr(row_idx, bytes((ctypes.c_uint32 * N)(*spark.row_idx)))
    _wr(col_idx, bytes((ctypes.c_uint32 * N)(*spark.col_idx)))
    return 0


def install() -> "emulated_device.EmulatedDevice":
    dev = emulated_device.install()
    dev.b200_spark_repr_dev = types.MethodType(b200_spark_repr_dev, dev)
    return dev


def uninstall():
    emulated_device.uninstall()

