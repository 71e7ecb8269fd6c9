"""The verifier's linear-time pieces by the C oracle (tests/verify_oracle.c on top of oracle/oracle.c), plus the
host build of the real verifier kernels (tests/hostcheck/simt_verify.cpp).  TEST INFRASTRUCTURE ONLY.

Shared objects are compiled on first use into the temporary directory, keyed by a hash of their sources, so that a
read-only checkout works and a changed source is never served stale."""
from __future__ import annotations

import ctypes
import hashlib
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "nova_b200", "csrc")
_LIBS = {}


def _build(name: str, sources: list, cmd) -> ctypes.CDLL:
    if name not in _LIBS:
        h = hashlib.sha256()
        for p in sources:
            with open(p, "rb") as f:
                h.update(f.read())
        so = os.path.join(tempfile.gettempdir(), f"nova_b200_{name}_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(cmd(tmp))
            os.replace(tmp, so)
        _LIBS[name] = ctypes.CDLL(so)
    return _LIBS[name]


def lib() -> ctypes.CDLL:
    src = os.path.join(ROOT, "tests", "verify_oracle.c")
    sources = [src, os.path.join(ROOT, "oracle", "oracle.c"), os.path.join(ROOT, "oracle", "field_constants.h")]
    return _build("verify_oracle", sources, lambda out: ["gcc", "-O3", "-std=gnu11", "-fPIC", "-fvisibility=hidden",
                                                         "-Wall", "-Wno-unused-function", "-shared", "-o", out, src,
                                                         "-lpthread"])


def simt() -> ctypes.CDLL:
    src = os.path.join(ROOT, "tests", "hostcheck", "simt_verify.cpp")
    sources = [src, os.path.join(ROOT, "tests", "hostcheck", "simt_host.h")] + sorted(
        os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh"))
    return _build("simt_verify", sources, lambda out: ["g++", "-O2", "-std=c++17", "-pthread", "-shared", "-fPIC",
                                                       "-x", "c++", src, "-o", out])


def _buf(b: bytes):
    return ctypes.create_string_buffer(bytes(b), max(len(b), 1))


def r1cs_eval(fid: int, data: bytes, indices, indptr, Tx: bytes, Ty: bytes, nthreads: int = 1) -> bytes:
    """sum_e T_x[row_e] T_y[col_e] val_e of one CSR matrix (Montgomery bytes in and out)"""
    rows = len(indptr) - 1
    idx = (ctypes.c_uint64 * max(len(indices), 1))(*indices)
    ip = (ctypes.c_uint64 * len(indptr))(*indptr)
    out = ctypes.create_string_buffer(32)
    assert lib().orc_r1cs_eval_par(fid, _buf(data), idx, ip, ctypes.c_size_t(rows), _buf(Tx), _buf(Ty), out,
                                   nthreads) == 0
    return out.raw


def ipa_s(fid: int, r: list, scale: int | None = None) -> bytes:
    """the reference's s for challenges r (ints), times scale; Montgomery bytes"""
    from oracle.pyref import FIELD_MODULUS, mont_bytes
    p = FIELD_MODULUS[fid]
    inv = [pow(x, -1, p) for x in r]
    ri = b"".join(mont_bytes(p, x) for x in inv)
    rs = b"".join(mont_bytes(p, x * x % p) for x in r)
    out = ctypes.create_string_buffer(32 << len(r))
    sc = _buf(mont_bytes(p, scale % p)) if scale is not None else None
    assert lib().orc_ipa_s(fid, _buf(ri), _buf(rs), len(r), sc, out) == 0
    return out.raw


def simt_r1cs_eval(fid: int, mats: list, Tx: bytes, Ty: bytes, grid: int, chunk: int = 0) -> bytes:
    """the real k_r1cs_eval + k_r1cs_final on host threads; mats = [(data, indices, indptr)] (k <= 3)"""
    k = len(mats)
    keep = []
    ips, cis, vals = (ctypes.c_void_p * k)(), (ctypes.c_void_p * k)(), (ctypes.c_void_p * k)()
    rows, nnz = (ctypes.c_size_t * k)(), (ctypes.c_size_t * k)()
    for y, (data, indices, indptr) in enumerate(mats):
        ip = (ctypes.c_uint32 * len(indptr))(*indptr)
        ci = (ctypes.c_uint32 * max(len(indices), 1))(*indices)
        dv = _buf(data)
        keep += [ip, ci, dv]
        ips[y], cis[y], vals[y] = ctypes.addressof(ip), ctypes.addressof(ci), ctypes.addressof(dv)
        rows[y], nnz[y] = len(indptr) - 1, len(indices)
    out = ctypes.create_string_buffer(32 * k)
    tx, ty = _buf(Tx), _buf(Ty)
    assert simt().hc_simt_r1cs_eval(fid, k, ips, cis, vals, rows, nnz, tx, ty, grid, ctypes.c_size_t(chunk), out) == 0
    return out.raw


def simt_ipa_s(fid: int, r_mont: bytes, r_inv_mont: bytes, L: int, scale_mont: bytes | None, direct_bits: int) -> bytes:
    out = ctypes.create_string_buffer(32 << L)
    rc = simt().hc_simt_ipa_s(fid, _buf(r_mont), _buf(r_inv_mont), L, _buf(scale_mont) if scale_mont else None,
                              direct_bits, out)
    assert rc == 0
    return out.raw


def cpp_mirror() -> str:
    """tests/cpp/verify_mirror_test built against the library (in the temporary directory, keyed by the sources and
    the library's modification time)"""
    src = os.path.join(ROOT, "tests", "cpp", "verify_mirror_test.cpp")
    libdir = os.path.join(ROOT, "nova_b200")
    sources = [src] + [os.path.join(ROOT, "include", f) for f in ("nova_b200.hpp", "nova_b200.h")]
    h = hashlib.sha256(str(os.path.getmtime(os.path.join(libdir, "libnova_b200.so"))).encode())
    for p in sources:
        with open(p, "rb") as f:
            h.update(f.read())
    exe = os.path.join(tempfile.gettempdir(), f"nova_b200_verify_mirror_{os.getuid()}_{h.hexdigest()[:16]}")
    if not os.path.exists(exe):
        tmp = f"{exe}.{os.getpid()}.tmp"
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", src, "-o", tmp, "-L" + libdir, "-lnova_b200",
                               "-Wl,-rpath," + libdir])
        os.replace(tmp, exe)
    return exe
