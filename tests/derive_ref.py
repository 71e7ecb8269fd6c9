"""ck_derive_by_address by the C oracle (tests/derive_oracle.c on top of oracle/oracle.c) and by the naive Python group
law of oracle/pyref.py.  TEST INFRASTRUCTURE ONLY.

The shared object is compiled on first use into the temporary directory, keyed by a hash of its sources, so that a
read-only checkout works and a changed source is never served stale."""
from __future__ import annotations

import ctypes
import hashlib
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCES = [os.path.join(ROOT, "tests", "derive_oracle.c"), os.path.join(ROOT, "oracle", "oracle.c"),
           os.path.join(ROOT, "oracle", "field_constants.h")]
_LIB = None

# return codes of orc_ck_derive_by_address -> the reference's outcome
IDENTITY_GENERATOR, KEY_LENGTH, INVALID_INDEX = 2, 3, 4


class DeriveError(Exception):
    def __init__(self, code: int, first_bad):
        super().__init__({IDENTITY_GENERATOR: "identity generator", KEY_LENGTH: "InvalidCommitmentKeyLength",
                          INVALID_INDEX: "InvalidIndex"}.get(code, f"error {code}"))
        self.code, self.first_bad = code, first_bad


def lib():
    global _LIB
    if _LIB is None:
        h = hashlib.sha256()
        for p in SOURCES:
            with open(p, "rb") as f:
                h.update(f.read())
        so = os.path.join(tempfile.gettempdir(), f"nova_b200_derive_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-O3", "-std=gnu11", "-fPIC", "-fvisibility=hidden", "-Wall",
                                   "-Wno-unused-function", "-shared", "-o", tmp, SOURCES[0], "-lpthread"])
            os.replace(tmp, so)
        _LIB = ctypes.CDLL(so)
    return _LIB


def derive(curve: int, bases: bytes, addresses, table_size: int) -> bytes:
    """derived bases (table_size x 64 B, affine Montgomery, identity = zeros); raises DeriveError like the reference"""
    m, n = len(addresses), len(bases) // 64
    arr = (ctypes.c_uint64 * max(m, 1))(*addresses)
    out = ctypes.create_string_buffer(max(64 * table_size, 1))
    bad = ctypes.c_size_t(0)
    rc = lib().orc_ck_derive_by_address(curve, ctypes.create_string_buffer(bytes(bases), max(len(bases), 1)),
                                        ctypes.c_size_t(n), arr, ctypes.c_size_t(m), ctypes.c_size_t(table_size), out,
                                        ctypes.byref(bad))
    if rc:
        raise DeriveError(rc, None if bad.value == ctypes.c_size_t(-1).value else bad.value)
    return out.raw[:64 * table_size]


def derive_naive(curve: int, bases: bytes, addresses, table_size: int) -> bytes:
    """the same sum with the Python big-int group law (small sizes)"""
    from oracle.pyref import CURVES
    c = CURVES[curve]
    pts = [c.affine_from_bytes(bases[64 * i:64 * i + 64]) for i in range(len(bases) // 64)]
    if any(P is None for P in pts):
        raise DeriveError(IDENTITY_GENERATOR, next(i for i, P in enumerate(pts) if P is None))
    if len(addresses) > len(pts):
        raise DeriveError(KEY_LENGTH, None)
    acc = [None] * table_size
    for i, a in enumerate(addresses):
        if a >= table_size:
            raise DeriveError(INVALID_INDEX, i)
        acc[a] = c.add(acc[a], pts[i])
    return b"".join(c.affine_bytes(P) for P in acc)
