"""Host-side mirror of the MicroSpartan (ppsnark) prover up to the batched opening claim
(src/spartan/ppsnark.rs:1056-1355), with every O(N) step on the device:

  R1CSShapeSparkRepr (::new, ::evaluation_oracles)             ppsnark.rs:113-198, 220-253
  MemorySumcheckInstance (::compute_oracles, engine)           ppsnark.rs:328-670
  InnerBatchedSumcheckInstance                                 ppsnark.rs:677-786
  WitnessBoundSumcheck (masked eq, polys/masked_eq.rs:65-76)   ppsnark.rs:270-325
  prove_helper (3 engines, 9 claims, one cubic per round)      ppsnark.rs:886-983
  prove_core = RelaxedR1CSSNARK::prove minus EE::prove         ppsnark.rs:1056-1355

The 16 size-N polynomials of the inner sum-check stay resident in HBM.  Per round the host enqueues
the nine reductions (2 linear, 2 eq-cubic-3, 2 eq-cubic-2, 1 cubic, 1 eq-quadratic-1, 1 quadratic)
into ONE result buffer, reads it back once (9 x 96 B), does the O(1) claim derivation / UniPoly /
transcript work on Python integers exactly as the Rust host would, uploads the challenge once and
enqueues the 16 binds.  The transcript is passed in (absorb_bytes / squeeze), as in spartan.py.
"""
from __future__ import annotations

import ctypes

from . import fields
from .native import check, lib
from .provider import CommitmentKey, _cbuf, _jac_to_affine
from .spartan import (SC_CUBIC, SC_EQ_CUBIC2, SC_EQ_CUBIC2_M1, SC_EQ_CUBIC3, SC_EQ_CUBIC3_M1, SC_EQ_QUAD1,
                      SC_EQ_QUAD1_M1, SC_LINEAR, SC_NOUT, SC_QUADRATIC, DeviceVec, EqSumCheckInstance,
                      SparseMatrix, SumcheckProof, UniPoly, _bind_all, _challenge_dev, _sc_eval_dev, _small_buf,
                      commit_many_dev, update_claim)


SCB_RAW3, SCB_LIN2, SCB_EQ_DEG2, SCB_EQ_DEG1 = range(4)  # b200_scb_desc.kind (include/nova_b200.h)
SCB_MAX_CLAIMS, SCB_MAX_EQ = 16, 4


class ScbDesc(ctypes.Structure):
    """b200_scb_desc"""
    _fields_ = [("nclaims", ctypes.c_int32), ("neq", ctypes.c_int32), ("kind", ctypes.c_int32 * SCB_MAX_CLAIMS),
                ("slot", ctypes.c_int32 * SCB_MAX_CLAIMS), ("slot_m1", ctypes.c_int32 * SCB_MAX_CLAIMS),
                ("eq_of", ctypes.c_int32 * SCB_MAX_CLAIMS), ("tau", ctypes.c_void_p * SCB_MAX_EQ),
                ("tau_inv", ctypes.c_void_p * SCB_MAX_EQ)]


SCP_MAX_TABLES = 24


class ScpProgram(ctypes.Structure):
    """b200_scp_program"""
    _fields_ = [("nclaims", ctypes.c_int32), ("neq", ctypes.c_int32), ("ntables", ctypes.c_int32),
                ("num_rounds", ctypes.c_int32), ("kind", ctypes.c_int32 * SCB_MAX_CLAIMS),
                ("form", ctypes.c_int32 * SCB_MAX_CLAIMS), ("form_m1", ctypes.c_int32 * SCB_MAX_CLAIMS),
                ("eq_of", ctypes.c_int32 * SCB_MAX_CLAIMS), ("tab", (ctypes.c_int32 * 3) * SCB_MAX_CLAIMS),
                ("tables", ctypes.c_void_p * SCP_MAX_TABLES), ("taus", ctypes.c_void_p * SCB_MAX_EQ)]


def to_repr(x: int) -> bytes:
    return int(x).to_bytes(32, "little")  # canonical little-endian (traits.rs:323-327)


class View:
    """`n` field elements starting `off` elements into a DeviceVec (keeps the allocation alive)."""

    def __init__(self, base: DeviceVec, off: int = 0):
        self.base = base
        self.ptr = ctypes.c_void_p(base.ptr.value + 32 * off)


def dev_zeros(n: int) -> DeviceVec:
    v = DeviceVec(32 * n)
    check(lib().b200_memset_dev(v.ptr, 0, 32 * n, None))
    return v


def dev_copy(src, n: int) -> DeviceVec:
    v = DeviceVec(32 * n)
    check(lib().b200_memcpy_d2d(v.ptr, src.ptr, 32 * n, None))
    return v


def dev_padded(src, n_src: int, n: int) -> DeviceVec:
    """padded() with e = 0 (ppsnark.rs:41-47)."""
    v = dev_zeros(n)
    check(lib().b200_memcpy_d2d(v.ptr, src.ptr, 32 * n_src, None))
    return v


def dev_scalar(fid: int, x: int) -> DeviceVec:
    return DeviceVec.from_bytes(fields.to_mont_bytes(fid, x))


def dev_from_u64(fid: int, xs) -> DeviceVec:
    """Small non-negative integers (numpy array / list of u64) -> Montgomery field vector, converted
    on the device: canonical rows [x, 0, 0, 0] are multiplied by R^2 (axpy with a = 0)."""
    import numpy as np
    a = np.zeros((len(xs), 4), dtype=np.uint64)
    a[:, 0] = np.asarray(xs, dtype=np.uint64)
    n = len(xs)
    raw = DeviceVec(32 * n)
    check(lib().b200_memcpy_h2d(raw.ptr, a.ctypes.data_as(ctypes.c_void_p), 32 * n))
    p = fields.MODULUS[fid]
    r2 = DeviceVec.from_bytes((fields.R * fields.R % p).to_bytes(32, "little"))
    zero = dev_zeros(n)
    out = DeviceVec(32 * n)
    check(lib().b200_axpy_dev(fid, zero.ptr, raw.ptr, r2.ptr, n, out.ptr, None))
    check(lib().b200_sync())
    return out


def _as_dev(x) -> DeviceVec:
    return x if hasattr(x, "ptr") else DeviceVec.from_bytes(x)


def dev_u32(xs) -> DeviceVec:
    if hasattr(xs, "ctypes"):  # numpy uint32 array
        v = DeviceVec(4 * max(len(xs), 1))
        check(lib().b200_memcpy_h2d(v.ptr, xs.ctypes.data_as(ctypes.c_void_p), 4 * len(xs)))
        return v
    raw = (ctypes.c_uint32 * max(len(xs), 1))(*xs)
    v = DeviceVec(4 * max(len(xs), 1))
    check(lib().b200_memcpy_h2d(v.ptr, raw, 4 * len(xs)))
    return v


class Shard:
    """Cyclic sharding of the sum-check tables over `world` ranks (SURVEY.md §8e): rank `rank` holds the global
    entries rank, rank + world, ...; `reduce(list of ints) -> list of ints` adds the ranks' partial sums."""

    def __init__(self, rank: int, world: int, reduce):
        self.rank, self.world, self.reduce = rank, world, reduce


def _sc_eval_one(shard, fid, form, A, B, C, length, L, R, shift) -> list:
    """one reduction read back at once (the tau = 0 third sums); `shard`: the engine's Shard or None"""
    if shard is None:
        return _sc_eval_dev(fid, form, A, B, C, length, L, R, shift)
    sums = RoundSums(fid, shard=shard)
    sums.add(form, A, B, C, length, L, R, shift)
    return sums.fetch()[0]


class RoundSums:
    """All reductions of one sum-check round in one result buffer, one read-back (and, when the tables are
    sharded, one exchange of the partial sums)."""

    def __init__(self, fid: int, cap: int = 16, shard: "Shard | None" = None):
        self.fid, self.out, self.nout, self.shard = fid, _small_buf("round_sums", 96 * cap), [], shard

    def add(self, form, A, B, C, length, L=None, R=None, shift=0) -> int:
        k = len(self.nout)
        dst = ctypes.c_void_p(self.out.ptr.value + 96 * k)
        a = (self.fid, form, A.ptr, B.ptr if B else None, C.ptr if C else None, length,
             L.ptr if L else None, R.ptr if R else None, shift)
        if self.shard is None:
            check(lib().b200_sc_eval_dev(*a, dst, None))
        else:  # local index j stands for the global index j * world + rank
            check(lib().b200_sc_eval_sharded_dev(*a, self.shard.world, self.shard.rank, dst, None))
        self.nout.append(SC_NOUT[form])
        return k

    def reset(self):
        """Forget the slots without reading them back (the device-transcript loop never fetches)."""
        self.nout = []

    def fetch(self):
        raw = self.out.to_bytes(96 * len(self.nout))
        res = [fields.unpack(self.fid, raw[96 * k:96 * k + 32 * n]) for k, n in enumerate(self.nout)]
        self.nout = []
        if self.shard is not None:
            flat = self.shard.reduce([x for r in res for x in r])
            it = iter(flat)
            res = [[next(it) for _ in r] for r in res]
        return res


def commit_dev(curve, ck: CommitmentKey, v, n: int):
    """CE::commit(ck, v, r = 0) of a device-resident vector -> affine (x, y) or None."""
    out = DeviceVec(96)
    check(lib().b200_commit_dev(ck.handle, v.ptr, n, None, out.ptr, None))
    return _jac_to_affine(curve, out.to_bytes(96))


def commitment_transcript_bytes(P) -> bytes:
    """pedersen.rs:103-117: x || y || is_infinity."""
    if P is None:
        return to_repr(0) + to_repr(0) + b"\x01"
    return to_repr(P[0]) + to_repr(P[1]) + b"\x00"


# ---------------------------------------------------------------------------------------------
class SparkRepr:
    """R1CSShapeSparkRepr::new (ppsnark.rs:113-198); vectors uploaded once, index arrays kept as
    u32 for the device gathers."""

    def __init__(self, fid: int, A, B, C, num_cons: int, num_vars: int):
        p = fields.MODULUS[fid]
        total = len(A) + len(B) + len(C)
        N = 1
        while N < max(total, 2 * num_vars, num_cons):
            N *= 2
        self.fid, self.N = fid, N
        row, col = [0] * N, [N - 1] * N
        for i, (r, c, _) in enumerate(list(A) + list(B) + list(C)):
            row[i], col[i] = r, c
        vals = [[0] * N for _ in range(3)]
        off = 0
        for k, M in enumerate((A, B, C)):
            for i, (_, _, v) in enumerate(M):
                vals[k][off + i] = v % p
            off += len(M)
        ts_row, ts_col = [0] * N, [0] * N
        for a in row:
            ts_row[a] += 1
        for a in col:
            ts_col[a] += 1
        up = lambda xs: DeviceVec.from_bytes(fields.pack(fid, xs))
        self.row, self.col, self.ts_row, self.ts_col = up(row), up(col), up(ts_row), up(ts_col)
        self.val_A, self.val_B, self.val_C = (up(v) for v in vals)
        self.row_idx, self.col_idx = dev_u32(row), dev_u32(col)

    @classmethod
    def from_numpy(cls, fid: int, rows, cols, vals_mont, num_cons: int, num_vars: int):
        """Same representation built with numpy for large synthetic shapes: rows/cols are uint32
        arrays over the concatenated entries of A, B, C; vals_mont = three (nnz_k, 4) uint64 arrays
        of Montgomery coefficients."""
        import numpy as np
        self = cls.__new__(cls)
        total = len(rows)
        N = 1
        while N < max(total, 2 * num_vars, num_cons):
            N *= 2
        self.fid, self.N = fid, N
        row = np.zeros(N, dtype=np.uint32)
        col = np.full(N, N - 1, dtype=np.uint32)
        row[:total], col[:total] = rows, cols
        self.row, self.col = dev_from_u64(fid, row), dev_from_u64(fid, col)
        self.ts_row = dev_from_u64(fid, np.bincount(row, minlength=N))
        self.ts_col = dev_from_u64(fid, np.bincount(col, minlength=N))
        off, vs = 0, []
        for v in vals_mont:
            buf = np.zeros((N, 4), dtype=np.uint64)
            buf[off:off + len(v)] = v
            off += len(v)
            d = DeviceVec(32 * N)
            check(lib().b200_memcpy_h2d(d.ptr, buf.ctypes.data_as(ctypes.c_void_p), 32 * N))
            vs.append(d)
        self.val_A, self.val_B, self.val_C = vs
        self.row_idx, self.col_idx = dev_u32(row), dev_u32(col)
        return self

    @classmethod
    def from_shape(cls, fid: int, S: dict):
        """The same representation built on the device from the three registered matrices of `S` (the dict
        `prove` takes: A/B/C `spartan.SparseMatrix`, num_cons, num_vars) by b200_spark_repr_dev: nothing is
        read back or uploaded but the pointers."""
        A, B, C = S["A"], S["B"], S["C"]
        if any(M.fid != fid for M in (A, B, C)):
            raise ValueError(f"the matrices are not over field {fid}")
        self = cls.__new__(cls)
        N = 1
        while N < max(A.nnz + B.nnz + C.nnz, 2 * S["num_vars"], S["num_cons"]):
            N *= 2
        self.fid, self.N = fid, N
        vecs = [DeviceVec(32 * N) for _ in range(7)]
        self.row, self.col, self.val_A, self.val_B, self.val_C, self.ts_row, self.ts_col = vecs
        self.row_idx, self.col_idx = DeviceVec(4 * N), DeviceVec(4 * N)
        ptrs = (ctypes.c_void_p * 7)(*[v.ptr.value for v in vecs])
        check(lib().b200_spark_repr_dev(A.handle, B.handle, C.handle, N, ptrs, self.row_idx.ptr, self.col_idx.ptr,
                                        None))
        return self

    def evaluation_oracles(self, r_outer_full: list, z, z_len: int):
        """ppsnark.rs:220-253 -> (mem_row, mem_col, L_row, L_col), all of length N on the device."""
        fid, N = self.fid, self.N
        assert (1 << len(r_outer_full)) == N
        mem_row = DeviceVec(32 * N)
        r_dev = DeviceVec.from_bytes(fields.pack(fid, r_outer_full))  # named: must outlive the launches below
        check(lib().b200_eq_table_dev(fid, r_dev.ptr, len(r_outer_full), mem_row.ptr, None))
        mem_col = dev_padded(z, z_len, N)
        L_row, L_col = DeviceVec(32 * N), DeviceVec(32 * N)
        check(lib().b200_gather_dev(mem_row.ptr, self.row_idx.ptr, N, L_row.ptr, None))
        check(lib().b200_gather_dev(mem_col.ptr, self.col_idx.ptr, N, L_col.ptr, None))
        check(lib().b200_sync())  # r_dev is released on return
        return mem_row, mem_col, L_row, L_col


def memory_compute_oracles(fid, r: int, gamma: int, N: int, mem_row, addr_row, L_row, ts_row, mem_col, addr_col,
                           L_col, ts_col):
    """MemorySumcheckInstance::compute_oracles without the commitments (ppsnark.rs:372-455).
    Returns ([t_inv_row, w_inv_row, t_inv_col, w_inv_col], [t_row, w_row, t_col, w_col]) as Views.
    Raises ValueError("InternalError") if an inversion meets zero (spartan/mod.rs:98-100)."""
    g, rr = dev_scalar(fid, gamma), dev_scalar(fid, r)
    flag = DeviceVec(4)
    oracles, aux = [], []
    for mem, addr, L, ts in ((mem_row, addr_row, L_row, ts_row), (mem_col, addr_col, L_col, ts_col)):
        tw = DeviceVec(64 * N)  # (T + r) || (W + r)
        check(lib().b200_logup_hash_dev(fid, mem.ptr, None, g.ptr, rr.ptr, N, tw.ptr, None))
        check(lib().b200_logup_hash_dev(fid, L.ptr, addr.ptr, g.ptr, rr.ptr, N, View(tw, N).ptr, None))
        inv = DeviceVec(64 * N)
        check(lib().b200_batch_invert_dev(fid, tw.ptr, 2 * N, inv.ptr, flag.ptr, None))
        if int.from_bytes(flag.to_bytes(4), "little"):
            raise ValueError("InternalError")
        check(lib().b200_vec_mul_dev(fid, inv.ptr, ts.ptr, N, inv.ptr, None))  # TS[i] / (T[i] + r)
        oracles += [View(inv, 0), View(inv, N)]
        aux += [View(tw, 0), View(tw, N)]
    return oracles, aux


# ---- the three engines ---------------------------------------------------------------------------
def _read1(view) -> bytes:
    out = ctypes.create_string_buffer(32)
    check(lib().b200_memcpy_d2h(out, view.ptr, 32))
    return out.raw


def _first(fid, v) -> int:
    return fields.unpack(fid, _read1(v))[0]


class _Engine:
    """One engine of the batched sum-check (ppsnark.rs:886-983), stated once as data by its subclass:

      CLAIMS  one row per claim: (b200_scb_desc kind SCB_*, sum form, third-sum form for a round whose tau is 0 or -1,
              the names of the three tables it reads (None for an unused one), the index of its eq instance in
              `eqs` or None)
      TABLES  every table, in bind order
      FINALS  the final claims, as groups of table names

    The constructor calls `_setup`.  The round's launches, the evaluation points, the binds and the final claims of the
    host loop, and the claims as data for the device loops, all follow from these three."""
    shard = None  # a Shard while prove_helper runs the rounds on this rank's shards of the tables

    def _setup(self, fid, n, claims, eqs=()):
        self.fid, self.p, self.len = fid, fields.MODULUS[fid], n
        self.claims = [c % self.p for c in claims]
        self.eqs = list(eqs)
        # running claims are needed by the eq claims only (their evaluation points); 0 for the others
        self.running = [c if row[4] is not None else 0 for c, row in zip(self.claims, self.CLAIMS)]
        self._finals = {}  # table name -> final value, when b200_sumcheck_batched returned them

    def _add(self, sums, form, names, g, tabs):
        A, B, C = (None if t is None else getattr(self, t) for t in names)
        return sums.add(form, A, B, C, self.len, *(() if g is None else tabs[g]))

    def enqueue(self, sums: RoundSums):
        tabs = [q._tables() for q in self.eqs]
        self.slots = [self._add(sums, form, names, g, tabs) for _, form, _, names, g in self.CLAIMS]

    def enqueue_m1(self, sums: RoundSums) -> list:
        """the third sums t(-1) of the eq claims whose tau is 0 in this round (sumcheck.rs:1082-1213): a slot or None
        per claim"""
        tabs = [q._tables() for q in self.eqs]
        zero = [q.taus[q.round - 1] % self.p == 0 for q in self.eqs]
        return [self._add(sums, form_m1, names, g, tabs) if g is not None and zero[g] else None
                for _, _, form_m1, names, g in self.CLAIMS]

    def _third_sum(self, form, names, g) -> int:
        A, B, C = (None if t is None else getattr(self, t) for t in names)
        return _sc_eval_one(self.shard, self.fid, form, A, B, C, self.len, *self.eqs[g]._tables())[0]

    def evaluation_points(self, res):
        """[e(0), lead, e(-1)] per claim from the round's sums `res` (indexed by the slots `enqueue` took)"""
        self.saved = []
        for (kind, _, form_m1, names, g), k, claim in zip(self.CLAIMS, self.slots, self.running):
            r = res[k]
            if kind == SCB_LIN2:
                ev = (r[0], 0, r[1])
            elif kind == SCB_RAW3:
                ev = tuple(r)
            else:  # SCB_EQ_DEG2: r = (t0, tinf); SCB_EQ_DEG1: r = (t0,)
                ev = self.eqs[g].evaluation_points(r[0], r[1] if kind == SCB_EQ_DEG2 else 0, claim,
                                                   lambda: self._third_sum(form_m1, names, g))
            self.saved.append(ev)
        return [list(ev) for ev in self.saved]

    def _bind(self, r_dev):
        _bind_all(self.fid, [getattr(self, t) for t in self.TABLES], self.len, r_dev)
        self.len //= 2

    def bound(self, r, r_dev):
        self.running = [0 if row[4] is None else update_claim(self.p, c, ev, r)
                        for c, ev, row in zip(self.running, self.saved, self.CLAIMS)]
        self._bind(r_dev)
        for q in self.eqs:
            q.bound(r)

    def bound_device(self, r_dev):
        """the binds of a round whose algebra ran on the device"""
        self._bind(r_dev)
        for q in self.eqs:
            q.round += 1

    def final_claims(self):
        """element 0 of the fully bound tables: from the values b200_sumcheck_batched returned, else read from the device"""
        got = self._finals
        return [[got[t] if t in got else _first(self.fid, getattr(self, t)) for t in group] for group in self.FINALS]


class MemorySumcheckInstance(_Engine):
    CLAIMS = ((SCB_LIN2, SC_LINEAR, -1, ("t_inv_row", "w_inv_row", None), None),
              (SCB_LIN2, SC_LINEAR, -1, ("t_inv_col", "w_inv_col", None), None),
              (SCB_EQ_DEG2, SC_EQ_CUBIC3, SC_EQ_CUBIC3_M1, ("t_inv_row", "t_row", "ts_row"), 0),
              (SCB_EQ_DEG2, SC_EQ_CUBIC2, SC_EQ_CUBIC2_M1, ("w_inv_row", "w_row", None), 0),
              (SCB_EQ_DEG2, SC_EQ_CUBIC3, SC_EQ_CUBIC3_M1, ("t_inv_col", "t_col", "ts_col"), 0),
              (SCB_EQ_DEG2, SC_EQ_CUBIC2, SC_EQ_CUBIC2_M1, ("w_inv_col", "w_col", None), 0))
    TABLES = ("t_row", "t_inv_row", "w_row", "w_inv_row", "ts_row", "t_col", "t_inv_col", "w_col", "w_inv_col", "ts_col")
    FINALS = (("t_inv_row", "w_inv_row", "ts_row"), ("t_inv_col", "w_inv_col", "ts_col"))

    def __init__(self, fid, N, polys_oracle, polys_aux, rhos, ts_row, ts_col):
        self.t_inv_row, self.w_inv_row, self.t_inv_col, self.w_inv_col = (dev_copy(v, N) for v in polys_oracle)
        self.t_row, self.w_row, self.t_col, self.w_col = polys_aux  # consumed (moved in the reference)
        self.ts_row, self.ts_col = dev_copy(ts_row, N), dev_copy(ts_col, N)
        self._setup(fid, N, [0] * 6, [EqSumCheckInstance(fid, rhos)])


class InnerBatchedSumcheckInstance(_Engine):
    CLAIMS = ((SCB_RAW3, SC_CUBIC, -1, ("L_row", "L_col", "val"), None),
              (SCB_EQ_DEG1, SC_EQ_QUAD1, SC_EQ_QUAD1_M1, ("E", None, None), 0))
    TABLES = ("L_row", "L_col", "val", "E")
    FINALS = (("L_row", "L_col"), ("E",))

    def __init__(self, fid, N, claim, L_row, L_col, val, claim_E, r_outer, E):
        self.L_row, self.L_col, self.val, self.E = dev_copy(L_row, N), dev_copy(L_col, N), val, dev_copy(E, N)
        self._setup(fid, N, [claim, claim_E], [EqSumCheckInstance(fid, r_outer)])


class WitnessBoundSumcheck(_Engine):
    CLAIMS = ((SCB_LIN2, SC_QUADRATIC, -1, ("masked_eq", "W", None), None),)
    TABLES = ("W", "masked_eq")
    FINALS = (("W", "masked_eq"),)

    def __init__(self, fid, N, tau: list, W_padded, num_vars: int):
        m = num_vars.bit_length() - 1
        assert m < N.bit_length() - 1  # ppsnark.rs:288
        self.W = dev_copy(W_padded, N)
        self.masked_eq = DeviceVec(32 * N)
        self._tau_dev = DeviceVec.from_bytes(fields.pack(fid, tau))  # kept: the eq kernels read it asynchronously
        check(lib().b200_eq_table_dev(fid, self._tau_dev.ptr, len(tau), self.masked_eq.ptr, None))
        check(lib().b200_memset_dev(self.masked_eq.ptr, 0, 32 << m, None))  # first 2^m entries -> 0
        self._setup(fid, N, [0])

    @classmethod
    def from_shards(cls, fid, n_local: int, W_local, masked_eq_local):
        """this rank's cyclic shard of W (padded) and of the masked eq table (ppsnark.rs:270-300)"""
        self = cls.__new__(cls)
        self.W, self.masked_eq = dev_copy(W_local, n_local), dev_copy(masked_eq_local, n_local)
        self._setup(fid, n_local, [0])
        return self


def _batching(fid, engines, transcript):
    """ppsnark.rs:909-921: the engines' initial claims combined with the powers of s -> (coefficients, combined claim)"""
    p = fields.MODULUS[fid]
    assert len({eng.len for eng in engines}) == 1
    claims = [c for eng in engines for c in eng.claims]
    s = transcript.squeeze(b"r")
    coeffs = [pow(s, i, p) for i in range(len(claims))]
    return coeffs, sum(c * k for c, k in zip(claims, coeffs)) % p


def prove_helper(fid, mem, inner, witness, transcript, rank: int = 0, world: int = 1, gather=None):
    """RelaxedR1CSSNARK::prove_helper (ppsnark.rs:886-983).

    With `world` > 1 (a power of two) the sixteen tables are sharded CYCLICALLY over `world` ranks: the engines are
    built from this rank's shards (local length N / world; the eq instances from the full point).  Per round every rank
    reduces its shard (nine sums; the eq weight uses the global index), the partial sums are exchanged with ONE
    all-gather (`gather(bytes) -> list of every rank's bytes`), the O(1) algebra and the transcript run replicated, and
    the binds need no exchange (i and i + len/2 are co-resident under the cyclic layout).  When one element per rank is
    left the tables are all-gathered (16 x world elements) and the last log2(world) rounds run replicated.  Every rank
    returns what the unsharded loop returns."""
    p = fields.MODULUS[fid]
    assert world & (world - 1) == 0
    engines = (mem, inner, witness)

    def reduce(vals):
        raw = b"".join(int(v).to_bytes(32, "little") for v in vals)
        parts = gather(raw)
        return [sum(int.from_bytes(q[32 * k:32 * k + 32], "little") for q in parts) % p for k in range(len(vals))]

    def replicate_tail():
        for eng in engines:
            for name in eng.TABLES:
                old = getattr(eng, name)
                setattr(eng, name, DeviceVec.from_bytes(b"".join(gather(_read1(old)))))
            eng.len = world

    n_rounds = (mem.len * world).bit_length() - 1
    coeffs, e = _batching(fid, engines, transcript)
    rs, polys = [], []
    shard = Shard(rank, world, reduce) if world > 1 else None
    sums = RoundSums(fid, shard=shard)
    for eng in engines:
        eng.shard = shard
    try:
        for _ in range(n_rounds):
            if shard is not None and mem.len == 1:
                replicate_tail()
                shard = sums.shard = None
                for eng in engines:
                    eng.shard = None
            for eng in engines:
                eng.enqueue(sums)
            res = sums.fetch()
            evals = [ev for eng in engines for ev in eng.evaluation_points(res)]
            c0 = sum(evals[i][0] * coeffs[i] for i in range(len(evals))) % p
            cb = sum(evals[i][1] * coeffs[i] for i in range(len(evals))) % p
            ci = sum(evals[i][2] * coeffs[i] for i in range(len(evals))) % p
            poly = UniPoly.from_evals_deg3(p, [c0, (e - c0) % p, cb, ci])
            transcript.absorb_bytes(b"p", poly.to_transcript_bytes())
            r = transcript.squeeze(b"c")
            rs.append(r)
            r_dev = _challenge_dev(fid, r)
            for eng in engines:
                eng.bound(r, r_dev)
            e = poly.evaluate(r)
            polys.append(poly.compress())
    finally:
        for eng in engines:
            eng.shard = None
    return polys, rs, mem.final_claims(), inner.final_claims(), witness.final_claims()


# the name the sharded callers know: prove_helper_sharded(fid, mem, inner, witness, transcript, rank, world, gather)
prove_helper_sharded = prove_helper


def _device_claims(fid, engines, transcript):
    """What both device loops start from: the number of rounds, the coefficients and the combined claim
    (`_batching`), every claim as (engine, CLAIMS row, its eq instance numbered across the engines or None), the eq
    instances in that numbering, and the running claims."""
    coeffs, e = _batching(fid, engines, transcript)
    claims, eqs = [], []
    for eng in engines:
        claims += [(eng, row, None if row[4] is None else len(eqs) + row[4]) for row in eng.CLAIMS]
        eqs += eng.eqs
    assert len(claims) <= SCB_MAX_CLAIMS and len(eqs) <= SCB_MAX_EQ
    running = [c for eng in engines for c in eng.running]
    return engines[0].len.bit_length() - 1, coeffs, e, claims, eqs, running


def prove_helper_device(fid, mem, inner, witness, transcript):
    """prove_helper (ppsnark.rs:886-983) as ONE library call (b200_sumcheck_batched): the engines' claims as data
    (b200_scp_program), the library runs every round -- all sums in two launches, the round kernel, one bind launch,
    the short rounds inside one kernel -- and the proof is read back once.
    `transcript` needs the serialisable fields `round`, `state`, `buf` (see spartan._device_loop)."""
    engines = (mem, inner, witness)
    nr, coeffs, e, claims, eqs, running = _device_claims(fid, engines, transcript)
    prog = ScpProgram()
    tables, index = [], {}

    def table(eng, name):
        if (eng, name) not in index:
            index[(eng, name)] = len(tables)
            tables.append(getattr(eng, name))
        return index[(eng, name)]
    for i, (eng, (kind, form, form_m1, names, _), g) in enumerate(claims):
        prog.kind[i], prog.form[i], prog.form_m1[i] = kind, form, form_m1
        prog.eq_of[i] = -1 if g is None else g
        for c, name in enumerate(names):
            prog.tab[i][c] = -1 if name is None else table(eng, name)
    for eng in engines:  # tables no claim reads are still bound every round (none today)
        for name in eng.TABLES:
            table(eng, name)
    assert len(tables) <= SCP_MAX_TABLES
    prog.nclaims, prog.neq, prog.ntables, prog.num_rounds = len(claims), len(eqs), len(tables), nr
    for t, Z in enumerate(tables):
        prog.tables[t] = Z.ptr.value
    tau_bufs = [_cbuf(fields.pack(fid, q.taus)) for q in eqs]
    for g, buf in enumerate(tau_bufs):
        prog.taus[g] = ctypes.addressof(buf)
    inputs = (_cbuf(fields.pack(fid, coeffs)), _cbuf(fields.to_mont_bytes(fid, e)), _cbuf(fields.pack(fid, running)))
    polys, rs, vals = SumcheckProof._device_loop(
        fid, transcript, lambda *io: lib().b200_sumcheck_batched(fid, ctypes.byref(prog), *inputs, *io), nr, 3,
        len(tables))
    for eng in engines:
        eng.len = 1
        eng._finals = {name: vals[t] for (owner, name), t in index.items() if owner is eng}
        for q in eng.eqs:
            q.round += nr
    return polys, rs, mem.final_claims(), inner.final_claims(), witness.final_claims()


def prove_helper_device_rounds(fid, mem, inner, witness, transcript):
    """prove_helper (ppsnark.rs:886-983) with the per-round algebra and the transcript on the device, one call per
    launch (the building blocks b200_sc_eval_dev / b200_sc_round_batched_dev / b200_bind_top_multi_dev):
    per round the nine reductions, one b200_sc_round_batched_dev and the sixteen binds are enqueued
    without reading anything back; proof, challenges and transcript state are read once at the end.
    `transcript` needs the serialisable fields `round`, `state`, `buf` (see spartan._device_loop)."""
    p = fields.MODULUS[fid]
    engines = (mem, inner, witness)
    nr, coeffs, e, claims, eqs, running = _device_claims(fid, engines, transcript)
    pad = lambda xs, n: list(xs) + [0] * (n - len(xs))
    head = (fields.to_mont_bytes(fid, e) + bytes(32) + int(transcript.round).to_bytes(8, "little")
            + bytes(transcript.state) + bytes(8))
    state = DeviceVec.from_bytes(head + fields.pack(fid, pad(coeffs, SCB_MAX_CLAIMS)) + fields.pack(fid, pad(running, SCB_MAX_CLAIMS))
                                 + fields.pack(fid, pad([1] * len(eqs), SCB_MAX_EQ)))
    assert state.nbytes == 1296
    tau_dev = [DeviceVec.from_bytes(fields.pack(fid, q.taus)) for q in eqs]
    tinv_dev = [DeviceVec.from_bytes(fields.pack(fid, [pow(t, -1, p) if t % p else 0 for t in q.taus])) for q in eqs]
    polys_dev, rs_dev = DeviceVec(96 * nr), DeviceVec(32 * nr)
    pending = bytes(transcript.buf)
    pend_dev = DeviceVec.from_bytes(pending) if pending else None
    sums = RoundSums(fid)
    L = lib()
    for j in range(nr):
        for eng in engines:
            eng.enqueue(sums)
        slots = [sl for eng in engines for sl in eng.slots]
        m1 = [sl for eng in engines for sl in eng.enqueue_m1(sums)]  # third sums for the eq instances whose tau is 0
        d = ScbDesc()
        d.nclaims, d.neq = len(claims), len(eqs)
        for i, (_, row, g) in enumerate(claims):
            d.kind[i], d.slot[i] = row[0], 3 * slots[i]
            d.slot_m1[i] = -1 if m1[i] is None else 3 * m1[i]
            d.eq_of[i] = -1 if g is None else g
        for g, q in enumerate(eqs):
            d.tau[g] = tau_dev[g].ptr.value + 32 * (q.round - 1)
            d.tau_inv[g] = tinv_dev[g].ptr.value + 32 * (q.round - 1)
        check(L.b200_sc_round_batched_dev(fid, ctypes.byref(d), sums.out.ptr, state.ptr, pend_dev.ptr if (pend_dev and j == 0) else None,
                                          len(pending) if j == 0 else 0, ord("p"), ord("c"), View(polys_dev, 3 * j).ptr,
                                          View(rs_dev, j).ptr, None))
        sums.reset()
        r_dev = View(rs_dev, j)
        for eng in engines:
            eng.bound_device(r_dev)
    raw_polys, raw_rs, raw_state = polys_dev.to_bytes(96 * nr), rs_dev.to_bytes(32 * nr), state.to_bytes(144)
    transcript.round = int.from_bytes(raw_state[64:72], "little")
    transcript.state = raw_state[72:136]
    transcript.buf = b""
    coeffs_out = [int.from_bytes(raw_polys[32 * i:32 * i + 32], "little") for i in range(3 * nr)]
    polys = [coeffs_out[3 * j:3 * j + 3] for j in range(nr)]
    return polys, fields.unpack(fid, raw_rs), mem.final_claims(), inner.final_claims(), witness.final_claims()


def _mle_eval(fid, Z, ell, r_dev) -> int:
    out = DeviceVec(32)
    check(lib().b200_mle_eval_dev(fid, Z.ptr, ell, r_dev.ptr, out.ptr, None))
    return fields.unpack(fid, out.to_bytes(32))[0]


def prove_core(curve, ck: CommitmentKey, S: dict, spark: SparkRepr, U: dict, W: dict, vk_digest: int, transcript,
               timings: dict | None = None, device_transcript: bool = False):
    """ppsnark.rs:1056-1355 up to (and excluding) EE::prove.

    S: dict(num_cons, num_vars, A, B, C) with A/B/C `spartan.SparseMatrix` (regular, padded shape).
    U: dict(comm_W, comm_E (affine or None), u, X: ints);  W: dict(W, E: Montgomery bytes or
    DeviceVec).  `timings`, if given, receives wall-clock seconds per phase (device synchronised
    at the phase boundaries).
    Returns every proof field plus the batched opening polynomial (DeviceVec) and its value.
    """
    import time
    t_last = [time.perf_counter()]

    def mark(name):
        if timings is not None:
            check(lib().b200_sync())
            now = time.perf_counter()
            timings[name] = timings.get(name, 0.0) + now - t_last[0]
            t_last[0] = now
    fid = curve.scalar_field
    p = fields.MODULUS[fid]
    num_cons, num_vars, N = S["num_cons"], S["num_vars"], spark.N
    tr = transcript
    tr.absorb_bytes(b"vk", to_repr(vk_digest % p))
    tr.absorb_bytes(b"U", commitment_transcript_bytes(U["comm_W"]) + commitment_transcript_bytes(U["comm_E"])
                    + to_repr(U["u"] % p) + b"".join(to_repr(x % p) for x in U["X"]))
    u_dev = dev_scalar(fid, U["u"])
    z_len = num_vars + 1 + len(U["X"])
    Wd, Ed = _as_dev(W["W"]), _as_dev(W["E"])
    z = DeviceVec(32 * z_len)
    check(lib().b200_memcpy_d2d(z.ptr, Wd.ptr, 32 * num_vars, None))
    check(lib().b200_memcpy_h2d(View(z, num_vars).ptr, _cbuf(fields.pack(fid, [U["u"]] + list(U["X"]))),
                                32 * (1 + len(U["X"]))))
    Az, Bz, Cz = (DeviceVec(32 * num_cons) for _ in range(3))
    for M, out in ((S["A"], Az), (S["B"], Bz), (S["C"], Cz)):
        check(lib().b200_spmv_dev(M.handle, z.ptr, None, out.ptr, None, None))
    nro, nri = num_cons.bit_length() - 1, N.bit_length() - 1
    tau = [tr.squeeze(b"t") for _ in range(nro)]
    uCz_E = DeviceVec(32 * num_cons)
    check(lib().b200_axpy_dev(fid, Ed.ptr, Cz.ptr, u_dev.ptr, num_cons, uCz_E.ptr, None))  # E + u*Cz
    mark("spmv")
    outer = (SumcheckProof.prove_cubic_with_three_inputs_device if device_transcript  # one call (b200_sumcheck_cubic3)
             else SumcheckProof.prove_cubic_with_three_inputs)
    sc_outer, r_outer, claims_outer = outer(fid, 0, tau, Az, Bz, uCz_E, tr)
    eAz, eBz = claims_outer[0], claims_outer[1]
    eCz = _mle_eval(fid, Cz, nro, DeviceVec.from_bytes(fields.pack(fid, r_outer)))
    eE_outer = (claims_outer[2] - U["u"] * eCz) % p
    tr.absorb_bytes(b"e", b"".join(to_repr(x) for x in (eAz, eBz, eCz, eE_outer)))
    mark("outer_sumcheck")
    r_pad = [tr.squeeze(b"p") for _ in range(nri - nro)]
    r_full = r_pad + r_outer
    factor = 1
    for x in r_pad:
        factor = factor * (1 - x) % p
    E_p, W_p = dev_padded(Ed, num_cons, N), dev_padded(Wd, num_vars, N)
    mem_row, mem_col, L_row, L_col = spark.evaluation_oracles(r_full, z, z_len)
    mark("evaluation_oracles")
    comm_L_row, comm_L_col = commit_many_dev(curve, ck, [L_row, L_col], [N, N])
    mark("commit_L")
    tr.absorb_bytes(b"e", commitment_transcript_bytes(comm_L_row) + commitment_transcript_bytes(comm_L_col))
    c = tr.squeeze(b"c")
    gamma = tr.squeeze(b"g")
    r = tr.squeeze(b"r")
    val = DeviceVec(32 * N)  # val_A + c val_B + c^2 val_C (ppsnark.rs:1183-1188)
    _rlc_dev(fid, [spark.val_A, spark.val_B, spark.val_C], [1, c, c * c % p], N, val)
    inner = InnerBatchedSumcheckInstance(fid, N, factor * (eAz + c * eBz + c * c * eCz), L_row, L_col, val,
                                         factor * eE_outer, r_full, E_p)
    mem_oracles, mem_aux = memory_compute_oracles(fid, r, gamma, N, mem_row, spark.row, L_row, spark.ts_row,
                                                  mem_col, spark.col, L_col, spark.ts_col)
    mark("memory_oracles")
    comm_mem = commit_many_dev(curve, ck, mem_oracles, [N] * 4)
    mark("commit_mem")
    tr.absorb_bytes(b"l", b"".join(commitment_transcript_bytes(P) for P in comm_mem))
    rho = [tr.squeeze(b"r") for _ in range(nri)]
    mem = MemorySumcheckInstance(fid, N, mem_oracles, mem_aux, rho, spark.ts_row, spark.ts_col)
    wit = WitnessBoundSumcheck(fid, N, r_full, W_p, num_vars)
    mark("engines_setup")
    sc_inner, r_inner, c_mem, c_inner, c_wit = (prove_helper_device if device_transcript else prove_helper)(
        fid, mem, inner, wit, tr)
    mark("inner_sumcheck")
    ev = {
        "eval_L_row": c_inner[0][0], "eval_L_col": c_inner[0][1], "eval_E": c_inner[1][0],
        "eval_t_plus_r_inv_row": c_mem[0][0], "eval_w_plus_r_inv_row": c_mem[0][1], "eval_ts_row": c_mem[0][2],
        "eval_t_plus_r_inv_col": c_mem[1][0], "eval_w_plus_r_inv_col": c_mem[1][1], "eval_ts_col": c_mem[1][2],
        "eval_W": c_wit[0][0],
    }
    ri_dev = DeviceVec.from_bytes(fields.pack(fid, r_inner))
    names = ("eval_val_A", "eval_val_B", "eval_val_C", "eval_row", "eval_col")
    from .spartan import mle_eval_multi_dev  # multi_evaluate_with, multilinear.rs:129-180: one pair of eq tables, one read-back
    ev.update(zip(names, mle_eval_multi_dev(fid, [spark.val_A, spark.val_B, spark.val_C, spark.row, spark.col], nri, ri_dev)))
    order = ["eval_W", "eval_E", "eval_L_row", "eval_L_col", "eval_val_A", "eval_val_B", "eval_val_C",
             "eval_t_plus_r_inv_row", "eval_row", "eval_w_plus_r_inv_row", "eval_ts_row",
             "eval_t_plus_r_inv_col", "eval_col", "eval_w_plus_r_inv_col", "eval_ts_col"]
    eval_vec = [ev[k] for k in order]
    poly_vec = [W_p, E_p, L_row, L_col, spark.val_A, spark.val_B, spark.val_C, mem_oracles[0], spark.row,
                mem_oracles[1], spark.ts_row, mem_oracles[2], spark.col, mem_oracles[3], spark.ts_col]
    tr.absorb_bytes(b"e", b"".join(to_repr(x) for x in eval_vec))
    cb = tr.squeeze(b"c")
    pw = [pow(cb, i, p) for i in range(len(poly_vec))]
    batched = DeviceVec(32 * N)  # PolyEvalWitness::batch (spartan/mod.rs:232-277)
    _rlc_dev(fid, poly_vec, pw, N, batched)
    mark("final_evals_rlc")
    out = dict(ev)
    out.update(comm_L_row=comm_L_row, comm_L_col=comm_L_col, comm_mem=comm_mem, sc_outer=sc_outer,
               r_outer=r_outer, eval_Az_at_r_outer=eAz, eval_Bz_at_r_outer=eBz, eval_Cz_at_r_outer=eCz,
               eval_E_at_r_outer=eE_outer, sc_inner_batched=sc_inner, r_inner_batched=r_inner,
               batched_poly=batched, batched_eval=sum(a * b for a, b in zip(pw, eval_vec)) % p, batch_challenge=cb)
    return out


SHAPE_COMMITMENTS = ("val_A", "val_B", "val_C", "row", "col", "ts_row", "ts_col")  # R1CSShapeSparkCommitment


def setup(curve, ck: CommitmentKey, S: dict):
    """The shape half of ppsnark's setup: R1CSShapeSparkRepr::new + ::commit (ppsnark.rs:117-217), both on the
    device -> (spark, S_comm).  `S` is the dict `prove` takes, already regular (padding stays the caller's);
    S_comm maps SHAPE_COMMITMENTS to the commitments (r = 0) of the seven N-element vectors, so `ck` needs N bases."""
    from .provider import Curve
    curve = Curve(curve)
    spark = SparkRepr.from_shape(curve.scalar_field, S)
    comms = commit_many_dev(curve, ck, [getattr(spark, k) for k in SHAPE_COMMITMENTS], [spark.N] * 7)
    return spark, dict(zip(SHAPE_COMMITMENTS, comms))


def _batched_commitment(curve, U: dict, S_comm: dict, out: dict):
    """PolyEvalInstance::batch, the commitment part (spartan/mod.rs:346-368): sum_i c^i C_i over the 15 commitments
    in ppsnark.rs's comm_vec order, c = the batch challenge."""
    from .provider import DlogGroup
    from .snark import _affine_bytes
    fid = curve.scalar_field
    p = fields.MODULUS[fid]
    cm = out["comm_mem"]
    comm_vec = [U["comm_W"], U["comm_E"], out["comm_L_row"], out["comm_L_col"], S_comm["val_A"], S_comm["val_B"],
                S_comm["val_C"], cm[0], S_comm["row"], cm[1], S_comm["ts_row"], cm[2], S_comm["col"], cm[3],
                S_comm["ts_col"]]
    c = out["batch_challenge"]
    return DlogGroup(curve).vartime_multiscalar_mul(fields.pack(fid, [pow(c, i, p) for i in range(len(comm_vec))]),
                                                    b"".join(_affine_bytes(curve, P) for P in comm_vec))


def prove(curve, ck: CommitmentKey, S: dict, spark: SparkRepr, U: dict, W: dict, vk_digest: int, transcript,
          timings: dict | None = None, device_transcript: bool = False, ee: str = "hyperkzg",
          S_comm: dict | None = None):
    """The whole RelaxedR1CSSNARK::prove of ppsnark.rs:1056-1385: prove_core, then EE::prove with the transcript
    on the batched polynomial at r_inner_batched.  -> proof fields + `eval_arg`.
      ee = "hyperkzg": hyperkzg.rs:926-1116.  (The batched commitment sum_i c^i C_i of PolyEvalInstance::batch
                       is only an input of EE::prove for the HyperKZG prover, which does not use it: the caller /
                       verifier forms it from the 15 commitments.)
      ee = "mercury":  mercury.rs:891-1268, which absorbs the batched commitment: `S_comm` must hold the seven
                       shape commitments (R1CSShapeSparkCommitment: val_A, val_B, val_C, row, col, ts_row, ts_col,
                       as `setup` returns them).
      ee = "ipa":      ipa_pc.rs:64-77, 174-285 -> eval_arg = (L_vec, R_vec, a_hat); absorbs the batched commitment
                       too, so it needs `S_comm`.  `ck` must carry the generator ck_c as its blinding base and at
                       least N bases.
    With `timings`, ee = "ipa" adds the phases "ipa_batch_commitment", "ipa_b_vec", "ipa_inner_products",
    "ipa_commit" and "ipa_fold" (ipa.InnerProductArgument.prove)."""
    if ee not in ("hyperkzg", "mercury", "ipa"):
        raise ValueError(f"unknown evaluation engine {ee!r}")
    if ee != "hyperkzg" and S_comm is None:
        raise ValueError(f"the {ee} evaluation argument needs the shape commitments S_comm")
    if ee == "ipa" and (not ck.has_h or len(ck) < spark.N):
        raise ValueError(f"the IPA needs a key with the generator ck_c and at least N = {spark.N} bases")
    out = prove_core(curve, ck, S, spark, U, W, vk_digest, transcript, timings, device_transcript)
    if ee == "hyperkzg":
        from .spartan import hyperkzg_prove
        out["eval_arg"] = hyperkzg_prove(curve, ck, out["batched_poly"], out["r_inner_batched"], transcript, timings)
        return out
    import time
    from .provider import Curve
    curve = Curve(curve)
    t0 = time.perf_counter()
    C = _batched_commitment(curve, U, S_comm, out)
    if ee == "mercury":
        from .mercury import mercury_prove
        out["eval_arg"] = mercury_prove(curve, ck, out["batched_poly"], out["r_inner_batched"], transcript, timings,
                                        comm=C, eval_=out["batched_eval"])
        return out
    if timings is not None:
        timings["ipa_batch_commitment"] = timings.get("ipa_batch_commitment", 0.0) + time.perf_counter() - t0
    from .ipa import prove_at_point
    out["eval_arg"] = prove_at_point(curve, ck, C, out["r_inner_batched"], out["batched_eval"], out["batched_poly"],
                                     transcript, timings)
    return out


def _rlc_dev(fid, polys, coeffs, n, out, lens=None):
    """out[0..n) = sum_i coeffs[i] polys[i], polynomial i read over its first lens[i] entries (default n) and
    zero-extended"""
    k = len(polys)
    ptrs = (ctypes.c_void_p * k)(*[v.ptr.value for v in polys])
    lens = (ctypes.c_size_t * k)(*([n] * k if lens is None else lens))
    cd = DeviceVec.from_bytes(fields.pack(fid, coeffs))
    check(lib().b200_rlc_dev(fid, ptrs, lens, k, cd.ptr, n, out.ptr, None))
    check(lib().b200_sync())  # `cd` and the pointer table must outlive the launch
