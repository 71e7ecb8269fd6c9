"""Shared bodies of the NeutronNova checks (GPU: tests/test_neutron_gpu.py; CPU with the emulated device:
tests/test_neutron_mirror_cpu.py), and the fixtures of tests/test_oracle_neutron.py.

Fixtures (oracle.neutron_ref.Shape, padded, with a generator of satisfying (W, X)):
  "cubic"     the tiny cubic R1CS x^3 + x + 5 = y of r1cs/mod.rs:1349-1413, padded from 3 to 4 variables
  "squaring"  32 constraints of repeated squaring (the NonTrivialCircuit pattern): x * x = w0, w_{i-1}^2 = w_i
  "boolean"   x * x = x on every variable (nifs.rs:534-585, generate_sample_r1cs), random bits, X = [0]

`run_sequence` restates execute_sequence (nifs.rs:366-435): default running pair -> fold instance 1 -> fold
instance 2; after each fold the oracle's verify reproduces the prover's U and is_sat holds.  With a device library
the mirror (nova_b200.neutron) runs the same sequence and is compared with the oracle field for field."""
from oracle import neutron_ref as nr
from oracle.poseidon_ref import PoseidonRO as OraclePoseidonRO
from oracle.pyref import CURVES, FIELD_MODULUS, SplitMix64, from_mont_bytes, mont_bytes
from test_oracle_nifs_fold import NUM_CONS, NUM_IO, NUM_VARS, csr, tiny_r1cs
from test_oracle_nifs_fold import witness as cubic_witness


def pack(p, xs):
    return b"".join(mont_bytes(p, x) for x in xs)


def ints(p, b):
    return [from_mont_bytes(p, b[i:i + 32]) for i in range(0, len(b), 32)]


def _identity(n, ones_col):
    return [1] * n, [ones_col(i) for i in range(n)], list(range(n + 1))


def fixture(kind, fid, log2n=None):
    """-> (padded Shape, fresh(rng) -> satisfying (W, X))"""
    p = FIELD_MODULUS[fid]
    if kind == "cubic":
        S = nr.Shape(fid, NUM_CONS, NUM_VARS, NUM_IO, *(csr(M, NUM_CONS) for M in tiny_r1cs()))
        Sp = nr.pad(S)

        def fresh(rng):
            W, X = cubic_witness(p, rng.field(p))
            return nr.pad_witness(Sp, W), X
        return Sp, fresh
    if kind == "squaring":
        n = 32
        x_col = n + 1  # z = (w_0 .. w_31, u, x)
        A = [1] * n, [x_col] + list(range(n - 1)), list(range(n + 1))
        C = _identity(n, lambda i: i)
        S = nr.Shape(fid, n, n, 1, A, A, C)

        def fresh(rng):
            x = rng.field(p)
            W, w = [], x
            for _ in range(n):
                w = w * w % p
                W.append(w)
            return W, [x]
        return nr.pad(S), fresh
    if kind == "boolean":
        n = 1 << log2n
        M = _identity(n, lambda i: i)
        S = nr.Shape(fid, n, n, 1, M, M, M)

        def fresh(rng):
            return [rng.next() & 1 for _ in range(n)], [0]
        return nr.pad(S), fresh
    raise ValueError(kind)


def device_shape(nb, cid, S):
    from nova_b200 import r1cs, spartan as sp
    p = FIELD_MODULUS[S.fid]
    ncols = S.num_vars + 1 + S.num_io
    mats = [sp.SparseMatrix(S.fid, pack(p, d), idx, ptr, ncols) for (d, idx, ptr) in (S.A, S.B, S.C)]
    return r1cs.R1CSShape(nb.Curve(cid), *mats, S.num_cons, S.num_vars, S.num_io)


def keys(nb, oracle, cid, n_key):
    bases = oracle.gen_bases(cid, n_key + 1)
    ck = nb.CommitmentKey(nb.Curve(cid), bases[:64 * n_key], bases[64 * n_key:]) if nb is not None else None
    return ck, (cid, bases[:64 * n_key], bases[64 * n_key:])


def oracle_ro(fid):
    return OraclePoseidonRO(FIELD_MODULUS[fid])


def _same(nb, st_dev, U, W, Uo, Wo, fid):
    """the mirror's folded pair equals the oracle's, field for field and byte for byte"""
    p = FIELD_MODULUS[fid]
    assert (U.comm_W, U.comm_E, U.T, U.u, U.X) == (Uo.comm_W, Uo.comm_E, Uo.T, Uo.u, Uo.X)
    assert W.W.to_bytes(32 * st_dev.S.num_vars) == pack(p, Wo.W)
    assert W.E.to_bytes(32 * (st_dev.left + st_dev.right)) == pack(p, Wo.E)
    assert (W.r_W, W.r_E) == (Wo.r_W, Wo.r_E)


def run_sequence(nb, oracle, cid, kind, log2n=None, mirror_ro=None, pp_digest=0, seed=1):
    """execute_sequence on the oracle, and on the mirror when `nb` is given (mirror_ro(fid) -> its RO2)"""
    c = CURVES[cid]
    fid, p = c.scalar_field, c.q
    S, fresh = fixture(kind, fid, log2n)
    st = nr.Structure.new(S)
    rng = SplitMix64(1000 * seed + 10 * cid + len(kind))
    n_key = max(S.num_vars, st.left + st.right)
    ck, ck_o = keys(nb, oracle, cid, n_key)
    if nb is not None:
        from nova_b200 import neutron as ne, r1cs, spartan as sp
        st_dev = ne.Structure(device_shape(nb, cid, S))
        assert (st_dev.ell, st_dev.left, st_dev.right) == (st.ell, st.left, st.right)
        U, W = ne.FoldedInstance.default(st_dev), ne.FoldedWitness.default(st_dev)
        assert ne.is_sat(ck, st_dev, U, W)
    Uo, Wo = nr.FoldedInstance.default(st), nr.FoldedWitness.default(st)
    assert nr.is_sat(ck_o, st, Uo, Wo)
    for _ in range(2):
        Wv, X = fresh(rng)
        r_W, r_E = rng.field(p), rng.field(p)
        U2o = nr.R1CSInstance(nr.commit(ck_o, fid, Wv, r_W), X)
        W2o = nr.R1CSWitness(Wv, r_W)
        nifs_o, (Uo_new, Wo_new) = nr.nifs_prove(ck_o, oracle_ro(fid), pp_digest, st, Uo, Wo, U2o, W2o, r_E)
        assert nr.nifs_verify(cid, p, nifs_o, oracle_ro(fid), pp_digest, Uo, U2o) == Uo_new
        assert nr.is_sat(ck_o, st, Uo_new, Wo_new)
        if nb is not None:
            U2 = r1cs.R1CSInstance(U2o.comm_W, list(X))
            W2 = r1cs.R1CSWitness(sp.DeviceVec.from_bytes(pack(p, Wv)), r_W)
            nifs, (U_new, W_new) = ne.nifs_prove(ck, mirror_ro(fid), pp_digest, st_dev, U, W, U2, W2, r_E)
            assert (nifs.comm_E, list(nifs.poly)) == (nifs_o.comm_E, nifs_o.poly)
            _same(nb, st_dev, U_new, W_new, Uo_new, Wo_new, fid)
            assert ne.verify(nb.Curve(cid), mirror_ro(fid), pp_digest, nifs, U, U2) == U_new
            assert ne.is_sat(ck, st_dev, U_new, W_new)
            U, W = U_new, W_new
        Uo, Wo = Uo_new, Wo_new
    if nb is not None:
        ck.release()
    return st, ck_o, (Uo, Wo)


# ---- single entry points -----------------------------------------------------------------------------------
def _vectors(fid, left, right, kind, seed):
    """e1, e2 (lists of left + right entries) and the six n-vectors (Montgomery bytes) for the evals checks"""
    from oracle import coracle as co
    p = FIELD_MODULUS[fid]
    n = left * right
    rng = SplitMix64(seed)
    rand_e = lambda: [rng.field(p) for _ in range(left + right)]
    if kind == "random":
        es, vec = (rand_e(), rand_e()), lambda k: co.gen_scalars(fid, seed + k, n)
    elif kind == "zero":
        es, vec = ([0] * (left + right),) * 2, lambda k: bytes(32 * n)
    elif kind == "last_row":  # the n-vectors are non-zero only in their last row
        es, vec = (rand_e(), rand_e()), lambda k: bytes(32 * (n - 1)) + mont_bytes(p, rng.field(p))
    elif kind == "p_minus_1":
        es, vec = ([p - 1] * (left + right),) * 2, lambda k: mont_bytes(p, p - 1) * n
    else:
        raise ValueError(kind)
    return es[0], [vec(k) for k in range(3)], es[1], [vec(k) for k in range(3, 6)]


def check_evals(L, oracle, fid, left, right, kind, seed=7):
    """b200_neutron_evals against the oracle: the C composition, and for n <= 2^12 also the literal loop"""
    import ctypes
    from nova_b200.provider import _cbuf
    p = FIELD_MODULUS[fid]
    e1, abc1, e2, abc2 = _vectors(fid, left, right, kind, seed + left + right)
    out = ctypes.create_string_buffer(32 * 5)
    rc = L.b200_neutron_evals(fid, _cbuf(pack(p, e1)), *map(_cbuf, abc1), _cbuf(pack(p, e2)), *map(_cbuf, abc2),
                              left, right, out)
    assert rc == 0, L.b200_last_error()
    exp = nr.evals_raw(fid, left, right, e1, *abc1, e2, *abc2)
    if left * right <= 1 << 12:
        assert exp == nr.prove_helper_raw(p, left, right, e1, *(ints(p, v) for v in abc1), e2,
                                          *(ints(p, v) for v in abc2))
    assert ints(p, out.raw) == exp, (fid, left, right, kind)


def check_pow_split(L, fid, left, right, seed=3):
    import ctypes
    from nova_b200.provider import _cbuf
    p = FIELD_MODULUS[fid]
    tau = SplitMix64(seed + left).field(p)
    out = ctypes.create_string_buffer(32 * (left + right))
    assert L.b200_pow_split_evals(fid, _cbuf(mont_bytes(p, tau)), left, right, out) == 0, L.b200_last_error()
    assert ints(p, out.raw) == nr.split_evals(p, tau, left, right)


def check_lerp(L, fid, n, aliased, seed=5):
    """b200_lerp_dev out of place, and with out == a"""
    from nova_b200 import spartan as sp
    from nova_b200.native import check
    p = FIELD_MODULUS[fid]
    a, b = (oracle_gen(fid, seed + k, n) for k in (0, 1))
    r = SplitMix64(seed).field(p)
    da, db, dr = sp.DeviceVec.from_bytes(a), sp.DeviceVec.from_bytes(b), sp.DeviceVec.from_bytes(mont_bytes(p, r))
    out = da if aliased else sp.DeviceVec(32 * n)
    check(L.b200_lerp_dev(fid, da.ptr, db.ptr, dr.ptr, n, out.ptr, None))
    got = out.to_bytes(32 * n)
    # a + r (b - a) = (1 - r) a + r b: two C-oracle axpy passes
    from oracle import coracle as co
    exp = co.axpy(fid, co.axpy(fid, bytes(32 * n), a, mont_bytes(p, (1 - r) % p)), b, mont_bytes(p, r))
    assert got == exp, (fid, n, aliased)


def oracle_gen(fid, seed, n):
    from oracle import coracle as co
    return co.gen_scalars(fid, seed, n)
