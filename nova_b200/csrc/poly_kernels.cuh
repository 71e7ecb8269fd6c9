// Sum-check, multilinear-extension, HyperKZG and sparse-matrix kernels (K5-K8 of SURVEY.md §2).
// All are HBM-bound streaming passes over 32-byte field elements; reductions produce 1-3 field
// elements through a two-stage (per-block partial, single-block final) tree.
//
// Reference functions restated here (the host keeps the O(1) algebra, transcript and control):
//   compute_eval_points_{quad_prod,linear,quadratic,cubic}   src/spartan/sumcheck.rs:165-186,352-443
//   EqSumCheckInstance::evaluation_points_* (t(0), t(inf), t(-1) sums)
//                                                            src/spartan/sumcheck.rs:900-1213
//   EqPolynomial::evals_from_points                          src/spartan/polys/eq.rs:54-73
//   MultilinearPolynomial::evaluate_with                     src/spartan/polys/multilinear.rs:98-127
//   batch_invert                                             src/spartan/mod.rs:54-145
//   PolyEvalWitness::batch (RLC of polynomials)              src/spartan/mod.rs:232-277
//   HyperKZG fold / Horner evaluation / divide by (X-u)      src/provider/hyperkzg.rs:1083-1095,
//                                                            1011-1019, 961-999
//   PrecomputedSparseMatrix::multiply_vec(_pair)             src/r1cs/sparse.rs:136-230
//   Mercury compute_h_poly / divide_by_binomial / make_s_polynomial
//                                                            src/provider/mercury.rs:369-386, 319-356, 391-475
#pragma once
#if !defined(NOVA_SIMT_HOST)  // tests/hostcheck/simt_host.h supplies the few CUDA names the kernels use
#include <cuda_runtime.h>
#endif
#include "field.cuh"

namespace nova {

// ------------------------------------------------------------------------------------------
// reduction framework
// ------------------------------------------------------------------------------------------
NOVA_D fe_t fe_shfl_down(const fe_t& a, int delta) {
  fe_t r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.l[i] = __shfl_down_sync(0xffffffffu, a.l[i], delta);
  return r;
}

// block-wide sum of NOUT accumulators; result valid in thread 0
template <class F, int NOUT>
NOVA_D void block_sum(fe_t (&acc)[NOUT], fe_t* sm /* [8][NOUT] */) {
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NOUT; k++) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc[k] = fe_add<F>(acc[k], fe_shfl_down(acc[k], d));
    if (lane == 0) sm[wid * NOUT + k] = acc[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int nw = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int k = 0; k < NOUT; k++) {
      fe_t s = sm[k];
      for (int w = 1; w < nw; w++) s = fe_add<F>(s, sm[w * NOUT + k]);
      acc[k] = s;
    }
  }
}

template <class F, int NOUT, class Form>
__global__ void __launch_bounds__(256) k_form_reduce(Form form, size_t count, void* partials) {
  __shared__ fe_t sm[8 * NOUT];
  fe_t acc[NOUT];
#pragma unroll
  for (int k = 0; k < NOUT; k++) acc[k] = fe_zero<F>();
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < count;
       id += (size_t)gridDim.x * blockDim.x)
    form(id, acc);
  block_sum<F, NOUT>(acc, sm);
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < NOUT; k++) fe_store(partials, (size_t)blockIdx.x * NOUT + k, acc[k]);
}

template <class F, int NOUT>
__global__ void __launch_bounds__(256) k_form_final(const void* partials, int nblocks, void* out) {
  __shared__ fe_t sm[8 * NOUT];
  fe_t acc[NOUT];
#pragma unroll
  for (int k = 0; k < NOUT; k++) acc[k] = fe_zero<F>();
  for (int b = threadIdx.x; b < nblocks; b += blockDim.x)
#pragma unroll
    for (int k = 0; k < NOUT; k++) acc[k] = fe_add<F>(acc[k], fe_load_rw(partials, (size_t)b * NOUT + k));
  block_sum<F, NOUT>(acc, sm);
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < NOUT; k++) fe_store(out, k, acc[k]);
}

// ------------------------------------------------------------------------------------------
// sum-check round forms.  `h` = half length; lo = P[id], hi = P[id + h].
// eq factor: f = eq_left[id >> shift] * eq_right[id & mask]  (first half of the rounds), or
//            f = eq_right[id] when eq_left == nullptr          (sumcheck.rs:1233-1251)
// ------------------------------------------------------------------------------------------
// When a polynomial is sharded cyclically over `id_mul` ranks (rank r holds entries r, r+N, ...)
// the local index j stands for the global index j*id_mul + id_add; binding the top variable then
// needs no data movement (pairs (i, i+h) are co-resident) and only the eq weight must use the
// global index.  Unsharded calls pass id_mul = 1, id_add = 0.
struct eq_factor {
  const void* left;
  const void* right;
  int shift;
  size_t mask;
  size_t id_mul, id_add;
  template <class F>
  NOVA_D fe_t get(size_t local_id) const {
    size_t id = local_id * id_mul + id_add;
    if (left == nullptr) return fe_load(right, id);
    return fe_mul<F>(fe_load(left, id >> shift), fe_load(right, id & mask));
  }
};

enum sc_form_id {
  SC_QUAD_PROD = 0,   // (sum A_lo B_lo, sum dA dB)                         sumcheck.rs:165-186
  SC_LINEAR = 1,      // (sum A_lo-B_lo, sum A(-1)-B(-1))                   sumcheck.rs:352-377
  SC_QUADRATIC = 2,   // (sum A_lo B_lo, sum A(-1) B(-1))                   sumcheck.rs:379-405
  SC_CUBIC = 3,       // (sum ABC lo, sum dA dB dC, sum A(-1)B(-1)C(-1))    sumcheck.rs:407-443
  SC_EQ_CUBIC3 = 4,   // t0 = sum f (A_lo B_lo - C_lo), tinf = sum f dA dB  sumcheck.rs:900-966
  SC_EQ_CUBIC2 = 5,   // t0 = sum f (A_lo B_lo - 1),    tinf = sum f dA dB  sumcheck.rs:972-1033
  SC_EQ_QUAD1 = 6,    // t0 = sum f A_lo                                    sumcheck.rs:1039-1080
  SC_EQ_CUBIC3_M1 = 7,  // t(-1) = sum f (A(-1)B(-1) - C(-1))   fallback     sumcheck.rs:1082-1130
  SC_EQ_CUBIC2_M1 = 8,  // t(-1) = sum f (A(-1)B(-1) - 1)       fallback     sumcheck.rs:1132-1178
  SC_EQ_QUAD1_M1 = 9,   // t(-1) = sum f A(-1)                  fallback     sumcheck.rs:1180-1213
  SC_DOT_EQ = 10,     // sum f Z[id]  (MLE evaluation, multilinear.rs:98-127; h unused)
  SC_DOT = 11,        // sum A[id] B[id]  (inner_product, provider/ipa_pc.rs:102-108)
};

// RW: the tables are read through the coherent path (fe_load_rw) -- for a kernel that also binds them (k_scb_tail)
template <class F, int FORM, bool RW = false>
struct sc_form {
  static NOVA_D fe_t ld(const void* base, size_t idx) {
    if constexpr (RW) return fe_load_rw(base, idx);
    else return fe_load(base, idx);
  }
  const void *A, *B, *C;
  size_t h;
  eq_factor eq;
  template <int N>
  NOVA_D void operator()(size_t id, fe_t (&acc)[N]) const {
    if constexpr (FORM == SC_DOT) {
      acc[0] = fe_add<F>(acc[0], fe_mul<F>(ld(A, id), ld(B, id)));
    } else if constexpr (FORM == SC_QUAD_PROD) {
      fe_t al = ld(A, id), ah = ld(A, id + h), bl = ld(B, id), bh = ld(B, id + h);
      acc[0] = fe_add<F>(acc[0], fe_mul<F>(al, bl));
      acc[1] = fe_add<F>(acc[1], fe_mul<F>(fe_sub<F>(ah, al), fe_sub<F>(bh, bl)));
    } else if constexpr (FORM == SC_LINEAR) {
      fe_t al = ld(A, id), ah = ld(A, id + h), bl = ld(B, id), bh = ld(B, id + h);
      acc[0] = fe_add<F>(acc[0], fe_sub<F>(al, bl));
      fe_t am = fe_sub<F>(fe_dbl<F>(al), ah), bm = fe_sub<F>(fe_dbl<F>(bl), bh);
      acc[1] = fe_add<F>(acc[1], fe_sub<F>(am, bm));
    } else if constexpr (FORM == SC_QUADRATIC) {
      fe_t al = ld(A, id), ah = ld(A, id + h), bl = ld(B, id), bh = ld(B, id + h);
      acc[0] = fe_add<F>(acc[0], fe_mul<F>(al, bl));
      fe_t am = fe_sub<F>(fe_dbl<F>(al), ah), bm = fe_sub<F>(fe_dbl<F>(bl), bh);
      acc[1] = fe_add<F>(acc[1], fe_mul<F>(am, bm));
    } else if constexpr (FORM == SC_CUBIC) {
      fe_t al = ld(A, id), ah = ld(A, id + h), bl = ld(B, id), bh = ld(B, id + h);
      fe_t cl = ld(C, id), ch = ld(C, id + h);
      fe_t da = fe_sub<F>(ah, al), db = fe_sub<F>(bh, bl), dc = fe_sub<F>(ch, cl);
      acc[0] = fe_add<F>(acc[0], fe_mul<F>(fe_mul<F>(al, bl), cl));
      acc[1] = fe_add<F>(acc[1], fe_mul<F>(fe_mul<F>(da, db), dc));
      acc[2] = fe_add<F>(acc[2], fe_mul<F>(fe_mul<F>(fe_sub<F>(al, da), fe_sub<F>(bl, db)),
                                           fe_sub<F>(cl, dc)));
    } else {  // eq-weighted forms: the un-weighted terms times f = eq(id)
      fe_t x[N];
      unweighted(id, x);
      fe_t f = eq.get<F>(id);
#pragma unroll
      for (int k = 0; k < N; k++) acc[k] = fe_add<F>(acc[k], fe_mul<F>(x[k], f));
    }
  }
  // the terms of an eq-weighted form before the weight: t0 / tinf (or the single t) of index `id`
  static constexpr bool eq_weighted = FORM >= SC_EQ_CUBIC3 && FORM <= SC_DOT_EQ;
  template <int N>
  NOVA_D void unweighted(size_t id, fe_t (&x)[N]) const {
    if constexpr (FORM == SC_EQ_CUBIC3 || FORM == SC_EQ_CUBIC2) {
      fe_t al = ld(A, id), ah = ld(A, id + h), bl = ld(B, id), bh = ld(B, id + h);
      fe_t e0 = fe_mul<F>(al, bl);
      if constexpr (FORM == SC_EQ_CUBIC3)
        e0 = fe_sub<F>(e0, ld(C, id));
      else
        e0 = fe_sub<F>(e0, fe_one<F>());
      x[0] = e0;
      x[1] = fe_mul<F>(fe_sub<F>(ah, al), fe_sub<F>(bh, bl));
    } else if constexpr (FORM == SC_EQ_QUAD1 || FORM == SC_DOT_EQ) {
      x[0] = ld(A, id);
    } else if constexpr (FORM == SC_EQ_CUBIC3_M1 || FORM == SC_EQ_CUBIC2_M1) {
      fe_t al = ld(A, id), ah = ld(A, id + h), bl = ld(B, id), bh = ld(B, id + h);
      fe_t am = fe_sub<F>(fe_dbl<F>(al), ah), bm = fe_sub<F>(fe_dbl<F>(bl), bh);
      fe_t e = fe_mul<F>(am, bm);
      if constexpr (FORM == SC_EQ_CUBIC3_M1) {
        fe_t cl = ld(C, id), ch = ld(C, id + h);
        e = fe_sub<F>(e, fe_sub<F>(fe_dbl<F>(cl), ch));
      } else {
        e = fe_sub<F>(e, fe_one<F>());
      }
      x[0] = e;
    } else if constexpr (FORM == SC_EQ_QUAD1_M1) {
      fe_t al = ld(A, id), ah = ld(A, id + h);
      x[0] = fe_sub<F>(fe_dbl<F>(al), ah);
    }
  }
};

// Segmented form of the same reduction for the eq-weighted sums (opt-in, NOVA_B200_SC_SEG=1; off by default, it showed
// no gain over the flat form for the cubic loop at 2^22):
//   sum_id left[id >> shift] right[id & mask] X(id)  =  sum_hi left[hi] * ( sum_lo right[lo] X(hi, lo) )
// -- the order the reference's split-eq loops use (sumcheck.rs:900-966).  A block walks whole segments of 2^shift
// indices, so the product left * right per index disappears (one product by left[hi] per thread and segment
// instead), and two indices share one Montgomery reduction through fe_mul2_add.  Field sums are exact, so the
// result is bit-identical to k_form_reduce's.  Needs the split tables (left != nullptr), an unsharded index
// (id_mul == 1) and segments of at least a few indices per thread; the launcher checks.
template <class F, int NOUT, class Form>
__global__ void __launch_bounds__(256) k_form_reduce_eqseg(Form form, size_t count, void* partials) {
  __shared__ fe_t sm[8 * NOUT];
  fe_t acc[NOUT];
#pragma unroll
  for (int k = 0; k < NOUT; k++) acc[k] = fe_zero<F>();
  const size_t seg = (size_t)1 << form.eq.shift;
  const size_t nseg = (count + seg - 1) / seg;
  const size_t T = blockDim.x;
  for (size_t s = blockIdx.x; s < nseg; s += gridDim.x) {
    const size_t base = s * seg;
    const size_t end = base + seg < count ? base + seg : count;
    fe_t in[NOUT];
#pragma unroll
    for (int k = 0; k < NOUT; k++) in[k] = fe_zero<F>();
    size_t id = base + threadIdx.x;
    for (; id + T < end; id += 2 * T) {  // indices id and id + T together
      fe_t xa[NOUT], xb[NOUT];
      form.unweighted(id, xa);
      form.unweighted(id + T, xb);
      const fe_t ra = fe_load(form.eq.right, id - base), rb = fe_load(form.eq.right, id + T - base);
#pragma unroll
      for (int k = 0; k < NOUT; k++) in[k] = fe_add<F>(in[k], fe_mul2_add<F>(xa[k], ra, xb[k], rb));
    }
    if (id < end) {
      fe_t xa[NOUT];
      form.unweighted(id, xa);
      const fe_t ra = fe_load(form.eq.right, id - base);
#pragma unroll
      for (int k = 0; k < NOUT; k++) in[k] = fe_add<F>(in[k], fe_mul<F>(xa[k], ra));
    }
    const fe_t lf = fe_load(form.eq.left, s);
#pragma unroll
    for (int k = 0; k < NOUT; k++) acc[k] = fe_add<F>(acc[k], fe_mul<F>(in[k], lf));
  }
  block_sum<F, NOUT>(acc, sm);
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < NOUT; k++) fe_store(partials, (size_t)blockIdx.x * NOUT + k, acc[k]);
}

NOVA_HD constexpr int sc_form_nout(int form) {
  return form == SC_CUBIC ? 3
         : (form == SC_EQ_QUAD1 || form == SC_DOT_EQ || form == SC_DOT || form >= SC_EQ_CUBIC3_M1) ? 1
                                                                                : 2;
}

// The nested eq tables of an EqSumCheckInstance (sumcheck.rs:606-664) in one launch: table k = eq(taus[hi-k .. hi)),
// 2^k entries at element offset 2^k - 1 of `out`, for k = 0 .. K.  Table k+1 is table k times (1 - t, t) with
// t = taus[hi-k-1] as the new TOP variable -- the recurrence of the reference's compute_eqs.  One block; K <= 12 here
// (longer tables come from k_eq_small / k_eq_outer, which split the work over the GPU).
template <class F>
__global__ void __launch_bounds__(1024) k_eq_prefix_tables(const void* __restrict__ taus, int hi, int K,
                                                           void* __restrict__ out) {
  if (threadIdx.x == 0) fe_store(out, 0, fe_one<F>());
  __syncthreads();
  for (int k = 0; k < K; k++) {
    const fe_t t = fe_load(taus, (size_t)(hi - k - 1));
    const size_t n = (size_t)1 << k;
    const void* src = (const char*)out + 32 * (n - 1);
    void* dst = (char*)out + 32 * (2 * n - 1);
    for (size_t i = threadIdx.x; i < n; i += blockDim.x) {
      const fe_t base = fe_load_rw(src, i);
      const fe_t up = fe_mul<F>(base, t);
      fe_store(dst, i, fe_sub<F>(base, up));
      fe_store(dst, i + n, up);
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------
// All sums of one round of a BATCHED sum-check in one launch (prove_helper, ppsnark.rs:886-983: nine claims over
// sixteen tables of one length): grid = (blocks, sums), block (x, y) reduces a slice of sum y.  Two launches per
// round (this + k_form_final_multi) instead of two per sum.  Forms 0..9 only (the pair forms: count = len / 2).
// ------------------------------------------------------------------------------------------
constexpr int SC_MULTI_MAX = 32;
struct multi_sum {
  int32_t form;   // sc_form_id
  int32_t shift;  // eq split (eq_factor)
  const void *A, *B, *C;
  const void *eq_left, *eq_right;
};
struct multi_args {
  int32_t n;      // sums
  size_t h;       // half length = index count of every sum
  size_t id_mul, id_add;
  multi_sum s[SC_MULTI_MAX];
};

template <class F, int FORM, bool RW>
NOVA_D void multi_run(const multi_sum& m, size_t h, size_t id_mul, size_t id_add, size_t first, size_t stride,
                      fe_t (&acc)[3]) {
  constexpr int NOUT = sc_form_nout(FORM);
  sc_form<F, FORM, RW> f;
  f.A = m.A;
  f.B = m.B;
  f.C = m.C;
  f.h = h;
  f.eq.left = m.eq_left;
  f.eq.right = m.eq_right;
  f.eq.shift = m.shift;
  f.eq.mask = ((size_t)1 << m.shift) - 1;
  f.eq.id_mul = id_mul;
  f.eq.id_add = id_add;
  fe_t x[NOUT];
#pragma unroll
  for (int k = 0; k < NOUT; k++) x[k] = fe_zero<F>();
  for (size_t id = first; id < h; id += stride) f(id, x);
#pragma unroll
  for (int k = 0; k < NOUT; k++) acc[k] = x[k];
}

// acc = this thread's share of sum m (unused outputs stay zero)
template <class F, bool RW>
NOVA_D void multi_dispatch(const multi_sum& m, size_t h, size_t id_mul, size_t id_add, size_t first, size_t stride,
                           fe_t (&acc)[3]) {
#define NOVA_MULTI_CASE(X) \
  case X: multi_run<F, X, RW>(m, h, id_mul, id_add, first, stride, acc); break
  switch (m.form) {
    NOVA_MULTI_CASE(SC_QUAD_PROD);
    NOVA_MULTI_CASE(SC_LINEAR);
    NOVA_MULTI_CASE(SC_QUADRATIC);
    NOVA_MULTI_CASE(SC_CUBIC);
    NOVA_MULTI_CASE(SC_EQ_CUBIC3);
    NOVA_MULTI_CASE(SC_EQ_CUBIC2);
    NOVA_MULTI_CASE(SC_EQ_QUAD1);
    NOVA_MULTI_CASE(SC_EQ_CUBIC3_M1);
    NOVA_MULTI_CASE(SC_EQ_CUBIC2_M1);
    NOVA_MULTI_CASE(SC_EQ_QUAD1_M1);
    default: break;
  }
#undef NOVA_MULTI_CASE
}

// partials[(y * gridDim.x + x) * 3 + k]
// MINB = resident blocks per SM the register allocation aims at (2: 124 registers, no spills; 3: 80 registers, the
// cubic form spills) -- NOVA_B200_SC_MULTI_OCC selects at run time
template <class F, int MINB = 2>
__global__ void __launch_bounds__(256, MINB) k_form_reduce_multi(const multi_args a, void* __restrict__ partials) {
  __shared__ fe_t sm[8 * 3];
  fe_t acc[3] = {fe_zero<F>(), fe_zero<F>(), fe_zero<F>()};
  multi_dispatch<F, false>(a.s[blockIdx.y], a.h, a.id_mul, a.id_add, (size_t)blockIdx.x * blockDim.x + threadIdx.x,
                           (size_t)gridDim.x * blockDim.x, acc);
  block_sum<F, 3>(acc, sm);
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < 3; k++) fe_store(partials, ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 3 + k, acc[k]);
}

// block y: out[3 y + k] = sum over the nblocks partials of sum y (all three slots are written; a form with fewer
// outputs leaves zeros behind them)
template <class F>
__global__ void __launch_bounds__(256) k_form_final_multi(const void* __restrict__ partials, int nblocks,
                                                          void* __restrict__ out) {
  __shared__ fe_t sm[8 * 3];
  fe_t acc[3] = {fe_zero<F>(), fe_zero<F>(), fe_zero<F>()};
  for (int b = threadIdx.x; b < nblocks; b += blockDim.x)
#pragma unroll
    for (int k = 0; k < 3; k++)
      acc[k] = fe_add<F>(acc[k], fe_load_rw(partials, ((size_t)blockIdx.y * nblocks + b) * 3 + k));
  block_sum<F, 3>(acc, sm);
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < 3; k++) fe_store(out, (size_t)blockIdx.y * 3 + k, acc[k]);
}

// ------------------------------------------------------------------------------------------
// eq tables (eq.rs:54-73): index bit (ell-1-k) <-> r[k]; built as an outer product of two
// sqrt-sized tables, each entry of which is a direct product over its bits.
// ------------------------------------------------------------------------------------------
template <class F>
__global__ void __launch_bounds__(256) k_eq_small(const void* __restrict__ r, int ell,
                                                  void* __restrict__ out) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= ((size_t)1 << ell)) return;
  fe_t acc = fe_one<F>();
  const fe_t one = fe_one<F>();
  for (int k = 0; k < ell; k++) {
    fe_t rk = fe_load(r, k);
    bool bit = (idx >> (ell - 1 - k)) & 1;
    acc = fe_mul<F>(acc, bit ? rk : fe_sub<F>(one, rk));
  }
  fe_store(out, idx, acc);
}

template <class F>
__global__ void __launch_bounds__(256) k_eq_outer(const void* __restrict__ left,
                                                  const void* __restrict__ right, int right_bits,
                                                  size_t n, void* __restrict__ out) {
  size_t mask = ((size_t)1 << right_bits) - 1;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x)
    fe_store(out, i, fe_mul<F>(fe_load(left, i >> right_bits), fe_load(right, i & mask)));
}

// ------------------------------------------------------------------------------------------
// batch inversion (spartan/mod.rs:54-145).  Each thread runs Montgomery's trick over a chunk;
// zero inputs are reported through *zero_flag (the reference returns Err(InternalError)).
// ------------------------------------------------------------------------------------------
// `chunk` elements per thread: one Fermat inversion (~380 products) is shared by a chunk, so an element costs
// 3 + 380 / chunk products.  The launcher keeps >= 32 Ki threads: chunk = n / 32768 clamped to [32, 128]
// (larger chunks were faster for the two 2^22-element batches inside ppsnark).
constexpr int BINV_CHUNK = 32, BINV_CHUNK_MAX = 128;
constexpr size_t BINV_MIN_THREADS = (size_t)1 << 15;
template <class F>
__global__ void __launch_bounds__(128) k_batch_invert(const void* __restrict__ in, size_t n,
                                                      void* __restrict__ out,
                                                      int* __restrict__ zero_flag, int chunk) {
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t lo = t * (size_t)chunk;
  if (lo >= n) return;
  size_t hi = lo + chunk < n ? lo + chunk : n;
  // pass 1: out[i] = product of in[lo..i)
  fe_t acc = fe_one<F>();
  for (size_t i = lo; i < hi; i++) {
    fe_store(out, i, acc);
    acc = fe_mul<F>(acc, fe_load(in, i));
  }
  if (fe_is_zero(acc)) {
    atomicExch(zero_flag, 1);
    return;
  }
  acc = fe_inv<F>(acc);
  for (size_t i = hi; i-- > lo;) {
    fe_t v = fe_load(in, i);
    fe_t pre = fe_load_rw(out, i);
    fe_store(out, i, fe_mul<F>(acc, pre));
    acc = fe_mul<F>(acc, v);
  }
}

// ------------------------------------------------------------------------------------------
// random linear combination  out[i] = sum_k coeff[k] * P_k[i]  with P_k zero-extended to n
// (PolyEvalWitness::batch / batch_diff_size, spartan/mod.rs:232-277; hyperkzg.rs:1028-1040)
// ------------------------------------------------------------------------------------------
constexpr int RLC_MAX = 32;
struct rlc_args {
  const void* p[RLC_MAX];
  size_t len[RLC_MAX];
  int k;
};
template <class F>
__global__ void __launch_bounds__(256) k_rlc(rlc_args a, const void* __restrict__ coeffs, size_t n,
                                             void* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x) {
    fe_t acc = fe_zero<F>();
    for (int k = 0; k < a.k; k++)
      if (i < a.len[k]) acc = fe_add<F>(acc, fe_mul<F>(fe_load(coeffs, k), fe_load(a.p[k], i)));
    fe_store(out, i, acc);
  }
}

// ------------------------------------------------------------------------------------------
// HyperKZG pieces
// ------------------------------------------------------------------------------------------
// fold: out[j] = x*(P[2j+1] - P[2j]) + P[2j]                      hyperkzg.rs:1085-1095
template <class F>
__global__ void __launch_bounds__(256) k_kzg_fold(const void* __restrict__ p,
                                                  const void* __restrict__ x_ptr, size_t half,
                                                  void* __restrict__ out) {
  const fe_t x = fe_load(x_ptr, 0);
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < half;
       j += (size_t)gridDim.x * blockDim.x) {
    fe_t a = fe_load(p, 2 * j), b = fe_load(p, 2 * j + 1);
    fe_store(out, j, fe_add<F>(fe_mul<F>(x, fe_sub<F>(b, a)), a));
  }
}


template <class F>
NOVA_D fe_t fe_pow_u64(fe_t base, uint64_t e) {
  fe_t acc = fe_one<F>();
  while (e) {
    if (e & 1) acc = fe_mul<F>(acc, base);
    base = fe_sqr<F>(base);
    e >>= 1;
  }
  return acc;
}

// Horner evaluation at NU points with COALESCED loads: thread t owns coefficients t, t+T, t+2T, ...
// and evaluates  A_t(y) = sum_k f[t + kT] y^k  with y = u^T by Horner (high k first); then
//   f(u) = sum_t u^t A_t(u^T).   (hyperkzg.rs:1011-1019 computes the same value serially.)
// Every coefficient is loaded once for all NU points; partials[blockIdx][q] feed k_form_final.
//
// The powers come from one small launch (k_poly_eval_powers) instead of two square-and-multiply
// ladders in every thread (which cost more than the Horner steps themselves once each thread owns
// only a few dozen coefficients, and ~180 dependent products of latency for short polynomials):
//   pw[q][0] = u_q^T,   pw[q][1 + b] = u_q^(256 b) for b < grid,   pw[q][1 + grid + j] = u_q^j, j < 256
// so u^t = pw[1 + blockIdx] * pw[1 + grid + threadIdx] is one product.
template <class F>
__global__ void __launch_bounds__(128) k_poly_eval_powers(const void* __restrict__ us, int nu,
                                                          int grid, uint64_t T,
                                                          void* __restrict__ pw) {
  const int per = 1 + grid + 256;
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nu * per) return;
  int q = idx / per, j = idx % per;
  uint64_t e = j == 0 ? T : (j <= grid ? (uint64_t)256 * (uint64_t)(j - 1) : (uint64_t)(j - 1 - grid));
  fe_store(pw, (size_t)idx, fe_pow_u64<F>(fe_load(us, q), e));
}

template <class F, int NU>
__global__ void __launch_bounds__(256) k_poly_eval_strided(const void* __restrict__ f, size_t n,
                                                           const void* __restrict__ pw,
                                                           void* __restrict__ partials) {
  __shared__ fe_t sm[8 * NU];
  const size_t T = (size_t)gridDim.x * blockDim.x;
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t per = 1 + gridDim.x + 256;
  fe_t acc[NU], y[NU];
#pragma unroll
  for (int q = 0; q < NU; q++) {
    y[q] = fe_load(pw, q * per);
    acc[q] = fe_zero<F>();
  }
  if (t < n) {
    size_t kmax = (n - 1 - t) / T;  // largest k with t + kT < n
    for (size_t k = kmax + 1; k-- > 0;) {
      fe_t c = fe_load(f, t + k * T);
#pragma unroll
      for (int q = 0; q < NU; q++) acc[q] = fe_add<F>(fe_mul<F>(acc[q], y[q]), c);
    }
#pragma unroll
    for (int q = 0; q < NU; q++) {
      fe_t ut = fe_mul<F>(fe_load(pw, q * per + 1 + blockIdx.x),
                          fe_load(pw, q * per + 1 + gridDim.x + threadIdx.x));
      acc[q] = fe_mul<F>(acc[q], ut);
    }
  }
  block_sum<F, NU>(acc, sm);
  if (threadIdx.x == 0)
#pragma unroll
    for (int q = 0; q < NU; q++) fe_store(partials, (size_t)blockIdx.x * NU + q, acc[q]);
}

// Several SHORT polynomials at the same NU points in one launch (the tail of the HyperKZG fold chain, hyperkzg.rs:1048-
// 1056: polynomials of 2^12 .. 2 coefficients, each of which would otherwise pay three launches).  Block b takes polynomial
// b; thread t owns coefficients t, t + 256, ...; its u^t and y = u^256 come from square-and-multiply ladders (16 products,
// nothing next to three launch latencies).  evals[(out_index[b]) * NU + q] = f_b(u_q).
constexpr int POLY_SMALL_MAX_LOG2 = 12;
struct poly_multi_args {
  const void* p[RLC_MAX];
  size_t len[RLC_MAX];
  int32_t out_index[RLC_MAX];
  int k;
};
template <class F, int NU>
__global__ void __launch_bounds__(256) k_poly_eval_small_multi(poly_multi_args a, const void* __restrict__ us,
                                                               void* __restrict__ evals) {
  __shared__ fe_t sm[8 * NU];
  const void* f = a.p[blockIdx.x];
  const size_t n = a.len[blockIdx.x], t = threadIdx.x, T = blockDim.x;
  fe_t acc[NU];
#pragma unroll
  for (int q = 0; q < NU; q++) acc[q] = fe_zero<F>();
  if (t < n) {
    fe_t y[NU];
#pragma unroll
    for (int q = 0; q < NU; q++) y[q] = fe_pow_u64<F>(fe_load(us, q), (uint64_t)T);
    const size_t kmax = (n - 1 - t) / T;
    for (size_t k = kmax + 1; k-- > 0;) {
      const fe_t c = fe_load(f, t + k * T);
#pragma unroll
      for (int q = 0; q < NU; q++) acc[q] = fe_add<F>(fe_mul<F>(acc[q], y[q]), c);
    }
#pragma unroll
    for (int q = 0; q < NU; q++) acc[q] = fe_mul<F>(acc[q], fe_pow_u64<F>(fe_load(us, q), (uint64_t)t));
  }
  block_sum<F, NU>(acc, sm);
  if (threadIdx.x == 0)
#pragma unroll
    for (int q = 0; q < NU; q++) fe_store(evals, (size_t)a.out_index[blockIdx.x] * NU + q, acc[q]);
}

constexpr int POLY_CHUNK = 64;
// The division kernels below take `cols` interleaved polynomials of n coefficients each: coefficient k
// of column j is b[k * cols + j] (divide_by_binomial, mercury.rs:319-356, divides every column of the
// row-major matrix f by (Y - alpha)).  cols = 1 is the plain polynomial of hyperkzg.rs:961-999.  Chunk
// values and carries are laid out [point][chunk][column], so neighbouring threads touch neighbouring
// columns and every load is coalesced.
//
// chunk values V_c = sum_{k<len_c} B[c*m + k] u^k  for each of the NU points (Horner per chunk)
template <class F>
__global__ void __launch_bounds__(128) k_poly_chunk_vals(const void* __restrict__ b, size_t n, size_t cols,
                                                         const void* __restrict__ us, int nu,
                                                         void* __restrict__ vals /* [nu][T][cols] */) {
  size_t T = (n + POLY_CHUNK - 1) / POLY_CHUNK;
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T * cols) return;
  size_t c = t / cols, j = t - c * cols;
  size_t lo = c * POLY_CHUNK, hi = lo + POLY_CHUNK < n ? lo + POLY_CHUNK : n;
  for (int q = 0; q < nu; q++) {
    fe_t u = fe_load(us, q);
    fe_t acc = fe_zero<F>();
    for (size_t i = hi; i-- > lo;) acc = fe_add<F>(fe_mul<F>(acc, u), fe_load(b, i * cols + j));
    fe_store(vals, (size_t)q * T * cols + t, acc);
  }
}

// one block per (point, column): suffix recurrence over chunk values
//   H_c = V_{c+1} + y * H_{c+1},  H_{T-1} = 0,  y = u^m      (carry into chunk c from above)
// and the polynomial value  P(u) = V_0 + y * H_0.  Affine maps x -> a*x + b are composed with a
// block-wide scan.  suffix[q][c][j] = H_c, evals[q][j] = P_j(u_q).
template <class F>
__global__ void __launch_bounds__(512) k_poly_suffix(const void* __restrict__ vals, size_t T, size_t cols,
                                                      const void* __restrict__ us,
                                                      void* __restrict__ suffix,
                                                      void* __restrict__ evals) {
  __shared__ fe_t sa[512], sb[512];
  const size_t q = blockIdx.x / cols, col = blockIdx.x - q * cols;
  // chunk c of this (point, column) at element (q * T + c) * cols + col of vals / suffix
  const void* v = (const char*)vals + 32 * (q * T * cols + col);
  void* sfx = (char*)suffix + 32 * (q * T * cols + col);
  const fe_t y = fe_pow_u64<F>(fe_load(us, q), POLY_CHUNK);
  const int nt = blockDim.x, tid = threadIdx.x;
  // thread tid owns chunk indices [clo, chi) ; processed from high to low
  size_t per = (T + nt - 1) / nt;
  size_t clo = (size_t)tid * per, chi = clo + per < T ? clo + per : T;
  if (clo > T) clo = T;
  // map for the thread's range: H_{clo-1}... we define g(x) = value entering below the range
  // given x = H_{chi-1} (carry entering the top chunk of the range).  For c from chi-1 down to clo:
  //   carry_below = V_c + y * carry_in
  fe_t a = fe_one<F>(), b = fe_zero<F>();  // identity map
  for (size_t c = chi; c-- > clo;) {
    // new = V_c + y * (a*x + b) = (y a) x + (y b + V_c)
    a = fe_mul<F>(y, a);
    b = fe_add<F>(fe_mul<F>(y, b), fe_load(v, c * cols));
  }
  sa[tid] = a;
  sb[tid] = b;
  __syncthreads();
  // inclusive scan from high tid to low tid: total_t = map_t o total_{t+1}
  for (int d = 1; d < nt; d <<= 1) {
    fe_t oa, ob;
    bool have = tid + d < nt;
    if (have) {
      oa = sa[tid + d];
      ob = sb[tid + d];
    }
    __syncthreads();
    if (have) {
      // combined(x) = mine(other(x)) = a*(oa x + ob) + b
      fe_t na = fe_mul<F>(sa[tid], oa);
      fe_t nb = fe_add<F>(fe_mul<F>(sa[tid], ob), sb[tid]);
      sa[tid] = na;
      sb[tid] = nb;
    }
    __syncthreads();
  }
  // carry entering the top of my range = total_{tid+1}(0) = sb[tid+1]
  fe_t carry = (tid + 1 < nt) ? sb[tid + 1] : fe_zero<F>();
  if (tid == 0) fe_store(evals, blockIdx.x, sb[0]);  // total_0(0) = P(u)
  for (size_t c = chi; c-- > clo;) {
    fe_store(sfx, c * cols, carry);
    carry = fe_add<F>(fe_load(v, c * cols), fe_mul<F>(y, carry));
  }
}

// y = u^e (single element), for the second scan level
template <class F>
__global__ void k_fe_pow(const void* __restrict__ u, uint64_t e, void* __restrict__ out) {
  if (blockIdx.x == 0 && threadIdx.x == 0) fe_store(out, 0, fe_pow_u64<F>(fe_load(u, 0), e));
}

// out[i] = u^i as a CANONICAL integer (not Montgomery), i < n: the scalars of the test SRS [tau^i] G
// (k_scalar_bases in msm_kernels.cuh; hyperkzg.rs:357-376)
template <class F>
__global__ void __launch_bounds__(128) k_powers_canonical(const void* __restrict__ u, size_t n,
                                                          void* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  fe_store(out, i, fe_from_mont<F>(fe_pow_u64<F>(fe_load(u, 0), (uint64_t)i)));
}

// quotient by (X - u): h[k-1] = B[k] + u*h[k], h[n-1] := 0  (hyperkzg.rs:961-999); chunk c starts
// from the carry H_c computed above.  out[k] = h[k] for k < out_len (n-1 for the quotient; n when the
// same recurrence is reused one level up to spread carries over the level-1 chunks).  Per column j of
// `cols` interleaved polynomials: h_j[k] lands at out[k * cols + j].
template <class F>
__global__ void __launch_bounds__(128) k_poly_div_apply(const void* __restrict__ b, size_t n, size_t cols,
                                                        const void* __restrict__ u_ptr,
                                                        const void* __restrict__ suffix,
                                                        size_t out_len, void* __restrict__ out) {
  size_t T = (n + POLY_CHUNK - 1) / POLY_CHUNK;
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T * cols) return;
  const fe_t u = fe_load(u_ptr, 0);
  size_t c = t / cols, j = t - c * cols;
  size_t lo = c * POLY_CHUNK, hi = lo + POLY_CHUNK < n ? lo + POLY_CHUNK : n;
  fe_t carry = fe_load(suffix, t);  // = h[hi-1]
  for (size_t k = hi; k-- > lo;) {
    // carry == h[k];  h[k-1] = B[k] + u*h[k]
    if (k < out_len) fe_store(out, k * cols + j, carry);
    carry = fe_add<F>(fe_load(b, k * cols + j), fe_mul<F>(u, carry));
  }
}

// ------------------------------------------------------------------------------------------
// Mercury prover pieces (provider/mercury.rs)
// ------------------------------------------------------------------------------------------
// compute_h_poly (mercury.rs:369-386): out[r] = sum_c f[r*cols + c] * v[c].  One block per row (grid-
// stride over rows), threads stride over the columns: coalesced reads of f, v stays in L2.
template <class F>
__global__ void __launch_bounds__(256) k_mat_vec_rows(const void* __restrict__ f, size_t rows, size_t cols,
                                                      const void* __restrict__ v, void* __restrict__ out) {
  __shared__ fe_t sm[8];
  for (size_t r = blockIdx.x; r < rows; r += gridDim.x) {
    fe_t acc[1] = {fe_zero<F>()};
    const void* row = (const char*)f + 32 * r * cols;
    for (size_t c = threadIdx.x; c < cols; c += blockDim.x)
      acc[0] = fe_add<F>(acc[0], fe_mul<F>(fe_load(row, c), fe_load(v, c)));
    block_sum<F, 1>(acc, sm);
    if (threadIdx.x == 0) fe_store(out, r, acc[0]);
    __syncthreads();  // sm is reused by the next row
  }
}

// make_s_polynomial (mercury.rs:391-475) without an NTT: s[k] is the coefficient of X^(k+1) (lag m = k+1)
// of a1(X) b1(1/X) + a1(1/X) b1(X) + gamma (a2(X) b2(1/X) + a2(1/X) b2(X)):
//   s[m-1] = sum_{j <= b-1-m} (a1[j+m] b1[j] + a1[j] b1[j+m]) + gamma * (the same over a2, b2),  1 <= m < b.
// Lag m has b - m terms, so block i takes the lags i+1 and b-1-i (b terms together, one lag when they meet).
template <class F>
__global__ void __launch_bounds__(256) k_mercury_s_poly(const void* __restrict__ a1, const void* __restrict__ b1,
                                                        const void* __restrict__ a2, const void* __restrict__ b2,
                                                        size_t b, const void* __restrict__ gamma_ptr,
                                                        void* __restrict__ out) {
  __shared__ fe_t sm[8 * 2];
  for (size_t i = blockIdx.x; i < b / 2; i += gridDim.x) {
    const int nl = i + 1 == b - 1 - i ? 1 : 2;
    for (int l = 0; l < nl; l++) {
      const size_t m = l == 0 ? i + 1 : b - 1 - i;
      fe_t acc[2] = {fe_zero<F>(), fe_zero<F>()};
      for (size_t j = threadIdx.x; j + m < b; j += blockDim.x) {
        acc[0] = fe_add<F>(acc[0], fe_add<F>(fe_mul<F>(fe_load(a1, j + m), fe_load(b1, j)),
                                             fe_mul<F>(fe_load(a1, j), fe_load(b1, j + m))));
        acc[1] = fe_add<F>(acc[1], fe_add<F>(fe_mul<F>(fe_load(a2, j + m), fe_load(b2, j)),
                                             fe_mul<F>(fe_load(a2, j), fe_load(b2, j + m))));
      }
      block_sum<F, 2>(acc, sm);
      if (threadIdx.x == 0) fe_store(out, m - 1, fe_add<F>(acc[0], fe_mul<F>(fe_load(gamma_ptr, 0), acc[1])));
      __syncthreads();
    }
  }
}

// ------------------------------------------------------------------------------------------
// sparse matrix (CSR) x dense vector, coefficient classes of sparse.rs:19-133
//   code  1 / -1      : add / subtract
//   code  +-2..+-7     : doubling/add chains (small_mul, sparse.rs:110-133)
//   code  0            : general coefficient, full field multiplication with vals[e]
// One thread per row (R1CS rows carry a handful of entries); z stays L2-resident.
// ------------------------------------------------------------------------------------------
template <class F>
__global__ void __launch_bounds__(256) k_spmv_classify(const void* __restrict__ vals, size_t nnz,
                                                       int8_t* __restrict__ codes) {
  size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nnz) return;
  fe_t v = fe_load(vals, e);
  fe_t k = fe_one<F>();
  const fe_t one = k;
  int8_t code = 0;
  for (int c = 1; c <= 7; c++) {
    if (fe_eq(v, k)) code = (int8_t)c;
    if (fe_eq(v, fe_neg<F>(k))) code = (int8_t)(-c);
    k = fe_add<F>(k, one);
  }
  codes[e] = code;
}

template <class F>
NOVA_D fe_t small_mul(int c, const fe_t& x) {  // sparse.rs:110-133
  int a = c < 0 ? -c : c;
  fe_t d = fe_dbl<F>(x), r;
  switch (a) {
    case 1: r = x; break;
    case 2: r = d; break;
    case 3: r = fe_add<F>(d, x); break;
    case 4: r = fe_dbl<F>(d); break;
    case 5: r = fe_add<F>(fe_dbl<F>(d), x); break;
    case 6: r = fe_add<F>(fe_dbl<F>(d), d); break;
    default: r = fe_add<F>(fe_add<F>(fe_dbl<F>(d), d), x); break;
  }
  return c < 0 ? fe_neg<F>(r) : r;
}

template <class F, int NV>
__global__ void __launch_bounds__(256) k_spmv(const uint32_t* __restrict__ indptr,
                                              const uint32_t* __restrict__ cols,
                                              const int8_t* __restrict__ codes,
                                              const void* __restrict__ vals, size_t rows,
                                              const void* __restrict__ z1,
                                              const void* __restrict__ z2, void* __restrict__ o1,
                                              void* __restrict__ o2) {
  for (size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows;
       r += (size_t)gridDim.x * blockDim.x) {
    fe_t s1 = fe_zero<F>(), s2 = fe_zero<F>();
    for (uint32_t e = indptr[r]; e < indptr[r + 1]; e++) {
      uint32_t col = cols[e];
      int c = codes[e];
      fe_t x1 = fe_load(z1, col), x2;
      if (NV == 2) x2 = fe_load(z2, col);
      if (c == 0) {
        fe_t v = fe_load(vals, e);
        s1 = fe_add<F>(s1, fe_mul<F>(v, x1));
        if (NV == 2) s2 = fe_add<F>(s2, fe_mul<F>(v, x2));
      } else {
        s1 = fe_add<F>(s1, small_mul<F>(c, x1));
        if (NV == 2) s2 = fe_add<F>(s2, small_mul<F>(c, x2));
      }
    }
    fe_store(o1, r, s1);
    if (NV == 2) fe_store(o2, r, s2);
  }
}

// transposed product  out[col] = sum_{(row,col,val) in M} rx[row] * val   (compute_eval_table_sparse,
// spartan/mod.rs:497-534: serial scatter in the reference; here one thread per COLUMN over the CSC
// view built at registration, so no atomics on 256-bit values are needed)
template <class F>
__global__ void __launch_bounds__(256) k_spmv_t(const uint32_t* __restrict__ tptr,
                                                const uint32_t* __restrict__ trow,
                                                const uint32_t* __restrict__ tperm,
                                                const int8_t* __restrict__ codes,
                                                const void* __restrict__ vals, size_t cols, size_t out_len,
                                                const void* __restrict__ rx, void* __restrict__ out) {
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < out_len;
       c += (size_t)gridDim.x * blockDim.x) {
    fe_t s = fe_zero<F>();
    if (c < cols) {
      for (uint32_t e = tptr[c]; e < tptr[c + 1]; e++) {
        uint32_t src = tperm[e];
        fe_t x = fe_load(rx, trow[e]);
        int code = codes[src];
        s = fe_add<F>(s, code == 0 ? fe_mul<F>(fe_load(vals, src), x) : small_mul<F>(code, x));
      }
    }
    fe_store(out, c, s);
  }
}

// out[i] = table[idx[i]]  (L_row / L_col of ppsnark.rs:236-250)
static __global__ void __launch_bounds__(256) k_gather32(const void* __restrict__ table,
                                                  const uint32_t* __restrict__ idx, size_t n,
                                                  void* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x)
    fe_store(out, i, fe_load(table, idx[i]));
}

// ------------------------------------------------------------------------------------------
// R1CSShapeSparkRepr::new (ppsnark.rs:117-190) from three registered matrices of one shape.
// Slot i < nnz_A + nnz_B + nnz_C is entry e of matrix k in CSR order; its row is found by binary
// search in that matrix' indptr.  Padding slots get row 0 and column N - 1 (ppsnark.rs:123).
// The timestamps need no scatter: ts_row[r] = sum_k (indptr_k[r+1] - indptr_k[r]) and ts_col[c]
// the same over the CSC pointers tptr_k, plus the N - total padding slots at ts_row[0] and
// ts_col[N-1].  One thread per slot writes row, col, ts_row and ts_col in Montgomery form and
// the u32 row / col gather indices.
// ------------------------------------------------------------------------------------------
struct spark_mats {
  const uint32_t* indptr[3];
  const uint32_t* colidx[3];
  const uint32_t* tptr[3];
  size_t nnz[3];
  size_t rows, cols;
};

template <class F>
NOVA_D fe_t fe_from_small(uint64_t x) {
  fe_t r = fe_zero<F>();
  r.l[0] = (uint32_t)x;
  r.l[1] = (uint32_t)(x >> 32);
  return fe_to_mont<F>(r);
}

template <class F>
__global__ void __launch_bounds__(256) k_spark_repr(const spark_mats m, size_t N, void* __restrict__ row,
                                                    void* __restrict__ col, void* __restrict__ ts_row,
                                                    void* __restrict__ ts_col, uint32_t* __restrict__ row_idx,
                                                    uint32_t* __restrict__ col_idx) {
  const size_t o1 = m.nnz[0], o2 = o1 + m.nnz[1], total = o2 + m.nnz[2], pad = N - total;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t r = 0, c = (uint32_t)(N - 1);
    if (i < total) {
      const int k = i < o1 ? 0 : (i < o2 ? 1 : 2);
      const size_t e = i - (k == 0 ? 0 : (k == 1 ? o1 : o2));
      const uint32_t* ip = k == 0 ? m.indptr[0] : (k == 1 ? m.indptr[1] : m.indptr[2]);
      const uint32_t* ci = k == 0 ? m.colidx[0] : (k == 1 ? m.colidx[1] : m.colidx[2]);
      size_t lo = 0, hi = m.rows;  // ip[lo] <= e < ip[hi]
      while (hi - lo > 1) {
        const size_t mid = (lo + hi) / 2;
        if (ip[mid] <= e) lo = mid;
        else hi = mid;
      }
      r = (uint32_t)lo;
      c = ci[e];
    }
    uint64_t tr = i == 0 ? pad : 0, tc = i == N - 1 ? pad : 0;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      if (i < m.rows) tr += m.indptr[k][i + 1] - m.indptr[k][i];
      if (i < m.cols) tc += m.tptr[k][i + 1] - m.tptr[k][i];
    }
    row_idx[i] = r;
    col_idx[i] = c;
    fe_store(row, i, fe_from_small<F>(r));
    fe_store(col, i, fe_from_small<F>(c));
    fe_store(ts_row, i, fe_from_small<F>(tr));
    fe_store(ts_col, i, fe_from_small<F>(tc));
  }
}

// ------------------------------------------------------------------------------------------
// The verifier's R1CS matrix evaluations (multi_evaluate, spartan/snark.rs:325-355):
//   out[y] = sum over the entries (row, col, val) of matrix y of T_x[row] * T_y[col] * val,   y < k <= 3.
// Work is split by ENTRY range, not by row: thread g of matrix y (grid.y) takes entries [g chunk, (g+1) chunk)
// (and every grid's worth of slices after it, should the launch not cover nnz),
// finds the row of its first entry by binary search in indptr (as k_spark_repr does), keeps a running row sum of
// T_y[col] * val and multiplies it by T_x[row] only when the row ends -- one product per row boundary plus one per
// general coefficient (codes +-1..7 cost adds, small_mul).  A long row spreads over many threads and a run of empty
// rows is skipped by one more search, so no thread's work depends on the row lengths.  Field sums are exact, so the
// split does not change the result.  partials[y * gridDim.x + x] feed k_r1cs_final.
// ------------------------------------------------------------------------------------------
constexpr int R1CS_MAX_MATS = 3;
struct r1cs_mats {
  const uint32_t* indptr[R1CS_MAX_MATS];
  const uint32_t* colidx[R1CS_MAX_MATS];
  const int8_t* codes[R1CS_MAX_MATS];
  const void* vals[R1CS_MAX_MATS];
  size_t rows[R1CS_MAX_MATS];
  size_t nnz[R1CS_MAX_MATS];
};

// the row holding entry e: the largest r in [lo, rows) with ip[r] <= e (ip[lo] <= e < ip[rows] = nnz)
NOVA_D size_t r1cs_row_of(const uint32_t* __restrict__ ip, size_t lo, size_t rows, size_t e) {
  size_t hi = rows;
  while (hi - lo > 1) {
    const size_t mid = (lo + hi) / 2;
    if (ip[mid] <= e) lo = mid;
    else hi = mid;
  }
  return lo;
}

template <class F>
__global__ void __launch_bounds__(256) k_r1cs_eval(const r1cs_mats m, const void* __restrict__ tx,
                                                   const void* __restrict__ ty, size_t chunk,
                                                   void* __restrict__ partials) {
  __shared__ fe_t sm[8];
  const int y = blockIdx.y;
  const uint32_t* ip = m.indptr[y];
  const uint32_t* ci = m.colidx[y];
  const int8_t* codes = m.codes[y];
  const void* vals = m.vals[y];
  const size_t nnz = m.nnz[y], rows = m.rows[y];
  fe_t acc[1] = {fe_zero<F>()};
  const size_t stride = (size_t)gridDim.x * blockDim.x * chunk;  // one slice per thread when the launch covers nnz
  // the entries are [ip[0], ip[rows]): registration allows an indptr that does not start at 0, and the reference
  // (par_windows over indptr) never reads the entries before ip[0]; rows == 0 gives ip[0] == nnz, no work
  for (size_t e0 = ip[0] + ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * chunk; e0 < nnz; e0 += stride) {
    const size_t e1 = e0 + chunk < nnz ? e0 + chunk : nnz;
    size_t row = r1cs_row_of(ip, 0, rows, e0);
    size_t next = ip[row + 1];
    fe_t s = fe_zero<F>();
    for (size_t e = e0; e < e1; e++) {
      if (e >= next) {  // row ends: weigh its sum, then find the row of e (the next one, or past a run of empty rows)
        acc[0] = fe_add<F>(acc[0], fe_mul<F>(fe_load(tx, row), s));
        s = fe_zero<F>();
        row = ip[row + 2] > e ? row + 1 : r1cs_row_of(ip, row + 1, rows, e);
        next = ip[row + 1];
      }
      const fe_t t = fe_load(ty, ci[e]);
      const int c = codes[e];
      s = fe_add<F>(s, c == 0 ? fe_mul<F>(fe_load(vals, e), t) : small_mul<F>(c, t));
    }
    acc[0] = fe_add<F>(acc[0], fe_mul<F>(fe_load(tx, row), s));
  }
  block_sum<F, 1>(acc, sm);
  if (threadIdx.x == 0) fe_store(partials, (size_t)blockIdx.y * gridDim.x + blockIdx.x, acc[0]);
}

// block y: out[y] = sum of the nblocks partials of matrix y
template <class F>
__global__ void __launch_bounds__(256) k_r1cs_final(const void* __restrict__ partials, int nblocks,
                                                    void* __restrict__ out) {
  __shared__ fe_t sm[8];
  fe_t acc[1] = {fe_zero<F>()};
  for (int b = threadIdx.x; b < nblocks; b += blockDim.x)
    acc[0] = fe_add<F>(acc[0], fe_load_rw(partials, (size_t)blockIdx.y * nblocks + b));
  block_sum<F, 1>(acc, sm);
  if (threadIdx.x == 0) fe_store(out, blockIdx.y, acc[0]);
}

// ------------------------------------------------------------------------------------------
// The IPA verifier's tensor vector (ipa_pc.rs:334-349): s[i] = scale * prod_j (bit j of i, MSB first ? r_j : r_j^-1),
// the reference's s[0] = prod r^-1, s[i] = s[i - 2^pos] r^2_{L-1-pos} written as one product per entry.  Built as
// an eq table is: each half table entry is a direct product over its bits (this kernel, `scale` folded into the
// left half only), and s is their outer product (k_eq_outer).
// ------------------------------------------------------------------------------------------
template <class F>
__global__ void __launch_bounds__(256) k_ipa_s_half(const void* __restrict__ r, const void* __restrict__ r_inv,
                                                    int bits, const void* __restrict__ scale_or_null,
                                                    void* __restrict__ out) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= ((size_t)1 << bits)) return;
  fe_t acc = scale_or_null ? fe_load(scale_or_null, 0) : fe_one<F>();
  for (int j = 0; j < bits; j++) {
    const bool bit = (idx >> (bits - 1 - j)) & 1;
    acc = fe_mul<F>(acc, fe_load(bit ? r : r_inv, j));
  }
  fe_store(out, idx, acc);
}

// ------------------------------------------------------------------------------------------
// NeutronNova folding prover pieces (neutron/nifs.rs, spartan/polys/power.rs)
// ------------------------------------------------------------------------------------------
// prove_helper (nifs.rs:29-186) before the rho factors.  Row k = i*left + j; with V_t = V1 + t (V2 - V1)
// for e (first `left` entries of e1/e2), f (the `right` entries after them), Az, Bz, Cz:
//   S_t = sum_i f_t[i] * sum_j e_t[j] (Az_t[k] Bz_t[k] - Cz_t[k]),   t in {0, 2, 3, 4, 5}.
// Each block owns a contiguous tile of rows and its threads stride through it by blockDim, so loads
// stay coalesced and a thread meets the same i for about left / blockDim rows in a row: the inner sums
// are kept per thread and multiplied by f_t[i] only when i changes (10 products per row plus 5 per
// change).  partials[block][t] feed k_form_final<F, 5>; field sums are exact, so the tiling does not
// change the result.
template <class F>
__global__ void __launch_bounds__(256) k_neutron_evals(const void* __restrict__ e1, const void* __restrict__ az1,
                                                       const void* __restrict__ bz1, const void* __restrict__ cz1,
                                                       const void* __restrict__ e2, const void* __restrict__ az2,
                                                       const void* __restrict__ bz2, const void* __restrict__ cz2,
                                                       size_t left, size_t right, size_t tile,
                                                       void* __restrict__ partials) {
  __shared__ fe_t sm[8 * 5];
  const size_t n = left * right;
  const size_t lo = (size_t)blockIdx.x * tile, hi = lo + tile < n ? lo + tile : n;
  fe_t acc[5], inner[5];
#pragma unroll
  for (int t = 0; t < 5; t++) acc[t] = inner[t] = fe_zero<F>();
  const void* f1 = (const char*)e1 + 32 * left;
  const void* f2 = (const char*)e2 + 32 * left;
  // inner[] -> acc[]: acc_t += f_t[i] * inner_t
  auto flush = [&](size_t i) {
    fe_t fv = fe_load(f1, i), fh = fe_load(f2, i), d = fe_sub<F>(fh, fv);
    acc[0] = fe_add<F>(acc[0], fe_mul<F>(fv, inner[0]));
    fv = fe_add<F>(fh, d);  // t = 2
#pragma unroll
    for (int t = 1; t < 5; t++) {
      acc[t] = fe_add<F>(acc[t], fe_mul<F>(fv, inner[t]));
      fv = fe_add<F>(fv, d);
    }
  };
  size_t cur = ~(size_t)0;
  for (size_t k = lo + threadIdx.x; k < hi; k += blockDim.x) {
    const size_t i = k / left, j = k - i * left;
    if (i != cur) {
      if (cur != ~(size_t)0) flush(cur);
#pragma unroll
      for (int t = 0; t < 5; t++) inner[t] = fe_zero<F>();
      cur = i;
    }
    fe_t e = fe_load(e1, j), a = fe_load(az1, k), b = fe_load(bz1, k), c = fe_load(cz1, k);
    const fe_t eh = fe_load(e2, j), ah = fe_load(az2, k), bh = fe_load(bz2, k), ch = fe_load(cz2, k);
    const fe_t de = fe_sub<F>(eh, e), da = fe_sub<F>(ah, a), db = fe_sub<F>(bh, b), dc = fe_sub<F>(ch, c);
    inner[0] = fe_add<F>(inner[0], fe_mul<F>(e, fe_sub<F>(fe_mul<F>(a, b), c)));
    // t = 2: 2 V2 - V1 = V2 + d; then one more d per step
    e = fe_add<F>(eh, de);
    a = fe_add<F>(ah, da);
    b = fe_add<F>(bh, db);
    c = fe_add<F>(ch, dc);
#pragma unroll
    for (int t = 1; t < 5; t++) {
      inner[t] = fe_add<F>(inner[t], fe_mul<F>(e, fe_sub<F>(fe_mul<F>(a, b), c)));
      e = fe_add<F>(e, de);
      a = fe_add<F>(a, da);
      b = fe_add<F>(b, db);
      c = fe_add<F>(c, dc);
    }
  }
  if (cur != ~(size_t)0) flush(cur);
  block_sum<F, 5>(acc, sm);
  if (threadIdx.x == 0)
#pragma unroll
    for (int t = 0; t < 5; t++) fe_store(partials, (size_t)blockIdx.x * 5 + t, acc[t]);
}

// PowPolynomial::split_evals (power.rs:62-86): out[j] = tau^j (j < left), out[left + i] = tau^(left i) (i < right).
template <class F>
__global__ void __launch_bounds__(128) k_pow_split_evals(const void* __restrict__ tau_ptr, size_t left, size_t right,
                                                         void* __restrict__ out) {
  const fe_t tau = fe_load(tau_ptr, 0);
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < left + right;
       x += (size_t)gridDim.x * blockDim.x)
    fe_store(out, x, fe_pow_u64<F>(tau, (uint64_t)(x < left ? x : left * (x - left))));
}

}  // namespace nova
