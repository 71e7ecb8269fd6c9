// Instantiates every kernel for one field and fills the launcher table (see ops.cuh).
#pragma once
#include "ops.cuh"
#include "msm_kernels.cuh"
#include "field_kernels.cuh"
#include "poly_kernels.cuh"
#include "transcript.cuh"
#include "transcript_batched.cuh"
#include "poseidon.cuh"
#include "sumcheck_tail.cuh"

namespace nova {

inline int stream_grid(size_t n, int block, int waves = 8) {
  // grid = multiple of the SM count, capped by the work available
  size_t need = (n + block - 1) / block;
  size_t cap = (size_t)NUM_SMS * waves;
  size_t g = need < cap ? need : cap;
  return (int)(g == 0 ? 1 : g);
}

// sum of n points (optionally gathered through idx): used by the 0/1-scalar and sparse paths
// (msm.rs:432-454 accumulate_bases, msm.rs:689-708 batch_add).  Two-level: each thread sums a
// strided slice with mixed adds, then a single block tree-sums the partials.
template <class F>
__global__ void __launch_bounds__(128) k_sum_points1(const void* __restrict__ tables,
                                                     const uint32_t* __restrict__ idx, size_t n,
                                                     void* __restrict__ partial) {
  size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t nthreads = (size_t)gridDim.x * blockDim.x;
  using PA = msm_arith<F>;
  typename PA::pt acc = PA::identity();
  for (size_t i = tid; i < n; i += nthreads) {
    typename PA::aff p = PA::load_table(tables, idx ? idx[i] : i);
    if (!PA::aff_is_identity(p)) PA::madd(acc, p);
  }
  PA::store(partial, tid, acc);
}

template <class F>
struct ops_impl {
  static void digits(cudaStream_t s, const void* scalars, const msm_plan& p) {
    digits_range(s, scalars, 0, p.n, p);
  }
  static void digits_range(cudaStream_t s, const void* scalars, size_t i0, size_t i1, const msm_plan& p) {
    if (i1 <= i0) return;
    int block = 256;
    size_t blocks = (i1 - i0 + block - 1) / block;
    int grid = (int)(blocks < SORT_HIST_BLOCKS ? blocks : SORT_HIST_BLOCKS);
    k_digits<F><<<grid, block, 0, s>>>(scalars, i0, i1, p.n, p.c, p.W, p.G, p.B, p.digits, p.sortctl, p.sp);
  }
  static void expand_key(cudaStream_t s, void* tables, size_t n_ck, int ntables, int shift) {
    int block = 128;
    int grid = (int)((n_ck + block - 1) / block);
    k_expand_key<F><<<grid, block, 0, s>>>(tables, n_ck, ntables, shift);
  }
  static void accumulate(cudaStream_t s, const void* tables, const msm_plan& p) {
    uint32_t K = (uint32_t)p.G * p.B;
    size_t max_entries = p.n * (size_t)p.W;
    size_t nseg = (max_entries + p.L - 1) / p.L;
    int block = 128;
    int grid = (int)((nseg + block - 1) / block);
#if !defined(NOVA_MSM_ARITH29)
    // run-time A/B: NOVA_B200_ACC_TMA=1 stages the gathered points in shared memory with cp.async.bulk + mbarrier
    static const bool use_tma = [] {
      const char* e = getenv("NOVA_B200_ACC_TMA");
      return e != nullptr && e[0] == '1';
    }();
    if (use_tma) {
      k_accumulate_tma<F><<<grid, block, 0, s>>>(p.entries, p.start, K, tables, p.L, p.buckets, p.parts, p.pkeys);
      return;
    }
#endif
    k_accumulate<F><<<grid, block, 0, s>>>(p.entries, p.start, K, tables, p.L, p.buckets, p.parts,
                                           p.pkeys);
  }
  static void fixup(cudaStream_t s, const msm_plan& p) {
    uint32_t K = (uint32_t)p.G * p.B;
    // expected partials per bucket = (entries / K) / L + 1; about 8 per lane (a lone thread up to 16),
    // at most a warp per key
    size_t entries = p.n * (size_t)p.W;
    size_t ppk = entries / ((size_t)K * p.L) + 1;
    int G = 1;
    while (G < 32 && (size_t)G * 8 < ppk) G <<= 1;
    if (ppk <= 16) G = 1;
    size_t threads = (size_t)K * G;
#if !defined(NOVA_MSM_ARITH29)
    if (G == 1) {  // few partials per bucket: one quad per key, cooperative adds
      threads = (size_t)K * 4;
      k_fixup_q<F><<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(p.start, K, p.L, p.heavy_min, p.parts,
                                                                     p.pkeys, p.buckets);
    } else
#endif
      k_fixup<F><<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(p.start, K, p.L, p.heavy_min, G, p.parts,
                                                                   p.pkeys, p.buckets);
    k_fixup_heavy1<F><<<NUM_SMS * 4, 256, 0, s>>>(p.start, p.L, p.heavy, p.parts, p.pkeys, p.hparts);
    k_fixup_heavy2<F><<<NUM_SMS, 32, 0, s>>>(p.heavy, p.hparts, p.buckets);
  }
  static void index_bases(cudaStream_t s, void* bases, size_t n, const void* gen, uint64_t k0) {
    k_index_bases<F><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(bases, n, gen, k0);
  }
  static void jacobian_sum(cudaStream_t s, const void* pts, int k, void* out_jac) {
#if !defined(NOVA_MSM_ARITH29)
    k_jacobian_sum_q<F><<<1, 32, 0, s>>>(pts, k, out_jac);
#else
    k_jacobian_sum<F><<<1, 32, 0, s>>>(pts, k, out_jac);
#endif
  }
  static void reduce(cudaStream_t s, const msm_plan& p, void* out_jac) {
    int bits = p.c - 1;  // bucket index bits
#if !defined(NOVA_MSM_ARITH29)
    // NOVA_B200_RED_FLAT=1 forces the round-1 form (every bucket read once per digit position), =0 the hierarchical
    // form; default: hierarchical from NOVA_B200_RED_HIER_BITS bucket-index bits on
    static const int flat_mode = [] {
      const char* e = getenv("NOVA_B200_RED_FLAT");
      return e == nullptr ? -1 : (e[0] == '1' ? 1 : 0);
    }();
    static const int hier_bits = [] {
      const char* e = getenv("NOVA_B200_RED_HIER_BITS");
      return e ? atoi(e) : 18;
    }();
    const bool flat = flat_mode == 1 || (flat_mode == -1 && bits < hier_bits);
    if (bits >= 1 && bits <= 24 && !flat) {  // hierarchical radix-16 digit sums (k_red_level_q)
      red_levels lv{};
      lv.nd = (bits + 3) / 4;
      size_t off = 0;  // in points (128 B) inside p.rparts
      uint32_t N = p.B;
      const void* X = p.buckets;
      for (int l = 0; l < lv.nd - 1; l++) {
        const uint32_t groups = N >> 4;
        int nsplit = (int)((groups + 511) / 512);  // ~8 serial additions per quad before the block tree
        if (nsplit < 1) nsplit = 1;
        lv.nsplit[l] = nsplit;
        lv.parts_off[l] = (unsigned)off;
        char* parts = (char*)p.rparts + off * 128;
        off += (size_t)p.G * 16 * nsplit;
        char* next = (char*)p.rparts + off * 128;
        const unsigned next_off = (unsigned)off;
        off += (size_t)p.G * groups;
        unsigned gx = (unsigned)nsplit, gb = (groups + 15) / 16;
        dim3 grid(gx > gb ? gx : gb, 17u, (unsigned)p.G);
        k_red_level_q<F><<<grid, 256, 0, s>>>(l == 0 ? p.start : nullptr, p.B, X, N, nsplit, parts, next);
        X = next;
        N = groups;
        lv.top_off = next_off;
      }
      if (lv.nd == 1) lv.top_off = 0xFFFFFFFFu;
      lv.top_n = N;
      char* merged = (char*)p.rparts + off * 128;
      dim3 g2((unsigned)(lv.nd * 16), (unsigned)p.G);
      k_red_merge_levels_q<F><<<g2, 256, 0, s>>>(p.rparts, lv, p.start, p.B, p.buckets, p.G, merged);
      k_red_final_q<F><<<1, 384, 0, s>>>(merged, p.G, bits, p.c, out_jac, p.peer);
      return;
    }
    if (bits >= 1 && bits <= 24) {  // radix-16 digit sums, quad-cooperative point operations
      int nd = (bits + 3) / 4;
      uint32_t count = p.B >> (bits < 4 ? bits : 4);  // buckets per digit value (full-width digits)
      int nsplit = (int)((count + 255) / 256);          // ~4 buckets per quad, then a 6-level tree
      if (nsplit < 1) nsplit = 1;
      if (nsplit > 4096) nsplit = 4096;
      char* merged = (char*)p.rparts + (size_t)p.G * nd * 16 * nsplit * 128;
      dim3 g1((unsigned)nsplit, (unsigned)(nd * 16), (unsigned)p.G);
      k_red_digits_q<F><<<g1, 256, 0, s>>>(p.start, p.B, bits, p.buckets, p.rparts);
      dim3 g2((unsigned)(nd * 16), (unsigned)p.G);
      k_red_merge_q<F><<<g2, 256, 0, s>>>(p.rparts, nd, nsplit, merged);
      k_red_final_q<F><<<1, 384, 0, s>>>(merged, p.G, bits, p.c, out_jac, p.peer);
      return;
    }
#endif
    if (bits >= 1 && bits <= 24) {  // radix-16 digit sums (msm_kernels.cuh)
      int nd = (bits + 3) / 4;
      dim3 g1(RED_NSPLIT, (unsigned)(nd * 16), (unsigned)p.G);
      k_red_digits<F><<<g1, 128, 0, s>>>(p.start, p.B, bits, p.buckets, p.rparts);
      k_red_final<F><<<1, 256, 0, s>>>(p.rparts, p.G, bits, p.c, out_jac);
      return;
    }
    uint32_t T = p.B / p.m;
    int block = 128;
    int grid = (int)(((size_t)T * p.G + block - 1) / block);
    k_reduce1<F><<<grid, block, 0, s>>>(p.start, p.B, p.G, p.m, p.buckets, p.rparts);
    k_reduce2<F><<<1, 256, 0, s>>>(p.rparts, T, p.G, p.c, out_jac);
  }
  static void sum_points(cudaStream_t s, const void* tables, const uint32_t* idx, size_t n,
                         void* scratch, void* out_jac) {
    // scratch must hold SUM_THREADS xyzz
    int block = 128, grid = NUM_SMS;
    k_sum_points1<F><<<grid, block, 0, s>>>(tables, idx, n, scratch);
    k_reduce2<F><<<1, 256, 0, s>>>(scratch, (uint32_t)(grid * block), 1, 0, out_jac);
  }
  static void cross_term(cudaStream_t s, const void* az, const void* bz, const void* cz,
                         const void* e1, const void* e2, const void* u, size_t n, void* t) {
    k_cross_term<F><<<stream_grid(n, 256), 256, 0, s>>>(az, bz, cz, e1, e2, u, n, t);
  }
  static void axpy(cudaStream_t s, const void* a, const void* b, const void* r, size_t n,
                   void* out) {
    k_axpy<F><<<stream_grid(n, 256), 256, 0, s>>>(a, b, r, n, out);
  }
  static void vec_add(cudaStream_t s, const void* a, const void* b, size_t n, void* out) {
    k_vec_add<F><<<stream_grid(n, 256), 256, 0, s>>>(a, b, n, out);
  }
  static void vec_mul(cudaStream_t s, const void* a, const void* b, size_t n, void* out) {
    k_vec_mul<F><<<stream_grid(n, 256), 256, 0, s>>>(a, b, n, out);
  }
  static void logup_hash(cudaStream_t s, const void* val, const void* addr, const void* gamma,
                         const void* r, size_t n, void* out) {
    k_logup_hash<F><<<stream_grid(n, 256), 256, 0, s>>>(val, addr, gamma, r, n, out);
  }
  static void bind_top(cudaStream_t s, void* z, size_t n, const void* r) {
    k_bind_top<F><<<stream_grid(n / 2, 256), 256, 0, s>>>(z, n / 2, r);
  }
  static void bind_top_multi(cudaStream_t s, void* const* zs, int k, size_t n, const void* r) {
    bind_multi_args a{};
    for (int i = 0; i < k; i++) a.z[i] = zs[i];
    int gx = stream_grid(n / 2, 256, 8);
    int per = (NUM_SMS * 8 + k - 1) / k;  // keep the whole launch near 8 waves of blocks
    if (gx > per) gx = per < 1 ? 1 : per;
    k_bind_top_multi<F><<<dim3((unsigned)gx, (unsigned)k), 256, 0, s>>>(a, n / 2, r);
  }
  static void fold_halves(cudaStream_t s, const void* v, size_t half, const void* x_lo, const void* x_hi,
                          void* out) {
    k_fold_halves<F><<<stream_grid(half, 256), 256, 0, s>>>(v, half, x_lo, x_hi, out);
  }
  static void ipa_scalars(cudaStream_t s, const void* a, const void* w, size_t n, size_t nk, void* sL,
                          void* sR) {
    k_ipa_scalars<F><<<stream_grid(n, 256), 256, 0, s>>>(a, w, n, nk, sL, sR);
  }
  static void ipa_weights(cudaStream_t s, void* w, size_t n, size_t nk, const void* r, const void* r_inv) {
    k_ipa_weights<F><<<stream_grid(n, 256), 256, 0, s>>>(w, n, nk, r, r_inv);
  }
  static void fill_one(cudaStream_t s, void* w, size_t n) {
    k_fill_one<F><<<stream_grid(n, 256), 256, 0, s>>>(w, n);
  }
  template <int FORM>
  static void sc_launch(cudaStream_t s, const void* A, const void* B, const void* C, size_t count,
                        size_t half, const void* eq_left, const void* eq_right, int shift,
                        size_t id_mul, size_t id_add, void* scratch, void* out) {
    constexpr int NOUT = sc_form_nout(FORM);
    sc_form<F, FORM> f;
    f.A = A;
    f.B = B;
    f.C = C;
    f.h = half;
    f.eq.left = eq_left;
    f.eq.right = eq_right;
    f.eq.shift = shift;
    f.eq.mask = ((size_t)1 << shift) - 1;
    f.eq.id_mul = id_mul;
    f.eq.id_add = id_add;
    size_t need = (count + 255) / 256;
    int grid = (int)(need < (size_t)SC_MAX_BLOCKS ? (need ? need : 1) : SC_MAX_BLOCKS);
    if constexpr (sc_form<F, FORM>::eq_weighted) {
      // opt-in segmented reduction (see k_form_reduce_eqseg): split tables, unsharded, >= 4 indices per thread
      if (sc_segmented_enabled() && eq_left != nullptr && id_mul == 1 && shift >= 10) {
        size_t nseg = (count + ((size_t)1 << shift) - 1) >> shift;
        grid = (int)(nseg < (size_t)SC_MAX_BLOCKS ? nseg : SC_MAX_BLOCKS);
        k_form_reduce_eqseg<F, NOUT, sc_form<F, FORM>><<<grid, 256, 0, s>>>(f, count, scratch);
        k_form_final<F, NOUT><<<1, 256, 0, s>>>(scratch, grid, out);
        return;
      }
    }
    k_form_reduce<F, NOUT, sc_form<F, FORM>><<<grid, 256, 0, s>>>(f, count, scratch);
    k_form_final<F, NOUT><<<1, 256, 0, s>>>(scratch, grid, out);
  }
  static void sc_reduce(cudaStream_t s, int form, const void* A, const void* B, const void* C,
                        size_t count, size_t half, const void* eq_left, const void* eq_right,
                        int shift, size_t id_mul, size_t id_add, void* scratch, void* out) {
#define SC_CASE(X) \
  case X: sc_launch<X>(s, A, B, C, count, half, eq_left, eq_right, shift, id_mul, id_add, scratch, out); break
    switch (form) {
      SC_CASE(SC_QUAD_PROD);
      SC_CASE(SC_LINEAR);
      SC_CASE(SC_QUADRATIC);
      SC_CASE(SC_CUBIC);
      SC_CASE(SC_EQ_CUBIC3);
      SC_CASE(SC_EQ_CUBIC2);
      SC_CASE(SC_EQ_QUAD1);
      SC_CASE(SC_EQ_CUBIC3_M1);
      SC_CASE(SC_EQ_CUBIC2_M1);
      SC_CASE(SC_EQ_QUAD1_M1);
      SC_CASE(SC_DOT_EQ);
      SC_CASE(SC_DOT);
      default: break;
    }
#undef SC_CASE
  }
  static void eq_small(cudaStream_t s, const void* r, int ell, void* out) {
    size_t n = (size_t)1 << ell;
    k_eq_small<F><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(r, ell, out);
  }
  static void eq_outer(cudaStream_t s, const void* left, const void* right, int right_bits, size_t n,
                       void* out) {
    k_eq_outer<F><<<stream_grid(n, 256), 256, 0, s>>>(left, right, right_bits, n, out);
  }
  static void batch_invert(cudaStream_t s, const void* in, size_t n, void* out, int* zero_flag) {
    static const int forced = [] {  // A/B: NOVA_B200_BINV_CHUNK=<elements per thread>
      const char* e = getenv("NOVA_B200_BINV_CHUNK");
      int v = e ? atoi(e) : 0;
      return v >= 1 && v <= 4096 ? v : 0;
    }();
    int chunk = (int)(n / BINV_MIN_THREADS);
    chunk = chunk < BINV_CHUNK ? BINV_CHUNK : (chunk > BINV_CHUNK_MAX ? BINV_CHUNK_MAX : chunk);
    if (forced) chunk = forced;
    size_t threads = (n + chunk - 1) / chunk;
    k_batch_invert<F><<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(in, n, out, zero_flag, chunk);
  }
  static void rlc(cudaStream_t s, const void* const* polys, const size_t* lens, int k,
                  const void* coeffs, size_t n, void* out) {
    rlc_args a;
    a.k = k;
    for (int i = 0; i < k; i++) {
      a.p[i] = polys[i];
      a.len[i] = lens[i];
    }
    k_rlc<F><<<stream_grid(n, 256), 256, 0, s>>>(a, coeffs, n, out);
  }
  static void kzg_fold(cudaStream_t s, const void* p, const void* x, size_t half, void* out) {
    k_kzg_fold<F><<<stream_grid(half, 256), 256, 0, s>>>(p, x, half, out);
  }
  template <int NU>
  static void poly_eval_n(cudaStream_t s, const void* f, size_t n, const void* us, void* scratch,
                          void* evals) {
    size_t need = (n + 255) / 256;
    int grid = (int)(need < (size_t)SC_MAX_BLOCKS ? (need ? need : 1) : SC_MAX_BLOCKS);
    void* pw = scratch;                                                     // NU x (1 + grid + 256)
    void* partials = (char*)scratch + (size_t)3 * (1 + SC_MAX_BLOCKS + 256) * 32;  // grid x NU
    int np = NU * (1 + grid + 256);
    k_poly_eval_powers<F><<<(np + 127) / 128, 128, 0, s>>>(us, NU, grid, (uint64_t)grid * 256, pw);
    k_poly_eval_strided<F, NU><<<grid, 256, 0, s>>>(f, n, pw, partials);
    k_form_final<F, NU><<<1, 256, 0, s>>>(partials, grid, evals);
  }
  static void poly_eval(cudaStream_t s, const void* f, size_t n, const void* us, int nu, void* scratch,
                        void* evals) {
    if (nu == 1) poly_eval_n<1>(s, f, n, us, scratch, evals);
    else if (nu == 2) poly_eval_n<2>(s, f, n, us, scratch, evals);
    else poly_eval_n<3>(s, f, n, us, scratch, evals);
  }
  // h = f / (X - u).  Level 1: chunk values V1 (Horner per 64 coefficients).  If there are few
  // chunks a single block scans them; otherwise the same two kernels run one level up (V1 as a
  // polynomial in y = u^64) so the single-block scan only ever sees <= ~n/4096 values.
  //
  // With cols > 1 the same kernels divide every column of a row-major matrix (divide_by_binomial,
  // mercury.rs:319-356): one thread per (chunk, column), one scan block per column.  One polynomial keeps
  // the 512-thread scan block; a column with few chunks gets a block just wide enough for them.
  static void poly_div(cudaStream_t s, const void* f, size_t n, size_t cols, const void* u, void* scratch, void* out,
                       void* rem) {
    static_assert(POLY_CHUNK == POLY_CHUNK_HOST, "chunk constants out of sync");
    size_t T1 = (n + POLY_CHUNK - 1) / POLY_CHUNK, T2 = (T1 + POLY_CHUNK - 1) / POLY_CHUNK;
    char* base = (char*)scratch;
    void* v1 = base;
    void* s1 = base + T1 * cols * 32;
    void* v2 = base + 2 * T1 * cols * 32;
    void* s2 = base + (2 * T1 + T2) * cols * 32;
    void* y = base + (2 * T1 + 2 * T2) * cols * 32;
    void* ev = rem ? rem : base + ((2 * T1 + 2 * T2) * cols + 1) * 32;
    unsigned g1 = (unsigned)((T1 * cols + 127) / 128), g2 = (unsigned)((T2 * cols + 127) / 128);
    auto scan_threads = [cols](size_t T) {
      unsigned nt = 32;
      while (cols > 1 && nt < 512 && nt < T) nt *= 2;
      return cols == 1 ? 512u : nt;
    };
    k_poly_chunk_vals<F><<<g1, 128, 0, s>>>(f, n, cols, u, 1, v1);
    if (T1 <= POLY_DIV_ONE_LEVEL_CHUNKS) {
      k_poly_suffix<F><<<(unsigned)cols, scan_threads(T1), 0, s>>>(v1, T1, cols, u, s1, ev);
    } else {
      k_fe_pow<F><<<1, 32, 0, s>>>(u, POLY_CHUNK, y);
      k_poly_chunk_vals<F><<<g2, 128, 0, s>>>(v1, T1, cols, y, 1, v2);
      k_poly_suffix<F><<<(unsigned)cols, scan_threads(T2), 0, s>>>(v2, T2, cols, y, s2, ev);
      k_poly_div_apply<F><<<g2, 128, 0, s>>>(v1, T1, cols, y, s2, T1, s1);  // carries into level-1 chunks
    }
    k_poly_div_apply<F><<<g1, 128, 0, s>>>(f, n, cols, u, s1, n - 1, out);
  }
  static void mat_vec_rows(cudaStream_t s, const void* f, size_t rows, size_t cols, const void* v, void* out) {
    unsigned grid = (unsigned)(rows < (size_t)NUM_SMS * 64 ? rows : (size_t)NUM_SMS * 64);
    if (grid) k_mat_vec_rows<F><<<grid, 256, 0, s>>>(f, rows, cols, v, out);
  }
  static void mercury_s_poly(cudaStream_t s, const void* a1, const void* b1, const void* a2, const void* b2, size_t b,
                             const void* gamma, void* out) {
    size_t pairs = b / 2;
    unsigned grid = (unsigned)(pairs < (size_t)NUM_SMS * 64 ? pairs : (size_t)NUM_SMS * 64);
    if (grid) k_mercury_s_poly<F><<<grid, 256, 0, s>>>(a1, b1, a2, b2, b, gamma, out);
  }
  static void neutron_evals(cudaStream_t s, const void* e1, const void* az1, const void* bz1, const void* cz1,
                            const void* e2, const void* az2, const void* bz2, const void* cz2, size_t left,
                            size_t right, void* scratch, void* out) {
    const size_t n = left * right, grid = neutron_evals_blocks(n), tile = (n + grid - 1) / grid;
    k_neutron_evals<F><<<(unsigned)grid, 256, 0, s>>>(e1, az1, bz1, cz1, e2, az2, bz2, cz2, left, right, tile,
                                                      scratch);
    k_form_final<F, 5><<<1, 256, 0, s>>>(scratch, (int)grid, out);
  }
  static void pow_split_evals(cudaStream_t s, const void* tau, size_t left, size_t right, void* out) {
    k_pow_split_evals<F><<<stream_grid(left + right, 128), 128, 0, s>>>(tau, left, right, out);
  }
  static void lerp(cudaStream_t s, const void* a, const void* b, const void* r, size_t n, void* out) {
    k_lerp<F><<<stream_grid(n, 256), 256, 0, s>>>(a, b, r, n, out);
  }
  static void spark_repr(cudaStream_t s, const spark_mats& m, size_t N, void* row, void* col, void* ts_row,
                         void* ts_col, uint32_t* row_idx, uint32_t* col_idx) {
    k_spark_repr<F><<<stream_grid(N, 256), 256, 0, s>>>(m, N, row, col, ts_row, ts_col, row_idx, col_idx);
  }
  static void spmv_classify(cudaStream_t s, const void* vals, size_t nnz, int8_t* codes) {
    k_spmv_classify<F><<<(unsigned)((nnz + 255) / 256), 256, 0, s>>>(vals, nnz, codes);
  }
  static void spmv(cudaStream_t s, const uint32_t* indptr, const uint32_t* cols, const int8_t* codes,
                   const void* vals, size_t rows, const void* z1, const void* z2, void* o1, void* o2) {
    if (z2)
      k_spmv<F, 2><<<stream_grid(rows, 256), 256, 0, s>>>(indptr, cols, codes, vals, rows, z1, z2, o1, o2);
    else
      k_spmv<F, 1><<<stream_grid(rows, 256), 256, 0, s>>>(indptr, cols, codes, vals, rows, z1, z1, o1, o1);
  }
  static void spmv_t(cudaStream_t s, const uint32_t* tptr, const uint32_t* trow, const uint32_t* tperm,
                     const int8_t* codes, const void* vals, size_t cols, size_t out_len, const void* rx,
                     void* out) {
    k_spmv_t<F><<<stream_grid(out_len, 256), 256, 0, s>>>(tptr, trow, tperm, codes, vals, cols, out_len, rx, out);
  }
  static void sc_round(cudaStream_t s, int kind, void* state, const void* res, const void* tau,
                       const void* tau_inv, const void* pending, uint32_t pending_len, int absorb_label,
                       int squeeze_label, void* out_poly, void* out_r) {
    k_sc_round<F><<<1, 32, 0, s>>>(kind, (sc_state*)state, res, tau, tau_inv, (const uint8_t*)pending,
                                   pending_len, (uint8_t)absorb_label, (uint8_t)squeeze_label, out_poly, out_r);
  }
  static void fe_inv_each(cudaStream_t s, const void* in, size_t n, void* out) {
    if (n) k_fe_inv_each<F><<<(unsigned)((n + 63) / 64), 64, 0, s>>>(in, n, out);
  }
  static void sc_round_batched(cudaStream_t s, const void* desc, void* state, const void* sums, const void* pending,
                               uint32_t pending_len, int absorb_label, int squeeze_label, void* out_poly, void* out_r) {
    k_sc_round_batched<F><<<1, 32, 0, s>>>(*(const scb_desc*)desc, (scb_state*)state, sums, (const uint8_t*)pending,
                                           pending_len, (uint8_t)absorb_label, (uint8_t)squeeze_label, out_poly, out_r);
  }
  static void eq_prefix_tables(cudaStream_t s, const void* taus, int hi, int K, void* out) {
    k_eq_prefix_tables<F><<<1, 1024, 0, s>>>(taus, hi, K, out);
  }
  static int sc_reduce_multi_partials(cudaStream_t s, const multi_args& a, void* scratch) {
    size_t need = (a.h + 255) / 256;
    unsigned gx = (unsigned)(need < (size_t)SC_MULTI_BLOCKS ? (need ? need : 1) : SC_MULTI_BLOCKS);
    static const bool occ3 = [] {
      const char* e = getenv("NOVA_B200_SC_MULTI_OCC");
      return e && e[0] == '3';
    }();
    if (occ3) k_form_reduce_multi<F, 3><<<dim3(gx, (unsigned)a.n), 256, 0, s>>>(a, scratch);
    else k_form_reduce_multi<F, 2><<<dim3(gx, (unsigned)a.n), 256, 0, s>>>(a, scratch);
    return (int)gx;
  }
  static void sc_round_batched_fused(cudaStream_t s, const void* desc, void* state, const void* partials, int nblocks,
                                     int nsums, const void* pending, uint32_t pending_len, int absorb_label,
                                     int squeeze_label, void* out_poly, void* out_r) {
    k_sc_round_batched_fused<F><<<1, 32 * nsums, 0, s>>>(*(const scb_desc*)desc, (scb_state*)state, partials, nblocks,
                                                       (const uint8_t*)pending, pending_len, (uint8_t)absorb_label,
                                                       (uint8_t)squeeze_label, out_poly, out_r);
  }
  static void poly_eval_small_multi(cudaStream_t s, const poly_multi_args& a, const void* us, int nu, void* evals) {
    if (nu == 1) k_poly_eval_small_multi<F, 1><<<a.k, 256, 0, s>>>(a, us, evals);
    else if (nu == 2) k_poly_eval_small_multi<F, 2><<<a.k, 256, 0, s>>>(a, us, evals);
    else k_poly_eval_small_multi<F, 3><<<a.k, 256, 0, s>>>(a, us, evals);
  }
  static void gather_heads(cudaStream_t s, void* const* zs, int k, void* out) {
    bind_multi_args a{};
    for (int i = 0; i < k; i++) a.z[i] = zs[i];
    k_gather_heads<F><<<1, BIND_MULTI_MAX, 0, s>>>(a, k, out);
  }
  static void sc_reduce_multi(cudaStream_t s, const multi_args& a, void* scratch, void* out) {
    size_t need = (a.h + 255) / 256;
    unsigned gx = (unsigned)(need < (size_t)SC_MULTI_BLOCKS ? (need ? need : 1) : SC_MULTI_BLOCKS);
    k_form_reduce_multi<F><<<dim3(gx, (unsigned)a.n), 256, 0, s>>>(a, scratch);
    k_form_final_multi<F><<<dim3(1, (unsigned)a.n), 256, 0, s>>>(scratch, (int)gx, out);
  }
  static void scb_tail(cudaStream_t s, const scb_tail_args& a, void* state, void* sums, const void* pending,
                       uint32_t pending_len, int absorb_label, int squeeze_label, void* polys, void* rs) {
    k_scb_tail<F><<<1, SCB_TAIL_THREADS, 0, s>>>(a, (scb_state*)state, sums, (const uint8_t*)pending, pending_len,
                                                (uint8_t)absorb_label, (uint8_t)squeeze_label, polys, rs);
  }
  static void on_curve(cudaStream_t s, const void* pts, size_t n, int b_small, uint32_t* first_bad) {
    if (n) k_on_curve<F><<<stream_grid(n, 256), 256, 0, s>>>(pts, n, b_small, first_bad);
  }
  static void powers_canonical(cudaStream_t s, const void* u, size_t n, void* out) {
    if (n) k_powers_canonical<F><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(u, n, out);
  }
  static void scalar_bases(cudaStream_t s, void* bases, size_t n, const void* gen, const void* scalars) {
    if (n) k_scalar_bases<F><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(bases, n, gen, scalars);
  }
  static void poseidon_ro(cudaStream_t s, int t, int r_f, int r_p, const void* rc, const void* mds, const void* elems,
                          uint32_t n, const void* tag, int num_bits, int start_with_one, void* out) {
    poseidon_desc d{t, r_f, r_p};
    k_poseidon_ro<F><<<1, 32 * t, 0, s>>>(d, rc, mds, elems, n, tag, num_bits, start_with_one, out);
  }
  static void to_mont(cudaStream_t s, const void* in, size_t n, void* out) {
    if (n) k_to_mont<F><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(in, n, out);
  }
  static void exchange_identity(cudaStream_t s, const msm_plan& p, void* out_jac) {
#if !defined(NOVA_MSM_ARITH29)
    k_red_final_q<F><<<1, 384, 0, s>>>(nullptr, 0, 4, 4, out_jac, p.peer);  // G = 0: the local partial is the identity
#endif
  }
  static void derive_check(cudaStream_t s, const void* tables, size_t n, const uint32_t* addr, size_t m,
                           size_t table_size, uint32_t* flags) {
    if (n) k_derive_check<F><<<stream_grid(n, 256), 256, 0, s>>>(tables, n, addr, m, table_size, flags);
  }
  static void derive_affine(cudaStream_t s, const uint32_t* start, uint32_t K, const void* buckets, void* out) {
    if (K) k_derive_affine<F><<<(unsigned)((K + 127) / 128), 128, 0, s>>>(start, K, buckets, out);
  }
  static void r1cs_eval(cudaStream_t s, const r1cs_mats& m, int k, const void* tx, const void* ty, void* scratch,
                        void* out) {
    size_t nnz = 0;
    for (int y = 0; y < k; y++) nnz = m.nnz[y] > nnz ? m.nnz[y] : nnz;
    const size_t want = (nnz + 256 * R1CS_MIN_CHUNK - 1) / (256 * R1CS_MIN_CHUNK);
    const unsigned gx = (unsigned)(want < 1 ? 1 : (want > R1CS_EVAL_BLOCKS ? R1CS_EVAL_BLOCKS : want));
    const size_t threads = (size_t)gx * 256, chunk = nnz ? (nnz + threads - 1) / threads : 1;
    k_r1cs_eval<F><<<dim3(gx, (unsigned)k), 256, 0, s>>>(m, tx, ty, chunk, scratch);
    k_r1cs_final<F><<<dim3(1, (unsigned)k), 256, 0, s>>>(scratch, (int)gx, out);
  }
  static void ipa_s(cudaStream_t s, const void* r, const void* r_inv, int L, const void* scale, void* scratch,
                    void* out) {
    if (L <= IPA_S_DIRECT_BITS) {
      k_ipa_s_half<F><<<(unsigned)((((size_t)1 << L) + 255) / 256), 256, 0, s>>>(r, r_inv, L, scale, out);
      return;
    }
    const int rb = L / 2, lb = L - rb;
    void* left = scratch;
    void* right = (char*)scratch + ((size_t)32 << lb);
    k_ipa_s_half<F><<<(unsigned)((((size_t)1 << lb) + 255) / 256), 256, 0, s>>>(r, r_inv, lb, scale, left);
    k_ipa_s_half<F><<<(unsigned)((((size_t)1 << rb) + 255) / 256), 256, 0, s>>>(
        (const char*)r + 32 * lb, (const char*)r_inv + 32 * lb, rb, nullptr, right);
    k_eq_outer<F><<<stream_grid((size_t)1 << L, 256), 256, 0, s>>>(left, right, rb, (size_t)1 << L, out);
  }
  static constexpr field_ops table() {
    return field_ops{F::ID,  digits,       expand_key, accumulate, fixup,   reduce,
                     sum_points, jacobian_sum, index_bases, cross_term, axpy,       vec_add, bind_top, bind_top_multi, vec_mul, logup_hash,
                     fold_halves, ipa_scalars, ipa_weights, fill_one,
                     sc_reduce, eq_small, eq_outer, batch_invert, rlc, kzg_fold, poly_eval, poly_div, spmv_classify, spmv, spmv_t,
                     sc_round, fe_inv_each, digits_range, sc_round_batched, on_curve,
                     powers_canonical, scalar_bases, poseidon_ro, to_mont, exchange_identity,
                     sc_round_batched_fused, sc_reduce_multi_partials, gather_heads, poly_eval_small_multi,
                     eq_prefix_tables, sc_reduce_multi, scb_tail, mat_vec_rows, mercury_s_poly,
                     neutron_evals, pow_split_evals, lerp, spark_repr, derive_check, derive_affine, r1cs_eval, ipa_s};
  }
};

}  // namespace nova
