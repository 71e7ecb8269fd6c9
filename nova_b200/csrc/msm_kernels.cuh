// Pippenger bucket MSM for sm_90a (K2/K3 of SURVEY.md §2).
//
// Replaces  src/provider/msm.rs:225-419 `msm` (+ the third-party
// halo2curves::msm::msm_best it delegates to at msm.rs:399-411,493-501) behind
// DlogGroupExt::vartime_multiscalar_mul (src/provider/traits.rs:77-117).
//
// Because a commitment key is fixed for the life of PublicParams (src/nova/mod.rs:55-58), the
// key is registered once and expanded into F tables  T_t[i] = 2^(c*G*t) * P_i  (affine).  A
// scalar's signed c-bit digit for window w = t*G + g then selects table t and bucket group g,
// so   sum_i s_i P_i = sum_g 2^(c g) * sum_b b * Bucket[g][b].   With F = W (full expansion)
// there is ONE bucket group and no serial doubling tail.
//
// Pipeline (all on one stream, no host sync):
//   k_digits      scalar (Montgomery) -> canonical -> sign-fold (s > p/2 => p-s, flip) ->
//                 signed c-bit digits; per-pass radix histograms of the bucket keys  [msm.rs:247-252 idea]
//   k_sort_pass   stable LSD radix sort of the (key, sign, table index) entries by key (msm_sort.cuh)
//   k_sort_starts bucket starts and the heavy-bucket list
//   k_accumulate  one thread per L consecutive sorted entries: XYZZ mixed adds
//                 (msm.rs:126-165); interior runs go straight to their bucket, the first/last
//                 run of a segment to a boundary-partial list
//   k_fixup       joins boundary partials of the same bucket (msm.rs:91-123 full add)
//   k_reduce1/2   sum_b b*Bucket[b] by chunked running sums (msm.rs:555-560 is the serial form),
//                 group Horner, XYZZ -> Jacobian
#pragma once
#include <cuda_runtime.h>
#include "curve29.cuh"
#include "coop.cuh"
#include "msm_sort.cuh"

namespace nova {

constexpr uint32_t KEY_INVALID = 0xffffffffu;

// Multi-GPU epilogue of the sharded MSM (SURVEY.md §8e "allreduce of partial sums"): every rank owns one
// exchange buffer that all peers can write over NVLink (CUDA IPC between processes, peer access inside one).
// Layout of a buffer:  slots[2][MSM_PEER_MAX] XYZZ (128 B each; the set is chosen by the epoch's parity), then
// flags[MSM_PEER_MAX] u64 (flag[r] = last epoch whose partial rank r has delivered), then one u64 error word.
constexpr int MSM_PEER_MAX = 8;
constexpr size_t MSM_PEER_FLAGS_OFF = (size_t)2 * MSM_PEER_MAX * 128;
constexpr size_t MSM_PEER_ERR_OFF = MSM_PEER_FLAGS_OFF + (size_t)MSM_PEER_MAX * 8;
constexpr size_t MSM_PEER_BUF_BYTES = MSM_PEER_ERR_OFF + 8;
struct msm_peer {
  int world = 1, rank = 0;
  unsigned long long epoch = 0;   // strictly increasing per call, the same on every rank
  void* buf[MSM_PEER_MAX] = {};   // buf[r] = rank r's exchange buffer as mapped in THIS process
};

struct msm_plan {
  // problem
  size_t n;            // scalars in this call
  size_t n_ck;         // points per table in the registered key
  size_t base_offset;  // first key point used
  size_t blind_i;      // scalar index whose base is the blinding generator h (SIZE_MAX: none)
  size_t h_index;      // position of h inside each table
  int c;               // window bits
  int W;               // number of windows = F*G
  int G;               // bucket groups
  uint32_t B;          // buckets per group = 2^(c-1)
  int L;               // entries per accumulate segment
  int m;               // buckets per reduce chunk
  // workspace (device)
  int32_t* digits;     // [W][n]
  uint32_t* sortctl;   // [SORT_CTL_WORDS]: per-pass radix histograms, then the per-pass tile counters
  sort_plan sp;        // radix passes over the keys [0, K), K = G*B
  uint32_t sort_tag;   // look-back tag of pass 0 (pass p uses sort_tag + p)
  unsigned long long* look;  // [ceil(n*W / SORT_TILE) * SORT_BINS] look-back words
  uint32_t* start;     // [K+1]
  uint64_t* entries;   // [n*W]   sorted by key
  uint64_t* entries_tmp;  // [n*W] the other buffer of the radix passes
  void* buckets;       // [K] xyzz
  void* parts;         // [2*nseg_max] xyzz
  uint32_t* pkeys;     // [2*nseg_max]
  void* rparts;        // [G*T] xyzz, T = B/m
  uint32_t* heavy;     // [0] = count, [1..] = keys whose bucket spans > heavy_min entries
  uint32_t heavy_min;  // entries; such buckets are joined by k_fixup_heavy1/2
  uint32_t heavy_cap;  // capacity of the heavy list
  void* hparts;        // [heavy_cap * HEAVY_SPLIT] xyzz: slice sums of the heavy buckets
  msm_peer peer;       // world > 1: the reduction's last kernel also exchanges and sums the ranks' partials
};

// ------------------------------------------------------------------------------------------
// digits + histogram   (templated on the SCALAR field)
// ------------------------------------------------------------------------------------------
// Processes scalars [i0, i1) of a vector of n (the digit array is [W][n]): a whole MSM passes
// (0, n); the streamed witness hand-off (b200_witness_append) passes each chunk as it arrives.
// Grid-stride over blocks of 256 scalars; the block's radix histograms are added to hist at the end.
template <class S>
__global__ void __launch_bounds__(256) k_digits(const void* __restrict__ scalars, size_t i0, size_t i1,
                                                size_t n, int c, int W, int G, uint32_t B,
                                                int32_t* __restrict__ digits,
                                                uint32_t* __restrict__ hist, const sort_plan sp) {
  __shared__ uint32_t s_hist[SORT_PASSES_MAX * SORT_BINS];
  sort_hist_clear(s_hist);
  for (size_t blk = i0 + (size_t)blockIdx.x * blockDim.x; blk < i1; blk += (size_t)gridDim.x * blockDim.x) {
    size_t i = blk + threadIdx.x;
    const bool live = i < i1;  // no early exit: the whole warp takes part in sort_hist_count
    fe_t s = live ? fe_from_mont<S>(fe_load(scalars, i)) : fe_zero<S>();
    // sign fold: use p - s when that is the smaller integer (msm.rs:1-8 "signed scalar
    // decomposition"); small negative witness values then cost one bucket add, not W.
    uint32_t p[8], t[8];
    load_p<S>(p);
    bool neg = false;
    if (!fe_is_zero(s)) {
      sub8(t, p, s.l);  // p - s, never borrows
      // compare t < s  <=> p - s < s
      uint32_t d[8];
      uint32_t lt = sub8(d, t, s.l);
      if (lt) {
        neg = true;
#pragma unroll
        for (int k = 0; k < 8; k++) s.l[k] = t[k];
      }
    }
    const uint32_t half = 1u << (c - 1);
    const uint32_t mask = (1u << c) - 1;
    uint32_t carry = 0;
    for (int w = 0; w < W; w++) {
      int bit = w * c;
      int limb = bit >> 5, sh = bit & 31;
      uint32_t v = 0;
      if (limb < 8) {
        uint64_t two = s.l[limb];
        if (limb + 1 < 8) two |= (uint64_t)s.l[limb + 1] << 32;
        v = (uint32_t)(two >> sh) & mask;
      }
      v += carry;
      int32_t dgt;
      if (v > half) {  // digits in [-(half-1), half]
        dgt = (int32_t)v - (int32_t)(1u << c);
        carry = 1;
      } else {
        dgt = (int32_t)v;
        carry = 0;
      }
      if (neg) dgt = -dgt;
      if (live) digits[(size_t)w * n + i] = dgt;
      uint32_t key = NO_KEY;
      if (dgt != 0) {
        uint32_t mag = dgt < 0 ? (uint32_t)(-dgt) : (uint32_t)dgt;
        key = (uint32_t)(w % G) * B + (mag - 1);
      }
      sort_hist_count(s_hist, key, sp);
    }
  }
  sort_hist_flush(s_hist, hist, sp);
}

// ------------------------------------------------------------------------------------------
// bucket accumulation   (templated on the BASE field)
// ------------------------------------------------------------------------------------------
template <class F>
__global__ void __launch_bounds__(128) k_accumulate(const uint64_t* __restrict__ entries,
                                                    const uint32_t* __restrict__ start, uint32_t K,
                                                    const void* __restrict__ tables, int L,
                                                    void* __restrict__ buckets,
                                                    void* __restrict__ parts,
                                                    uint32_t* __restrict__ pkeys) {
  using PA = msm_arith<F>;
  const uint32_t M = start[K];
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t seg_start = t * (size_t)L;
  if (seg_start >= M) return;
  size_t seg_end = seg_start + L < M ? seg_start + L : M;

  typename PA::pt acc = PA::identity();
  uint64_t ent = entries[seg_start];
  uint32_t cur_key = (uint32_t)(ent >> 32);
  bool first = true;
  typename PA::aff pt = PA::load_table(tables, (uint32_t)ent & 0x7fffffffu);
  for (size_t e = seg_start; e < seg_end; e++) {
    uint32_t key = (uint32_t)(ent >> 32);
    bool sign = (ent >> 31) & 1;
    typename PA::aff cur = pt;
    // prefetch the next entry's point while this one is being added
    if (e + 1 < seg_end) {
      ent = entries[e + 1];
      pt = PA::load_table(tables, (uint32_t)ent & 0x7fffffffu);
    }
    if (key != cur_key) {
      if (first) {
        PA::store(parts, 2 * t, acc);
        pkeys[2 * t] = cur_key;
        first = false;
      } else {
        PA::store(buckets, cur_key, acc);
      }
      acc = PA::identity();
      cur_key = key;
    }
    if (!PA::aff_is_identity(cur)) {  // identity bases are skipped (msm.rs:247)
      if (sign) PA::neg_aff(cur);
      PA::madd(acc, cur);
    }
  }
  if (first) {
    PA::store(parts, 2 * t, acc);
    pkeys[2 * t] = cur_key;
    pkeys[2 * t + 1] = KEY_INVALID;
  } else {
    PA::store(parts, 2 * t + 1, acc);
    pkeys[2 * t + 1] = cur_key;
  }
}

// ------------------------------------------------------------------------------------------
// The same accumulation with the gathered points STAGED IN SHARED MEMORY BY THE TMA UNIT
// (north_star: "TMA staging of bucket windows into shared memory").  Every lane owns one 64-byte
// slot per pipeline stage; it issues `cp.async.bulk.shared.global` (1-D bulk copy, 64 B, 16-B
// aligned on both sides) for the table point of entry k + ACC_TMA_DEPTH - 1 while it adds entry
// k, and the copies of one warp and stage complete on one mbarrier (expect_tx = 64 B x issuing
// lanes, one arrival by the elected lane).  The point then comes from shared memory (4 x
// LDS.128) instead of living in 16 registers across the previous addition.
// Stage reuse needs no "empty" barrier: a lane refills slot (k + D - 1) % D only after the
// addition of entry k - 1 -- the last reader of that slot -- has issued, and a lane reads and
// writes only its own slots.
// Run-time A/B against k_accumulate: NOVA_B200_ACC_TMA=1 (ops_impl.cuh); DESIGN.md §4 has the
// measured verdict.
// ------------------------------------------------------------------------------------------
constexpr int ACC_TMA_DEPTH = 3;
#if defined(__CUDACC__) && !defined(NOVA_MSM_ARITH29)
NOVA_D uint32_t smem_addr_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
NOVA_D void mbar_init(uint64_t* bar, uint32_t arrivals) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr_u32(bar)), "r"(arrivals) : "memory");
}
NOVA_D void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr_u32(bar)), "r"(bytes)
               : "memory");
}
NOVA_D void mbar_wait_parity(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "MBAR_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra MBAR_DONE;\n"
      "bra MBAR_WAIT;\n"
      "MBAR_DONE:\n"
      "}\n" ::"r"(smem_addr_u32(bar)),
      "r"(parity)
      : "memory");
}
// 1-D bulk copy global -> shared through the TMA unit; completion is signalled on `bar` (complete_tx)
NOVA_D void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_addr_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_addr_u32(bar))
               : "memory");
}

template <class F>
__global__ void __launch_bounds__(128) k_accumulate_tma(const uint64_t* __restrict__ entries,
                                                        const uint32_t* __restrict__ start, uint32_t K,
                                                        const void* __restrict__ tables, int L,
                                                        void* __restrict__ buckets, void* __restrict__ parts,
                                                        uint32_t* __restrict__ pkeys) {
  using PA = msm_arith<F>;
  static_assert(sizeof(typename PA::aff) == 64, "one table point = one 64-byte bulk copy");
  __shared__ __align__(128) uint4 slots[ACC_TMA_DEPTH][128][4];  // [stage][thread][64 B]
  __shared__ __align__(8) uint64_t bars[4][ACC_TMA_DEPTH];       // [warp][stage]
  const uint32_t M = start[K];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0)
    for (int st = 0; st < ACC_TMA_DEPTH; st++) mbar_init(&bars[warp][st], 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncwarp();
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t seg_start = t * (size_t)L;
  const bool active = seg_start < M;
  size_t seg_end = seg_start + L < M ? seg_start + L : M;
  const int len = active ? (int)(seg_end - seg_start) : 0;
  // trip count of the warp = its longest segment (all lanes run the barrier protocol together)
  int wlen = len;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    int o = __shfl_xor_sync(0xffffffffu, wlen, d);
    wlen = o > wlen ? o : wlen;
  }
  if (wlen == 0) return;

  // issue the copy of entry j (if this lane has one) into stage j % D; returns the entry
  auto issue = [&](int j) -> uint64_t {
    const bool mine = j < len;
    uint64_t ent = mine ? entries[seg_start + j] : 0;
    const int st = j % ACC_TMA_DEPTH;  // (callers pass consecutive j: strength-reduced by the compiler)
    unsigned who = __ballot_sync(0xffffffffu, mine);
    if (who) {
      if (lane == (int)(__ffs(who) - 1)) mbar_arrive_expect_tx(&bars[warp][st], 64u * (uint32_t)__popc(who));
      __syncwarp();
      if (mine)
        tma_load_1d(&slots[st][threadIdx.x][0],
                    (const char*)tables + (size_t)((uint32_t)ent & 0x7fffffffu) * 64, 64, &bars[warp][st]);
    }
    return ent;
  };

  // entries in flight (key | sign | table index), oldest first; rotated by register moves so that the
  // loop body -- one inlined mixed addition, ~37 KB of code -- exists once
  static_assert(ACC_TMA_DEPTH == 3, "the rotation below is written for three stages");
  uint64_t e0 = issue(0), e1 = issue(1);

  typename PA::pt acc = PA::identity();
  uint32_t cur_key = active ? (uint32_t)(e0 >> 32) : 0;
  bool first = true;
  int st = 0;  // k % ACC_TMA_DEPTH
  uint32_t phase = 0;  // (k / ACC_TMA_DEPTH) & 1
#pragma unroll 1
  for (int k = 0; k < wlen; k++) {
    const uint64_t e2 = issue(k + 2);  // refills the stage that entry k - 1 used
    // a stage is armed only if some lane had an entry for it: the ballot is warp-uniform
    if (__ballot_sync(0xffffffffu, k < len)) mbar_wait_parity(&bars[warp][st], phase);
    if (k < len) {
      const uint64_t ent = e0;
      const uint32_t key = (uint32_t)(ent >> 32);
      const bool sign = (ent >> 31) & 1;
      typename PA::aff cur;
      {
        const uint4* sp = &slots[st][threadIdx.x][0];
        uint4 a = sp[0], b = sp[1], c = sp[2], d = sp[3];
        cur.x.l[0] = a.x; cur.x.l[1] = a.y; cur.x.l[2] = a.z; cur.x.l[3] = a.w;
        cur.x.l[4] = b.x; cur.x.l[5] = b.y; cur.x.l[6] = b.z; cur.x.l[7] = b.w;
        cur.y.l[0] = c.x; cur.y.l[1] = c.y; cur.y.l[2] = c.z; cur.y.l[3] = c.w;
        cur.y.l[4] = d.x; cur.y.l[5] = d.y; cur.y.l[6] = d.z; cur.y.l[7] = d.w;
      }
      if (key != cur_key) {
        if (first) {
          PA::store(parts, 2 * t, acc);
          pkeys[2 * t] = cur_key;
          first = false;
        } else {
          PA::store(buckets, cur_key, acc);
        }
        acc = PA::identity();
        cur_key = key;
      }
      if (!PA::aff_is_identity(cur)) {  // identity bases are skipped (msm.rs:247)
        if (sign) PA::neg_aff(cur);
        PA::madd(acc, cur);
      }
    }
    e0 = e1;
    e1 = e2;
    if (++st == ACC_TMA_DEPTH) {
      st = 0;
      phase ^= 1u;
    }
  }
  if (!active) return;
  if (first) {
    PA::store(parts, 2 * t, acc);
    pkeys[2 * t] = cur_key;
    pkeys[2 * t + 1] = KEY_INVALID;
  } else {
    PA::store(parts, 2 * t + 1, acc);
    pkeys[2 * t + 1] = cur_key;
  }
}
#endif  // __CUDACC__ && !NOVA_MSM_ARITH29

// G threads per bucket key (G a power of two <= 32, chosen by the host from the expected number of
// partials per bucket): join the boundary partials of that bucket.  The bucket's entries span
// segments t0..t1, so its partials can only sit in slots 2*t0 .. 2*t1+1; the G lanes stride over
// that range and combine with a shuffle tree.  A bucket whose entries are interior to one segment
// finds no matching slot (it was stored directly by k_accumulate); buckets above heavy_min are
// left to k_fixup_heavy1/2.
template <class F>
__global__ void __launch_bounds__(128) k_fixup(const uint32_t* __restrict__ start, uint32_t K,
                                               int L, uint32_t heavy_min, int G,
                                               const void* __restrict__ parts,
                                               const uint32_t* __restrict__ pkeys,
                                               void* __restrict__ buckets) {
  using PA = msm_arith<F>;
  uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t key = gtid / G, sub = gtid % G;
  bool live = key < K;
  uint32_t s0 = 0, s1 = 0;
  if (live) {
    s0 = start[key];
    s1 = start[key + 1];
    live = s1 != s0 && s1 - s0 <= heavy_min;
  }
  typename PA::pt acc = PA::identity();
  bool found = false;
  if (live) {
    size_t j0 = 2 * ((size_t)s0 / L), j1 = 2 * (((size_t)s1 - 1) / L) + 1;
    for (size_t j = j0 + sub; j <= j1; j += G) {
      if (pkeys[j] == key) {
        typename PA::pt o = PA::load(parts, j);
        PA::add(acc, o);
        found = true;
      }
    }
  }
  // all 32 lanes take part in the shuffles (groups are aligned sub-warps)
  for (int d = G / 2; d > 0; d >>= 1) {
    typename PA::pt o = PA::shfl_down(acc, d, G);
    bool of = __shfl_down_sync(0xffffffffu, (int)found, d, G) != 0;
    if (sub + d < (uint32_t)G && of) {
      PA::add(acc, o);
      found = true;
    }
  }
  if (live && sub == 0 && found) PA::store(buckets, key, acc);
}

// Heavy buckets (skewed scalars: 0/1 witnesses, padding, one value repeated a million times) hold
// thousands of boundary partials.  Stage 1 gives each heavy bucket HEAVY_SPLIT blocks: the threads
// stride over one slice of the bucket's partial slots and tree-sum through shared memory into
// hparts[h][slice]; stage 2 joins the HEAVY_SPLIT slice sums with a shuffle tree.  A lone warp
// needs ~9 us per XYZZ addition, so the point is the length of the dependent chain: 16 K partials
// are 4 strided adds + 8 tree levels + 4 join levels instead of 64 + 8.
constexpr int HEAVY_SPLIT = 16;
template <class F>
__global__ void __launch_bounds__(256) k_fixup_heavy1(const uint32_t* __restrict__ start, int L,
                                                      const uint32_t* __restrict__ heavy,
                                                      const void* __restrict__ parts,
                                                      const uint32_t* __restrict__ pkeys,
                                                      void* __restrict__ hparts) {
  using PA = msm_arith<F>;
  __shared__ typename msm_arith<F>::pt sm[256];
  const uint32_t nitems = heavy[0] * HEAVY_SPLIT;
  for (uint32_t it = blockIdx.x; it < nitems; it += gridDim.x) {
    uint32_t h = it / HEAVY_SPLIT, sl = it % HEAVY_SPLIT;
    uint32_t key = heavy[1 + h];
    size_t s0 = 2 * ((size_t)start[key] / L);
    size_t s1 = 2 * (((size_t)start[key + 1] - 1) / L) + 2;  // one past the last slot
    size_t per = (s1 - s0 + HEAVY_SPLIT - 1) / HEAVY_SPLIT;
    size_t lo = s0 + sl * per, hi = lo + per < s1 ? lo + per : s1;
    typename PA::pt acc = PA::identity();
    for (size_t k = lo + threadIdx.x; k < hi; k += blockDim.x) {
      if (pkeys[k] == key) {
        typename PA::pt o = PA::load(parts, k);
        PA::add(acc, o);
      }
    }
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
      if ((int)threadIdx.x < s) {
        typename PA::pt a = sm[threadIdx.x];
        PA::add(a, sm[threadIdx.x + s]);
        sm[threadIdx.x] = a;
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) PA::store(hparts, it, sm[0]);
    __syncthreads();
  }
}

template <class F>
__global__ void __launch_bounds__(32) k_fixup_heavy2(const uint32_t* __restrict__ heavy,
                                                     const void* __restrict__ hparts,
                                                     void* __restrict__ buckets) {
  using PA = msm_arith<F>;
  static_assert(HEAVY_SPLIT <= 32 && (HEAVY_SPLIT & (HEAVY_SPLIT - 1)) == 0, "one warp joins the slices");
  const uint32_t nheavy = heavy[0];
  for (uint32_t h = blockIdx.x; h < nheavy; h += gridDim.x) {
    typename PA::pt acc = PA::identity();
    if (threadIdx.x < HEAVY_SPLIT) acc = PA::load(hparts, (size_t)h * HEAVY_SPLIT + threadIdx.x);
    for (int d = HEAVY_SPLIT / 2; d > 0; d >>= 1) {
      typename PA::pt o = PA::shfl_down(acc, d, 32);
      if ((int)threadIdx.x < d) PA::add(acc, o);
    }
    if (threadIdx.x == 0) PA::store(buckets, heavy[1 + h], acc);
  }
}

// ------------------------------------------------------------------------------------------
// bucket reduction
// ------------------------------------------------------------------------------------------
// thread (g, k): chunk of m buckets [k*m, (k+1)*m) of group g ->
//   rparts[g*T + k] = sum_{b in chunk} (b+1) * Bucket[g][b]
template <class F>
__global__ void __launch_bounds__(128) k_reduce1(const uint32_t* __restrict__ start, uint32_t B,
                                                 int G, int m, const void* __restrict__ buckets,
                                                 void* __restrict__ rparts) {
  using PA = msm_arith<F>;
  uint32_t T = B / m;
  uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= T * (uint32_t)G) return;
  uint32_t g = tid / T, k = tid % T;
  uint32_t lo = k * m;
  typename PA::pt run = PA::identity(), tot = PA::identity();
  for (int b = m - 1; b >= 0; b--) {
    uint32_t key = g * B + lo + b;
    if (start[key + 1] > start[key]) {
      typename PA::pt bk = PA::load(buckets, key);
      PA::add(run, bk);
    }
    PA::add(tot, run);
  }
  if (lo != 0) {
    typename PA::pt sc = PA::mul_small(run, lo);
    PA::add(tot, sc);
  }
  PA::store(rparts, tid, tot);
}

// single block: per group tree-sum of T partials, Horner over groups (c doublings each),
// plus an optional extra XYZZ addend, then Jacobian out (3 x fe_t).
template <class F>
__global__ void __launch_bounds__(256) k_reduce2(const void* __restrict__ rparts, uint32_t T, int G,
                                                 int c, void* __restrict__ out_jac) {
  using PA = msm_arith<F>;
  __shared__ typename msm_arith<F>::pt sm[256];
  typename PA::pt total = PA::identity();
  for (int g = G - 1; g >= 0; g--) {
    typename PA::pt acc = PA::identity();
    for (uint32_t k = threadIdx.x; k < T; k += blockDim.x) {
      typename PA::pt o = PA::load(rparts, (size_t)g * T + k);
      PA::add(acc, o);
    }
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
      if ((int)threadIdx.x < s) {
        typename PA::pt a = sm[threadIdx.x];
        PA::add(a, sm[threadIdx.x + s]);
        sm[threadIdx.x] = a;
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      if (g != G - 1)
        for (int d = 0; d < c; d++) PA::dbl(total);
      PA::add(total, sm[0]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    fe_t X, Y, Z;
    PA::to_jacobian_std(total, X, Y, Z);
    fe_store(out_jac, 0, X);
    fe_store(out_jac, 1, Y);
    fe_store(out_jac, 2, Z);
  }
}

// ------------------------------------------------------------------------------------------
// Radix-16 digit-sum bucket reduction.  Write the bucket index b in base 16, b = sum_d 16^d v_d:
//     sum_b (b+1) B_b  =  S_all  +  sum_d 16^d  sum_{v=1}^{15} v * S_d[v],
//     S_d[v] = sum of the buckets whose digit d equals v,   S_all = sum_b B_b = sum_v S_d[v].
// k_red_digits computes the (at most 6 x 16) digit sums with plain tree sums spread over the whole
// GPU (every bucket is read once per digit position); k_red_final turns each 16-entry array into
// its weighted sum with a shuffle suffix-scan (sum_v v S_v = sum_{j>=1} sum_{v>=j} S_v), scales by
// 16^d with 4d doublings in parallel across digit positions, and adds up.  No scalar
// multiplications, no long serial running sums: ~25 dependent point operations in total, each
// executed with at most a few warps per SM (a lone warp needs ~4 us per point addition because one
// field product occupies the integer-multiply pipe for ~550 cycles).
// ------------------------------------------------------------------------------------------
constexpr int RED_NSPLIT = 4;
template <class F>
__global__ void __launch_bounds__(128) k_red_digits(const uint32_t* __restrict__ start, uint32_t B,
                                                    int bits, const void* __restrict__ buckets,
                                                    void* __restrict__ parts /* [G][nd][16][NSPLIT] */) {
  using PA = msm_arith<F>;
  __shared__ typename PA::pt sm[128];
  const int nd = (bits + 3) / 4;
  const int x = blockIdx.x, d = blockIdx.y / 16, v = blockIdx.y % 16, g = blockIdx.z;
  const int width = bits - 4 * d < 4 ? bits - 4 * d : 4;
  typename PA::pt acc = PA::identity();
  if (v < (1 << width)) {
    const uint32_t count = B >> width;  // buckets whose digit d equals v
    const uint32_t per = (count + RED_NSPLIT - 1) / RED_NSPLIT;
    const uint32_t lo = x * per, hi = lo + per < count ? lo + per : count;
    const uint32_t lowmask = (1u << (4 * d)) - 1;
    for (uint32_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
      uint32_t b = ((i >> (4 * d)) << (4 * d + width)) | ((uint32_t)v << (4 * d)) | (i & lowmask);
      uint32_t key = g * B + b;
      if (start[key + 1] > start[key]) {
        typename PA::pt o = PA::load(buckets, key);
        PA::add(acc, o);
      }
    }
  }
  sm[threadIdx.x] = acc;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) {
      typename PA::pt a = sm[threadIdx.x];
      PA::add(a, sm[threadIdx.x + s]);
      sm[threadIdx.x] = a;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) PA::store(parts, (((size_t)g * nd + d) * 16 + v) * RED_NSPLIT + x, sm[0]);
}

// one block, 32 threads per digit position (16 active lanes each)
template <class F>
__global__ void __launch_bounds__(256) k_red_final(const void* __restrict__ parts, int G, int bits, int c,
                                                   void* __restrict__ out_jac) {
  using PA = msm_arith<F>;
  __shared__ typename PA::pt sm[8];
  const int nd = (bits + 3) / 4;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  typename PA::pt total = PA::identity();
  for (int g = G - 1; g >= 0; g--) {
    typename PA::pt S = PA::identity();
    if (w < nd && lane < 16)
      for (int x = 0; x < RED_NSPLIT; x++) {
        typename PA::pt o = PA::load(parts, (((size_t)g * nd + w) * 16 + lane) * RED_NSPLIT + x);
        PA::add(S, o);
      }
    // suffix scan over the 16 digit values: T_v = sum_{k >= v} S_k
    for (int d = 1; d < 16; d <<= 1) {
      typename PA::pt o = PA::shfl_down(S, d, 16);
      if (lane < 16 && lane + d < 16) PA::add(S, o);
    }
    // weighted sum  sum_{v>=1} T_v  (lane 0 keeps T_0 = S_all aside)
    typename PA::pt T0 = S;
    typename PA::pt X = (lane >= 1 && lane < 16) ? S : PA::identity();
    for (int d = 8; d > 0; d >>= 1) {
      typename PA::pt o = PA::shfl_down(X, d, 16);
      if (lane < 16 && lane + d < 16) PA::add(X, o);
    }
    if (lane == 0 && w < nd) {
      for (int k = 0; k < 4 * w; k++) PA::dbl(X);  // * 16^w
      if (w == 0) PA::add(X, T0);                   // + S_all
      sm[w] = X;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      if (g != G - 1)
        for (int k = 0; k < c; k++) PA::dbl(total);
      for (int k = 0; k < nd; k++) PA::add(total, sm[k]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    fe_t X, Y, Z;
    PA::to_jacobian_std(total, X, Y, Z);
    fe_store(out_jac, 0, X);
    fe_store(out_jac, 1, Y);
    fe_store(out_jac, 2, Z);
  }
}

// ------------------------------------------------------------------------------------------
// Quad-cooperative versions of the latency-bound tail (coop.cuh): four lanes share every point
// operation.  Used with the default 8x32-bit arithmetic (pa32); same mathematics as k_fixup /
// k_red_digits / k_red_final above.
// ------------------------------------------------------------------------------------------
#if !defined(NOVA_MSM_ARITH29)
NOVA_D xyzz_t xyzz_load_q(const void* base, size_t idx) { return xyzz_load(base, idx); }

// one quad per bucket key: serial cooperative adds over the key's boundary partials
template <class F>
__global__ void __launch_bounds__(128) k_fixup_q(const uint32_t* __restrict__ start, uint32_t K, int L,
                                                 uint32_t heavy_min, const void* __restrict__ parts,
                                                 const uint32_t* __restrict__ pkeys,
                                                 void* __restrict__ buckets) {
  quad_comm_dev cm;
  uint32_t key = (blockIdx.x * blockDim.x + threadIdx.x) >> 2;
  bool live = key < K;
  uint32_t s0 = 0, s1 = 0;
  if (live) {
    s0 = start[key];
    s1 = start[key + 1];
    live = s1 != s0 && s1 - s0 <= heavy_min;
  }
  // all lanes of the warp stay in the loop structure; quads whose key is dead add nothing
  size_t j0 = live ? 2 * ((size_t)s0 / L) : 1, j1 = live ? 2 * (((size_t)s1 - 1) / L) + 1 : 0;
  xyzz_t acc = xyzz_identity<F>();
  bool found = false;
  for (size_t j = j0; j <= j1; j++) {
    if (pkeys[j] == key) {  // uniform within the quad
      xyzz_t o = xyzz_load(parts, j);
      coop_add<F>(acc, o, cm);
      found = true;
    }
  }
  if (live && found && cm.lane() == 0) xyzz_store(buckets, key, acc);
}

// Stage 1: block (x, d*16+v, g), 64 quads, sums its slice of the buckets whose digit d equals v.
// nsplit = gridDim.x is chosen by the host so that a quad adds ~4 buckets before the tree.
template <class F>
__global__ void __launch_bounds__(256) k_red_digits_q(const uint32_t* __restrict__ start, uint32_t B,
                                                      int bits, const void* __restrict__ buckets,
                                                      void* __restrict__ parts /* [G][nd][16][nsplit] */) {
  __shared__ xyzz_t sm[64];
  quad_comm_dev cm;
  const int nd = (bits + 3) / 4;
  const int nsplit = gridDim.x;
  const int x = blockIdx.x, d = blockIdx.y / 16, v = blockIdx.y % 16, g = blockIdx.z;
  const int width = bits - 4 * d < 4 ? bits - 4 * d : 4;
  const int quad = threadIdx.x >> 2;
  xyzz_t acc = xyzz_identity<F>();
  if (v < (1 << width)) {
    const uint32_t count = B >> width;
    const uint32_t per = (count + nsplit - 1) / nsplit;
    const uint32_t lo = x * per, hi = lo + per < count ? lo + per : count;
    const uint32_t lowmask = (1u << (4 * d)) - 1;
    for (uint32_t i = lo + quad; i < hi; i += 64) {
      uint32_t b = ((i >> (4 * d)) << (4 * d + width)) | ((uint32_t)v << (4 * d)) | (i & lowmask);
      uint32_t key = g * B + b;
      if (start[key + 1] > start[key]) {  // uniform within the quad
        xyzz_t o = xyzz_load(buckets, key);
        coop_add<F>(acc, o, cm);
      }
    }
  }
  if (cm.lane() == 0) sm[quad] = acc;
  __syncthreads();
  for (int s = 32; s > 0; s >>= 1) {
    if (quad < s) {
      xyzz_t o = sm[quad + s];
      coop_add<F>(acc, o, cm);
    }
    __syncthreads();
    if (quad < s && cm.lane() == 0) sm[quad] = acc;
    __syncthreads();
  }
  if (threadIdx.x == 0) xyzz_store(parts, (((size_t)g * nd + d) * 16 + v) * nsplit + x, acc);
}

// Stage 2: block (d*16+v, g) tree-sums the nsplit partials of one digit value -> merged[g][d][v]
template <class F>
__global__ void __launch_bounds__(256) k_red_merge_q(const void* __restrict__ parts, int nd, int nsplit,
                                                     void* __restrict__ merged) {
  __shared__ xyzz_t sm[64];
  quad_comm_dev cm;
  const int dv = blockIdx.x, g = blockIdx.y;
  const int quad = threadIdx.x >> 2;
  const size_t base = ((size_t)g * nd * 16 + dv) * nsplit;
  xyzz_t acc = xyzz_identity<F>();
  for (int x = quad; x < nsplit; x += 64) {
    xyzz_t o = xyzz_load(parts, base + x);
    coop_add<F>(acc, o, cm);
  }
  if (cm.lane() == 0) sm[quad] = acc;
  __syncthreads();
  for (int s = 32; s > 0; s >>= 1) {
    if (quad < s && s < nsplit) {  // uniform per block level: skip levels beyond the partial count
      xyzz_t o = sm[quad + s];
      coop_add<F>(acc, o, cm);
    }
    __syncthreads();
    if (quad < s && cm.lane() == 0) sm[quad] = acc;
    __syncthreads();
  }
  if (threadIdx.x == 0) xyzz_store(merged, (size_t)g * nd * 16 + dv, acc);
}

// ------------------------------------------------------------------------------------------
// Hierarchical form of the radix-16 digit sums (default; the flat k_red_digits_q above reads every
// bucket once per digit position = nd additions per bucket, this one does 2 + 2/16 + ...):
//   level l works on X^(l) (X^(0) = the buckets, N_l = 2^(bits - 4 l) points) and produces
//     pass A   S_l[v]   = sum_j X^(l)[16 j + v]           (the digit sums of position l)
//     pass B   X^(l+1)[j] = sum_v X^(l)[16 j + v]          (the input of the next level)
//   the top level (N <= 16) IS its own digit-sum array.
// sum_b (b+1) B_b = S_all + sum_l 16^l sum_v v S_l[v]  as before (k_red_final_q is unchanged).
// One launch per level: blockIdx.y < 16 -> pass A for digit value v = blockIdx.y (blockIdx.x = slice of the
// groups, 64 quads stride over it and tree-sum), blockIdx.y == 16 -> pass B (four quads per group: 3 serial
// cooperative additions each, then a 2-level tree), blockIdx.z = bucket group.
// ------------------------------------------------------------------------------------------
template <class F>
__global__ void __launch_bounds__(256) k_red_level_q(const uint32_t* __restrict__ start_or_null, uint32_t key_base_stride,
                                                     const void* __restrict__ X, uint32_t N, int nsplit,
                                                     void* __restrict__ parts /* [G][16][nsplit] */,
                                                     void* __restrict__ next /* [G][N/16] */) {
  __shared__ xyzz_t sm[64];
  quad_comm_dev cm;
  const int quad = threadIdx.x >> 2;
  const uint32_t g = blockIdx.z;
  const uint32_t groups = N >> 4;
  const size_t xbase = (size_t)g * N;
  // level 0 reads the bucket array, where an empty bucket holds stale data: its emptiness comes from the offsets
  auto load = [&](uint32_t i) -> xyzz_t {
    if (start_or_null) {
      const uint32_t key = g * key_base_stride + i;
      if (start_or_null[key + 1] == start_or_null[key]) return xyzz_identity<F>();
    }
    return xyzz_load(X, xbase + i);
  };
  if (blockIdx.y == 16) {  // pass B: group sums, four quads per group (3 serial additions each, then a 2-level tree)
    const uint32_t j = blockIdx.x * 16 + (quad >> 2);
    const int sub = quad & 3;
    const bool live = j < groups;  // uniform within a quad
    xyzz_t acc = xyzz_identity<F>();
    if (live) {
      acc = load(16 * j + 4 * sub);
      for (int k = 1; k < 4; k++) {
        xyzz_t o = load(16 * j + 4 * sub + k);
        coop_add<F>(acc, o, cm);
      }
    }
    if (cm.lane() == 0) sm[quad] = acc;
    __syncthreads();
    if (live && sub < 2) {
      xyzz_t o = sm[quad + 2];
      coop_add<F>(acc, o, cm);
    }
    __syncthreads();
    if (sub < 2 && cm.lane() == 0) sm[quad] = acc;
    __syncthreads();
    if (live && sub == 0) {
      xyzz_t o = sm[quad + 1];
      coop_add<F>(acc, o, cm);
      if (cm.lane() == 0) xyzz_store(next, (size_t)g * groups + j, acc);
    }
    return;
  }
  if ((int)blockIdx.x >= nsplit) return;
  const uint32_t v = blockIdx.y;
  const uint32_t per = (groups + nsplit - 1) / nsplit;
  const uint32_t lo = blockIdx.x * per, hi = lo + per < groups ? lo + per : groups;
  xyzz_t acc = xyzz_identity<F>();
  for (uint32_t j = lo + quad; j < hi; j += 64) {
    xyzz_t o = load(16 * j + v);
    coop_add<F>(acc, o, cm);
  }
  if (cm.lane() == 0) sm[quad] = acc;
  __syncthreads();
  for (int s = 32; s > 0; s >>= 1) {
    if (quad < s) {
      xyzz_t o = sm[quad + s];
      coop_add<F>(acc, o, cm);
    }
    __syncthreads();
    if (quad < s && cm.lane() == 0) sm[quad] = acc;
    __syncthreads();
  }
  if (threadIdx.x == 0) xyzz_store(parts, ((size_t)g * 16 + v) * nsplit + blockIdx.x, acc);
}

// merged[g][d][v] for all digit positions: d < nd - 1 -> tree sum of level d's nsplit[d] partials; d = nd - 1 (the top
// level, N_top <= 16 points) -> the point itself.  Block (d * 16 + v, g).
struct red_levels {
  int nd;
  int nsplit[8];          // per level (unused for the top level)
  unsigned parts_off[8];  // offset (in points) of level d's parts inside the scratch area
  unsigned top_off;       // offset of X^(nd-1) (dense), or 0xFFFFFFFF when the top level is level 0 (= the buckets)
  unsigned top_n;         // N of the top level
};
template <class F>
__global__ void __launch_bounds__(256) k_red_merge_levels_q(const void* __restrict__ scratch, const red_levels lv,
                                                            const uint32_t* __restrict__ start, uint32_t B,
                                                            const void* __restrict__ buckets, int G,
                                                            void* __restrict__ merged) {
  __shared__ xyzz_t sm[64];
  quad_comm_dev cm;
  const int d = blockIdx.x >> 4, v = blockIdx.x & 15, g = blockIdx.y;
  const int quad = threadIdx.x >> 2;
  xyzz_t acc = xyzz_identity<F>();
  if (d == lv.nd - 1) {
    if (threadIdx.x == 0) {
      if ((unsigned)v < lv.top_n) {
        if (lv.top_off == 0xFFFFFFFFu) {
          uint32_t key = (uint32_t)g * B + v;
          if (start[key + 1] > start[key]) acc = xyzz_load(buckets, key);
        } else {
          acc = xyzz_load(scratch, (size_t)lv.top_off + (size_t)g * lv.top_n + v);
        }
      }
      xyzz_store(merged, ((size_t)g * lv.nd + d) * 16 + v, acc);
    }
    return;
  }
  const int nsplit = lv.nsplit[d];
  const size_t base = (size_t)lv.parts_off[d] + ((size_t)g * 16 + v) * nsplit;
  for (int x = quad; x < nsplit; x += 64) {
    xyzz_t o = xyzz_load(scratch, base + x);
    coop_add<F>(acc, o, cm);
  }
  if (cm.lane() == 0) sm[quad] = acc;
  __syncthreads();
  for (int s = 32; s > 0; s >>= 1) {
    if (quad < s && s < nsplit) {
      xyzz_t o = sm[quad + s];
      coop_add<F>(acc, o, cm);
    }
    __syncthreads();
    if (quad < s && cm.lane() == 0) sm[quad] = acc;
    __syncthreads();
  }
  if (threadIdx.x == 0) xyzz_store(merged, ((size_t)g * lv.nd + d) * 16 + v, acc);
}

// Fused compute + collective epilogue of the sharded MSM.  Called by the whole (single) block of
// k_red_final_q with quad 0 holding this rank's partial sum:
//   publish  lanes r < world store the partial into rank r's slot[epoch & 1][rank] (peer stores over NVLink for
//            r != rank), fence at system scope, then set rank r's flag[rank] = epoch
//   wait     lane r spins (acquire, system scope) until the LOCAL flag[r] reaches the epoch
//   sum      quad q < world loads slot q from the local buffer; a fixed binary tree of cooperative additions over
//            the ranks gives every rank bit-identical coordinates
// No NCCL call and no extra launch on the critical path.  Two slot sets suffice: a peer can only deliver epoch
// e + 2 after it has seen this rank's epoch e + 1, which this rank publishes after it finished summing epoch e.
// A peer that never delivers trips the bounded spin: the error word is set (b200 reports B200_E_PEER at the next
// host read) instead of hanging the GPU.
template <class F>
NOVA_D xyzz_t peer_exchange_sum(const xyzz_t& mine, const msm_peer& peer, xyzz_t* sm /* >= MSM_PEER_MAX */,
                                const quad_comm_dev& cm) {
  const int tid = threadIdx.x, quad = tid >> 2;
  const int set = (int)(peer.epoch & 1ull);
  if (tid == 0) sm[0] = mine;
  __syncthreads();
  if (tid < peer.world) {
    char* dst = (char*)peer.buf[tid];
    xyzz_store(dst, (size_t)set * MSM_PEER_MAX + peer.rank, sm[0]);
    __threadfence_system();
    volatile unsigned long long* flag = (volatile unsigned long long*)(dst + MSM_PEER_FLAGS_OFF) + peer.rank;
    *flag = peer.epoch;
    // wait for rank `tid`'s partial in the local buffer
    char* loc = (char*)peer.buf[peer.rank];
    const unsigned long long* lflag = (const unsigned long long*)(loc + MSM_PEER_FLAGS_OFF) + tid;
    unsigned long long seen = 0;
    long long t0 = clock64();
    for (;;) {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(lflag) : "memory");
      if (seen >= peer.epoch) break;
      if (clock64() - t0 > (1ll << 32)) {  // ~2 s at 1.9 GHz
        *(volatile unsigned long long*)(loc + MSM_PEER_ERR_OFF) = peer.epoch;
        break;
      }
    }
  }
  __syncthreads();
  xyzz_t acc = xyzz_identity<F>();
  if (quad < peer.world) acc = xyzz_load((const char*)peer.buf[peer.rank], (size_t)set * MSM_PEER_MAX + quad);
  for (int s = MSM_PEER_MAX / 2; s > 0; s >>= 1) {
    if (quad < 2 * s && cm.lane() == 0) sm[quad] = acc;
    __syncthreads();
    if (quad < s && quad + s < peer.world) {
      xyzz_t o = sm[quad + s];
      coop_add<F>(acc, o, cm);
    }
    __syncthreads();
  }
  return acc;  // quad 0 holds the total
}

// Stage 3: one block, one quad per (d, v), d < nd <= 6: weighted sums, 16^d scaling, combine
template <class F>
__global__ void __launch_bounds__(384) k_red_final_q(const void* __restrict__ merged, int G, int bits, int c,
                                                     void* __restrict__ out_jac, const msm_peer peer) {
  __shared__ xyzz_t sm[96];
  quad_comm_dev cm;
  const int nd = (bits + 3) / 4;  // <= 6
  const int quad = threadIdx.x >> 2;
  const int d = quad >> 4, v = quad & 15;
  xyzz_t total = xyzz_identity<F>();
  for (int g = G - 1; g >= 0; g--) {
    xyzz_t acc = xyzz_identity<F>();
    if (d < nd) acc = xyzz_load(merged, ((size_t)g * nd + d) * 16 + v);  // S_d[v]
    if (cm.lane() == 0) sm[quad] = acc;
    __syncthreads();
    // suffix scan over v: T_v = sum_{j>=v} S_j
    for (int dd = 1; dd < 16; dd <<= 1) {
      bool have = v + dd < 16;
      xyzz_t o = xyzz_identity<F>();
      if (have) o = sm[quad + dd];
      __syncthreads();
      if (have) coop_add<F>(acc, o, cm);
      if (cm.lane() == 0) sm[quad] = acc;
      __syncthreads();
    }
    // W_d = sum_{v>=1} T_v (tree over v); S_all = T_0 of digit 0
    xyzz_t t0 = acc;
    if (v == 0) acc = xyzz_identity<F>();
    if (cm.lane() == 0) sm[quad] = acc;
    __syncthreads();
    for (int s = 8; s > 0; s >>= 1) {
      bool have = v < s;
      xyzz_t o = xyzz_identity<F>();
      if (have) o = sm[quad + s];
      __syncthreads();
      if (have) coop_add<F>(acc, o, cm);
      if (cm.lane() == 0) sm[quad] = acc;
      __syncthreads();
    }
    // quad (d, 0): W_d * 16^d ; digit 0 also adds S_all
    if (v == 0 && d < nd) {
      for (int i = 0; i < 4 * d; i++) coop_dbl<F>(acc, cm);
      if (d == 0) coop_add<F>(acc, t0, cm);
      if (cm.lane() == 0) sm[quad] = acc;
    }
    __syncthreads();
    if (quad == 0) {  // combine the digits and (for un-expanded keys) the window groups
      if (g != G - 1)
        for (int i = 0; i < c; i++) coop_dbl<F>(total, cm);
      for (int dd = 0; dd < nd; dd++) {
        xyzz_t o = sm[dd * 16];
        coop_add<F>(total, o, cm);
      }
    }
    __syncthreads();
  }
  if (peer.world > 1) total = peer_exchange_sum<F>(total, peer, sm, cm);  // every rank leaves with the same sum
  if (threadIdx.x == 0) {
    fe_t X, Y, Z;
    xyzz_to_jacobian<F>(total, X, Y, Z);
    fe_store(out_jac, 0, X);
    fe_store(out_jac, 1, Y);
    fe_store(out_jac, 2, Z);
  }
}
#endif  // !NOVA_MSM_ARITH29

// sum of k Jacobian points (the per-GPU partial MSMs after the all-gather, SURVEY.md §8e);
// k is tiny (= number of GPUs), one thread.
template <class F>
__global__ void k_jacobian_sum(const void* __restrict__ pts, int k, void* __restrict__ out_jac) {
  using PA = msm_arith<F>;
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  typename PA::pt acc = PA::identity();
  for (int i = 0; i < k; i++) {
    fe_t X = fe_load(pts, 3 * (size_t)i), Y = fe_load(pts, 3 * (size_t)i + 1),
         Z = fe_load(pts, 3 * (size_t)i + 2);
    typename PA::pt p = PA::from_jacobian_std(X, Y, Z);  // Jacobian (X,Y,Z) == XYZZ (X, Y, Z^2, Z^3)
    PA::add(acc, p);
  }
  fe_t X, Y, Z;
  PA::to_jacobian_std(acc, X, Y, Z);
  fe_store(out_jac, 0, X);
  fe_store(out_jac, 1, Y);
  fe_store(out_jac, 2, Z);
}

#if !defined(NOVA_MSM_ARITH29)
// the same with quad-cooperative additions: 8 quads stride over the points, then a 3-level tree (one block of 32
// threads).  4 points cost 2 dependent cooperative additions (~6 us) instead of 3 full ones on a lone thread (~27 us).
template <class F>
__global__ void __launch_bounds__(32) k_jacobian_sum_q(const void* __restrict__ pts, int k, void* __restrict__ out_jac) {
  __shared__ xyzz_t sm[8];
  quad_comm_dev cm;
  const int quad = threadIdx.x >> 2;
  xyzz_t acc = xyzz_identity<F>();
  for (int i = quad; i < k; i += 8) {  // uniform within a quad
    fe_t X = fe_load(pts, 3 * (size_t)i), Y = fe_load(pts, 3 * (size_t)i + 1), Z = fe_load(pts, 3 * (size_t)i + 2);
    xyzz_t p = xyzz_identity<F>();
    if (!fe_is_zero(Z)) {
      p.x = X;
      p.y = Y;
      p.zz = fe_sqr<F>(Z);
      p.zzz = fe_mul<F>(p.zz, Z);
    }
    coop_add<F>(acc, p, cm);
  }
  for (int s = 4; s > 0; s >>= 1) {
    if (quad < 2 * s && cm.lane() == 0) sm[quad] = acc;
    __syncwarp();
    if (quad < s) {
      xyzz_t o = sm[quad + s];
      coop_add<F>(acc, o, cm);
    }
    __syncwarp();
  }
  if (threadIdx.x == 0) {
    fe_t X, Y, Z;
    xyzz_to_jacobian<F>(acc, X, Y, Z);
    fe_store(out_jac, 0, X);
    fe_store(out_jac, 1, Y);
    fe_store(out_jac, 2, Z);
  }
}
#endif

// Synthetic key for tests/benches: bases[i] = (k0 + i) * G, affine.  Plays the role of the
// reference's test-only key generators (hyperkzg.rs:357-376 `setup_from_rng`, the
// "P0 + i*G" bases of curve_property_tests.rs:186-194); real keys come from the host.
template <class F>
__global__ void __launch_bounds__(128) k_index_bases(void* __restrict__ bases, size_t n,
                                                     const void* __restrict__ gen, uint64_t k0) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  fe_t gx = fe_load(gen, 0), gy = fe_load(gen, 1);
  uint64_t k = k0 + i;
  xyzz_t acc = xyzz_identity<F>();
  for (int b = 63; b >= 0; b--) {
    xyzz_dbl<F>(acc);
    if ((k >> b) & 1) xyzz_madd<F>(acc, gx, gy);
  }
  fe_t x = fe_zero<F>(), y = fe_zero<F>();
  if (!xyzz_is_identity(acc)) {
    fe_t iz3 = fe_inv<F>(acc.zzz);
    fe_t iz2 = fe_mul<F>(fe_sqr<F>(acc.zz), fe_sqr<F>(iz3));
    x = fe_mul<F>(acc.x, iz2);
    y = fe_mul<F>(acc.y, iz3);
  }
  fe_store(bases, 2 * i, x);
  fe_store(bases, 2 * i + 1, y);
}

// Test/bench SRS: bases[i] = [s_i] G for canonical (non-Montgomery) 256-bit scalars s_i, affine.  With
// s_i = tau^i this is the reference's test-only KZG setup (hyperkzg.rs:357-376 `setup_from_rng`:
// powers of a sampled tau times the generator), which lets a bench-scale proof be checked by the
// restated verifier with the pairing replaced by L = [tau] R.  254 doublings + ~127 mixed adds +
// one inversion per point; a 2^22-point key costs ~0.3 s.
template <class F>
__global__ void __launch_bounds__(128) k_scalar_bases(void* __restrict__ bases, size_t n,
                                                      const void* __restrict__ gen,
                                                      const void* __restrict__ scalars) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  fe_t gx = fe_load(gen, 0), gy = fe_load(gen, 1);
  fe_t k = fe_load(scalars, i);
  xyzz_t acc = xyzz_identity<F>();
  for (int b = 255; b >= 0; b--) {
    xyzz_dbl<F>(acc);
    if ((k.l[b >> 5] >> (b & 31)) & 1u) xyzz_madd<F>(acc, gx, gy);
  }
  fe_t x = fe_zero<F>(), y = fe_zero<F>();
  if (!xyzz_is_identity(acc)) {
    fe_t iz3 = fe_inv<F>(acc.zzz);
    fe_t iz2 = fe_mul<F>(fe_sqr<F>(acc.zz), fe_sqr<F>(iz3));
    x = fe_mul<F>(acc.x, iz2);
    y = fe_mul<F>(acc.y, iz3);
  }
  fe_store(bases, 2 * i, x);
  fe_store(bases, 2 * i + 1, y);
}

// ------------------------------------------------------------------------------------------
// key expansion:  tables[t][i] = 2^(shift*t) * bases[i]  (affine; identity stays (0,0))
// ------------------------------------------------------------------------------------------
// In: table 0 holds the host's bases in the BOUNDARY format.  Out: every table in the arithmetic
// policy's own table format (table 0 is converted in place).
template <class F>
__global__ void __launch_bounds__(128) k_expand_key(void* __restrict__ tables, size_t n_ck,
                                                    int ntables, int shift) {
  using PA = msm_arith<F>;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_ck) return;
  fe_t bx = fe_load_rw(tables, 2 * i), by = fe_load_rw(tables, 2 * i + 1);
  if (fe_is_zero(bx) && fe_is_zero(by)) {  // identity base: stays (0,0) in every table
    for (int t = 1; t < ntables; t++) PA::store_table_identity(tables, (size_t)t * n_ck + i);
    return;
  }
  typename PA::aff p = PA::from_std_affine(bx, by);
  PA::store_table(tables, i, p);
  for (int t = 1; t < ntables; t++) {
    typename PA::pt q = PA::identity();
    PA::madd(q, p);
    for (int d = 0; d < shift; d++) PA::dbl(q);
    p = PA::to_affine(q);
    PA::store_table(tables, (size_t)t * n_ck + i, p);
  }
}

// Key validation (hyperkzg.rs:113-119, ptau.rs:372-392): the smallest index of a base that has a non-canonical
// coordinate or is not on the curve is left in *first_bad (initialised to 0xFFFFFFFF by the caller).  64 B read per point, 3 products.
template <class F>
__global__ void __launch_bounds__(256) k_on_curve(const void* __restrict__ pts, size_t n, int b_small,
                                                  uint32_t* __restrict__ first_bad) {
  const fe_t b = fe_from_small_int<F>(b_small);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    affine_t p;
    p.x = fe_load(pts, 2 * i);
    p.y = fe_load(pts, 2 * i + 1);
    if (!affine_valid_raw<F>(p, b)) atomicMin(first_bad, (uint32_t)i);
  }
}

// ------------------------------------------------------------------------------------------
// ck_derive_by_address (traits/commitment.rs:177-194, pedersen.rs:360-382, hyperkzg.rs:731-749):
//   derived[j] = sum_{i < m, addr[i] = j} ck[i]
// is the bucket stage of a one-window MSM whose scalars are all 1, with the address as the bucket:
// k_address_entries (msm_sort.cuh), the radix passes, k_sort_starts, k_accumulate over the source's
// table 0 and the fix-up kernels, then k_derive_affine in place of the reduction.
// ------------------------------------------------------------------------------------------
// The checks of one derivation in one pass: flags[0] = smallest index of an identity generator among the n bases of
// table 0 (ck_to_group_elements' assertion), flags[1] = smallest position i < m of an address >= table_size
// (NovaError::InvalidIndex).  The caller presets both to 0xFFFFFFFF and passes m <= n.  64 + 4 B read per base.
template <class F>
__global__ void __launch_bounds__(256) k_derive_check(const void* __restrict__ tables, size_t n,
                                                      const uint32_t* __restrict__ addr, size_t m,
                                                      size_t table_size, uint32_t* __restrict__ flags) {
  using PA = msm_arith<F>;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (PA::aff_is_identity(PA::load_table(tables, i))) atomicMin(&flags[0], (uint32_t)i);
    if (i < m && addr[i] >= table_size) atomicMin(&flags[1], (uint32_t)i);
  }
}

// bucket k -> derived base k in the BOUNDARY format (affine Montgomery, identity (0,0)), the layout register_key
// takes: a slot no address points to, or whose sum is the identity (P + (-P)), is (0,0).  One inversion per slot;
// 128 B read and 64 B written.
template <class F>
__global__ void __launch_bounds__(128) k_derive_affine(const uint32_t* __restrict__ start, uint32_t K,
                                                       const void* __restrict__ buckets, void* __restrict__ out) {
  using PA = msm_arith<F>;
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  fe_t x = fe_zero<F>(), y = fe_zero<F>();
  if (start[k + 1] > start[k]) {  // an empty bucket holds stale data
    fe_t X, Y, Z;
    PA::to_jacobian_std(PA::load(buckets, k), X, Y, Z);
    if (!fe_is_zero(Z)) {
      const fe_t zi = fe_inv<F>(Z), zi2 = fe_sqr<F>(zi);
      x = fe_mul<F>(X, zi2);
      y = fe_mul<F>(Y, fe_mul<F>(zi2, zi));
    }
  }
  fe_store(out, 2 * (size_t)k, x);
  fe_store(out, 2 * (size_t)k + 1, y);
}

}  // namespace nova
