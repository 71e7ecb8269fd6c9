// Bucket sort of the MSM: a stable LSD radix sort of the (key, sign, table index) entries by bucket key.
//
//   digit stage   (k_digits<S>, k_digits_small) writes digits[W][n] and, per block in shared memory, the
//                 histogram of every pass's radix digit over the non-zero digits; each block adds its
//                 histogram to sortctl's hist[pass][bin] (a few hundred atomics per block).  Histograms are
//                 additive, so the digits of one vector may be produced chunk by chunk.
//   k_sort_pass   one launch per pass.  A tile of SORT_TILE inputs (pass 0: the flattened [W][n] digit array,
//                 zero digits dropped and the entry built on the fly; later passes: the previous pass's
//                 entries) is ranked in shared memory by the pass's radix digit -- per-warp counters, and
//                 within a warp one ballot per digit bit, so a tile holding a single key costs no more than a
//                 uniform one -- and written out in bin order.  The tile's global offset per bin is the bin's
//                 base (exclusive scan of hist[pass]) plus the counts of the tiles before it, obtained by
//                 decoupled look-back: every tile publishes its per-bin count, then its inclusive prefix, in
//                 one 64-bit word per (tile, bin).  Tile ids come from an atomic counter, so a tile only ever
//                 waits on tiles that are already running.
//   k_sort_starts start[k] = first position of key >= k (binary search inside the key's top-digit range,
//                 which the last pass's histogram gives exactly), start[K] = M; keys with more than
//                 heavy_min entries go to the heavy list.
// Entries are generated in (window, index) order and every pass is stable, so the order inside a bucket, and
// with it every bit of the MSM output, does not depend on scheduling.  No pass does a per-entry global atomic.
//
// The kernels also compile for the CPU through tests/hostcheck/simt_host.h, which runs them as written.
#pragma once
#if !defined(NOVA_SIMT_HOST)
#include <cuda_runtime.h>
#endif
#include <cstddef>
#include <cstdint>
#include "field.cuh"  // NOVA_D

namespace nova {

constexpr uint32_t NO_KEY = 0xFFFFFFFFu;

constexpr int SORT_THREADS = 256;
constexpr int SORT_WARPS = SORT_THREADS / 32;
constexpr int SORT_ITEMS = 16;                          // inputs per thread and tile
constexpr int SORT_TILE = SORT_THREADS * SORT_ITEMS;    // 4096
constexpr int SORT_RADIX_MAX = 8;                       // bits per pass
constexpr int SORT_BINS = 1 << SORT_RADIX_MAX;          // 256 = one bin per thread
constexpr int SORT_PASSES_MAX = 4;                      // keys of up to 32 bits
constexpr int SORT_CTL_WORDS = SORT_PASSES_MAX * SORT_BINS + SORT_PASSES_MAX;  // hist[pass][bin], tile counter[pass]
constexpr unsigned SORT_HIST_BLOCKS = 1024;             // grid cap of the digit kernels (each block flushes once)
constexpr int SORT_LOOK_WINDOW = 4;                     // look-back words read per round trip
// k_sort_pass is latency-bound (load, rank, look-back and write-out of a tile run one after the other): three
// resident blocks per SM instead of two cut a 2^20 MSM's two passes from 385 to 342 us on an H100 SXM (700 W),
// although ptxas then spills a few words of the 80-register budget
constexpr int SORT_MIN_BLOCKS = 3;
static_assert(SORT_BINS == SORT_THREADS, "the per-bin steps run one bin per thread");

struct sort_plan {
  int passes;  // ceil(key_bits / SORT_RADIX_MAX)
  int bits;    // radix bits per pass (<= SORT_RADIX_MAX); pass p sorts by key bits [p * bits, (p + 1) * bits)
};

// passes for keys in [0, K): as few as 8-bit digits allow, with the bits spread evenly over them
inline sort_plan make_sort_plan(uint64_t K) {
  int kb = 1;
  while (kb < 32 && ((uint64_t)1 << kb) < K) kb++;
  sort_plan sp;
  sp.passes = (kb + SORT_RADIX_MAX - 1) / SORT_RADIX_MAX;
  sp.bits = (kb + sp.passes - 1) / sp.passes;
  return sp;
}

// what pass 0 needs to build an entry from a digit's position (w, i) in the [W][n] digit array
struct sort_args {
  uint32_t n;            // scalars
  uint32_t count;        // n * W digits
  int W, G;
  uint32_t B;            // buckets per group: key = (w % G) * B + |digit| - 1
  uint32_t n_ck;         // points per table: table index = (w / G) * n_ck + base
  uint32_t base_offset;  // base of scalar i = base_offset + i ...
  uint32_t blind_i;      // ... except scalar blind_i (NO_KEY: none), whose base is h_index
  uint32_t h_index;
  sort_plan sp;
};

// ---- digit-stage histogram ------------------------------------------------------------------
NOVA_D void sort_hist_clear(uint32_t* sh /* [SORT_PASSES_MAX * SORT_BINS] */) {
  for (int i = threadIdx.x; i < SORT_PASSES_MAX * SORT_BINS; i += blockDim.x) sh[i] = 0;
  __syncthreads();
}

// all 32 lanes call; key = NO_KEY for lanes without an entry.  A warp whose entries share one key (0/1 witnesses,
// padding, a repeated value) adds its count with one shared atomic per pass instead of 32 on one counter.
NOVA_D void sort_hist_count(uint32_t* sh, uint32_t key, const sort_plan sp) {
  const bool live = key != NO_KEY;
  const unsigned live_mask = __ballot_sync(0xFFFFFFFFu, live);
  if (live_mask == 0) return;
  const unsigned lane = threadIdx.x & 31u, leader = (unsigned)(__ffs(live_mask) - 1);
  const uint32_t lead_key = __shfl_sync(0xFFFFFFFFu, key, (int)leader);
  const bool same = __ballot_sync(0xFFFFFFFFu, live && key != lead_key) == 0;
  const uint32_t mask = (1u << sp.bits) - 1;
  for (int p = 0; p < sp.passes; p++) {
    const uint32_t bin = (key >> (p * sp.bits)) & mask;
    if (same) {
      if (lane == leader) atomicAdd(&sh[p * SORT_BINS + bin], (uint32_t)__popc(live_mask));
    } else if (live) {
      atomicAdd(&sh[p * SORT_BINS + bin], 1u);
    }
  }
}

NOVA_D void sort_hist_flush(const uint32_t* sh, uint32_t* hist, const sort_plan sp) {
  __syncthreads();
  for (int i = threadIdx.x; i < sp.passes * SORT_BINS; i += blockDim.x) {
    const uint32_t v = sh[i];
    if (v) atomicAdd(&hist[i], v);
  }
}

// integer scalars (msm.rs:469-503): unsigned little-endian elements of 1/2/4/8 bytes -> the same signed c-bit
// digit stream and histograms as k_digits; zero scalars produce no entries (msm.rs:512,545)
static __global__ void __launch_bounds__(256) k_digits_small(const void* __restrict__ scalars, int elem_bytes,
                                                             size_t n, int c, int W, int G, uint32_t B,
                                                             int32_t* __restrict__ digits, uint32_t* __restrict__ hist,
                                                             const sort_plan sp) {
  __shared__ uint32_t s_hist[SORT_PASSES_MAX * SORT_BINS];
  sort_hist_clear(s_hist);
  for (size_t blk = (size_t)blockIdx.x * blockDim.x; blk < n; blk += (size_t)gridDim.x * blockDim.x) {
    const size_t i = blk + threadIdx.x;
    const bool live = i < n;  // no early exit: the whole warp takes part in sort_hist_count
    uint64_t v64 = 0;
    if (live) switch (elem_bytes) {
      case 1: v64 = ((const uint8_t*)scalars)[i]; break;
      case 2: v64 = ((const uint16_t*)scalars)[i]; break;
      case 4: v64 = ((const uint32_t*)scalars)[i]; break;
      default: v64 = ((const uint64_t*)scalars)[i]; break;
    }
    const uint32_t half = 1u << (c - 1);
    const uint64_t mask = (1ull << c) - 1;
    uint32_t carry = 0;
    for (int w = 0; w < W; w++) {
      int bit = w * c;
      uint32_t v = bit < 64 ? (uint32_t)((v64 >> bit) & mask) : 0u;
      v += carry;
      int32_t dgt;
      if (v > half) {
        dgt = (int32_t)v - (int32_t)(1u << c);
        carry = 1;
      } else {
        dgt = (int32_t)v;
        carry = 0;
      }
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

// The address stage of ck_derive_by_address (traits/commitment.rs:177-194), in place of the digit stage: a one-window
// MSM whose scalars are all 1 and whose bucket is the address.  Entry i = (key addr[i], sign 0, table index i), written
// in index order, and the radix histograms of the keys.  Every radix pass then reads entries (k_sort_pass<false>), so
// the order inside a bucket is the index order.  The caller has checked addr[i] < K <= 2^31 (no key is NO_KEY).
static __global__ void __launch_bounds__(256) k_address_entries(const uint32_t* __restrict__ addr, size_t m,
                                                                uint64_t* __restrict__ entries,
                                                                uint32_t* __restrict__ hist, const sort_plan sp) {
  __shared__ uint32_t s_hist[SORT_PASSES_MAX * SORT_BINS];
  sort_hist_clear(s_hist);
  for (size_t blk = (size_t)blockIdx.x * blockDim.x; blk < m; blk += (size_t)gridDim.x * blockDim.x) {
    const size_t i = blk + threadIdx.x;
    const bool live = i < m;  // no early exit: the whole warp takes part in sort_hist_count
    const uint32_t key = live ? addr[i] : NO_KEY;
    if (live) entries[i] = ((uint64_t)key << 32) | (uint32_t)i;
    sort_hist_count(s_hist, key, sp);
  }
  sort_hist_flush(s_hist, hist, sp);
}

// exclusive scan over the SORT_THREADS threads of a block; *total = sum of all v.  s_tmp: SORT_WARPS words.
NOVA_D uint32_t sort_block_scan(uint32_t v, uint32_t* s_tmp, uint32_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, inc, d);
    if (lane >= d) inc += o;
  }
  if (lane == 31) s_tmp[warp] = inc;
  __syncthreads();
  uint32_t before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < SORT_WARPS; w++) {
    const uint32_t t = s_tmp[w];
    before += w < warp ? t : 0u;
    all += t;
  }
  __syncthreads();  // s_tmp may be reused
  *total = all;
  return before + inc - v;
}

// look-back word: high half = (tag << 1) | inclusive, low half = count.  A word from an earlier pass or call has
// another tag and reads as "not published yet"; the buffer starts zeroed and tags are never 0.
constexpr unsigned long long LOOK_INCLUSIVE = 1ull << 32;
NOVA_D unsigned long long look_word(uint32_t tag, bool inclusive, uint32_t v) {
  return ((unsigned long long)tag << 33) | (inclusive ? LOOK_INCLUSIVE : 0ull) | v;
}

// one LSD pass.  FIRST: input = digits [W][n] (a.count of them, zeros dropped); else input = in[0 .. M) with M the
// total of the pass-0 histogram.  out[] receives the pass's input stably sorted by key bits [pass * bits, ...).
template <bool FIRST>
__global__ void __launch_bounds__(SORT_THREADS, SORT_MIN_BLOCKS) k_sort_pass(const int32_t* __restrict__ digits,
                                                            const uint64_t* __restrict__ in,
                                                            uint64_t* __restrict__ out, const sort_args a, int pass,
                                                            uint32_t* __restrict__ ctl,
                                                            unsigned long long* __restrict__ look, uint32_t tag) {
  __shared__ uint64_t s_items[SORT_TILE];                // the tile in bin order
  __shared__ uint32_t s_warp[SORT_WARPS][SORT_BINS];     // per-warp bin counts, then per-warp bin offsets in the tile
  __shared__ uint32_t s_glob[SORT_BINS];                 // out index of tile position 0 of each bin
  __shared__ uint32_t s_tmp[SORT_WARPS];
  __shared__ uint32_t s_tile;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  const int shift = pass * a.sp.bits;
  const uint32_t mask = (1u << a.sp.bits) - 1u;

  if (tid == 0) s_tile = atomicAdd(&ctl[SORT_PASSES_MAX * SORT_BINS + pass], 1u);
#pragma unroll
  for (int w = 0; w < SORT_WARPS; w++) s_warp[w][tid] = 0;
  // bin bases of this pass; the total is the number of entries M
  uint32_t M;
  const uint32_t bin_base = sort_block_scan(ctl[pass * SORT_BINS + tid], s_tmp, &M);  // (ends with a barrier)
  const uint32_t tile = s_tile;
  const uint32_t count = FIRST ? a.count : M;
  if ((uint64_t)tile * SORT_TILE >= count) return;  // uniform: no tile with a smaller id is past the end
  const uint32_t wbase = tile * SORT_TILE + warp * 32 * SORT_ITEMS + lane;

  // load (warp-striped: item j of lane l is input wbase + 32 j, so (warp, j, lane) order is input order)
  uint64_t item[SORT_ITEMS];
#pragma unroll
  for (int j = 0; j < SORT_ITEMS; j++) {
    const uint32_t idx = wbase + 32u * j;
    if (FIRST) item[j] = idx < count ? (uint64_t)(uint32_t)digits[idx] : 0ull;
    else item[j] = idx < count ? in[idx] : 0ull;
  }
  // rank: rank[j] = position among the tile's items of the same bin and warp, in input order
  uint32_t rank[SORT_ITEMS];
#pragma unroll
  for (int j = 0; j < SORT_ITEMS; j++) {
    const uint32_t idx = wbase + 32u * j;
    bool valid;
    if (FIRST) {
      const int32_t dgt = (int32_t)(uint32_t)item[j];
      valid = idx < count && dgt != 0;
      if (valid) {
        const uint32_t w = idx / a.n, i = idx - w * a.n;
        const uint32_t sign = dgt < 0 ? 1u : 0u;
        const uint32_t mag = sign ? (uint32_t)(-dgt) : (uint32_t)dgt;
        const uint32_t key = (w % (uint32_t)a.G) * a.B + (mag - 1);
        // the blinding scalar r rides along as one more (scalar, base) pair whose base is h
        const uint32_t bi = i == a.blind_i ? a.h_index : a.base_offset + i;
        const uint32_t tix = (w / (uint32_t)a.G) * a.n_ck + bi;
        item[j] = ((uint64_t)key << 32) | ((uint64_t)sign << 31) | tix;
      }
    } else {
      valid = idx < count;
    }
    const uint32_t bin = (uint32_t)(item[j] >> (32 + shift)) & mask;
    unsigned peers = __ballot_sync(0xFFFFFFFFu, valid);
    rank[j] = NO_KEY;
    if (peers) {  // warp-uniform
      for (int b = 0; b < a.sp.bits; b++) {
        const unsigned m = __ballot_sync(0xFFFFFFFFu, (bin >> b) & 1u);
        peers &= ((bin >> b) & 1u) ? m : ~m;
      }
      const uint32_t before = valid ? s_warp[warp][bin] : 0u;
      __syncwarp();
      if (valid) {
        rank[j] = before + (uint32_t)__popc(peers & lt_mask);
        if ((peers & lt_mask) == 0) s_warp[warp][bin] = before + (uint32_t)__popc(peers);
      }
      __syncwarp();
    }
  }
  __syncthreads();

  // per bin (one per thread): tile count, offsets of the warps inside the bin
  uint32_t run = 0;
#pragma unroll
  for (int w = 0; w < SORT_WARPS; w++) {
    const uint32_t c = s_warp[w][tid];
    s_warp[w][tid] = run;
    run += c;
  }
  volatile unsigned long long* vlook = look;
  const size_t slot = (size_t)tile * SORT_BINS + tid;
  vlook[slot] = look_word(tag, tile == 0, run);  // publish early: the aggregate is all a successor needs
  uint32_t tile_total;
  const uint32_t tile_off = sort_block_scan(run, s_tmp, &tile_total);
  // look-back over the tiles before this one, SORT_LOOK_WINDOW words per round trip: tiles t-1, t-2, ... are added
  // until one carries its inclusive prefix; an unpublished word ends the round and is read again
  uint32_t excl = 0;
  for (uint32_t t = tile; t > 0;) {
    unsigned long long v[SORT_LOOK_WINDOW];
#pragma unroll
    for (int q = 0; q < SORT_LOOK_WINDOW; q++)
      v[q] = (uint32_t)q < t ? vlook[(size_t)(t - 1 - q) * SORT_BINS + tid] : 0ull;
    bool go = true;
#pragma unroll
    for (int q = 0; q < SORT_LOOK_WINDOW; q++) {
      go = go && t > 0 && (uint32_t)(v[q] >> 33) == tag;
      if (go) {
        excl += (uint32_t)v[q];
        t = (v[q] & LOOK_INCLUSIVE) ? 0u : t - 1;
      }
    }
  }
  if (tile != 0) vlook[slot] = look_word(tag, true, excl + run);
  s_glob[tid] = bin_base + excl - tile_off;
#pragma unroll
  for (int w = 0; w < SORT_WARPS; w++) s_warp[w][tid] += tile_off;
  __syncthreads();

  // the tile in bin order through shared memory, then out in per-bin runs
#pragma unroll
  for (int j = 0; j < SORT_ITEMS; j++) {
    if (rank[j] != NO_KEY) {
      const uint32_t bin = (uint32_t)(item[j] >> (32 + shift)) & mask;
      s_items[s_warp[warp][bin] + rank[j]] = item[j];
    }
  }
  __syncthreads();
  for (uint32_t k = tid; k < tile_total; k += SORT_THREADS) {
    const uint64_t e = s_items[k];
    const uint32_t bin = (uint32_t)(e >> (32 + shift)) & mask;
    out[s_glob[bin] + k] = e;
  }
}

// start[k] for k in [0, K] and the heavy list, from the sorted entries.  One thread per key.
static __global__ void __launch_bounds__(SORT_THREADS) k_sort_starts(const uint64_t* __restrict__ entries,
                                                              const uint32_t* __restrict__ ctl, const sort_plan sp,
                                                              uint32_t K, uint32_t* __restrict__ start,
                                                              uint32_t* __restrict__ heavy, uint32_t heavy_min,
                                                              uint32_t heavy_cap) {
  __shared__ uint32_t s_base[SORT_BINS + 1];  // entries of the last pass's bin b: [s_base[b], s_base[b + 1])
  __shared__ uint32_t s_start[SORT_THREADS + 1];
  __shared__ uint32_t s_tmp[SORT_WARPS];
  const int tid = threadIdx.x;
  const int last = sp.passes - 1, shift = last * sp.bits;
  uint32_t M;
  s_base[tid] = sort_block_scan(ctl[last * SORT_BINS + tid], s_tmp, &M);
  if (tid == 0) s_base[SORT_BINS] = M;
  __syncthreads();
  auto lower_bound = [&](uint32_t k) -> uint32_t {
    if (k >= K) return M;
    const uint32_t top = k >> shift;
    uint32_t lo = s_base[top], hi = s_base[top + 1];
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if ((uint32_t)(entries[mid] >> 32) < k) lo = mid + 1;
      else hi = mid;
    }
    return lo;
  };
  const uint32_t k = blockIdx.x * SORT_THREADS + tid;
  s_start[tid] = lower_bound(k);
  if (tid == SORT_THREADS - 1) s_start[SORT_THREADS] = lower_bound(k + 1);
  __syncthreads();
  if (k <= K) start[k] = s_start[tid];
  if (k < K && s_start[tid + 1] - s_start[tid] > heavy_min) {  // at most M / heavy_min such keys (heavy_cap)
    const uint32_t slot = atomicAdd(&heavy[0], 1u);
    if (slot < heavy_cap) heavy[1 + slot] = k;
  }
}

}  // namespace nova
