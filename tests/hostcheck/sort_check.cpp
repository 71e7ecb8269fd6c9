// The bucket sort of the MSM (nova_b200/csrc/msm_sort.cuh) on the CPU through the SIMT shim (simt_host.h with the
// extra intrinsics of simt_host_sort.h): the integer-scalar digit kernel with its block histograms, every radix pass
// with its tile ranking and decoupled look-back, and the bucket-start kernel run as written, launched as
// msm_common.cu msm_sort launches them.
#include <cstring>
#include <vector>
#include "simt_host_sort.h"
#include "../../nova_b200/csrc/msm_sort.cuh"
using namespace nova;

// One bucket sort of the [W][n] digit array.  small_scalars != null: the digits (written to digits) and histograms
// come from k_digits_small over those u64 scalars, on `digit_blocks` blocks; otherwise digits is the input and the
// histograms are counted here.  The sort runs twice on the same look-back words (tags 1.. and then fresh ones),
// as two consecutive MSMs on one workspace do; both results must agree, and the second is returned.
extern "C" int hc_sort_run(int32_t* digits, const uint64_t* small_scalars, unsigned digit_blocks, uint32_t n, int c,
                           int W, int G, uint32_t n_ck, uint32_t base_offset, uint32_t blind_i, uint32_t h_index,
                           uint32_t heavy_min, uint32_t heavy_cap, uint64_t* entries_out, uint32_t* start_out,
                           uint32_t* heavy_out, int* passes_out) {
  const uint32_t B = 1u << (c - 1);
  const uint32_t K = (uint32_t)G * B;
  const sort_plan sp = make_sort_plan(K);
  *passes_out = sp.passes;
  std::vector<uint32_t> ctl(SORT_CTL_WORDS, 0);
  if (small_scalars) {
    simt_launch_grid(digit_blocks, 256, [&] {
      k_digits_small(small_scalars, 8, n, c, W, G, B, digits, ctl.data(), sp);
    });
  } else {
    const uint32_t mask = (1u << sp.bits) - 1;
    for (size_t x = 0; x < (size_t)n * W; x++) {
      const int32_t d = digits[x];
      if (d == 0) continue;
      const uint32_t w = (uint32_t)(x / n);
      const uint32_t key = (w % (uint32_t)G) * B + (uint32_t)(d < 0 ? -d : d) - 1;
      for (int p = 0; p < sp.passes; p++) ctl[p * SORT_BINS + ((key >> (p * sp.bits)) & mask)]++;
    }
  }
  sort_args a;
  a.n = n;
  a.count = n * (uint32_t)W;
  a.W = W;
  a.G = G;
  a.B = B;
  a.n_ck = n_ck;
  a.base_offset = base_offset;
  a.blind_i = blind_i;
  a.h_index = h_index;
  a.sp = sp;
  const unsigned tiles = (a.count + SORT_TILE - 1) / SORT_TILE;
  std::vector<unsigned long long> look((size_t)tiles * SORT_BINS, 0);
  std::vector<uint64_t> ent(a.count), tmp(a.count), first;
  std::vector<uint32_t> start(K + 1), first_start;
  std::vector<uint32_t> heavy(1 + heavy_cap), first_heavy;
  uint32_t tag = 1;
  for (int run = 0; run < 2; run++) {
    for (int p = 0; p < SORT_PASSES_MAX; p++) ctl[SORT_PASSES_MAX * SORT_BINS + p] = 0;
    std::fill(ent.begin(), ent.end(), ~0ull);
    std::fill(tmp.begin(), tmp.end(), ~0ull);
    std::fill(heavy.begin(), heavy.end(), 0u);
    const uint64_t* in = nullptr;
    for (int pass = 0; pass < sp.passes; pass++) {
      uint64_t* out = ((sp.passes - 1 - pass) & 1) ? tmp.data() : ent.data();
      const uint32_t t = tag + (uint32_t)pass;
      simt_launch_grid(tiles, SORT_THREADS, [&] {
        if (pass == 0) k_sort_pass<true>(digits, nullptr, out, a, 0, ctl.data(), look.data(), t);
        else k_sort_pass<false>(nullptr, in, out, a, pass, ctl.data(), look.data(), t);
      });
      in = out;
    }
    tag += (uint32_t)sp.passes;
    simt_launch_grid((K + 1 + SORT_THREADS - 1) / SORT_THREADS, SORT_THREADS, [&] {
      k_sort_starts(ent.data(), ctl.data(), sp, K, start.data(), heavy.data(), heavy_min, heavy_cap);
    });
    if (run == 0) {
      first = ent;
      first_start = start;
      first_heavy = heavy;
    } else if (first != ent || first_start != start || first_heavy[0] != heavy[0]) {
      return 2;
    }
  }
  memcpy(entries_out, ent.data(), ent.size() * 8);
  memcpy(start_out, start.data(), start.size() * 4);
  memcpy(heavy_out, heavy.data(), heavy.size() * 4);
  return 0;
}
