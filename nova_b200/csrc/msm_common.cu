// Field-independent MSM stages: the integer-scalar digit kernel and the radix sort of the entries.
#include "ops.cuh"
#include "msm_kernels.cuh"

namespace nova {

void msm_digits_small(cudaStream_t s, const void* scalars, int elem_bytes, const msm_plan& p) {
  size_t blocks = (p.n + 255) / 256;
  unsigned grid = (unsigned)(blocks < SORT_HIST_BLOCKS ? blocks : SORT_HIST_BLOCKS);
  k_digits_small<<<grid, 256, 0, s>>>(scalars, elem_bytes, p.n, p.c, p.W, p.G, p.B, p.digits, p.sortctl, p.sp);
}

sort_args make_sort_args(const msm_plan& p) {
  sort_args a;
  a.n = (uint32_t)p.n;
  a.count = (uint32_t)(p.n * (size_t)p.W);
  a.W = p.W;
  a.G = p.G;
  a.B = p.B;
  a.n_ck = (uint32_t)p.n_ck;
  a.base_offset = (uint32_t)p.base_offset;
  a.blind_i = p.blind_i == SIZE_MAX ? NO_KEY : (uint32_t)p.blind_i;
  a.h_index = (uint32_t)p.h_index;
  a.sp = p.sp;
  return a;
}

// the radix passes (pass 0 reads the digits; the last pass writes p.entries), then the bucket starts;
// returns the number of kernels launched
int msm_sort(cudaStream_t s, const msm_plan& p) {
  const sort_args a = make_sort_args(p);
  const unsigned tiles = (unsigned)((a.count + SORT_TILE - 1) / SORT_TILE);
  const int P = p.sp.passes;
  const uint64_t* in = nullptr;
  for (int pass = 0; pass < P; pass++) {
    uint64_t* out = ((P - 1 - pass) & 1) ? p.entries_tmp : p.entries;
    if (pass == 0)
      k_sort_pass<true><<<tiles, SORT_THREADS, 0, s>>>(p.digits, nullptr, out, a, 0, p.sortctl, p.look, p.sort_tag);
    else
      k_sort_pass<false><<<tiles, SORT_THREADS, 0, s>>>(nullptr, in, out, a, pass, p.sortctl, p.look,
                                                        p.sort_tag + (uint32_t)pass);
    in = out;
  }
  const uint32_t K = (uint32_t)p.G * p.B;
  k_sort_starts<<<(K + 1 + SORT_THREADS - 1) / SORT_THREADS, SORT_THREADS, 0, s>>>(
      p.entries, p.sortctl, p.sp, K, p.start, p.heavy, p.heavy_min, p.heavy_cap);
  return P + 1;
}

// ck_derive_by_address: the address stage writes the entries into the buffer the first pass reads (the last pass
// writes p.entries), then every pass reads entries; then the bucket starts.  Returns the number of kernels launched.
int derive_sort(cudaStream_t s, const uint32_t* addr, const msm_plan& p) {
  sort_args a = make_sort_args(p);
  a.count = (uint32_t)p.n;
  const unsigned tiles = (unsigned)((p.n + SORT_TILE - 1) / SORT_TILE);
  const int P = p.sp.passes;
  uint64_t* in = (P & 1) ? p.entries_tmp : p.entries;
  const size_t blocks = (p.n + 255) / 256;
  k_address_entries<<<(unsigned)(blocks < SORT_HIST_BLOCKS ? blocks : SORT_HIST_BLOCKS), 256, 0, s>>>(
      addr, p.n, in, p.sortctl, p.sp);
  for (int pass = 0; pass < P; pass++) {
    uint64_t* out = ((P - 1 - pass) & 1) ? p.entries_tmp : p.entries;
    k_sort_pass<false><<<tiles, SORT_THREADS, 0, s>>>(nullptr, in, out, a, pass, p.sortctl, p.look,
                                                      p.sort_tag + (uint32_t)pass);
    in = out;
  }
  const uint32_t K = (uint32_t)p.G * p.B;
  k_sort_starts<<<(K + 1 + SORT_THREADS - 1) / SORT_THREADS, SORT_THREADS, 0, s>>>(
      p.entries, p.sortctl, p.sp, K, p.start, p.heavy, p.heavy_min, p.heavy_cap);
  return P + 2;
}

}  // namespace nova
