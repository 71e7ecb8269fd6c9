// The verifier kernels of nova_b200/csrc/poly_kernels.cuh on the CPU through the SIMT shim (simt_host.h): the REAL
// k_r1cs_eval (entry-range slices, the binary search for a slice's first row, the running row sums, the warp and
// shared-memory reduction) and k_r1cs_final with grid.y emulated by a loop, launched as ops_impl.cuh r1cs_eval does
// but with a grid and slice length of the caller's choosing; and k_ipa_s_half + k_eq_outer as ops_impl.cuh ipa_s.
// TEST INFRASTRUCTURE: tests/test_verify_kernels_host.py compiles it and compares with tests/verify_oracle.c.
#include <cstring>
#include <vector>
#include "simt_host.h"
#include "../../nova_b200/csrc/poly_kernels.cuh"
using namespace nova;

template <class F>
static void classify(const void* vals, size_t nnz, int8_t* codes) {
  const unsigned grid = (unsigned)((nnz + 255) / 256);
  if (grid) simt_launch_grid(grid, 256, [&] { k_spmv_classify<F>(vals, nnz, codes); });
}

// k matrices in CSR (u32 indptr / colidx, Montgomery vals) -> out[k]; `grid` blocks of 256 threads per matrix,
// `chunk` entries per thread (0: as many as needed to cover the longest matrix with `grid` blocks)
template <class F>
static void r1cs_eval_t(int k, const uint32_t* const* indptr, const uint32_t* const* colidx, const void* const* vals,
                        const size_t* rows, const size_t* nnz, const void* tx, const void* ty, unsigned grid,
                        size_t chunk, void* out) {
  r1cs_mats m{};
  std::vector<std::vector<int8_t>> codes(k);
  size_t longest = 0;
  for (int y = 0; y < k; y++) {
    codes[y].assign(nnz[y] ? nnz[y] : 1, 0);
    classify<F>(vals[y], nnz[y], codes[y].data());
    m.indptr[y] = indptr[y];
    m.colidx[y] = colidx[y];
    m.codes[y] = codes[y].data();
    m.vals[y] = vals[y];
    m.rows[y] = rows[y];
    m.nnz[y] = nnz[y];
    longest = nnz[y] > longest ? nnz[y] : longest;
  }
  if (chunk == 0) chunk = longest ? (longest + (size_t)grid * 256 - 1) / ((size_t)grid * 256) : 1;
  std::vector<fe_t> partials((size_t)k * grid);
  for (int y = 0; y < k; y++)
    simt_launch_grid(grid, 256, [&] {
      blockIdx.y = (unsigned)y;
      k_r1cs_eval<F>(m, tx, ty, chunk, partials.data());
    });
  for (int y = 0; y < k; y++)
    simt_launch_grid(1, 256, [&] {
      blockIdx.y = (unsigned)y;
      k_r1cs_final<F>(partials.data(), (int)grid, out);
    });
}

extern "C" int hc_simt_r1cs_eval(int fid, int k, const uint32_t* const* indptr, const uint32_t* const* colidx,
                                 const void* const* vals, const size_t* rows, const size_t* nnz, const void* tx,
                                 const void* ty, unsigned grid, size_t chunk, void* out) {
  if (k < 1 || k > R1CS_MAX_MATS || grid == 0) return 1;
  switch (fid) {
    case 0: r1cs_eval_t<BN254_FR>(k, indptr, colidx, vals, rows, nnz, tx, ty, grid, chunk, out); return 0;
    case 1: r1cs_eval_t<BN254_FQ>(k, indptr, colidx, vals, rows, nnz, tx, ty, grid, chunk, out); return 0;
    case 2: r1cs_eval_t<PALLAS_FP>(k, indptr, colidx, vals, rows, nnz, tx, ty, grid, chunk, out); return 0;
    case 3: r1cs_eval_t<PALLAS_FQ>(k, indptr, colidx, vals, rows, nnz, tx, ty, grid, chunk, out); return 0;
    default: return 1;
  }
}

// s of 2^L entries: one direct pass for L <= direct_bits, else the two half tables and their outer product
template <class F>
static void ipa_s_t(const void* r, const void* r_inv, int L, const void* scale, int direct_bits, void* out) {
  if (L <= direct_bits) {
    simt_launch_grid((unsigned)((((size_t)1 << L) + 255) / 256), 256,
                     [&] { k_ipa_s_half<F>(r, r_inv, L, scale, out); });
    return;
  }
  const int rb = L / 2, lb = L - rb;
  std::vector<fe_t> left((size_t)1 << lb), right((size_t)1 << rb);
  simt_launch_grid((unsigned)((left.size() + 255) / 256), 256,
                   [&] { k_ipa_s_half<F>(r, r_inv, lb, scale, left.data()); });
  simt_launch_grid((unsigned)((right.size() + 255) / 256), 256, [&] {
    k_ipa_s_half<F>((const char*)r + 32 * lb, (const char*)r_inv + 32 * lb, rb, nullptr, right.data());
  });
  const size_t n = (size_t)1 << L;
  simt_launch_grid(2, 256, [&] { k_eq_outer<F>(left.data(), right.data(), rb, n, out); });
}

extern "C" int hc_simt_ipa_s(int fid, const void* r, const void* r_inv, int L, const void* scale, int direct_bits,
                             void* out) {
  switch (fid) {
    case 0: ipa_s_t<BN254_FR>(r, r_inv, L, scale, direct_bits, out); return 0;
    case 1: ipa_s_t<BN254_FQ>(r, r_inv, L, scale, direct_bits, out); return 0;
    case 2: ipa_s_t<PALLAS_FP>(r, r_inv, L, scale, direct_bits, out); return 0;
    case 3: ipa_s_t<PALLAS_FQ>(r, r_inv, L, scale, direct_bits, out); return 0;
    default: return 1;
  }
}
