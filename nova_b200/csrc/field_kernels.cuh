// Streaming prime-field vector kernels (K4 of SURVEY.md §2).  All HBM-bound: one element per
// thread-iteration, 2 x 128-bit loads per operand, grid-stride over a grid sized in
// multiples of the SM count.
//
//   k_cross_term  T = Az o Bz - u*Cz - E1 (- E2)      src/r1cs/mod.rs:614-620, 650-657
//   k_axpy        out = a + r*b                        src/r1cs/mod.rs:1044-1073 (W, E folds)
//   k_lerp        out = a + r*(b - a)                  src/neutron/relation.rs:139-153 (W, E folds)
//   k_vec_add     out = a + b                          src/r1cs/mod.rs:589-609 (Z = Z1 + Z2)
//   k_bind_top    Z[i] += r*(Z[i+n/2] - Z[i])          src/spartan/polys/multilinear.rs:65-84
//   k_vec_mul     out = a o b                          src/spartan/ppsnark.rs:446-449 (inv o TS)
//   k_logup_hash  out = val*gamma + addr + r           src/spartan/ppsnark.rs:386-435 (T+r, W+r)
#pragma once
#include <cuda_runtime.h>
#include "field.cuh"

namespace nova {

template <class F>
__global__ void __launch_bounds__(256) k_cross_term(const void* __restrict__ az,
                                                    const void* __restrict__ bz,
                                                    const void* __restrict__ cz,
                                                    const void* __restrict__ e1,
                                                    const void* __restrict__ e2,
                                                    const void* __restrict__ u_ptr, size_t n,
                                                    void* __restrict__ t) {
  const fe_t u = fe_load(u_ptr, 0);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x) {
    fe_t a = fe_load(az, i), b = fe_load(bz, i), c = fe_load(cz, i), e = fe_load(e1, i);
    fe_t r = fe_sub<F>(fe_sub<F>(fe_mul<F>(a, b), fe_mul<F>(u, c)), e);
    if (e2 != nullptr) r = fe_sub<F>(r, fe_load(e2, i));
    fe_store(t, i, r);
  }
}

template <class F>
__global__ void __launch_bounds__(256) k_axpy(const void* __restrict__ a,
                                              const void* __restrict__ b,
                                              const void* __restrict__ r_ptr, size_t n,
                                              void* __restrict__ out) {
  const fe_t r = fe_load(r_ptr, 0);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x) {
    fe_t x = fe_load(a, i), y = fe_load(b, i);
    fe_store(out, i, fe_add<F>(x, fe_mul<F>(r, y)));
  }
}

// out = a + r*(b - a).  out may alias a: each element is read and then written by one thread, and `a`
// goes through the coherent load path because the kernel writes that buffer.
template <class F>
__global__ void __launch_bounds__(256) k_lerp(const void* a, const void* __restrict__ b,
                                              const void* __restrict__ r_ptr, size_t n, void* out) {
  const fe_t r = fe_load(r_ptr, 0);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x) {
    fe_t x = fe_load_rw(a, i), y = fe_load(b, i);
    fe_store(out, i, fe_add<F>(x, fe_mul<F>(r, fe_sub<F>(y, x))));
  }
}

template <class F>
__global__ void __launch_bounds__(256) k_vec_add(const void* __restrict__ a,
                                                 const void* __restrict__ b, size_t n,
                                                 void* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x) {
    fe_store(out, i, fe_add<F>(fe_load(a, i), fe_load(b, i)));
  }
}

template <class F>
__global__ void __launch_bounds__(256) k_vec_mul(const void* __restrict__ a,
                                                 const void* __restrict__ b, size_t n,
                                                 void* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x) {
    fe_store(out, i, fe_mul<F>(fe_load(a, i), fe_load(b, i)));
  }
}

// LogUp fingerprint with the challenge shift folded in (MemorySumcheckInstance::compute_oracles,
// ppsnark.rs:386-435): out[i] = val[i]*gamma + addr[i] + r, where addr == nullptr means the
// memory's own address i (T[i] = mem[i]*gamma + i, `E::Scalar::from(i as u64)` at :394).
template <class F>
__global__ void __launch_bounds__(256) k_logup_hash(const void* __restrict__ val,
                                                    const void* __restrict__ addr,
                                                    const void* __restrict__ gamma_ptr,
                                                    const void* __restrict__ r_ptr, size_t n,
                                                    void* __restrict__ out) {
  const fe_t gamma = fe_load(gamma_ptr, 0), r = fe_load(r_ptr, 0);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x) {
    fe_t a;
    if (addr != nullptr) {
      a = fe_load(addr, i);
    } else {
      fe_t c = fe_zero<F>();
      c.l[0] = (uint32_t)i;
      c.l[1] = (uint32_t)((uint64_t)i >> 32);
      a = fe_to_mont<F>(c);
    }
    fe_store(out, i, fe_add<F>(fe_add<F>(fe_mul<F>(fe_load(val, i), gamma), a), r));
  }
}

// in place on the low half; the caller truncates to n/2 (multilinear.rs:82)
template <class F>
__global__ void __launch_bounds__(256) k_bind_top(void* z, size_t half,
                                                  const void* __restrict__ r_ptr) {
  const fe_t r = fe_load(r_ptr, 0);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half;
       i += (size_t)gridDim.x * blockDim.x) {
    fe_t lo = fe_load_rw(z, i), hi = fe_load_rw(z, i + half);
    fe_store(z, i, fe_add<F>(lo, fe_mul<F>(r, fe_sub<F>(hi, lo))));
  }
}

// the same for up to BIND_MULTI_MAX tables of one length in ONE launch (blockIdx.y = table): a batched sum-check binds
// 16 polynomials per round (ppsnark.rs:960-966) -- sixteen launches per round are pure launch latency once the tables are short
constexpr int BIND_MULTI_MAX = 32;
struct bind_multi_args {
  void* z[BIND_MULTI_MAX];
};
template <class F>
__global__ void __launch_bounds__(256) k_bind_top_multi(bind_multi_args a, size_t half, const void* __restrict__ r_ptr) {
  const fe_t r = fe_load(r_ptr, 0);
  void* z = a.z[blockIdx.y];
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
    fe_t lo = fe_load_rw(z, i), hi = fe_load_rw(z, i + half);
    fe_store(z, i, fe_add<F>(lo, fe_mul<F>(r, fe_sub<F>(hi, lo))));
  }
}

// out[t] = element 0 of table t (the final evaluations of a sum-check: one read-back instead of one per table)
template <class F>
__global__ void __launch_bounds__(BIND_MULTI_MAX) k_gather_heads(bind_multi_args a, int k, void* __restrict__ out) {
  if ((int)threadIdx.x < k) fe_store(out, threadIdx.x, fe_load_rw(a.z[threadIdx.x], 0));
}

// ---- inner-product argument helpers (provider/ipa_pc.rs:174-285, restated without key folding) --
// out[i] = v[i]*x_lo + v[i+half]*x_hi   (a' = a_L r + r^-1 a_R ; b' = b_L r^-1 + r b_R, ipa_pc.rs:244-254)
template <class F>
__global__ void __launch_bounds__(256) k_fold_halves(const void* __restrict__ v, size_t half,
                                                     const void* __restrict__ x_lo,
                                                     const void* __restrict__ x_hi, void* __restrict__ out) {
  const fe_t xl = fe_load(x_lo, 0), xh = fe_load(x_hi, 0);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half;
       i += (size_t)gridDim.x * blockDim.x)
    fe_store(out, i, fe_add<F>(fe_mul<F>(fe_load_rw(v, i), xl), fe_mul<F>(fe_load_rw(v, i + half), xh)));
}
// The folded key of round k is G^(k)_i = sum_m w[i + m nk] G_{i + m nk} over the ORIGINAL key, so
//   L = <a_L, ck_R^(k)> = MSM(original key, sL),  sL[j] = [j & nk/2] a[j mod nk/2] w[j]
//   R = <a_R, ck_L^(k)> = MSM(original key, sR),  sR[j] = [!(j & nk/2)] a[(j mod nk/2) + nk/2] w[j]
// and the key itself is never folded (pedersen.rs:484-497 `fold` is what this replaces).
template <class F>
__global__ void __launch_bounds__(256) k_ipa_scalars(const void* __restrict__ a, const void* __restrict__ w,
                                                     size_t n, size_t nk, void* __restrict__ sL,
                                                     void* __restrict__ sR) {
  const size_t half = nk / 2;
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < n;
       j += (size_t)gridDim.x * blockDim.x) {
    size_t i = j & (half - 1);
    bool hi = (j & half) != 0;
    fe_t wj = fe_load_rw(w, j);
    fe_t prod = fe_mul<F>(fe_load_rw(a, hi ? i : i + half), wj);
    fe_store(sL, j, hi ? prod : fe_zero<F>());
    fe_store(sR, j, hi ? fe_zero<F>() : prod);
  }
}
// w[j] *= (j & nk/2) ? r : r^-1   (ck.fold(&r_inverse, &r): first half r^-1, second half r)
template <class F>
__global__ void __launch_bounds__(256) k_ipa_weights(void* __restrict__ w, size_t n, size_t nk,
                                                     const void* __restrict__ r,
                                                     const void* __restrict__ r_inv) {
  const size_t half = nk / 2;
  const fe_t rr = fe_load(r, 0), ri = fe_load(r_inv, 0);
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < n;
       j += (size_t)gridDim.x * blockDim.x)
    fe_store(w, j, fe_mul<F>(fe_load_rw(w, j), (j & half) ? rr : ri));
}
template <class F>
__global__ void __launch_bounds__(256) k_fill_one(void* __restrict__ w, size_t n) {
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < n;
       j += (size_t)gridDim.x * blockDim.x)
    fe_store(w, j, fe_one<F>());
}

}  // namespace nova
