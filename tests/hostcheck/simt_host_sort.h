// The warp intrinsics and atomics the MSM bucket sort (nova_b200/csrc/msm_sort.cuh) uses beyond what simt_host.h
// supplies: `__shfl_up_sync` and `__ballot_sync` as exchanges through simt_host.h's per-warp slots, `__popc`,
// `__ffs`, and `atomicAdd` on u32 (shared and global memory alike).  Include after simt_host.h, BEFORE the
// headers under test.
#pragma once
#include "simt_host.h"

// every lane of the warp must call it (full mask), as in the kernels under test
inline uint32_t __shfl_up_sync(unsigned, uint32_t v, int delta) {
  simt_block* b = simt_current_block();
  unsigned w = threadIdx.x >> 5, l = threadIdx.x & 31;
  b->slots[w][l] = v;
  b->warps[w]->wait();
  uint32_t r = l >= (unsigned)delta ? b->slots[w][l - delta] : v;
  b->warps[w]->wait();
  return r;
}
// bit l of the result = pred of lane l (every lane of the warp must call it)
inline unsigned __ballot_sync(unsigned, bool pred) {
  simt_block* b = simt_current_block();
  unsigned w = threadIdx.x >> 5, l = threadIdx.x & 31;
  b->slots[w][l] = pred ? 1u : 0u;
  b->warps[w]->wait();
  unsigned r = 0;
  for (unsigned k = 0; k < 32 && w * 32 + k < blockDim.x; k++) r |= b->slots[w][k] << k;
  b->warps[w]->wait();
  return r;
}
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __ffs(unsigned x) { return __builtin_ffs((int)x); }
inline uint32_t atomicAdd(uint32_t* p, uint32_t v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
