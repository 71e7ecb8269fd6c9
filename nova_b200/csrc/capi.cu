// C ABI of nova_b200 (include/nova_b200.h): handles, workspaces, streams, error reporting.
// Template-free: all kernels are reached through the per-field launcher tables (ops.cuh).
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <map>
#include <memory>
#include <mutex>
#include <vector>

#include "../../include/nova_b200.h"
#include "msm_kernels.cuh"
#include "field_kernels.cuh"
#include "ops.cuh"
#include "poly_kernels.cuh"
#include "transcript.cuh"
#include "transcript_batched.cuh"
#include "sumcheck_tail.cuh"

using namespace nova;

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

#define CU(call)                                                                        \
  do {                                                                                  \
    cudaError_t e_ = (call);                                                            \
    if (e_ != cudaSuccess)                                                              \
      return fail(e_ == cudaErrorMemoryAllocation ? B200_E_NOMEM : B200_E_CUDA,         \
                  "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

struct curve_info {
  int base_fid, scalar_fid;
};
const curve_info CURVES[4] = {
    {B200_FIELD_BN254_FQ, B200_FIELD_BN254_FR},   // BN254 G1   (bn256_grumpkin.rs:35-41)
    {B200_FIELD_BN254_FR, B200_FIELD_BN254_FQ},   // Grumpkin   (bn256_grumpkin.rs:80-86)
    {B200_FIELD_PALLAS_FP, B200_FIELD_PALLAS_FQ}, // Pallas     (pasta.rs:33-39)
    {B200_FIELD_PALLAS_FQ, B200_FIELD_PALLAS_FP}, // Vesta      (pasta.rs:41-47)
};
const int FIELD_BITS[4] = {254, 254, 255, 255};

struct device_state {
  std::mutex mu;
  bool ready = false;
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t aux = nullptr;  // short side jobs forked from `stream` and joined through events
  bool pool = true;
} g_dev;

int ensure_init() {
  std::lock_guard<std::mutex> lk(g_dev.mu);
  if (g_dev.ready) {
    CU(cudaSetDevice(g_dev.device));
    return B200_OK;
  }
  int cnt = 0;
  cudaError_t e = cudaGetDeviceCount(&cnt);
  if (e != cudaSuccess || cnt == 0)
    return fail(B200_E_CUDA, "no usable CUDA device (%s); nova_b200 has no CPU fallback",
                e == cudaSuccess ? "count = 0" : cudaGetErrorString(e));
  CU(cudaSetDevice(g_dev.device));
  CU(cudaStreamCreateWithFlags(&g_dev.stream, cudaStreamNonBlocking));
  CU(cudaStreamCreateWithFlags(&g_dev.aux, cudaStreamNonBlocking));
  // b200_dev_alloc / b200_dev_free and the library's own temporaries (dev_buf) come from the device's stream-ordered
  // pool (cudaMallocAsync on the library stream, or on the stream a temporary is used on): a prover allocates and drops dozens of vectors per proof, and
  // cudaMalloc / cudaFree cost milliseconds each and synchronise the device (for HyperKZG 2^22 the pool is worth
  // an order of magnitude per proof).  The pool keeps what it has been given (release threshold = max).  NOVA_B200_POOL=0
  // restores plain cudaMalloc / cudaFree.
  const char* pe = getenv("NOVA_B200_POOL");
  g_dev.pool = !(pe && pe[0] == '0');
  if (g_dev.pool) {
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, g_dev.device) == cudaSuccess) {
      uint64_t keep = UINT64_MAX;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    } else {
      g_dev.pool = false;
      cudaGetLastError();
    }
  }
  g_dev.ready = true;
  return B200_OK;
}

inline cudaStream_t pick_stream(void* stream) { return stream ? (cudaStream_t)stream : g_dev.stream; }

cudaError_t pool_alloc(void** p, size_t bytes, cudaStream_t s) {
  return g_dev.pool ? cudaMallocAsync(p, bytes ? bytes : 1, s) : cudaMalloc(p, bytes ? bytes : 1);
}
cudaError_t pool_free(void* p, cudaStream_t s) { return g_dev.pool ? cudaFreeAsync(p, s) : cudaFree(p); }

// Scratch owned by one call, allocated and freed in the order of the stream `s` that uses it (pool_alloc).
struct dev_buf {
  void* p = nullptr;
  cudaStream_t s;
  explicit dev_buf(cudaStream_t st) : s(st) {}
  dev_buf(const dev_buf&) = delete;
  dev_buf& operator=(const dev_buf&) = delete;
  ~dev_buf() {
    if (p) pool_free(p, s);
  }
  int alloc(size_t bytes) {
    CU(pool_alloc(&p, bytes, s));
    return B200_OK;
  }
};

// ---------------------------------------------------------------------------------------------
// commitment-key context
// ---------------------------------------------------------------------------------------------
struct workspace {
  size_t cap_n = 0;  // scalars the buffers are sized for
  void* scalars = nullptr;
  int32_t* digits = nullptr;
  uint32_t *sortctl = nullptr, *start = nullptr;
  uint64_t *entries = nullptr, *entries_tmp = nullptr;
  unsigned long long* look = nullptr;  // look-back words of the radix passes
  uint32_t sort_epoch = 0;             // last look-back tag used on these buffers
  void *buckets = nullptr, *parts = nullptr, *rparts = nullptr, *sumscratch = nullptr;
  uint32_t* pkeys = nullptr;
  uint32_t* heavy = nullptr;
  uint32_t heavy_cap = 0;
  void* hparts = nullptr;
  void* d_out = nullptr;   // result slots (device)
  void* h_out = nullptr;   // pinned mirror
  size_t out_slots = 0;
  uint32_t* idx32 = nullptr;
  size_t idx_cap = 0;
  // stream hand-off: the last stream that enqueued work on these buffers and an event recorded after it.  A call
  // that arrives on ANOTHER stream waits for that event first (two *_dev calls on one key with different caller
  // streams, or a *_dev call followed by a host-pointer call on the library stream, never overlap on the buffers).
  cudaStream_t last_stream = nullptr;
  cudaEvent_t busy = nullptr;
  void release() {
    if (busy) cudaEventDestroy(busy);
    void* ptrs[] = {scalars, digits, sortctl, start, entries, entries_tmp, look, buckets,
                    parts, rparts, sumscratch, pkeys, heavy, hparts, d_out, idx32};
    for (void* p : ptrs)
      if (p) cudaFree(p);
    if (h_out) cudaFreeHost(h_out);
    *this = workspace();
  }
};

struct ck_ctx {
  std::mutex mu;
  int curve = 0;
  size_t n = 0;       // usable bases
  size_t stride = 0;  // points per table = n (+1 when the blinding generator h is present)
  bool has_h = false;
  int c = 0, W = 0, F = 0, G = 0;
  uint32_t B = 0;
  int m = 4;
  void* tables = nullptr;  // [F][n] affine
  workspace ws;
  // extra (stream, workspace) lanes for calls that carry several independent MSMs
  // (b200_commit_many_dev, b200_msm_batch): the latency-bound tails of short MSMs overlap with
  // the next vector's sort / accumulate, and host->device staging overlaps with compute
  struct lane {
    workspace ws;
    cudaStream_t s = nullptr;
    cudaEvent_t done = nullptr;
  };
  static constexpr int NLANES = 4;
  lane lanes[NLANES];
  // host-pointer calls (b200_msm / b200_commit / b200_msm_small) each take one of these slots -- own workspace, own
  // stream pair -- and hold only the slot's mutex: the 4-7 commitments the reference issues concurrently from rayon
  // threads (src/spartan/ppsnark.rs:457-470, src/r1cs/mod.rs:509-512) overlap on the device (uploads, sorts and the
  // latency-bound tails of one call under the accumulation of another) instead of queueing on one key-wide mutex.
  struct host_slot {
    std::mutex mu;
    workspace ws;
    cudaStream_t s = nullptr, side = nullptr;
  };
  static constexpr int NSLOTS = 4;
  host_slot slots[NSLOTS];
  unsigned next_slot = 0;  // guarded by mu
  // Keys wide enough for 20-bit windows also carry 17-bit-window tables over their first 2^21
  // bases: the same key commits vectors of very different lengths (W, E, T, the halving
  // polynomials of HyperKZG, hyperkzg.rs:1083-1100), and a short MSM should not pay the
  // 2^19-bucket reduction of the wide tables.
  std::shared_ptr<ck_ctx> small;
  ~ck_ctx() {
    if (tables) cudaFree(tables);
    ws.release();
    for (lane& l : lanes) {
      l.ws.release();
      if (l.done) cudaEventDestroy(l.done);
      if (l.s) cudaStreamDestroy(l.s);
    }
    for (host_slot& h : slots) {
      h.ws.release();
      if (h.s) cudaStreamDestroy(h.s);
      if (h.side) cudaStreamDestroy(h.side);
    }
  }
};

// ---- optional per-stage device timing + launch accounting (for bench.py's roofline) ---------
enum { ST_DIGITS = 0, ST_SORT, ST_ACCUMULATE, ST_FIXUP, ST_REDUCE, ST_COUNT };
// sort: the bucket starts (+ one per radix pass, added per call); reduce: merge + final (+ one per level, likewise)
const int STAGE_KERNELS[ST_COUNT] = {1, 1, 1, 3, 2};
struct profile_state {
  std::mutex mu;
  bool enabled = false;
  // a ring of event sets, so that the host may run PROF_RING - 1 MSMs ahead of the device while
  // timing is on (folding set k waits for the MSM that used it PROF_RING calls ago)
  static constexpr int PROF_RING = 4;
  cudaEvent_t ev[PROF_RING][ST_COUNT + 1] = {};
  bool have_events = false;
  bool pending[PROF_RING] = {};  // event set not folded in yet
  int next = 0;
  double ms[ST_COUNT] = {};    // accumulated
  uint64_t msms = 0;
  uint64_t launches = 0;       // kernels launched by this library (always counted)
} g_prof;

void prof_fold_set_locked(int k) {  // caller holds g_prof.mu
  if (!g_prof.pending[k]) return;
  if (cudaEventSynchronize(g_prof.ev[k][ST_COUNT]) == cudaSuccess) {
    for (int i = 0; i < ST_COUNT; i++) {
      float t = 0;
      if (cudaEventElapsedTime(&t, g_prof.ev[k][i], g_prof.ev[k][i + 1]) == cudaSuccess) g_prof.ms[i] += t;
    }
    g_prof.msms++;
  }
  g_prof.pending[k] = false;
}
void prof_fold_locked() {
  for (int k = 0; k < profile_state::PROF_RING; k++) prof_fold_set_locked(k);
}

void count_launch(int k) {
  std::lock_guard<std::mutex> lk(g_prof.mu);
  g_prof.launches += k;
}

std::mutex g_handles_mu;
std::map<uint64_t, std::shared_ptr<ck_ctx>> g_handles;
uint64_t g_next_handle = 1;

std::shared_ptr<ck_ctx> get_ck(uint64_t h) {
  std::lock_guard<std::mutex> lk(g_handles_mu);
  auto it = g_handles.find(h);
  return it == g_handles.end() ? nullptr : it->second;
}

constexpr size_t XYZZ_BYTES = 144;  // 36 words (pa29); pa32 uses the first 128
constexpr int SUM_THREADS = NUM_SMS * 128;
constexpr int L_MIN = 32;        // sizing bound of the segment length
constexpr int L_FLOOR_DEFAULT = 16;  // default floor: 2^17-pair shards run faster with 16 than with 32
// accumulate threads are sized to ~3 full waves of NUM_SMS SMs x 16 warps x 32 lanes
constexpr size_t ACC_THREADS = (size_t)NUM_SMS * 16 * 32 * 3;
constexpr uint32_t HEAVY_PARTS = 96;  // buckets spanning more segments than this get a block

size_t acc_threads() {
  // tuning hook: NOVA_B200_ACC_WAVES overrides the number of full-GPU waves of accumulate threads
  static const size_t threads = [] {
    const char* e = getenv("NOVA_B200_ACC_WAVES");
    double w = e ? atof(e) : 0.0;
    return w > 0.0 ? (size_t)((double)NUM_SMS * 16 * 32 * w) : ACC_THREADS;
  }();
  return threads;
}
size_t acc_lmin() {
  // tuning hook: NOVA_B200_ACC_LMIN lowers the floor of the segment length for small MSMs (8 .. L_MIN)
  static const size_t lmin = [] {
    const char* e = getenv("NOVA_B200_ACC_LMIN");
    int v = e ? atoi(e) : L_FLOOR_DEFAULT;
    return (size_t)(v < 8 ? 8 : (v > L_MIN ? L_MIN : v));
  }();
  return lmin;
}
int segment_len(size_t entries) {
  size_t L = (entries + acc_threads() - 1) / acc_threads();
  return (int)(L < acc_lmin() ? acc_lmin() : L);
}
// upper bound of the number of segments of ANY MSM with at most `entries` entries: L grows with the entry count
// once the thread target is met, so the count saturates at the thread target
size_t max_segments(size_t entries) {
  size_t by_floor = (entries + acc_lmin() - 1) / acc_lmin();
  size_t cap = acc_threads() + 256;
  return by_floor < cap ? by_floor : cap;
}

// order stream `s` after the last user of `w` (no-op when that was `s` itself)
int ws_acquire(workspace& w, cudaStream_t s) {
  if (w.busy && w.last_stream != s) CU(cudaStreamWaitEvent(s, w.busy, 0));
  return B200_OK;
}
int ws_release(workspace& w, cudaStream_t s) {
  if (!w.busy) CU(cudaEventCreateWithFlags(&w.busy, cudaEventDisableTiming));
  CU(cudaEventRecord(w.busy, s));
  w.last_stream = s;
  return B200_OK;
}

int ensure_workspace(ck_ctx& ck, workspace& w, size_t n, size_t out_slots) {
  if (out_slots > w.out_slots) {
    if (w.d_out) cudaFree(w.d_out);
    if (w.h_out) cudaFreeHost(w.h_out);
    w.d_out = w.h_out = nullptr;
    CU(cudaMalloc(&w.d_out, out_slots * 96));
    CU(cudaMallocHost(&w.h_out, out_slots * 96));
    w.out_slots = out_slots;
  }
  if (n <= w.cap_n) return B200_OK;
  // entries, bucket starts and the sort's positions are 32-bit (table indices 31-bit)
  if (n * (size_t)ck.W > 0x7FFFFFFFu)
    return fail(B200_E_RANGE, "%zu scalars x %d windows exceed 2^31 bucket entries", n, ck.W);
  // grow: release the size-dependent buffers and reallocate (after draining any asynchronous
  // *_dev work that may still be using them)
  CU(cudaDeviceSynchronize());
  void** szbufs[] = {&w.scalars, (void**)&w.digits, (void**)&w.entries, (void**)&w.entries_tmp, (void**)&w.look,
                     &w.parts, (void**)&w.pkeys, (void**)&w.heavy, &w.hparts};
  for (void** p : szbufs)
    if (*p) {
      cudaFree(*p);
      *p = nullptr;
    }
  size_t K = (size_t)ck.G * ck.B;
  size_t entries = n * (size_t)ck.W;
  size_t nseg = max_segments(entries);  // upper bound over every L this key will use
  w.heavy_cap = (uint32_t)(nseg / HEAVY_PARTS + 2);
  CU(cudaMalloc((void**)&w.heavy, ((size_t)w.heavy_cap + 1) * 4));
  CU(cudaMalloc(&w.hparts, (size_t)w.heavy_cap * HEAVY_SPLIT * XYZZ_BYTES));
  CU(cudaMalloc(&w.scalars, n * 32));
  CU(cudaMalloc((void**)&w.digits, entries * sizeof(int32_t)));
  CU(cudaMalloc((void**)&w.entries, entries * sizeof(uint64_t)));
  CU(cudaMalloc((void**)&w.entries_tmp, entries * sizeof(uint64_t)));
  // zeroed once: a zero word carries no valid tag (see msm_sort.cuh)
  const size_t look_bytes = (entries + SORT_TILE - 1) / SORT_TILE * SORT_BINS * sizeof(unsigned long long);
  CU(cudaMalloc((void**)&w.look, look_bytes));
  CU(cudaMemset(w.look, 0, look_bytes));
  w.sort_epoch = 0;
  CU(cudaMalloc(&w.parts, 2 * nseg * XYZZ_BYTES));
  CU(cudaMalloc((void**)&w.pkeys, 2 * nseg * sizeof(uint32_t)));
  if (!w.sortctl) {
    CU(cudaMalloc((void**)&w.sortctl, SORT_CTL_WORDS * 4));
    CU(cudaMalloc((void**)&w.start, (K + 1) * 4));
    CU(cudaMalloc(&w.buckets, K * XYZZ_BYTES));
    // chunk partials of the running-sum reduce, or [G][NR+NC] row/column sums + [G][2] of the
    // two-level reduce (NR + NC <= 2 * sqrt(2B) + 1 <= B / m + 514)
    CU(cudaMalloc(&w.rparts, ((size_t)ck.G * (ck.B / ck.m + 4096)) * XYZZ_BYTES));
    CU(cudaMalloc(&w.sumscratch, (size_t)SUM_THREADS * XYZZ_BYTES));
  }
  w.cap_n = n;
  return B200_OK;
}

int ensure_workspace(ck_ctx& ck, size_t n, size_t out_slots) {
  return ensure_workspace(ck, ck.ws, n, out_slots);
}

msm_plan make_plan(ck_ctx& ck, workspace& ws, size_t base_offset, size_t n) {
  msm_plan p;
  p.n = n;
  p.n_ck = ck.stride;
  p.base_offset = base_offset;
  p.blind_i = SIZE_MAX;
  p.h_index = ck.n;
  p.c = ck.c;
  p.W = ck.W;
  p.G = ck.G;
  p.B = ck.B;
  p.L = segment_len(n * (size_t)ck.W);
  p.m = ck.m;
  p.heavy = ws.heavy;
  p.heavy_min = HEAVY_PARTS * (uint32_t)p.L;
  p.heavy_cap = ws.heavy_cap;
  p.hparts = ws.hparts;
  p.digits = ws.digits;
  p.sortctl = ws.sortctl;
  p.sp = make_sort_plan((uint64_t)ck.G * ck.B);
  p.sort_tag = 0;  // set per call by enqueue_msm
  p.look = ws.look;
  p.start = ws.start;
  p.entries = ws.entries;
  p.entries_tmp = ws.entries_tmp;
  p.buckets = ws.buckets;
  p.parts = ws.parts;
  p.pkeys = ws.pkeys;
  p.rparts = ws.rparts;
  return p;
}

// enqueue one full-width MSM on `s`; scalars and out are device pointers
int enqueue_msm(ck_ctx& ck, workspace& ws, size_t base_offset, const void* d_scalars, size_t n,
                void* d_out, cudaStream_t s, int small_elem_bytes = 0, bool blinded = false,
                bool digits_done = false, const msm_peer* peer = nullptr, bool profile_ok = true) {
  // blinded: d_scalars holds n-1 vector entries followed by r, whose base is h
  // digits_done: ws.digits and the radix histograms of ws.sortctl were already filled chunk by chunk
  // (b200_witness_append, the chunked upload of b200_commit)
  const field_ops* sops = ops_for_field(CURVES[ck.curve].scalar_fid);
  const field_ops* bops = ops_for_field(CURVES[ck.curve].base_fid);
  {
    int arc = ws_acquire(ws, s);
    if (arc) return arc;
  }
  if (n == 0) {  // identity (msm.rs:228-230): z = 0
    if (peer && peer->world > 1) {  // the peers still wait for this rank's (empty) partial
      msm_plan p0 = make_plan(ck, ws, base_offset, 0);
      p0.peer = *peer;
      bops->exchange_identity(s, p0, d_out);
      count_launch(1);
      CU(cudaGetLastError());
      return B200_OK;
    }
    CU(cudaMemsetAsync(d_out, 0, 96, s));
    return B200_OK;
  }
  msm_plan p = make_plan(ck, ws, base_offset, n);
  if (peer) p.peer = *peer;
  if (blinded) p.blind_i = n - 1;
  // histograms and tile counters; only the tile counters when the digit stage already ran
  if (!digits_done) CU(cudaMemsetAsync(p.sortctl, 0, SORT_CTL_WORDS * 4, s));
  else CU(cudaMemsetAsync(p.sortctl + SORT_PASSES_MAX * SORT_BINS, 0, SORT_PASSES_MAX * 4, s));
  CU(cudaMemsetAsync(p.heavy, 0, 4, s));
  // look-back tags: fresh for every pass of every call on these buffers; the (practically unreachable) wrap of the
  // 31-bit tag space re-zeroes the words so that no stale word can carry a live tag
  if (ws.sort_epoch > 0x7FFFFFFFu - SORT_PASSES_MAX) {
    CU(cudaMemsetAsync(ws.look, 0, (ws.cap_n * (size_t)ck.W + SORT_TILE - 1) / SORT_TILE * SORT_BINS * 8, s));
    ws.sort_epoch = 0;
  }
  p.sort_tag = ws.sort_epoch + 1;
  ws.sort_epoch += (uint32_t)p.sp.passes;
  std::lock_guard<std::mutex> plk(g_prof.mu);
  const bool prof = g_prof.enabled && profile_ok;  // (the stage events belong to the library's own device)
  const int pset = g_prof.next;
  if (prof) {
    if (!g_prof.have_events) {
      for (auto& set : g_prof.ev)
        for (auto& e : set) CU(cudaEventCreate(&e));
      g_prof.have_events = true;
    }
    prof_fold_set_locked(pset);
    g_prof.next = (pset + 1) % profile_state::PROF_RING;
  }
#define STAGE_MARK(i) \
  if (prof) CU(cudaEventRecord(g_prof.ev[pset][i], s))
  STAGE_MARK(ST_DIGITS);
  if (digits_done)
    ;
  else if (small_elem_bytes)
    msm_digits_small(s, d_scalars, small_elem_bytes, p);
  else
    sops->digits(s, d_scalars, p);
  STAGE_MARK(ST_SORT);
  const int sort_launches = msm_sort(s, p);
  STAGE_MARK(ST_ACCUMULATE);
  bops->accumulate(s, ck.tables, p);
  STAGE_MARK(ST_FIXUP);
  bops->fixup(s, p);
  STAGE_MARK(ST_REDUCE);
  bops->reduce(s, p, d_out);
  STAGE_MARK(ST_COUNT);
#undef STAGE_MARK
  if (prof) g_prof.pending[pset] = true;
  for (int i = 0; i < ST_COUNT; i++) g_prof.launches += STAGE_KERNELS[i];
  g_prof.launches += sort_launches - STAGE_KERNELS[ST_SORT];  // the radix passes
  g_prof.launches += (ck.c - 1 + 3) / 4 - 1;  // the hierarchical reduction launches one kernel per level below the top
  CU(cudaGetLastError());
  return ws_release(ws, s);
}

int enqueue_msm(ck_ctx& ck, size_t base_offset, const void* d_scalars, size_t n, void* d_out,
                cudaStream_t s, int small_elem_bytes = 0, bool blinded = false) {
  return enqueue_msm(ck, ck.ws, base_offset, d_scalars, n, d_out, s, small_elem_bytes, blinded);
}

constexpr size_t SMALL_KEY_MAX = (size_t)1 << 21;
constexpr int SMALL_KEY_WINDOW = 17;

int choose_window(size_t n) {
  int lg = 0;
  while (((size_t)1 << lg) < n) lg++;
  int c = lg;
  if (c < 8) c = 8;
  if (c > 16) c = 16;
  // large keys: 13 windows of 20 bits instead of 16 of 16 (-19 % bucket additions); the 2^19-bucket
  // reduction costs ~1 ms, so this only pays from 2^22 points
  if (lg >= 22) c = 20;
  else if (lg >= 19) c = 17;  // 15 windows; the 65536-bucket reduction still fits the fast tail
  return c;
}

// b of y^2 = x^3 + b per curve id (bn256_grumpkin.rs:35-41,80-86; pasta.rs:33-47)
constexpr int CURVE_B_SMALL[4] = {3, -17, 5, 5};

// first_bad != nullptr: validate the raw points (bases, then h) where they land in HBM, before the tables are
// built from them; an invalid point ends the registration with B200_E_POINT and its index in *first_bad.
int register_key(int curve_id, const void* bases, bool bases_on_device, size_t n, const void* h,
                 int window_bits, bool expand, std::shared_ptr<ck_ctx>& out, size_t* first_bad = nullptr,
                 cudaStream_t st = nullptr, size_t src_pitch_points = 0, size_t src_block_points = 0) {
  // st: the stream of the CURRENT device the key is built on (nullptr = the library stream).
  // src_pitch_points / src_block_points != 0: `bases` is a strided view -- block i of src_block_points points sits at
  // bases + i * src_pitch_points * 64 (the block-cyclic slice one device of a multi-GPU key owns); the last block
  // may be short.
  if (!st) st = g_dev.stream;
  if (curve_id < 0 || curve_id > 3) return fail(B200_E_ARG, "unknown curve id %d", curve_id);
  if (bases == nullptr || n == 0) return fail(B200_E_ARG, "empty commitment key");
  if (window_bits != 0 && (window_bits < 2 || window_bits > 24))
    return fail(B200_E_ARG, "window_bits %d out of range [2,24]", window_bits);
  auto ck = std::make_shared<ck_ctx>();
  ck->curve = curve_id;
  ck->n = n;
  ck->has_h = h != nullptr;
  ck->stride = n + (h ? 1 : 0);
  ck->c = window_bits ? window_bits : choose_window(n);
  int bits = FIELD_BITS[CURVES[curve_id].scalar_fid];
  ck->W = (bits + ck->c - 1) / ck->c;
  ck->F = expand ? ck->W : 1;
  ck->G = expand ? 1 : ck->W;
  ck->B = 1u << (ck->c - 1);
  ck->m = ck->B >= 4 ? 4 : 1;
  if ((size_t)ck->F * ck->stride >= ((size_t)1 << 31))
    return fail(B200_E_RANGE, "key too large for 31-bit table indices (%zu x %d)", n, ck->F);
  CU(cudaMalloc(&ck->tables, (size_t)ck->F * ck->stride * 64));
  const cudaMemcpyKind kind = bases_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  if (src_block_points == 0) {
    CU(cudaMemcpyAsync(ck->tables, bases, n * 64, kind, st));
  } else {
    const size_t full = n / src_block_points, rest = n % src_block_points;
    if (full)
      CU(cudaMemcpy2DAsync(ck->tables, src_block_points * 64, bases, src_pitch_points * 64, src_block_points * 64, full,
                           kind, st));
    if (rest)
      CU(cudaMemcpyAsync((char*)ck->tables + full * src_block_points * 64,
                         (const char*)bases + full * src_pitch_points * 64, rest * 64, kind, st));
  }
  if (h)
    CU(cudaMemcpyAsync((char*)ck->tables + n * 64, h, 64, cudaMemcpyHostToDevice, st));
  if (first_bad) {
    *first_bad = SIZE_MAX;
    dev_buf flag(st);
    if (int rc = flag.alloc(4)) return rc;
    CU(cudaMemsetAsync(flag.p, 0xFF, 4, st));
    ops_for_field(CURVES[curve_id].base_fid)
        ->on_curve(st, ck->tables, ck->stride, CURVE_B_SMALL[curve_id], (uint32_t*)flag.p);
    count_launch(1);
    CU(cudaGetLastError());
    uint32_t bad = 0;
    CU(cudaMemcpyAsync(&bad, flag.p, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (bad != 0xFFFFFFFFu) {
      *first_bad = bad;
      return fail(B200_E_POINT, "key point %u%s has a non-canonical coordinate or is not on the curve", bad,
                  (h && bad == n) ? " (the blinding generator)" : "");
    }
  }
  {  // converts table 0 to the kernels' table format and builds tables 1..F-1
    const field_ops* bops = ops_for_field(CURVES[curve_id].base_fid);
    bops->expand_key(st, ck->tables, ck->stride, ck->F, ck->c * ck->G);
    CU(cudaGetLastError());
  }
  CU(cudaStreamSynchronize(st));
  if (expand && window_bits == 0 && ck->c >= 20) {
    size_t ns = n < SMALL_KEY_MAX ? n : SMALL_KEY_MAX;
    if (src_block_points) return fail(B200_E_ARG, "strided keys carry one table set");
    int rc = register_key(curve_id, bases, bases_on_device, ns, h, SMALL_KEY_WINDOW, true, ck->small, nullptr, st);
    if (rc) return rc;
  }
  out = ck;
  return B200_OK;
}

// the table set an MSM over ck[base_offset .. base_offset + n) runs on
ck_ctx& route(ck_ctx& ck, size_t base_offset, size_t n) {
  if (ck.small && base_offset + n <= ck.small->n) return *ck.small;
  return ck;
}

template <class Fn>
int with_field(int field_id, Fn fn) {
  int rc = ensure_init();
  if (rc) return rc;
  const field_ops* ops = ops_for_field(field_id);
  if (!ops) return fail(B200_E_ARG, "unknown field id %d", field_id);
  return fn(ops);
}

inline size_t pad256(size_t b) { return (b + 255) & ~(size_t)255; }

// One device region of a host-pointer call: `src` is uploaded into it before the device form runs, and `dst` is
// downloaded from it afterwards.  The region holds at least `bytes`, `src_bytes` and `dst_bytes`.
struct host_piece {
  const void* src;
  size_t src_bytes;
  void* dst;
  size_t dst_bytes;
  size_t bytes;
};
inline host_piece up(const void* src, size_t bytes) { return {src, bytes, nullptr, 0, 0}; }
inline host_piece down(void* dst, size_t bytes, size_t region = 0) { return {nullptr, 0, dst, bytes, region}; }

// The host-pointer form of a device entry: one pool block on the library stream, one 256-byte aligned region per
// piece, the uploads, dev(d, s) with d[i] the region of piece i, the downloads, one synchronisation.  A piece without
// a host pointer gives dev a null pointer, so dev's own checks decide the status; any other piece gets a region, even
// for 0 bytes.  When dev fails its status is returned and nothing is downloaded.
template <class Fn>
int via_device(const std::vector<host_piece>& pieces, Fn dev) {
  auto region = [](const host_piece& p) {
    return pad256(std::max({p.src_bytes, p.dst_bytes, p.bytes, (size_t)1}));
  };
  size_t total = 0;
  for (const host_piece& p : pieces)
    if (p.src || p.dst) total += region(p);
  const cudaStream_t s = g_dev.stream;
  dev_buf buf(s);
  int rc = buf.alloc(total);
  if (rc) return rc;
  std::vector<void*> d(pieces.size(), nullptr);
  char* next = (char*)buf.p;
  for (size_t i = 0; i < pieces.size(); i++) {
    const host_piece& p = pieces[i];
    if (!p.src && !p.dst) continue;
    d[i] = next;
    next += region(p);
    if (p.src && p.src_bytes) CU(cudaMemcpyAsync(d[i], p.src, p.src_bytes, cudaMemcpyHostToDevice, s));
  }
  if ((rc = dev(d.data(), s))) return rc;
  for (size_t i = 0; i < pieces.size(); i++)
    if (pieces[i].dst && pieces[i].dst_bytes)
      CU(cudaMemcpyAsync(pieces[i].dst, d[i], pieces[i].dst_bytes, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  return B200_OK;
}

}  // namespace

// =============================================================================================
extern "C" {

const char* b200_last_error(void) { return g_err; }
const char* b200_version(void) { return "nova_b200 0.1 (sm_90a)"; }

int b200_init(int device) {
  {
    std::lock_guard<std::mutex> lk(g_dev.mu);
    if (!g_dev.ready) g_dev.device = device;
  }
  return ensure_init();
}

int b200_device_count(int* count) {
  if (!count) return fail(B200_E_ARG, "null count");
  cudaError_t e = cudaGetDeviceCount(count);
  if (e != cudaSuccess) {
    *count = 0;
    return fail(B200_E_CUDA, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
  }
  return B200_OK;
}

int b200_host_alloc(size_t bytes, void** ptr) {
  int rc = ensure_init();
  if (rc) return rc;
  CU(cudaMallocHost(ptr, bytes ? bytes : 1));
  return B200_OK;
}
int b200_host_free(void* ptr) {
  CU(cudaFreeHost(ptr));
  return B200_OK;
}
int b200_dev_alloc(size_t bytes, void** dptr) {
  int rc = ensure_init();
  if (rc) return rc;
  CU(pool_alloc(dptr, bytes, g_dev.stream));
  return B200_OK;
}
int b200_dev_free(void* dptr) {
  if (!dptr) return B200_OK;
  int rc = ensure_init();
  if (rc) return rc;
  CU(pool_free(dptr, g_dev.stream));
  return B200_OK;
}
int b200_memcpy_h2d(void* dptr, const void* hptr, size_t bytes) {
  int rc = ensure_init();
  if (rc) return rc;
  CU(cudaMemcpyAsync(dptr, hptr, bytes, cudaMemcpyHostToDevice, g_dev.stream));
  CU(cudaStreamSynchronize(g_dev.stream));
  return B200_OK;
}
int b200_memcpy_d2h(void* hptr, const void* dptr, size_t bytes) {
  int rc = ensure_init();
  if (rc) return rc;
  CU(cudaMemcpyAsync(hptr, dptr, bytes, cudaMemcpyDeviceToHost, g_dev.stream));
  CU(cudaStreamSynchronize(g_dev.stream));
  return B200_OK;
}
int b200_memcpy_d2d(void* dst, const void* src, size_t bytes, void* stream) {
  int rc = ensure_init();
  if (rc) return rc;
  if (bytes == 0) return B200_OK;
  if (!dst || !src) return fail(B200_E_ARG, "null pointer");
  CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, pick_stream(stream)));
  return B200_OK;
}
int b200_memset_dev(void* dptr, int byte, size_t bytes, void* stream) {
  int rc = ensure_init();
  if (rc) return rc;
  if (bytes == 0) return B200_OK;
  if (!dptr) return fail(B200_E_ARG, "null pointer");
  CU(cudaMemsetAsync(dptr, byte, bytes, pick_stream(stream)));
  return B200_OK;
}
int b200_sync(void) {
  int rc = ensure_init();
  if (rc) return rc;
  CU(cudaDeviceSynchronize());
  return B200_OK;
}

// ---- profiling / accounting --------------------------------------------------------------------
int b200_profile_enable(int on) {
  std::lock_guard<std::mutex> lk(g_prof.mu);
  g_prof.enabled = on != 0;
  return B200_OK;
}
int b200_profile_reset(void) {
  std::lock_guard<std::mutex> lk(g_prof.mu);
  prof_fold_locked();
  for (double& m : g_prof.ms) m = 0;
  g_prof.msms = 0;
  g_prof.launches = 0;
  return B200_OK;
}
int b200_profile_read(double* stage_ms, int nstages, uint64_t* msms, uint64_t* launches) {
  std::lock_guard<std::mutex> lk(g_prof.mu);
  prof_fold_locked();
  for (int i = 0; i < nstages && i < ST_COUNT; i++)
    if (stage_ms) stage_ms[i] = g_prof.ms[i];
  if (msms) *msms = g_prof.msms;
  if (launches) *launches = g_prof.launches;
  return B200_OK;
}

int b200_jacobian_sum_dev(int curve_id, const void* d_points, size_t k, void* d_out, void* stream) {
  int rc = ensure_init();
  if (rc) return rc;
  if (curve_id < 0 || curve_id > 3) return fail(B200_E_ARG, "unknown curve id %d", curve_id);
  if (!d_out || (k && !d_points)) return fail(B200_E_ARG, "null pointer");
  const field_ops* bops = ops_for_field(CURVES[curve_id].base_fid);
  bops->jacobian_sum(pick_stream(stream), d_points, (int)k, d_out);
  {
    std::lock_guard<std::mutex> lk(g_prof.mu);
    g_prof.launches += 1;
  }
  CU(cudaGetLastError());
  return B200_OK;
}

// ---- keys -------------------------------------------------------------------------------------
int b200_ck_register(int curve_id, const void* bases, size_t n, const void* h, int window_bits,
                     uint64_t* handle) {
  int rc = ensure_init();
  if (rc) return rc;
  if (!handle) return fail(B200_E_ARG, "null handle pointer");
  std::shared_ptr<ck_ctx> ck;
  rc = register_key(curve_id, bases, false, n, h, window_bits, true, ck);
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g_handles_mu);
  *handle = g_next_handle++;
  g_handles[*handle] = ck;
  return B200_OK;
}

int b200_ck_register_checked(int curve_id, const void* bases, size_t n, const void* h, int window_bits,
                             uint64_t* handle, size_t* first_bad) {
  int rc = ensure_init();
  if (rc) return rc;
  if (!handle || !first_bad) return fail(B200_E_ARG, "null pointer");
  *handle = 0;
  std::shared_ptr<ck_ctx> ck;
  rc = register_key(curve_id, bases, false, n, h, window_bits, true, ck, first_bad);
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g_handles_mu);
  *handle = g_next_handle++;
  g_handles[*handle] = ck;
  return B200_OK;
}

int b200_ck_setup_synthetic(int curve_id, const void* gen_affine, uint64_t k0, size_t n, int with_h,
                            int window_bits, uint64_t* handle) {
  int rc = ensure_init();
  if (rc) return rc;
  if (curve_id < 0 || curve_id > 3) return fail(B200_E_ARG, "unknown curve id %d", curve_id);
  if (!gen_affine || !handle || n == 0) return fail(B200_E_ARG, "bad argument");
  size_t total = n + (with_h ? 1 : 0);
  dev_buf bases(g_dev.stream), gen(g_dev.stream);
  if ((rc = bases.alloc(total * 64))) return rc;
  if ((rc = gen.alloc(64))) return rc;
  CU(cudaMemcpyAsync(gen.p, gen_affine, 64, cudaMemcpyHostToDevice, g_dev.stream));
  const field_ops* bops = ops_for_field(CURVES[curve_id].base_fid);
  bops->index_bases(g_dev.stream, bases.p, total, gen.p, k0);
  CU(cudaGetLastError());
  std::vector<char> h(64);
  if (with_h)
    CU(cudaMemcpyAsync(h.data(), (char*)bases.p + n * 64, 64, cudaMemcpyDeviceToHost, g_dev.stream));
  CU(cudaStreamSynchronize(g_dev.stream));
  std::shared_ptr<ck_ctx> ck;
  rc = register_key(curve_id, bases.p, true, n, with_h ? h.data() : nullptr, window_bits, true, ck);
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g_handles_mu);
  *handle = g_next_handle++;
  g_handles[*handle] = ck;
  return B200_OK;
}

int b200_ck_setup_tau(int curve_id, const void* gen_affine, const void* tau_mont, size_t n, int window_bits,
                      uint64_t* handle) {
  int rc = ensure_init();
  if (rc) return rc;
  if (curve_id < 0 || curve_id > 3) return fail(B200_E_ARG, "unknown curve id %d", curve_id);
  if (!gen_affine || !tau_mont || !handle || n == 0) return fail(B200_E_ARG, "bad argument");
  dev_buf bases(g_dev.stream), gen(g_dev.stream), tau(g_dev.stream), pw(g_dev.stream);
  if ((rc = bases.alloc(n * 64)) || (rc = gen.alloc(64)) || (rc = tau.alloc(32)) || (rc = pw.alloc(n * 32))) return rc;
  CU(cudaMemcpyAsync(gen.p, gen_affine, 64, cudaMemcpyHostToDevice, g_dev.stream));
  CU(cudaMemcpyAsync(tau.p, tau_mont, 32, cudaMemcpyHostToDevice, g_dev.stream));
  ops_for_field(CURVES[curve_id].scalar_fid)->powers_canonical(g_dev.stream, tau.p, n, pw.p);
  ops_for_field(CURVES[curve_id].base_fid)->scalar_bases(g_dev.stream, bases.p, n, gen.p, pw.p);
  count_launch(2);
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(g_dev.stream));
  std::shared_ptr<ck_ctx> ck;
  rc = register_key(curve_id, bases.p, true, n, nullptr, window_bits, true, ck);
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g_handles_mu);
  *handle = g_next_handle++;
  g_handles[*handle] = ck;
  return B200_OK;
}

int b200_ck_export_bases(uint64_t handle, size_t offset, size_t n, void* out_host) {
  int rc = ensure_init();
  if (rc) return rc;
  auto ck = get_ck(handle);
  if (!ck) return fail(B200_E_HANDLE, "unknown key handle %llu", (unsigned long long)handle);
  if (offset + n > ck->n) return fail(B200_E_RANGE, "export [%zu, %zu) exceeds key length %zu", offset, offset + n, ck->n);
  if (n == 0) return B200_OK;
  if (!out_host) return fail(B200_E_ARG, "null pointer");
#if defined(NOVA_MSM_ARITH29)
  return fail(B200_E_ARG, "b200_ck_export_bases: table 0 is not in the boundary format in this build");
#else
  std::lock_guard<std::mutex> lk(ck->mu);
  CU(cudaMemcpyAsync(out_host, (const char*)ck->tables + offset * 64, n * 64, cudaMemcpyDeviceToHost, g_dev.stream));
  CU(cudaStreamSynchronize(g_dev.stream));
  return B200_OK;
#endif
}

// ck_derive_by_address: reads only the source's table 0 and its h slot, through the shared_ptr (a concurrent release
// is safe) and without the source's workspace or mutex; every temporary comes from the stream-ordered pool, sized by m
// and table_size.
int b200_ck_derive_by_address_dev(uint64_t ck_handle, const uint32_t* d_addresses, size_t m, size_t table_size,
                                  int window_bits, uint64_t* out_handle, size_t* first_bad, void* stream) {
  int rc = ensure_init();
  if (rc) return rc;
  if (!out_handle || (m && !d_addresses)) return fail(B200_E_ARG, "null pointer");
  if (window_bits != 0 && (window_bits < 2 || window_bits > 24))
    return fail(B200_E_ARG, "window_bits %d out of range [2,24]", window_bits);
  if (first_bad) *first_bad = SIZE_MAX;
  auto src = get_ck(ck_handle);
  if (!src) return fail(B200_E_HANDLE, "unknown key handle %llu", (unsigned long long)ck_handle);
#if defined(NOVA_MSM_ARITH29)
  return fail(B200_E_ARG, "b200_ck_derive_by_address: table 0 is not in the boundary format in this build");
#else
  const cudaStream_t s = pick_stream(stream);
  const field_ops* bops = ops_for_field(CURVES[src->curve].base_fid);
  // identity generators and out-of-range addresses in one pass; one read-back, together with h
  dev_buf flags(s);
  if ((rc = flags.alloc(8))) return rc;
  CU(cudaMemsetAsync(flags.p, 0xFF, 8, s));
  bops->derive_check(s, src->tables, src->n, d_addresses, m <= src->n ? m : 0, table_size, (uint32_t*)flags.p);
  count_launch(1);
  CU(cudaGetLastError());
  uint32_t bad[2];
  std::vector<char> h(64);
  CU(cudaMemcpyAsync(bad, flags.p, 8, cudaMemcpyDeviceToHost, s));
  if (src->has_h) CU(cudaMemcpyAsync(h.data(), (const char*)src->tables + src->n * 64, 64, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  if (bad[0] != 0xFFFFFFFFu) {
    if (first_bad) *first_bad = bad[0];
    return fail(B200_E_POINT, "generator %u of the key is the identity", bad[0]);
  }
  if (m > src->n)
    return fail(B200_E_RANGE, "InvalidCommitmentKeyLength: %zu addresses, key has %zu bases", m, src->n);
  if (bad[1] != 0xFFFFFFFFu) {
    if (first_bad) *first_bad = bad[1];
    return fail(B200_E_INDEX, "InvalidIndex: address at position %u is outside the table of %zu", bad[1], table_size);
  }
  if (table_size == 0) return fail(B200_E_ARG, "table_size = 0: a key of no bases cannot be registered");
  const int c = window_bits ? window_bits : choose_window(table_size);
  const size_t ntables = (size_t)(FIELD_BITS[CURVES[src->curve].scalar_fid] + c - 1) / c;
  if (table_size >= ((size_t)1 << 31) || ntables * (table_size + (src->has_h ? 1 : 0)) >= ((size_t)1 << 31))
    return fail(B200_E_RANGE, "table of %zu bases too large for 31-bit table indices (%zu tables)", table_size, ntables);

  const uint32_t K = (uint32_t)table_size;
  dev_buf bases(s);
  if ((rc = bases.alloc((size_t)K * 64))) return rc;
  if (m == 0) {
    CU(cudaMemsetAsync(bases.p, 0, (size_t)K * 64, s));
  } else {
    // a one-window MSM plan over m entries and K buckets; no digits and no reduction
    msm_plan p{};
    p.n = m;
    p.n_ck = src->stride;
    p.blind_i = SIZE_MAX;
    p.h_index = src->n;
    p.W = p.G = 1;
    p.B = K;
    p.L = segment_len(m);
    p.m = 1;
    const size_t nseg = (m + p.L - 1) / p.L;
    p.heavy_min = HEAVY_PARTS * (uint32_t)p.L;
    p.heavy_cap = (uint32_t)(nseg / HEAVY_PARTS + 2);
    p.sp = make_sort_plan(K);
    p.sort_tag = 1;  // fresh look-back words
    const size_t look_bytes = (m + SORT_TILE - 1) / SORT_TILE * SORT_BINS * sizeof(unsigned long long);
    dev_buf ctl(s), look(s), start(s), ent(s), ent_tmp(s), buckets(s), parts(s), pkeys(s), heavy(s), hparts(s);
    if ((rc = ctl.alloc(SORT_CTL_WORDS * 4)) || (rc = look.alloc(look_bytes)) || (rc = start.alloc(((size_t)K + 1) * 4)) ||
        (rc = ent.alloc(m * 8)) || (rc = ent_tmp.alloc(m * 8)) || (rc = buckets.alloc((size_t)K * XYZZ_BYTES)) ||
        (rc = parts.alloc(2 * nseg * XYZZ_BYTES)) || (rc = pkeys.alloc(2 * nseg * 4)) ||
        (rc = heavy.alloc(((size_t)p.heavy_cap + 1) * 4)) || (rc = hparts.alloc((size_t)p.heavy_cap * HEAVY_SPLIT * XYZZ_BYTES)))
      return rc;
    CU(cudaMemsetAsync(ctl.p, 0, SORT_CTL_WORDS * 4, s));
    CU(cudaMemsetAsync(look.p, 0, look_bytes, s));
    CU(cudaMemsetAsync(heavy.p, 0, 4, s));
    p.sortctl = (uint32_t*)ctl.p;
    p.look = (unsigned long long*)look.p;
    p.start = (uint32_t*)start.p;
    p.entries = (uint64_t*)ent.p;
    p.entries_tmp = (uint64_t*)ent_tmp.p;
    p.buckets = buckets.p;
    p.parts = parts.p;
    p.pkeys = (uint32_t*)pkeys.p;
    p.heavy = (uint32_t*)heavy.p;
    p.hparts = hparts.p;
    const int sort_launches = derive_sort(s, d_addresses, p);
    bops->accumulate(s, src->tables, p);  // every sign positive: the sum of the bases of each address
    bops->fixup(s, p);
    bops->derive_affine(s, p.start, K, p.buckets, bases.p);
    count_launch(sort_launches + 1 + STAGE_KERNELS[ST_FIXUP] + 1);
    CU(cudaGetLastError());
  }
  std::shared_ptr<ck_ctx> ck;
  rc = register_key(src->curve, bases.p, true, K, src->has_h ? h.data() : nullptr, window_bits, true, ck, nullptr, s);
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g_handles_mu);
  *out_handle = g_next_handle++;
  g_handles[*out_handle] = ck;
  return B200_OK;
#endif
}

int b200_ck_derive_by_address(uint64_t ck_handle, const uint64_t* addresses, size_t m, size_t table_size,
                              int window_bits, uint64_t* out_handle, size_t* first_bad) {
  int rc = ensure_init();
  if (rc) return rc;
  if (m && !addresses) return fail(B200_E_ARG, "null pointer");
  // The device form takes u32 addresses.  An address at or past table_size becomes 0xFFFFFFFF, which is past every
  // table size the device form is given (a table of 2^32 - 1 bases fails the 31-bit limit anyway), so it is reported
  // at its own position and never wraps onto a slot; an in-range address of 2^32 or more (only possible when the
  // table is too large to register) is clamped below that.
  const size_t ts = std::min(table_size, (size_t)0xFFFFFFFFu);
  std::vector<uint32_t> a32(m);
  for (size_t i = 0; i < m; i++)
    a32[i] = addresses[i] >= table_size ? 0xFFFFFFFFu : (uint32_t)std::min<uint64_t>(addresses[i], 0xFFFFFFFEu);
  return via_device({up(a32.data(), m * 4)}, [&](void** d, cudaStream_t s) {
    return b200_ck_derive_by_address_dev(ck_handle, (const uint32_t*)d[0], m, ts, window_bits, out_handle, first_bad, s);
  });
}

int b200_ck_release(uint64_t handle) {
  std::shared_ptr<ck_ctx> ck;
  {
    std::lock_guard<std::mutex> lk(g_handles_mu);
    auto it = g_handles.find(handle);
    if (it == g_handles.end()) return fail(B200_E_HANDLE, "unknown key handle %llu",
                                           (unsigned long long)handle);
    ck = it->second;
    g_handles.erase(it);
  }
  std::lock_guard<std::mutex> lk(ck->mu);  // wait for in-flight calls
  for (ck_ctx* t : {ck.get(), ck->small.get()})
    if (t)
      for (ck_ctx::host_slot& h : t->slots) std::lock_guard<std::mutex> wait(h.mu);
  cudaSetDevice(g_dev.device);
  return B200_OK;
}

int b200_ck_len(uint64_t handle, size_t* n, int* window_bits, int* num_tables) {
  auto ck = get_ck(handle);
  if (!ck) return fail(B200_E_HANDLE, "unknown key handle %llu", (unsigned long long)handle);
  if (n) *n = ck->n;
  if (window_bits) *window_bits = ck->c;
  if (num_tables) *num_tables = ck->F;
  return B200_OK;
}

// ---- MSM --------------------------------------------------------------------------------------
// Lane streams carry DECREASING priority with the lane index: when several MSMs are in flight, the latency-bound tail
// kernels (a handful of blocks) of the MSM on lane j are dispatched ahead of the thousands of queued accumulate blocks
// of the MSM on lane j + 1 instead of behind them -- without this the block scheduler serialises the lanes.
static int lane_stream(ck_ctx::lane& ln, int index) {
  if (ln.s) return B200_OK;
  int least = 0, greatest = 0;
  CU(cudaDeviceGetStreamPriorityRange(&least, &greatest));  // numerically lower = higher priority
  int prio = greatest + index;
  if (prio > least) prio = least;
  CU(cudaStreamCreateWithPriority(&ln.s, cudaStreamNonBlocking, prio));
  CU(cudaEventCreateWithFlags(&ln.done, cudaEventDisableTiming));
  return B200_OK;
}

static int msm_host(ck_ctx& ck, size_t base_offset, const void* scalars, size_t n, void* out,
                    const void* blind = nullptr) {
  int rc = B200_OK;
  // Tuning hook: NOVA_B200_H2D_CHUNKS=k splits the upload into k pieces
  // and runs the digit / histogram stage of piece i on a side stream while piece i+1 is still on the bus --
  // the same chunked path b200_witness_append uses.  At most the digit stage (~0.12 ms of a 2^20 MSM) can hide.
  static const int h2d_chunks = [] {
    const char* e = getenv("NOVA_B200_H2D_CHUNKS");
    int k = e ? atoi(e) : 4;  // default 4: a little faster end to end at 2^20 and 2^22
    return k < 1 ? 1 : (k > 64 ? 64 : k);
  }();
  // Slice pipeline (n >= 2^23): the vector is cut into k index ranges, each a complete MSM on its own lane (stream +
  // workspace) that starts as soon as ITS bytes have landed, so that the pipeline of slice j overlaps the upload of
  // slice j+1; the k partial points are added by one small kernel.  It pays at 2^24 from pinned memory; at
  // 2^20 - 2^22 it loses (a quarter-size MSM runs at lower efficiency and the lanes' kernels do not overlap -- each accumulate grid already fills the GPU for several waves),
  // so smaller vectors take the single-shot path with the chunked upload below.  NOVA_B200_E2E_SLICES=1 disables it.
  static const int e2e_slices = [] {
    const char* e = getenv("NOVA_B200_E2E_SLICES");
    int k = e ? atoi(e) : 4;
    return k < 1 ? 1 : (k > ck_ctx::NLANES ? ck_ctx::NLANES : k);
  }();
  if (e2e_slices > 1 && n >= ((size_t)1 << 23)) {
    std::lock_guard<std::mutex> lk(ck.mu);  // the lanes belong to the key
    cudaStream_t s = g_dev.stream;
    const int k = e2e_slices;
    rc = ensure_workspace(ck, 1, (size_t)k + 1);
    if (rc) return rc;
    if ((rc = ws_acquire(ck.ws, s))) return rc;
    cudaEvent_t ev = nullptr;
    CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    CU(cudaEventRecord(ev, s));
    const size_t per = (n + k - 1) / k;
    int used = 0;
    for (int j = 0; j < k && rc == B200_OK; j++) {
      const size_t lo = (size_t)j * per, hi = lo + per < n ? lo + per : n;
      if (lo >= hi) break;
      const bool last = hi == n;
      ck_ctx::lane& ln = ck.lanes[j];
      if ((rc = lane_stream(ln, j))) break;
      CU(cudaStreamWaitEvent(ln.s, ev, 0));
      rc = ensure_workspace(ck, ln.ws, hi - lo + 1, 1);
      if (rc) break;
      if ((rc = ws_acquire(ln.ws, ln.s))) break;
      CU(cudaMemcpyAsync(ln.ws.scalars, (const char*)scalars + 32 * lo, 32 * (hi - lo), cudaMemcpyHostToDevice, ln.s));
      const bool with_blind = last && blind != nullptr;
      if (with_blind)
        CU(cudaMemcpyAsync((char*)ln.ws.scalars + 32 * (hi - lo), blind, 32, cudaMemcpyHostToDevice, ln.s));
      rc = enqueue_msm(ck, ln.ws, base_offset + lo, ln.ws.scalars, hi - lo + (with_blind ? 1 : 0),
                       (char*)ck.ws.d_out + 96 * (j + 1), ln.s, 0, with_blind);
      used = j + 1;
    }
    for (int j = 0; j < used; j++) {
      cudaEventRecord(ck.lanes[j].done, ck.lanes[j].s);
      cudaStreamWaitEvent(s, ck.lanes[j].done, 0);
    }
    cudaEventDestroy(ev);
    if (rc) return rc;
    ops_for_field(CURVES[ck.curve].base_fid)->jacobian_sum(s, (char*)ck.ws.d_out + 96, used, ck.ws.d_out);
    count_launch(1);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(ck.ws.h_out, ck.ws.d_out, 96, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    memcpy(out, ck.ws.h_out, 96);
    return B200_OK;
  }
  // one host slot per call: a free one if there is any, else wait for the next in turn
  ck_ctx::host_slot* slot = nullptr;
  for (ck_ctx::host_slot& h : ck.slots)
    if (h.mu.try_lock()) {
      slot = &h;
      break;
    }
  if (!slot) {
    unsigned turn;
    {
      std::lock_guard<std::mutex> lk(ck.mu);
      turn = ck.next_slot++ % ck_ctx::NSLOTS;
    }
    slot = &ck.slots[turn];
    slot->mu.lock();
  }
  std::lock_guard<std::mutex> slk(slot->mu, std::adopt_lock);
  if (!slot->s) {
    CU(cudaStreamCreateWithFlags(&slot->s, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&slot->side, cudaStreamNonBlocking));
  }
  workspace& W = slot->ws;
  cudaStream_t s = slot->s;
  if ((rc = ensure_workspace(ck, W, n + 1, 1))) return rc;
  if (h2d_chunks > 1 && n >= ((size_t)1 << 16)) {
    cudaStream_t side = slot->side;
    const size_t total = n + (blind ? 1 : 0);
    const field_ops* sops = ops_for_field(CURVES[ck.curve].scalar_fid);
    msm_plan p = make_plan(ck, W, base_offset, total);
    cudaEvent_t ev = nullptr;
    CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    CU(cudaEventRecord(ev, s));  // order the side stream after earlier users of this workspace
    CU(cudaStreamWaitEvent(side, ev, 0));
    CU(cudaMemsetAsync(p.sortctl, 0, SORT_CTL_WORDS * 4, side));
    const size_t per = (n + h2d_chunks - 1) / h2d_chunks;
    auto piece = [&](const void* src, size_t lo, size_t hi) -> int {
      CU(cudaMemcpyAsync((char*)W.scalars + 32 * lo, src, 32 * (hi - lo), cudaMemcpyHostToDevice, s));
      CU(cudaEventRecord(ev, s));
      CU(cudaStreamWaitEvent(side, ev, 0));
      sops->digits_range(side, W.scalars, lo, hi, p);
      count_launch(1);
      return B200_OK;
    };
    for (size_t lo = 0; lo < n && rc == B200_OK; lo += per)
      rc = piece((const char*)scalars + 32 * lo, lo, lo + per < n ? lo + per : n);
    if (blind && rc == B200_OK) rc = piece(blind, n, n + 1);
    if (rc) {
      cudaEventDestroy(ev);
      return rc;
    }
    CU(cudaEventRecord(ev, side));
    CU(cudaStreamWaitEvent(s, ev, 0));
    cudaEventDestroy(ev);
    rc = enqueue_msm(ck, W, base_offset, W.scalars, total, W.d_out, s, 0, blind != nullptr, /*digits_done=*/true);
  } else {
    if (n) CU(cudaMemcpyAsync(W.scalars, scalars, n * 32, cudaMemcpyHostToDevice, s));
    if (blind) CU(cudaMemcpyAsync((char*)W.scalars + n * 32, blind, 32, cudaMemcpyHostToDevice, s));
    rc = enqueue_msm(ck, W, base_offset, W.scalars, n + (blind ? 1 : 0), W.d_out, s, 0, blind != nullptr);
  }
  if (rc) return rc;
  CU(cudaMemcpyAsync(W.h_out, W.d_out, 96, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  memcpy(out, W.h_out, 96);
  return B200_OK;
}

int b200_msm(uint64_t handle, size_t base_offset, const void* scalars, size_t n, void* out) {
  int rc = ensure_init();
  if (rc) return rc;
  auto ck = get_ck(handle);
  if (!ck) return fail(B200_E_HANDLE, "unknown key handle %llu", (unsigned long long)handle);
  if (!out || (n && !scalars)) return fail(B200_E_ARG, "null pointer");
  if (base_offset + n > ck->n)
    return fail(B200_E_RANGE, "msm slice [%zu, %zu) exceeds key length %zu", base_offset,
                base_offset + n, ck->n);
  return msm_host(route(*ck, base_offset, n), base_offset, scalars, n, out);
}

int b200_commit(uint64_t handle, const void* scalars, size_t n, const void* r, void* out) {
  int rc = ensure_init();
  if (rc) return rc;
  auto ck = get_ck(handle);
  if (!ck) return fail(B200_E_HANDLE, "unknown key handle %llu", (unsigned long long)handle);
  if (!out || (n && !scalars)) return fail(B200_E_ARG, "null pointer");
  if (n > ck->n)  // pedersen.rs:264 assert!(ck.ck.len() >= v.len())
    return fail(B200_E_RANGE, "commit of %zu scalars exceeds key length %zu", n, ck->n);
  if (r && !ck->has_h) return fail(B200_E_ARG, "key was registered without a blinding generator");
  return msm_host(route(*ck, 0, n), 0, scalars, n, out, r);
}

int b200_msm_dev(uint64_t handle, size_t base_offset, const void* d_scalars, size_t n, void* d_out,
                 void* stream) {
  int rc = ensure_init();
  if (rc) return rc;
  auto ck = get_ck(handle);
  if (!ck) return fail(B200_E_HANDLE, "unknown key handle %llu", (unsigned long long)handle);
  if (!d_out || (n && !d_scalars)) return fail(B200_E_ARG, "null pointer");
  if (base_offset + n > ck->n)
    return fail(B200_E_RANGE, "msm slice [%zu, %zu) exceeds key length %zu", base_offset,
                base_offset + n, ck->n);
  ck_ctx& t = route(*ck, base_offset, n);
  std::lock_guard<std::mutex> lk(t.mu);
  rc = ensure_workspace(t, n ? n : 1, 1);
  if (rc) return rc;
  return enqueue_msm(t, base_offset, d_scalars, n, d_out, pick_stream(stream));
}

int b200_commit_dev(uint64_t handle, const void* d_scalars, size_t n, const void* d_blind_or_null,
                    void* d_out, void* stream) {
  int rc = ensure_init();
  if (rc) return rc;
  auto ck = get_ck(handle);
  if (!ck) return fail(B200_E_HANDLE, "unknown key handle %llu", (unsigned long long)handle);
  if (!d_out || (n && !d_scalars)) return fail(B200_E_ARG, "null pointer");
  if (n > ck->n) return fail(B200_E_RANGE, "commit of %zu scalars exceeds key length %zu", n, ck->n);
  if (d_blind_or_null && !ck->has_h)
    return fail(B200_E_ARG, "key was registered without a blinding generator");
  ck_ctx& t = route(*ck, 0, n);
  std::lock_guard<std::mutex> lk(t.mu);
  rc = ensure_workspace(t, n + 1, 1);
  if (rc) return rc;
  cudaStream_t s = pick_stream(stream);
  if (!d_blind_or_null) return enqueue_msm(t, 0, d_scalars, n, d_out, s);
  if ((rc = ws_acquire(t.ws, s))) return rc;
  // the blinding scalar must follow the vector in one buffer: stage both in the workspace
  if (n) CU(cudaMemcpyAsync(t.ws.scalars, d_scalars, n * 32, cudaMemcpyDeviceToDevice, s));
  CU(cudaMemcpyAsync((char*)t.ws.scalars + n * 32, d_blind_or_null, 32, cudaMemcpyDeviceToDevice, s));
  return enqueue_msm(t, 0, t.ws.scalars, n + 1, d_out, s, 0, true);
}

// k independent MSMs over prefixes of one key, spread round-robin over the key's lanes.  Vector j
// is read from vecs[j] (device memory, or host memory staged through the lane's workspace when
// `from_host`); result j goes to d_out + 96 j.  Ordered after prior work on `s`; on return `s`
// waits for every lane.  Caller holds ck.mu.
static int enqueue_many(ck_ctx& ck, const void* const* vecs, const size_t* lens, size_t k,
                        bool from_host, void* d_out, cudaStream_t s, const size_t* offsets = nullptr) {
  std::unique_lock<std::mutex> lsmall;
  if (ck.small) lsmall = std::unique_lock<std::mutex>(ck.small->mu);  // lock order: wide, narrow
  cudaEvent_t start_ev = nullptr;
  CU(cudaEventCreateWithFlags(&start_ev, cudaEventDisableTiming));
  CU(cudaEventRecord(start_ev, s));
  bool used[2][ck_ctx::NLANES] = {};
  size_t next[2] = {0, 0};
  int rc = B200_OK;
  for (size_t j = 0; j < k && rc == B200_OK; j++) {
    const size_t off = offsets ? offsets[j] : 0;
    ck_ctx& t = route(ck, off, lens[j]);
    int which = &t == &ck ? 0 : 1;
    int li = (int)(next[which]++ % ck_ctx::NLANES);
    ck_ctx::lane& ln = t.lanes[li];
    if ((rc = lane_stream(ln, li))) break;
    if (!used[which][li]) {
      CU(cudaStreamWaitEvent(ln.s, start_ev, 0));
      used[which][li] = true;
    }
    rc = ensure_workspace(t, ln.ws, lens[j] ? lens[j] : 1, 1);
    if (rc) break;
    const void* src = vecs[j];
    if ((rc = ws_acquire(ln.ws, ln.s))) break;
    if (from_host && lens[j]) {
      CU(cudaMemcpyAsync(ln.ws.scalars, vecs[j], lens[j] * 32, cudaMemcpyHostToDevice, ln.s));
      src = ln.ws.scalars;
    }
    rc = enqueue_msm(t, ln.ws, off, src, lens[j], (char*)d_out + 96 * j, ln.s);
  }
  for (int which = 0; which < 2; which++) {
    ck_ctx* t = which == 0 ? &ck : ck.small.get();
    for (int li = 0; t && li < ck_ctx::NLANES; li++)
      if (used[which][li]) {
        cudaEventRecord(t->lanes[li].done, t->lanes[li].s);
        cudaStreamWaitEvent(s, t->lanes[li].done, 0);
      }
  }
  cudaEventDestroy(start_ev);
  return rc;
}

static int check_many(ck_ctx& ck, const void* const* vecs, const size_t* lens, size_t k) {
  if (!vecs || !lens) return fail(B200_E_ARG, "null pointer");
  for (size_t j = 0; j < k; j++) {
    if (lens[j] > ck.n)
      return fail(B200_E_RANGE, "batch vector %zu has %zu scalars, key has %zu", j, lens[j], ck.n);
    if (lens[j] && !vecs[j]) return fail(B200_E_ARG, "null scalar vector %zu", j);
  }
  return B200_OK;
}

int b200_msm_batch(uint64_t handle, const void* const* scalars, const size_t* lens, size_t k,
                   void* out) {
  int rc = ensure_init();
  if (rc) return rc;
  auto ck = get_ck(handle);
  if (!ck) return fail(B200_E_HANDLE, "unknown key handle %llu", (unsigned long long)handle);
  if (k == 0) return B200_OK;
  if (!out) return fail(B200_E_ARG, "null pointer");
  if ((rc = check_many(*ck, scalars, lens, k))) return rc;
  std::lock_guard<std::mutex> lk(ck->mu);
  rc = ensure_workspace(*ck, 1, k);
  if (rc) return rc;
  cudaStream_t s = g_dev.stream;
  rc = enqueue_many(*ck, scalars, lens, k, /*from_host=*/true, ck->ws.d_out, s);
  if (rc) return rc;
  CU(cudaMemcpyAsync(ck->ws.h_out, ck->ws.d_out, 96 * k, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  memcpy(out, ck->ws.h_out, 96 * k);
  return B200_OK;
}

int b200_commit_many_dev(uint64_t handle, const void* const* d_scalars, const size_t* lens, size_t k,
                         void* d_out, void* stream) {
  int rc = ensure_init();
  if (rc) return rc;
  auto ck = get_ck(handle);
  if (!ck) return fail(B200_E_HANDLE, "unknown key handle %llu", (unsigned long long)handle);
  if (k == 0) return B200_OK;
  if (!d_out) return fail(B200_E_ARG, "null pointer");
  if ((rc = check_many(*ck, d_scalars, lens, k))) return rc;
  std::lock_guard<std::mutex> lk(ck->mu);
  return enqueue_many(*ck, d_scalars, lens, k, /*from_host=*/false, d_out, pick_stream(stream));
}

int b200_msm_many_dev(uint64_t handle, const size_t* base_offsets, const void* const* d_scalars, const size_t* lens,
                      size_t k, void* d_out, void* stream) {
  int rc = ensure_init();
  if (rc) return rc;
  auto ck = get_ck(handle);
  if (!ck) return fail(B200_E_HANDLE, "unknown key handle %llu", (unsigned long long)handle);
  if (k == 0) return B200_OK;
  if (!d_out || !base_offsets || !d_scalars || !lens) return fail(B200_E_ARG, "null pointer");
  for (size_t j = 0; j < k; j++) {
    if (base_offsets[j] + lens[j] > ck->n)
      return fail(B200_E_RANGE, "msm %zu: slice [%zu, %zu) exceeds key length %zu", j, base_offsets[j],
                  base_offsets[j] + lens[j], ck->n);
    if (lens[j] && !d_scalars[j]) return fail(B200_E_ARG, "null scalar vector %zu", j);
  }
  std::lock_guard<std::mutex> lk(ck->mu);
  return enqueue_many(*ck, d_scalars, lens, k, /*from_host=*/false, d_out,
                      pick_stream(stream), base_offsets);
}

int b200_msm_small(uint64_t handle, size_t base_offset, const void* scalars, int elem_bytes, size_t n,
                   int max_bits, void* out) {
  int rc = ensure_init();
  if (rc) return rc;
  auto ck = get_ck(handle);
  if (!ck) return fail(B200_E_HANDLE, "unknown key handle %llu", (unsigned long long)handle);
  if (!out || (n && !scalars)) return fail(B200_E_ARG, "null pointer");
  if (elem_bytes != 1 && elem_bytes != 2 && elem_bytes != 4 && elem_bytes != 8)
    return fail(B200_E_ARG, "elem_bytes must be 1, 2, 4 or 8 (got %d)", elem_bytes);
  if (max_bits < 0 || max_bits > 64) return fail(B200_E_ARG, "max_bits %d out of range", max_bits);
  if (base_offset + n > ck->n)
    return fail(B200_E_RANGE, "msm slice [%zu, %zu) exceeds key length %zu", base_offset,
                base_offset + n, ck->n);
  // max_bits only selects the algorithm in the reference (msm.rs:487-502); the digit stream
  // below skips zero windows, so every width takes the same path here.
  ck_ctx& t = route(*ck, base_offset, n);
  std::lock_guard<std::mutex> lk(t.mu);
  rc = ensure_workspace(t, n ? n : 1, 1);
  if (rc) return rc;
  cudaStream_t s = g_dev.stream;
  if ((rc = ws_acquire(t.ws, s))) return rc;
  if (n) CU(cudaMemcpyAsync(t.ws.scalars, scalars, n * elem_bytes, cudaMemcpyHostToDevice, s));
  rc = enqueue_msm(t, base_offset, t.ws.scalars, n, t.ws.d_out, s, elem_bytes);
  if (rc) return rc;
  CU(cudaMemcpyAsync(t.ws.h_out, t.ws.d_out, 96, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  memcpy(out, t.ws.h_out, 96);
  return B200_OK;
}

int b200_msm_indices(uint64_t handle, const uint64_t* idx, size_t m, void* out) {
  int rc = ensure_init();
  if (rc) return rc;
  auto ck = get_ck(handle);
  if (!ck) return fail(B200_E_HANDLE, "unknown key handle %llu", (unsigned long long)handle);
  if (!out || (m && !idx)) return fail(B200_E_ARG, "null pointer");
  std::vector<uint32_t> idx32(m);
  for (size_t j = 0; j < m; j++) {
    if (idx[j] >= ck->n) return fail(B200_E_RANGE, "index %llu outside key of %zu",
                                     (unsigned long long)idx[j], ck->n);
    idx32[j] = (uint32_t)idx[j];
  }
  std::lock_guard<std::mutex> lk(ck->mu);
  rc = ensure_workspace(*ck, 1, 1);
  if (rc) return rc;
  workspace& w = ck->ws;
  if (m > w.idx_cap) {
    if (w.idx32) cudaFree(w.idx32);
    w.idx32 = nullptr;
    CU(cudaMalloc((void**)&w.idx32, m * 4));
    w.idx_cap = m;
  }
  cudaStream_t s = g_dev.stream;
  if (m) CU(cudaMemcpyAsync(w.idx32, idx32.data(), m * 4, cudaMemcpyHostToDevice, s));
  const field_ops* bops = ops_for_field(CURVES[ck->curve].base_fid);
  bops->sum_points(s, ck->tables, w.idx32, m, w.sumscratch, w.d_out);
  count_launch(2);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(w.h_out, w.d_out, 96, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  memcpy(out, w.h_out, 96);
  return B200_OK;
}

int b200_msm_adhoc(int curve_id, const void* bases, const void* scalars, size_t n, void* out) {
  int rc = ensure_init();
  if (rc) return rc;
  if (!out) return fail(B200_E_ARG, "null out");
  if (n == 0) {
    memset(out, 0, 96);
    return B200_OK;
  }
  if (!bases || !scalars) return fail(B200_E_ARG, "null pointer");
  std::shared_ptr<ck_ctx> ck;
  rc = register_key(curve_id, bases, false, n, nullptr, 0, /*expand=*/false, ck);
  if (rc) return rc;
  return msm_host(route(*ck, 0, n), 0, scalars, n, out);
}

// ---- host-side Keccak-256 for the transcript mirror ---------------------------------------------------
// The Fiat-Shamir transcript (src/provider/keccak.rs:31-160) stays on the HOST between device calls (HyperKZG,
// ppsnark, NIFS); in the Rust integration the `sha3` crate does this.  The Python / C++ host layers call this
// function instead of hashing in the interpreter (a pure-Python permutation costs ~0.5 ms; a HyperKZG proof
// absorbs ~4 KB).  Plain C, no device work; pinned by keccak.rs:279-288 through nova_b200/transcript.py's tests.
int b200_keccak256(const void* data, size_t len, void* out32) {
  if (!out32 || (len && !data)) return fail(B200_E_ARG, "null pointer");
  const size_t rate = 136;
  uint64_t st[25] = {};
  const uint8_t* p = (const uint8_t*)data;
  auto absorb_block = [&](const uint8_t* blk) {
    for (size_t i = 0; i < rate / 8; i++) {
      uint64_t w;
      memcpy(&w, blk + 8 * i, 8);  // little-endian host (x86-64 / aarch64)
      st[i] ^= w;
    }
    nova::keccak_f1600(st);  // the permutation the device transcript uses, compiled for the host (transcript.cuh)
  };
  while (len >= rate) {
    absorb_block(p);
    p += rate;
    len -= rate;
  }
  uint8_t last[136] = {};
  if (len) memcpy(last, p, len);
  last[len] ^= 0x01;        // original Keccak padding (sha3::Keccak256, not SHA3-256's 0x06)
  last[rate - 1] ^= 0x80;
  absorb_block(last);
  memcpy(out32, st, 32);
  return B200_OK;
}

// ---- sharded MSM with the collective fused into the reduction ---------------------------------------
namespace {
struct peer_group {
  std::mutex mu;
  msm_peer desc;
};
std::mutex g_groups_mu;
std::map<uint64_t, std::shared_ptr<peer_group>> g_groups;
uint64_t g_next_group = 1;
}  // namespace

int b200_peer_buffer_alloc(void** dptr) {
  int rc = ensure_init();
  if (rc) return rc;
  if (!dptr) return fail(B200_E_ARG, "null pointer");
  CU(cudaMalloc(dptr, MSM_PEER_BUF_BYTES));
  CU(cudaMemset(*dptr, 0, MSM_PEER_BUF_BYTES));
  return B200_OK;
}
int b200_peer_buffer_free(void* dptr) {
  if (dptr) CU(cudaFree(dptr));
  return B200_OK;
}
int b200_ipc_export(const void* dptr, void* handle64_out) {
  int rc = ensure_init();
  if (rc) return rc;
  if (!dptr || !handle64_out) return fail(B200_E_ARG, "null pointer");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "the ABI carries IPC handles as 64 bytes");
  cudaIpcMemHandle_t h;
  CU(cudaIpcGetMemHandle(&h, const_cast<void*>(dptr)));
  memcpy(handle64_out, &h, 64);
  return B200_OK;
}
int b200_ipc_open(const void* handle64, void** dptr) {
  int rc = ensure_init();
  if (rc) return rc;
  if (!handle64 || !dptr) return fail(B200_E_ARG, "null pointer");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  CU(cudaIpcOpenMemHandle(dptr, h, cudaIpcMemLazyEnablePeerAccess));
  return B200_OK;
}
int b200_ipc_close(void* dptr) {
  if (!dptr) return B200_OK;
  CU(cudaIpcCloseMemHandle(dptr));
  return B200_OK;
}
int b200_peer_group_create(int rank, int world, void* const* bufs, uint64_t* group) {
  int rc = ensure_init();
  if (rc) return rc;
  if (!bufs || !group) return fail(B200_E_ARG, "null pointer");
  if (world < 1 || world > MSM_PEER_MAX || rank < 0 || rank >= world)
    return fail(B200_E_ARG, "peer group of %d ranks (rank %d): world must be 1..%d", world, rank, MSM_PEER_MAX);
  auto g = std::make_shared<peer_group>();
  g->desc.world = world;
  g->desc.rank = rank;
  for (int r = 0; r < world; r++) {
    if (!bufs[r]) return fail(B200_E_ARG, "null exchange buffer for rank %d", r);
    g->desc.buf[r] = bufs[r];
  }
  std::lock_guard<std::mutex> lk(g_groups_mu);
  *group = g_next_group++;
  g_groups[*group] = g;
  return B200_OK;
}
int b200_peer_group_release(uint64_t group) {
  std::lock_guard<std::mutex> lk(g_groups_mu);
  if (!g_groups.erase(group)) return fail(B200_E_HANDLE, "unknown peer group %llu", (unsigned long long)group);
  return B200_OK;
}
static std::shared_ptr<peer_group> get_group(uint64_t h) {
  std::lock_guard<std::mutex> lk(g_groups_mu);
  auto it = g_groups.find(h);
  return it == g_groups.end() ? nullptr : it->second;
}
int b200_peer_group_status(uint64_t group) {
  int rc = ensure_init();
  if (rc) return rc;
  auto g = get_group(group);
  if (!g) return fail(B200_E_HANDLE, "unknown peer group %llu", (unsigned long long)group);
  unsigned long long err = 0;
  CU(cudaMemcpy(&err, (const char*)g->desc.buf[g->desc.rank] + MSM_PEER_ERR_OFF, 8, cudaMemcpyDeviceToHost));
  if (err) return fail(B200_E_PEER, "a peer never delivered its partial sum (epoch %llu): exchange timed out", err);
  return B200_OK;
}

int b200_msm_sharded_dev(uint64_t handle, size_t base_offset, const void* d_scalars, size_t n, uint64_t group,
                         void* d_out, void* stream) {
  int rc = ensure_init();
  if (rc) return rc;
  auto ck = get_ck(handle);
  if (!ck) return fail(B200_E_HANDLE, "unknown key handle %llu", (unsigned long long)handle);
  auto g = get_group(group);
  if (!g) return fail(B200_E_HANDLE, "unknown peer group %llu", (unsigned long long)group);
  if (!d_out || (n && !d_scalars)) return fail(B200_E_ARG, "null pointer");
  if (base_offset + n > ck->n)
    return fail(B200_E_RANGE, "msm slice [%zu, %zu) exceeds key length %zu", base_offset, base_offset + n, ck->n);
#if defined(NOVA_MSM_ARITH29)
  return fail(B200_E_ARG, "the fused exchange needs the default (8x32-bit) arithmetic build");
#else
  ck_ctx& t = route(*ck, base_offset, n);
  std::lock_guard<std::mutex> glk(g->mu);
  std::lock_guard<std::mutex> lk(t.mu);
  rc = ensure_workspace(t, n ? n : 1, 1);
  if (rc) return rc;
  msm_peer peer = g->desc;
  peer.epoch = ++g->desc.epoch;
  return enqueue_msm(t, t.ws, base_offset, d_scalars, n, d_out, pick_stream(stream), 0, false, false, &peer);
#endif
}

// ---- Poseidon random oracle on the device (SURVEY.md §8f-3; src/provider/poseidon.rs:41-127) ---------------
namespace {
struct poseidon_ctx {
  int fid = 0, t = 0, r_f = 0, r_p = 0;
  void *rc = nullptr, *mds = nullptr;
  ~poseidon_ctx() {
    if (rc) cudaFree(rc);
    if (mds) cudaFree(mds);
  }
};
std::mutex g_pos_mu;
std::map<uint64_t, std::shared_ptr<poseidon_ctx>> g_pos;
uint64_t g_next_pos = 1;

// IOPattern([Absorb(n), Squeeze(1)]).value(0) (sponge/api.rs:27-109): u128 arithmetic mod 2^128
void poseidon_tag(uint32_t n, unsigned char out32[32]) {
  typedef unsigned __int128 u128;
  const u128 base = (u128)0 - 159;
  u128 x_i = 1, state = 0;
  auto update = [&](uint32_t a) {
    x_i *= base;
    state += x_i * (u128)a;
  };
  if (n) update(n + (1u << 31));  // Absorb(n); a zero-count op is skipped (finish_op)
  update(1);                      // Squeeze(1)
  update(0);                      // domain separator
  memset(out32, 0, 32);
  memcpy(out32, &state, 16);
}
}  // namespace

int b200_poseidon_register(int fid, int arity, int r_f, int r_p, const void* rc_mont, const void* mds_mont, uint64_t* handle) {
  int rc = ensure_init();
  if (rc) return rc;
  if (!ops_for_field(fid)) return fail(B200_E_ARG, "unknown field id %d", fid);
  if (arity < 1 || arity + 1 > 25 || r_f < 2 || (r_f & 1) || r_p < 0 || !rc_mont || !mds_mont || !handle)
    return fail(B200_E_ARG, "bad Poseidon parameters (arity %d, R_F %d, R_P %d)", arity, r_f, r_p);
  auto c = std::make_shared<poseidon_ctx>();
  c->fid = fid;
  c->t = arity + 1;
  c->r_f = r_f;
  c->r_p = r_p;
  const size_t nrc = (size_t)(r_f + r_p) * c->t, nm = (size_t)c->t * c->t;
  CU(cudaMalloc(&c->rc, nrc * 32));
  CU(cudaMalloc(&c->mds, nm * 32));
  CU(cudaMemcpyAsync(c->rc, rc_mont, nrc * 32, cudaMemcpyHostToDevice, g_dev.stream));
  CU(cudaMemcpyAsync(c->mds, mds_mont, nm * 32, cudaMemcpyHostToDevice, g_dev.stream));
  CU(cudaStreamSynchronize(g_dev.stream));
  std::lock_guard<std::mutex> lk(g_pos_mu);
  *handle = g_next_pos++;
  g_pos[*handle] = c;
  return B200_OK;
}
int b200_poseidon_release(uint64_t handle) {
  std::lock_guard<std::mutex> lk(g_pos_mu);
  if (!g_pos.erase(handle)) return fail(B200_E_HANDLE, "unknown Poseidon handle %llu", (unsigned long long)handle);
  return B200_OK;
}
int b200_poseidon_ro_dev(uint64_t handle, const void* d_elems, size_t n, int num_bits, int start_with_one, void* d_out96,
                         void* stream) {
  int rc = ensure_init();
  if (rc) return rc;
  std::shared_ptr<poseidon_ctx> c;
  {
    std::lock_guard<std::mutex> lk(g_pos_mu);
    auto it = g_pos.find(handle);
    if (it == g_pos.end()) return fail(B200_E_HANDLE, "unknown Poseidon handle %llu", (unsigned long long)handle);
    c = it->second;
  }
  if (!d_out96 || (n && !d_elems)) return fail(B200_E_ARG, "null pointer");
  if (num_bits < 1 || num_bits > 250) return fail(B200_E_ARG, "num_bits %d outside 1..250", num_bits);
  if (n >= (1u << 31)) return fail(B200_E_ARG, "too many elements");
  cudaStream_t s = pick_stream(stream);
  unsigned char tag[32];
  poseidon_tag((uint32_t)n, tag);
  dev_buf d_tag(s);
  if ((rc = d_tag.alloc(32))) return rc;
  CU(cudaMemcpyAsync(d_tag.p, tag, 32, cudaMemcpyHostToDevice, s));  // (pageable source: staged before the call returns)
  ops_for_field(c->fid)->poseidon_ro(s, c->t, c->r_f, c->r_p, c->rc, c->mds, d_elems, (uint32_t)n, d_tag.p, num_bits,
                                     start_with_one, d_out96);
  count_launch(1);
  CU(cudaGetLastError());
  return B200_OK;
}
int b200_poseidon_ro(uint64_t handle, const void* elems_mont, size_t n, int num_bits, int start_with_one, void* out96) {
  int rc = ensure_init();
  if (rc) return rc;
  return via_device({up(elems_mont, 32 * n), down(out96, 96)}, [&](void* const* d, cudaStream_t s) {
    return b200_poseidon_ro_dev(handle, d[0], n, num_bits, start_with_one, d[1], s);
  });
}
int b200_to_mont_dev(int fid, const void* d_canonical, size_t n, void* d_out, void* stream) {
  return with_field(fid, [&](const field_ops* ops) {
    if (n && (!d_canonical || !d_out)) return fail(B200_E_ARG, "null pointer");
    ops->to_mont(pick_stream(stream), d_canonical, n, d_out);
    count_launch(1);
    CU(cudaGetLastError());
    return (int)B200_OK;
  });
}

// ---- ONE process, N GPUs: a commitment key sharded over the devices behind a single call -----------------
// What SURVEY.md §8b asked of the boundary: a Rust host calls DlogGroupExt::vartime_multiscalar_mul /
// CommitmentEngine::commit ONCE (src/provider/traits.rs:77-117, pedersen.rs:263-270) and the node's GPUs share the
// work.  The key is distributed BLOCK-CYCLICALLY (blocks of MGPU_BLOCK points: device d owns blocks d, d + D, ...),
// so every prefix ck[..n] -- the reference commits prefixes of one key all the time -- is balanced over the devices,
// and a device's scalars are a strided view of the caller's vector: one cudaMemcpy2DAsync per device.  One host thread
// drives all devices (every step is asynchronous); the partial sums are exchanged by peer stores inside each device's
// last reduction kernel (peer_exchange_sum, peer access enabled between all pairs) and every device ends with the sum.
namespace {
constexpr size_t MGPU_BLOCK = 4096;
struct mgpu_state {
  std::mutex mu;
  bool ready = false;
  int ndev = 0;
  int dev[MSM_PEER_MAX] = {};
  cudaStream_t stream[MSM_PEER_MAX] = {};
  void* xbuf[MSM_PEER_MAX] = {};
  void* out_dev[MSM_PEER_MAX] = {};  // 96-byte result slot per device
  void* out_host = nullptr;          // pinned
  unsigned long long epoch = 0;
} g_mgpu;
struct mgpu_key {
  int curve = 0;
  size_t n = 0;
  bool has_h = false;
  std::shared_ptr<ck_ctx> part[MSM_PEER_MAX];
};
std::mutex g_mkeys_mu;
std::map<uint64_t, std::shared_ptr<mgpu_key>> g_mkeys;
uint64_t g_next_mkey = 1;

// points of the first n that device d of D owns under the block-cyclic distribution
size_t mgpu_count(size_t n, int d, int D) {
  const size_t round = MGPU_BLOCK * (size_t)D;
  const size_t rem = n % round;
  size_t extra = rem > (size_t)d * MGPU_BLOCK ? rem - (size_t)d * MGPU_BLOCK : 0;
  if (extra > MGPU_BLOCK) extra = MGPU_BLOCK;
  return (n / round) * MGPU_BLOCK + extra;
}
struct device_guard {  // restores the library's own device on every exit path
  ~device_guard() { cudaSetDevice(g_dev.device); }
};
}  // namespace

int b200_mgpu_init(int ndev, const int* devices_or_null) {
  int rc = ensure_init();
  if (rc) return rc;
  if (ndev < 1 || ndev > MSM_PEER_MAX) return fail(B200_E_ARG, "ndev %d outside 1..%d", ndev, MSM_PEER_MAX);
  std::lock_guard<std::mutex> lk(g_mgpu.mu);
  if (g_mgpu.ready) {
    if (g_mgpu.ndev != ndev) return fail(B200_E_ARG, "already initialised with %d devices", g_mgpu.ndev);
    return B200_OK;
  }
  int have = 0;
  CU(cudaGetDeviceCount(&have));
  device_guard guard;
  for (int d = 0; d < ndev; d++) {
    int id = devices_or_null ? devices_or_null[d] : d;
    if (id < 0 || id >= have) return fail(B200_E_ARG, "device %d not present (%d visible)", id, have);
    g_mgpu.dev[d] = id;
  }
  for (int d = 0; d < ndev; d++) {
    CU(cudaSetDevice(g_mgpu.dev[d]));
    CU(cudaStreamCreateWithFlags(&g_mgpu.stream[d], cudaStreamNonBlocking));
    CU(cudaMalloc(&g_mgpu.xbuf[d], MSM_PEER_BUF_BYTES));
    CU(cudaMemset(g_mgpu.xbuf[d], 0, MSM_PEER_BUF_BYTES));
    CU(cudaMalloc(&g_mgpu.out_dev[d], 96));
    for (int e = 0; e < ndev; e++) {
      if (g_mgpu.dev[e] == g_mgpu.dev[d]) continue;
      int can = 0;
      CU(cudaDeviceCanAccessPeer(&can, g_mgpu.dev[d], g_mgpu.dev[e]));
      if (!can) return fail(B200_E_CUDA, "device %d cannot access device %d (no NVLink / P2P path)", g_mgpu.dev[d], g_mgpu.dev[e]);
      cudaError_t pe = cudaDeviceEnablePeerAccess(g_mgpu.dev[e], 0);
      if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled)
        return fail(B200_E_CUDA, "cudaDeviceEnablePeerAccess(%d -> %d): %s", g_mgpu.dev[d], g_mgpu.dev[e], cudaGetErrorString(pe));
      cudaGetLastError();
    }
  }
  CU(cudaMallocHost(&g_mgpu.out_host, 96));
  g_mgpu.ndev = ndev;
  g_mgpu.ready = true;
  return B200_OK;
}

int b200_mgpu_ck_register(int curve_id, const void* bases, size_t n, const void* h, int window_bits, uint64_t* key) {
  int rc = ensure_init();
  if (rc) return rc;
  if (!g_mgpu.ready) return fail(B200_E_ARG, "b200_mgpu_init has not been called");
  if (curve_id < 0 || curve_id > 3) return fail(B200_E_ARG, "unknown curve id %d", curve_id);
  if (!bases || !key || n == 0) return fail(B200_E_ARG, "bad argument");
  std::lock_guard<std::mutex> lk(g_mgpu.mu);
  device_guard guard;
  auto mk = std::make_shared<mgpu_key>();
  mk->curve = curve_id;
  mk->n = n;
  mk->has_h = h != nullptr;
  const int D = g_mgpu.ndev;
  for (int d = 0; d < D; d++) {
    size_t nd = mgpu_count(n, d, D);
    if (nd == 0 && !(d == 0 && h)) continue;  // this device owns nothing of this (tiny) key
    CU(cudaSetDevice(g_mgpu.dev[d]));
    if (nd == 0) return fail(B200_E_ARG, "key of %zu points is too small to carry a blinding generator on %d devices", n, D);
    rc = register_key(curve_id, (const char*)bases + (size_t)d * MGPU_BLOCK * 64, false, nd, d == 0 ? h : nullptr,
                      window_bits, true, mk->part[d], nullptr, g_mgpu.stream[d], MGPU_BLOCK * (size_t)D, MGPU_BLOCK);
    if (rc) return rc;
  }
  std::lock_guard<std::mutex> lk2(g_mkeys_mu);
  *key = g_next_mkey++;
  g_mkeys[*key] = mk;
  return B200_OK;
}

int b200_mgpu_ck_release(uint64_t key) {
  std::shared_ptr<mgpu_key> mk;
  {
    std::lock_guard<std::mutex> lk(g_mkeys_mu);
    auto it = g_mkeys.find(key);
    if (it == g_mkeys.end()) return fail(B200_E_HANDLE, "unknown multi-GPU key %llu", (unsigned long long)key);
    mk = it->second;
    g_mkeys.erase(it);
  }
  std::lock_guard<std::mutex> lk(g_mgpu.mu);  // wait for an in-flight call
  device_guard guard;
  for (int d = 0; d < g_mgpu.ndev; d++) {
    cudaSetDevice(g_mgpu.dev[d]);
    cudaStreamSynchronize(g_mgpu.stream[d]);
  }
  return B200_OK;
}

int b200_mgpu_commit(uint64_t key, const void* scalars, size_t n, const void* r, void* out) {
  int rc = ensure_init();
  if (rc) return rc;
  if (!g_mgpu.ready) return fail(B200_E_ARG, "b200_mgpu_init has not been called");
  std::shared_ptr<mgpu_key> mk;
  {
    std::lock_guard<std::mutex> lk(g_mkeys_mu);
    auto it = g_mkeys.find(key);
    if (it == g_mkeys.end()) return fail(B200_E_HANDLE, "unknown multi-GPU key %llu", (unsigned long long)key);
    mk = it->second;
  }
  if (!out || (n && !scalars)) return fail(B200_E_ARG, "null pointer");
  if (n > mk->n) return fail(B200_E_RANGE, "commit of %zu scalars exceeds key length %zu", n, mk->n);
  if (r && !mk->has_h) return fail(B200_E_ARG, "key was registered without a blinding generator");
#if defined(NOVA_MSM_ARITH29)
  return fail(B200_E_ARG, "the fused exchange needs the default (8x32-bit) arithmetic build");
#else
  std::lock_guard<std::mutex> lk(g_mgpu.mu);
  device_guard guard;
  const int D = g_mgpu.ndev;
  msm_peer peer;
  peer.world = D;
  peer.epoch = ++g_mgpu.epoch;
  for (int d = 0; d < D; d++) peer.buf[d] = g_mgpu.xbuf[d];
  const field_ops* bops = ops_for_field(CURVES[mk->curve].base_fid);
  // workspaces first: a (re)allocation synchronises its device, and by then the other devices' last kernels may
  // already be spinning on this device's partial
  for (int d = 0; d < D; d++) {
    ck_ctx* part = mk->part[d].get();
    const size_t nd = mgpu_count(n, d, D);
    if (!part || (nd == 0 && !(d == 0 && r))) continue;
    CU(cudaSetDevice(g_mgpu.dev[d]));
    std::lock_guard<std::mutex> plk(part->mu);
    if ((rc = ensure_workspace(*part, part->ws, nd + 1, 1))) return rc;
  }
  for (int d = 0; d < D; d++) {
    CU(cudaSetDevice(g_mgpu.dev[d]));
    cudaStream_t s = g_mgpu.stream[d];
    peer.rank = d;
    const size_t nd = mgpu_count(n, d, D);
    const bool blind = d == 0 && r != nullptr;
    ck_ctx* part = mk->part[d].get();
    if ((nd == 0 && !blind) || !part) {  // nothing here: deliver the identity so that the peers' sums complete
      msm_plan p0{};
      p0.peer = peer;
      bops->exchange_identity(s, p0, g_mgpu.out_dev[d]);
      count_launch(1);
      CU(cudaGetLastError());
      continue;
    }
    std::lock_guard<std::mutex> plk(part->mu);
    rc = ensure_workspace(*part, part->ws, nd + 1, 1);
    if (rc) return rc;
    if ((rc = ws_acquire(part->ws, s))) return rc;
    const size_t full = nd / MGPU_BLOCK, rest = nd % MGPU_BLOCK;
    const char* src = (const char*)scalars + (size_t)d * MGPU_BLOCK * 32;
    if (full)
      CU(cudaMemcpy2DAsync(part->ws.scalars, MGPU_BLOCK * 32, src, MGPU_BLOCK * (size_t)D * 32, MGPU_BLOCK * 32, full,
                           cudaMemcpyHostToDevice, s));
    if (rest)
      CU(cudaMemcpyAsync((char*)part->ws.scalars + full * MGPU_BLOCK * 32, src + full * MGPU_BLOCK * (size_t)D * 32,
                         rest * 32, cudaMemcpyHostToDevice, s));
    if (blind) CU(cudaMemcpyAsync((char*)part->ws.scalars + nd * 32, r, 32, cudaMemcpyHostToDevice, s));
    rc = enqueue_msm(*part, part->ws, 0, part->ws.scalars, nd + (blind ? 1 : 0), g_mgpu.out_dev[d], s, 0, blind, false,
                     &peer, /*profile_ok=*/false);
    if (rc) return rc;
  }
  CU(cudaSetDevice(g_mgpu.dev[0]));
  CU(cudaMemcpyAsync(g_mgpu.out_host, g_mgpu.out_dev[0], 96, cudaMemcpyDeviceToHost, g_mgpu.stream[0]));
  for (int d = 0; d < D; d++) {  // the caller's buffer is free again and every device has finished its part
    CU(cudaSetDevice(g_mgpu.dev[d]));
    CU(cudaStreamSynchronize(g_mgpu.stream[d]));
  }
  unsigned long long err = 0;
  CU(cudaSetDevice(g_mgpu.dev[0]));
  CU(cudaMemcpy(&err, (const char*)g_mgpu.xbuf[0] + MSM_PEER_ERR_OFF, 8, cudaMemcpyDeviceToHost));
  if (err) return fail(B200_E_PEER, "a device never delivered its partial sum (epoch %llu)", err);
  memcpy(out, g_mgpu.out_host, 96);
  return B200_OK;
#endif
}

// ---- field vectors ------------------------------------------------------------------------------
int b200_cross_term_dev(int fid, const void* az, const void* bz, const void* cz, const void* e1,
                        const void* e2, const void* u, size_t n, void* t, void* stream) {
  return with_field(fid, [&](const field_ops* ops) {
    if (n == 0) return (int)B200_OK;
    if (!az || !bz || !cz || !e1 || !u || !t) return fail(B200_E_ARG, "null pointer");
    ops->cross_term(pick_stream(stream), az, bz, cz, e1, e2, u, n, t);
    count_launch(1);
    CU(cudaGetLastError());
    return (int)B200_OK;
  });
}
int b200_axpy_dev(int fid, const void* a, const void* b, const void* r, size_t n, void* out,
                  void* stream) {
  return with_field(fid, [&](const field_ops* ops) {
    if (n == 0) return (int)B200_OK;
    if (!a || !b || !r || !out) return fail(B200_E_ARG, "null pointer");
    ops->axpy(pick_stream(stream), a, b, r, n, out);
    count_launch(1);
    CU(cudaGetLastError());
    return (int)B200_OK;
  });
}
int b200_vec_mul_dev(int fid, const void* a, const void* b, size_t n, void* out, void* stream) {
  return with_field(fid, [&](const field_ops* ops) {
    if (n == 0) return (int)B200_OK;
    if (!a || !b || !out) return fail(B200_E_ARG, "null pointer");
    ops->vec_mul(pick_stream(stream), a, b, n, out);
    count_launch(1);
    CU(cudaGetLastError());
    return (int)B200_OK;
  });
}
int b200_logup_hash_dev(int fid, const void* val, const void* addr_or_null, const void* gamma,
                        const void* r, size_t n, void* out, void* stream) {
  return with_field(fid, [&](const field_ops* ops) {
    if (n == 0) return (int)B200_OK;
    if (!val || !gamma || !r || !out) return fail(B200_E_ARG, "null pointer");
    ops->logup_hash(pick_stream(stream), val, addr_or_null, gamma, r, n, out);
    count_launch(1);
    CU(cudaGetLastError());
    return (int)B200_OK;
  });
}
int b200_vec_add_dev(int fid, const void* a, const void* b, size_t n, void* out, void* stream) {
  return with_field(fid, [&](const field_ops* ops) {
    if (n == 0) return (int)B200_OK;
    if (!a || !b || !out) return fail(B200_E_ARG, "null pointer");
    ops->vec_add(pick_stream(stream), a, b, n, out);
    count_launch(1);
    CU(cudaGetLastError());
    return (int)B200_OK;
  });
}
int b200_bind_top_dev(int fid, void* z, size_t n, const void* r, void* stream) {
  return with_field(fid, [&](const field_ops* ops) {
    if (n < 2) return (int)B200_OK;
    if (n & 1) return fail(B200_E_ARG, "bind_top needs an even length, got %zu", n);
    if (!z || !r) return fail(B200_E_ARG, "null pointer");
    ops->bind_top(pick_stream(stream), z, n, r);
    count_launch(1);
    CU(cudaGetLastError());
    return (int)B200_OK;
  });
}

int b200_bind_top_multi_dev(int fid, void* const* zs, size_t k, size_t n, const void* r, void* stream) {
  return with_field(fid, [&](const field_ops* ops) {
    if (k == 0 || n < 2) return (int)B200_OK;
    if (n & 1) return fail(B200_E_ARG, "bind_top needs an even length, got %zu", n);
    if (!zs || !r) return fail(B200_E_ARG, "null pointer");
    cudaStream_t s = pick_stream(stream);
    for (size_t j = 0; j < k; j += BIND_MULTI_MAX) {
      const int cnt = (int)(k - j < (size_t)BIND_MULTI_MAX ? k - j : (size_t)BIND_MULTI_MAX);
      for (int i = 0; i < cnt; i++)
        if (!zs[j + i]) return fail(B200_E_ARG, "null table %zu", j + i);
      ops->bind_top_multi(s, zs + j, cnt, n, r);
      count_launch(1);
    }
    CU(cudaGetLastError());
    return (int)B200_OK;
  });
}

// host-pointer forms: the _dev forms above, staged through via_device
int b200_cross_term(int fid, const void* az, const void* bz, const void* cz, const void* e1,
                    const void* e2, const void* u, size_t n, void* t) {
  int rc = ensure_init();
  if (rc || n == 0) return rc;
  const size_t vec = 32 * n;
  return via_device({up(az, vec), up(bz, vec), up(cz, vec), up(e1, vec), up(e2, vec), up(u, 32), down(t, vec)},
                    [&](void* const* d, cudaStream_t s) {
                      return b200_cross_term_dev(fid, d[0], d[1], d[2], d[3], d[4], d[5], n, d[6], s);
                    });
}

int b200_axpy(int fid, const void* a, const void* b, const void* r, size_t n, void* out) {
  int rc = ensure_init();
  if (rc || n == 0) return rc;
  return via_device({up(a, 32 * n), up(b, 32 * n), up(r, 32), down(out, 32 * n)}, [&](void* const* d, cudaStream_t s) {
    return b200_axpy_dev(fid, d[0], d[1], d[2], n, d[3], s);
  });
}

int b200_vec_add(int fid, const void* a, const void* b, size_t n, void* out) {
  int rc = ensure_init();
  if (rc || n == 0) return rc;
  return via_device({up(a, 32 * n), up(b, 32 * n), down(out, 32 * n)}, [&](void* const* d, cudaStream_t s) {
    return b200_vec_add_dev(fid, d[0], d[1], n, d[2], s);
  });
}

// in place: all n elements go up, the bound first half comes back
int b200_bind_top(int fid, void* z, size_t n, const void* r) {
  int rc = ensure_init();
  if (rc || n < 2) return rc;
  return via_device({{z, 32 * n, z, 16 * n, 0}, up(r, 32)}, [&](void* const* d, cudaStream_t s) {
    return b200_bind_top_dev(fid, d[0], n, d[1], s);
  });
}

}  // extern "C"

#include "capi_poly.inc"
#include "capi_sumcheck.inc"
#include "capi_stream.inc"
#include "capi_neutron.inc"
