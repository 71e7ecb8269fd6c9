// Per-field launcher table.  Every kernel in this library is a template over one prime field
// (point kernels over the curve's BASE field, digit/field-vector kernels over the field the
// vector lives in); each ops_<field>.cu instantiates the whole set once and exports it through
// a `field_ops` table so the C ABI (capi.cu) is template-free and the four translation units
// compile in parallel.
#pragma once
#include <cstdlib>
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>

namespace nova {

struct msm_plan;
struct multi_args;     // poly_kernels.cuh
struct poly_multi_args;
struct scb_tail_args;  // sumcheck_tail.cuh
struct spark_mats;     // poly_kernels.cuh
struct r1cs_mats;      // poly_kernels.cuh

struct field_ops {
  int field_id;
  // --- MSM stages -------------------------------------------------------------------------
  // scalar-field side
  void (*digits)(cudaStream_t, const void* scalars, const msm_plan&);
  // base-field side
  void (*expand_key)(cudaStream_t, void* tables, size_t n_ck, int ntables, int shift);
  void (*accumulate)(cudaStream_t, const void* tables, const msm_plan&);
  void (*fixup)(cudaStream_t, const msm_plan&);
  void (*reduce)(cudaStream_t, const msm_plan&, void* out_jac);
  // small helpers on points (base field)
  void (*sum_points)(cudaStream_t, const void* tables, const uint32_t* idx_or_null, size_t n,
                     void* scratch_xyzz, void* out_jac);
  void (*jacobian_sum)(cudaStream_t, const void* pts, int k, void* out_jac);
  void (*index_bases)(cudaStream_t, void* bases, size_t n, const void* gen_affine, uint64_t k0);
  // --- field-vector kernels (K4..K8) --------------------------------------------------------
  void (*cross_term)(cudaStream_t, const void* az, const void* bz, const void* cz, const void* e1,
                     const void* e2_or_null, const void* u, size_t n, void* t);
  void (*axpy)(cudaStream_t, const void* a, const void* b, const void* r, size_t n, void* out);
  void (*vec_add)(cudaStream_t, const void* a, const void* b, size_t n, void* out);
  void (*bind_top)(cudaStream_t, void* z, size_t n, const void* r);
  void (*bind_top_multi)(cudaStream_t, void* const* zs, int k, size_t n, const void* r);  // k <= 32 tables of length n
  void (*vec_mul)(cudaStream_t, const void* a, const void* b, size_t n, void* out);
  void (*logup_hash)(cudaStream_t, const void* val, const void* addr_or_null, const void* gamma,
                     const void* r, size_t n, void* out);
  void (*fold_halves)(cudaStream_t, const void* v, size_t half, const void* x_lo, const void* x_hi, void* out);
  void (*ipa_scalars)(cudaStream_t, const void* a, const void* w, size_t n, size_t nk, void* sL, void* sR);
  void (*ipa_weights)(cudaStream_t, void* w, size_t n, size_t nk, const void* r, const void* r_inv);
  void (*fill_one)(cudaStream_t, void* w, size_t n);
  // --- sum-check / MLE / HyperKZG / SpMV (poly_kernels.cuh) ----------------------------------
  // form: sc_form_id; writes sc_form_nout(form) elements to out; scratch >= SC_MAX_BLOCKS*3*32 B
  void (*sc_reduce)(cudaStream_t, int form, const void* A, const void* B, const void* C, size_t count,
                    size_t half, const void* eq_left, const void* eq_right, int shift, size_t id_mul,
                    size_t id_add, void* scratch, void* out);
  void (*eq_small)(cudaStream_t, const void* r, int ell, void* out);
  void (*eq_outer)(cudaStream_t, const void* left, const void* right, int right_bits, size_t n,
                   void* out);
  void (*batch_invert)(cudaStream_t, const void* in, size_t n, void* out, int* zero_flag);
  void (*rlc)(cudaStream_t, const void* const* polys, const size_t* lens, int k, const void* coeffs,
              size_t n, void* out);
  void (*kzg_fold)(cudaStream_t, const void* p, const void* x, size_t half, void* out);
  // evals[q] = f(us[q]), q < nu <= 3, coalesced strided Horner; scratch >= POLY_EVAL_SCRATCH_ELEMS*32 B
  void (*poly_eval)(cudaStream_t, const void* f, size_t n, const void* us, int nu, void* scratch,
                    void* evals);
  // quotient f / (X - u) (n-1 coefficients) of each of `cols` interleaved polynomials of n coefficients
  // (coefficient k of column j at f[k * cols + j], quotient likewise in out); rem_or_null receives the
  // cols remainders f_j(u).  scratch >= poly_div_scratch_elems(n, cols) * 32 B
  void (*poly_div)(cudaStream_t, const void* f, size_t n, size_t cols, const void* u, void* scratch, void* out,
                   void* rem_or_null);
  void (*spmv_classify)(cudaStream_t, const void* vals, size_t nnz, int8_t* codes);
  void (*spmv)(cudaStream_t, const uint32_t* indptr, const uint32_t* cols, const int8_t* codes,
               const void* vals, size_t rows, const void* z1, const void* z2_or_null, void* o1,
               void* o2_or_null);
  void (*spmv_t)(cudaStream_t, const uint32_t* tptr, const uint32_t* trow, const uint32_t* tperm,
                 const int8_t* codes, const void* vals, size_t cols, size_t out_len, const void* rx,
                 void* out);
  // one sum-check round of O(1) prover algebra + Fiat-Shamir on the device (transcript.cuh):
  // round polynomial from the reduction results, Keccak transcript absorb/squeeze, challenge,
  // new claim / eq bound.  kind: sc_round_kind; state: b200_sc_state (144 B, device)
  void (*sc_round)(cudaStream_t, int kind, void* state, const void* res, const void* tau,
                   const void* tau_inv, const void* pending, uint32_t pending_len, int absorb_label,
                   int squeeze_label, void* out_poly, void* out_r);
  void (*fe_inv_each)(cudaStream_t, const void* in, size_t n, void* out);  // 0 -> 0
  // digits + histogram of scalars [i0, i1) of a p.n-long vector (streamed witness hand-off)
  void (*digits_range)(cudaStream_t, const void* scalars, size_t i0, size_t i1, const msm_plan&);
  // one round of a batched sum-check (ppsnark prove_helper) on the device (transcript_batched.cuh);
  // desc: scb_desc by value, state: scb_state (1296 B, device)
  void (*sc_round_batched)(cudaStream_t, const void* desc, void* state, const void* sums, const void* pending,
                           uint32_t pending_len, int absorb_label, int squeeze_label, void* out_poly, void* out_r);
  // key validation: *first_bad = min index of an off-curve base (caller presets 0xFFFFFFFF)
  void (*on_curve)(cudaStream_t, const void* pts, size_t n, int b_small, uint32_t* first_bad);
  // test SRS (hyperkzg.rs:357-376): out[i] = u^i canonical (scalar field) ; bases[i] = [scalars[i]] G (base field)
  void (*powers_canonical)(cudaStream_t, const void* u_mont, size_t n, void* out);
  void (*scalar_bases)(cudaStream_t, void* bases, size_t n, const void* gen_affine, const void* scalars_canonical);
  // Poseidon RO squeeze on the device (poseidon.cuh): t, r_f, r_p; rc / mds Montgomery; out = [hash, challenge, canonical challenge]
  void (*poseidon_ro)(cudaStream_t, int t, int r_f, int r_p, const void* rc, const void* mds, const void* elems, uint32_t n,
                      const void* tag_canonical, int num_bits, int start_with_one, void* out);
  void (*to_mont)(cudaStream_t, const void* in_canonical, size_t n, void* out);
  // sharded MSM whose rank has no pairs: publish the identity and sum the peers' partials (plan.peer)
  void (*exchange_identity)(cudaStream_t, const msm_plan&, void* out_jac);
  // the round with the final stage of the reductions folded in: partials = k_form_reduce_multi's output for the
  // nsums <= 32 sums of the round (desc.slot[i] = 3 * index of claim i's sum)
  void (*sc_round_batched_fused)(cudaStream_t, const void* desc, void* state, const void* partials, int nblocks,
                                 int nsums, const void* pending, uint32_t pending_len, int absorb_label,
                                 int squeeze_label, void* out_poly, void* out_r);
  // first stage only of sc_reduce_multi; returns the blocks per sum (the nblocks of sc_round_batched_fused)
  int (*sc_reduce_multi_partials)(cudaStream_t, const multi_args&, void* scratch);
  void (*gather_heads)(cudaStream_t, void* const* zs, int k, void* out);  // out[t] = zs[t][0], k <= 32
  // <= 32 polynomials of <= 2^POLY_SMALL_MAX_LOG2 coefficients at the same nu <= 3 points, one launch
  void (*poly_eval_small_multi)(cudaStream_t, const poly_multi_args&, const void* us, int nu, void* evals);
  // nested eq tables eq(taus[hi-k .. hi)), k = 0 .. K <= EQ_PREFIX_MAX_K, table k at element 2^k - 1 of out
  void (*eq_prefix_tables)(cudaStream_t, const void* taus, int hi, int K, void* out);
  // all sums of a batched sum-check round in two launches: out[3 y + k] = output k of sum y;
  // scratch >= sc_multi_scratch_elems(n sums) * 32 B
  void (*sc_reduce_multi)(cudaStream_t, const multi_args&, void* scratch, void* out);
  // every remaining round of a batched sum-check in one CTA (sumcheck_tail.cuh); sums: 6 * 16 elements of scratch
  void (*scb_tail)(cudaStream_t, const scb_tail_args&, void* state, void* sums, const void* pending,
                   uint32_t pending_len, int absorb_label, int squeeze_label, void* polys, void* rs);
  // Mercury (mercury.rs): out[r] = sum_c f[r*cols + c] v[c]; the s polynomial (b - 1 coefficients, k_mercury_s_poly)
  void (*mat_vec_rows)(cudaStream_t, const void* f, size_t rows, size_t cols, const void* v, void* out);
  void (*mercury_s_poly)(cudaStream_t, const void* a1, const void* b1, const void* a2, const void* b2, size_t b,
                         const void* gamma, void* out);
  // NeutronNova (neutron/nifs.rs, relation.rs): the five raw sums of prove_helper (k_neutron_evals; scratch >=
  // neutron_evals_scratch_elems(left * right) * 32 B), split_evals of the power polynomial, out = a + r (b - a)
  void (*neutron_evals)(cudaStream_t, const void* e1, const void* az1, const void* bz1, const void* cz1,
                        const void* e2, const void* az2, const void* bz2, const void* cz2, size_t left, size_t right,
                        void* scratch, void* out);
  void (*pow_split_evals)(cudaStream_t, const void* tau, size_t left, size_t right, void* out);
  void (*lerp)(cudaStream_t, const void* a, const void* b, const void* r, size_t n, void* out);
  // R1CSShapeSparkRepr::new (k_spark_repr): row, col, ts_row, ts_col (Montgomery) and the u32 row / col indices
  void (*spark_repr)(cudaStream_t, const spark_mats&, size_t N, void* row, void* col, void* ts_row, void* ts_col,
                     uint32_t* row_idx, uint32_t* col_idx);
  // ck_derive_by_address (msm_kernels.cuh): flags[0] = first identity base of table 0, flags[1] = first address
  // >= table_size among addr[0 .. m), m <= n (caller presets 0xFFFFFFFF); buckets [0, K) -> boundary-format bases
  void (*derive_check)(cudaStream_t, const void* tables, size_t n, const uint32_t* addr, size_t m, size_t table_size,
                       uint32_t* flags);
  void (*derive_affine)(cudaStream_t, const uint32_t* start, uint32_t K, const void* buckets, void* out_bases);
  // the verifier's matrix evaluations (k_r1cs_eval + k_r1cs_final): out[y] = sum_e T_x[row_e] T_y[col_e] val_e over
  // matrix y < k <= 3; scratch >= r1cs_eval_scratch_elems(k) * 32 B
  void (*r1cs_eval)(cudaStream_t, const r1cs_mats&, int k, const void* tx, const void* ty, void* scratch, void* out);
  // the IPA verifier's s (k_ipa_s_half, k_eq_outer): out[i] = scale * prod_j (bit j of i, MSB first ? r_j : r_inv_j),
  // i < 2^L; scratch >= ipa_s_scratch_elems(L) * 32 B
  void (*ipa_s)(cudaStream_t, const void* r, const void* r_inv, int L, const void* scale_or_null, void* scratch,
                void* out);
};
// SM count of the H100 SXM (sm_90a): grids below are sized in whole waves of it
constexpr int NUM_SMS = 132;
constexpr int SC_MAX_BLOCKS = NUM_SMS * 4;
constexpr int EQ_PREFIX_MAX_K = 12;
constexpr int SC_MULTI_BLOCKS = NUM_SMS * 2;  // blocks per sum of sc_reduce_multi (times <= 32 sums in grid.y)
inline size_t sc_multi_scratch_elems(int nsums) { return (size_t)nsums * SC_MULTI_BLOCKS * 3; }
// NOVA_B200_SC_SEG=1 selects the segmented reduction of the eq-weighted sum-check forms (k_form_reduce_eqseg)
inline bool sc_segmented_enabled() {
  static const bool on = [] {
    const char* e = getenv("NOVA_B200_SC_SEG");
    return e != nullptr && e[0] == '1';
  }();
  return on;
}
constexpr size_t POLY_EVAL_SCRATCH_ELEMS = (size_t)3 * (1 + SC_MAX_BLOCKS + 256) + (size_t)3 * SC_MAX_BLOCKS;
constexpr int POLY_CHUNK_HOST = 64;  // must equal POLY_CHUNK in poly_kernels.cuh
inline size_t poly_div_scratch_elems(size_t n, size_t cols = 1) {
  size_t t1 = (n + POLY_CHUNK_HOST - 1) / POLY_CHUNK_HOST, t2 = (t1 + POLY_CHUNK_HOST - 1) / POLY_CHUNK_HOST;
  return cols * (2 * t1 + 2 * t2 + 1) + 8;
}
// above this many chunks per polynomial the carries are scanned in two levels
constexpr size_t POLY_DIV_ONE_LEVEL_CHUNKS = 8192;
// k_neutron_evals: one block per tile of at least NEUTRON_ROWS_PER_BLOCK rows, at most NEUTRON_MAX_BLOCKS blocks
constexpr size_t NEUTRON_ROWS_PER_BLOCK = 1024;
constexpr size_t NEUTRON_MAX_BLOCKS = (size_t)NUM_SMS * 8;
inline size_t neutron_evals_blocks(size_t n) {
  size_t g = (n + NEUTRON_ROWS_PER_BLOCK - 1) / NEUTRON_ROWS_PER_BLOCK;
  return g < 1 ? 1 : (g > NEUTRON_MAX_BLOCKS ? NEUTRON_MAX_BLOCKS : g);
}
inline size_t neutron_evals_scratch_elems(size_t n) { return 5 * neutron_evals_blocks(n); }
// k_r1cs_eval: at least R1CS_MIN_CHUNK entries per thread, at most R1CS_EVAL_BLOCKS blocks of 256 threads per matrix
constexpr size_t R1CS_MIN_CHUNK = 16;
constexpr unsigned R1CS_EVAL_BLOCKS = NUM_SMS * 2;
inline size_t r1cs_eval_scratch_elems(int k) { return (size_t)k * R1CS_EVAL_BLOCKS; }
// k_ipa_s_half writes the whole s directly up to IPA_S_DIRECT_BITS bits; above, two half tables and their outer product
constexpr int IPA_S_DIRECT_BITS = 10;
inline size_t ipa_s_scratch_elems(int L) {
  return L <= IPA_S_DIRECT_BITS ? 0 : ((size_t)1 << (L - L / 2)) + ((size_t)1 << (L / 2));
}

extern const field_ops OPS_BN254_FR, OPS_BN254_FQ, OPS_PALLAS_FP, OPS_PALLAS_FQ;

inline const field_ops* ops_for_field(int fid) {
  switch (fid) {
    case 0: return &OPS_BN254_FR;
    case 1: return &OPS_BN254_FQ;
    case 2: return &OPS_PALLAS_FP;
    case 3: return &OPS_PALLAS_FQ;
    default: return nullptr;
  }
}

// field-independent MSM stages (msm_common.cu)
int msm_sort(cudaStream_t, const msm_plan&);  // returns the number of kernels launched
void msm_digits_small(cudaStream_t, const void* scalars, int elem_bytes, const msm_plan&);
// ck_derive_by_address: the address stage (k_address_entries) and the radix passes over p.n = m entries, then the
// starts of the p.B buckets; returns the number of kernels launched
int derive_sort(cudaStream_t, const uint32_t* addr, const msm_plan&);

}  // namespace nova
