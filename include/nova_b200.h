/* nova_b200 -- C ABI of the H100-native (sm_90a) Nova prover hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8b): the entry points a `provider/b200.rs` module in
 * nova-snark would bind through a `nova-b200-sys` crate, exactly as `provider/blitzar.rs:7-40`
 * binds the blitzar library today.  Plain pointers and sizes only; no C++/torch types.
 *
 * Conventions (mirroring the reference's call sites):
 *   - field element  = 32 B = 4 x u64 little-endian limbs, Montgomery form, R = 2^256
 *                      (halo2curves 0.9.0 in-memory layout; blitzar.rs:10-16 precedent)
 *   - affine point   = {x, y} 64 B; identity = all-zero coordinates
 *   - group result   = Jacobian {x, y, z} 96 B (x_aff = x/z^2, y_aff = y/z^3); identity has z = 0
 *   - inputs are borrowed and never mutated; outputs are caller-owned; the library keeps no
 *     host pointer after return (src/provider/traits.rs:77-117 take slices, return by value)
 *   - every function returns 0 on success, a B200_E_* code otherwise; it never throws and never
 *     calls back.  b200_last_error() gives a thread-local message.  The reference's MSM/commit
 *     are infallible (`assert!` on length mismatch, msm.rs:226, pedersen.rs:264): the Rust shim
 *     panics on non-zero for those and maps to NovaError::GpuError (errors.rs:84-86) for the
 *     Result-returning sites (r1cs/mod.rs:411-413).
 *   - all entry points are thread-safe and re-entrant: the reference calls commits concurrently
 *     from rayon workers (r1cs/mod.rs:509-512, ppsnark.rs:1155-1158, hyperkzg.rs:1062-1065).
 *   - `*_dev` variants take DEVICE pointers (on the key's device) and a cudaStream_t passed as
 *     void* (NULL = the library's stream); they are asynchronous and are what a device-resident
 *     pipeline (fused Z1+Z2 -> SpMV -> T -> MSM(T)) chains together.
 *   - THERE IS NO CPU FALLBACK: if no CUDA device is usable every call returns B200_E_CUDA.
 */
#ifndef NOVA_B200_H
#define NOVA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* field ids (moduli: bn256_grumpkin.rs:39-40,84-85; pasta.rs:37-38,45-46) */
enum { B200_FIELD_BN254_FR = 0, B200_FIELD_BN254_FQ = 1, B200_FIELD_PALLAS_FP = 2, B200_FIELD_PALLAS_FQ = 3 };
/* curve ids: (base field, scalar field) = G1:(FQ,FR) Grumpkin:(FR,FQ) Pallas:(FP,FQ) Vesta:(FQ,FP) */
enum { B200_CURVE_BN254_G1 = 0, B200_CURVE_GRUMPKIN = 1, B200_CURVE_PALLAS = 2, B200_CURVE_VESTA = 3 };

enum {
  B200_OK = 0,
  B200_E_ARG = 1,      /* bad argument (null pointer, unknown id, length mismatch: msm.rs:226) */
  B200_E_CUDA = 2,     /* CUDA runtime failure or no device (maps to NovaError::GpuError) */
  B200_E_HANDLE = 3,   /* unknown / released handle */
  B200_E_NOMEM = 4,    /* device memory exhausted */
  B200_E_RANGE = 5,    /* slice outside the registered key (pedersen.rs:264 assert) */
  B200_E_ZERO = 6,     /* batch_invert met a zero (NovaError::InternalError, spartan/mod.rs:98-100) */
  B200_E_PEER = 8,     /* a peer GPU never delivered its partial sum to the exchange buffer (multi-GPU MSM) */
  B200_E_POINT = 7,    /* a key point is non-canonical or off the curve (NovaError::InvalidCommitmentKey,
                          hyperkzg.rs:113-119; PtauFileError::PointNotOnCurve, ptau.rs:386-388) */
  B200_E_INDEX = 9     /* an address outside the derived table (NovaError::InvalidIndex, b200_ck_derive_by_address) */
};

/* ---- library / device ------------------------------------------------------------------ */
int b200_init(int device);                 /* idempotent; selects the device for this process */
int b200_device_count(int* count);
const char* b200_last_error(void);         /* thread-local */
const char* b200_version(void);

/* pinned host buffers + raw device buffers, so a host language can stage witnesses for DMA and
 * keep folded vectors (W, E, T) resident between calls (SURVEY.md §7 step 7) */
int b200_host_alloc(size_t bytes, void** ptr);
int b200_host_free(void* ptr);
int b200_dev_alloc(size_t bytes, void** dptr);
int b200_dev_free(void* dptr);
int b200_memcpy_h2d(void* dptr, const void* hptr, size_t bytes);
int b200_memcpy_d2h(void* hptr, const void* dptr, size_t bytes);
/* asynchronous on `stream` (NULL = the library's stream) */
int b200_memcpy_d2d(void* dst, const void* src, size_t bytes, void* stream);
int b200_memset_dev(void* dptr, int byte, size_t bytes, void* stream);
int b200_sync(void);

/* per-stage device timing of the MSM pipeline (CUDA events on the launching stream) and a count
 * of the kernels this library launched; used by bench.py for the roofline line.  Stages:
 * 0 digits, 1 sort (scan + scatter), 2 bucket accumulate, 3 boundary fix-up, 4 bucket reduce. */
int b200_profile_enable(int on);
int b200_profile_reset(void);
int b200_profile_read(double* stage_ms, int nstages, uint64_t* msms, uint64_t* launches);

/* ---- commitment keys -------------------------------------------------------------------
 * Replaces holding `CommitmentKey{ck: Vec<Affine>, h}` (pedersen.rs:32-38, hyperkzg.rs:76-84) on
 * the host only: the bases are uploaded ONCE, expanded into the 2^(c*t)*P window tables, and stay
 * resident.  `h` is the blinding generator (CommitmentKey.h); NULL if the caller never blinds.
 * window_bits = 0 picks c from n.  Keys are immutable after registration. */
int b200_ck_register(int curve_id, const void* bases_affine_mont, size_t n,
                     const void* h_affine_mont_or_null, int window_bits, uint64_t* ck_handle);
/* The same registration for points that arrive from OUTSIDE the process -- CommitmentEngine::load_setup ->
 * read_ptau -> read_points (hyperkzg.rs:658-675, ptau.rs:372-438): every G1 point must have canonical
 * coordinates (read_raw) and lie on the curve, else PtauFileError::PointNotOnCurve.  The raw section bytes of
 * a PTAU file ARE this library's base layout (write_raw = in-memory Montgomery limbs, ptau.rs:197-208), so the
 * section goes to HBM unchanged, is validated there (one pass, 64 B and three products per point) and only then
 * expanded.  On an invalid point: B200_E_POINT, *first_bad = its index (n = the blinding generator), no key. */
int b200_ck_register_checked(int curve_id, const void* bases_affine_mont, size_t n,
                             const void* h_affine_mont_or_null, int window_bits, uint64_t* ck_handle,
                             size_t* first_bad);
/* test/bench key: bases[i] = (k0 + i) * G generated on the device (the analogue of the
 * reference's test-only setups, hyperkzg.rs:357-376 / curve_property_tests.rs:186-194);
 * with_h != 0 appends h = (k0 + n) * G as the blinding generator. */
int b200_ck_setup_synthetic(int curve_id, const void* generator_affine_mont, uint64_t k0, size_t n,
                            int with_h, int window_bits, uint64_t* ck_handle);
/* test/bench SRS: bases[i] = [tau^i] G generated on the device -- the reference's test-only KZG setup
 * (hyperkzg.rs:357-376 `setup_from_rng`: powers of a sampled tau).  A prover run at benchmark scale over such a
 * key can be checked by the restated verifier with the pairing replaced by L = [tau] R (oracle/hyperkzg_ref.py). */
int b200_ck_setup_tau(int curve_id, const void* generator_affine_mont, const void* tau_mont, size_t n,
                      int window_bits, uint64_t* ck_handle);
/* copies ck[offset .. offset + n) (affine, Montgomery: the layout b200_ck_register takes) back to host memory;
 * what `CommitmentKey::ck()` (traits.rs / hyperkzg.rs:98-110) gives a Rust caller.  The tests hand a
 * device-generated key to the CPU oracle with it. */
int b200_ck_export_bases(uint64_t ck_handle, size_t offset, size_t n, void* out_host);
/* ck_derive_by_address (traits/commitment.rs:177-194, pedersen.rs:360-382, hyperkzg.rs:731-749):
 *   derived[j] = sum_{i < m, addresses[i] = j} ck[i],  j < table_size   (a slot no address points to: the identity)
 * so that Comm(T[addresses], ck[..m]) = Comm(T, derived) for a lookup table T: a prover holding the derived key commits
 * to the table-sized vector in place of the lookup-sized one.  The derivation runs on the device (the bucket stage of a
 * one-window MSM whose scalars are all 1, with the address as the bucket) and the result is a new, independent resident
 * key of table_size bases, with its window tables built as b200_ck_register builds them (window_bits = 0 picks c from
 * table_size; a key of 2^22 bases or more also gets its 17-bit table set).  It carries the source key's h when the
 * source has one (HyperKZG's tau_H stays with the caller).  The call returns once the key is built; the source key may
 * be released right after, and other calls may use the source key meanwhile.
 * Errors, in the reference's order (nothing is registered and *out_handle is untouched on any of them; *first_bad,
 * when given, is SIZE_MAX unless noted):
 *   B200_E_HANDLE  unknown ck_handle
 *   B200_E_POINT   an identity generator anywhere in ck[0 .. n), *first_bad = its index (the reference panics:
 *                  ck_to_group_elements)
 *   B200_E_RANGE   m > n (NovaError::InvalidCommitmentKeyLength; a prefix m < n is allowed)
 *   B200_E_INDEX   an address >= table_size (NovaError::InvalidIndex), *first_bad = the smallest such position
 *   B200_E_ARG     table_size = 0 (the reference returns an empty key for m = 0; a key of no bases cannot be
 *                  registered here, as in b200_ck_register)
 *   B200_E_RANGE   table_size too large for the 31-bit table indices (the limit of b200_ck_register)
 * Null pointers and a window_bits outside {0} u [2, 24] give B200_E_ARG before any of these.  The host form checks the
 * 64-bit addresses before it narrows them: an address of 2^32 + 3 is reported at its position, never taken as slot 3.
 * Builds with -DNOVA_MSM_ARITH29 (table 0 not in the boundary format) return B200_E_ARG. */
int b200_ck_derive_by_address_dev(uint64_t ck_handle, const uint32_t* d_addresses, size_t m, size_t table_size,
                                  int window_bits, uint64_t* out_handle, size_t* first_bad_or_null, void* stream);
int b200_ck_derive_by_address(uint64_t ck_handle, const uint64_t* addresses, size_t m, size_t table_size,
                              int window_bits, uint64_t* out_handle, size_t* first_bad_or_null);
int b200_ck_release(uint64_t ck_handle);
int b200_ck_len(uint64_t ck_handle, size_t* n, int* window_bits, int* num_tables);

/* ---- MSM  (DlogGroupExt, src/provider/traits.rs:77-117; msm.rs:225) ---------------------- */
/* out = sum_i scalars[i] * ck[base_offset + i],  i < n.   n == 0 -> identity (msm.rs:228-230).
 * Replaces DlogGroupExt::vartime_multiscalar_mul(scalars, &ck.ck[..n]) (pedersen.rs:263-270,
 * hyperkzg.rs:584-591). */
int b200_msm(uint64_t ck_handle, size_t base_offset, const void* scalars_mont, size_t n,
             void* out_jacobian_mont);
int b200_msm_dev(uint64_t ck_handle, size_t base_offset, const void* d_scalars_mont, size_t n,
                 void* d_out_jacobian_mont, void* stream);
/* CommitmentEngineTrait::commit(ck, v, r) = MSM(v, ck[..n]) + r*h in ONE pass
 * (pedersen.rs:263-270, hyperkzg.rs:584-591).  r_or_null == NULL means r = 0 (benches/commit.rs:30).
 * Needs a key registered with h unless r is NULL. */
int b200_commit(uint64_t ck_handle, const void* scalars_mont, size_t n, const void* r_mont_or_null,
                void* out_jacobian_mont);
int b200_commit_dev(uint64_t ck_handle, const void* d_scalars_mont, size_t n,
                    const void* d_blind_mont_or_null, void* d_out_jacobian_mont, void* stream);
/* k commitments (r = 0) of device-resident vectors over prefixes of one key, spread over the key's
 * internal (stream, workspace) lanes so that the latency-bound tails of short MSMs overlap with the
 * next vector's work -- HyperKZG's ell-1 halving polynomials (hyperkzg.rs:1099-1100), the L / R pair
 * of an IPA round (ipa_pc.rs:222-238), the four memory oracles of ppsnark (ppsnark.rs:457-471).
 * d_out = k x 96 B; ordered after prior work on `stream`, which waits for every lane on return. */
/* the same for slices that do not start at the front of the key: MSM j runs over ck[base_offsets[j] .. + lens[j]).
 * What a rank of the sharded HyperKZG prover needs (its slice of every fold level sits at a different offset;
 * nova_b200/sharding.py), and the three quotient commitments of one proof. */
int b200_msm_many_dev(uint64_t ck_handle, const size_t* base_offsets, const void* const* d_scalars_mont,
                      const size_t* lens, size_t k, void* d_out_jacobian_mont, void* stream);
int b200_commit_many_dev(uint64_t ck_handle, const void* const* d_scalars_mont, const size_t* lens,
                         size_t k, void* d_out_jacobian_mont, void* stream);
/* k MSMs over prefixes of the same key: vector j uses ck[..lens[j]] (traits.rs:82-90,
 * blitzar.rs:23-40, hyperkzg.rs:594-612 batch_commit).  out = k x 96 B. */
int b200_msm_batch(uint64_t ck_handle, const void* const* scalars_mont, const size_t* lens,
                   size_t k, void* out_jacobian_mont);
/* integer scalars (msm.rs:469-503 msm_small / msm_small_with_max_num_bits): elem_bytes in
 * {1,2,4,8} little-endian unsigned; max_bits = 0 computes it from the data (msm.rs:473). */
int b200_msm_small(uint64_t ck_handle, size_t base_offset, const void* scalars_uint,
                   int elem_bytes, size_t n, int max_bits, void* out_jacobian_mont);
/* sum of ck[idx[j]] (msm.rs:689-708 batch_add; pedersen.rs commit_sparse_binary) */
int b200_msm_indices(uint64_t ck_handle, const uint64_t* idx, size_t m, void* out_jacobian_mont);
/* one-shot MSM over bases that are not a registered key (pedersen.rs:418-420,492,505) */
int b200_msm_adhoc(int curve_id, const void* bases_affine_mont, const void* scalars_mont, size_t n,
                   void* out_jacobian_mont);

/* out = sum of k Jacobian points (device pointers): the local combine after the all-gather of
 * per-GPU partial MSMs (SURVEY.md §8e; NCCL has no group-law reduction operator) */
int b200_jacobian_sum_dev(int curve_id, const void* d_points_jacobian, size_t k,
                          void* d_out_jacobian, void* stream);

/* ---- host-side Keccak-256 (no device work) ---------------------------------------------------------------
 * The digest the reference's transcript is built from (sha3::Keccak256, src/provider/keccak.rs:14, 66-95; known answer
 * keccak.rs:279-288).  The transcript stays on the host between device calls; the Python and C++ host layers hash
 * through this entry point.  A Rust host uses its own `sha3` crate and never calls it. */
int b200_keccak256(const void* data, size_t len, void* out32);

/* ---- the sharded MSM with its collective fused into the reduction (SURVEY.md §8e; traits.rs:77-117 over N GPUs) --
 * One process per GPU (or one host thread per GPU): every rank holds a key over ITS index range of the bases and an
 * exchange buffer all peers can write over NVLink.  b200_msm_sharded_dev runs the local Pippenger pipeline and its
 * last kernel writes the rank's partial sum straight into every peer's buffer (peer stores), waits for the peers'
 * partials and adds them in a fixed order: every rank ends with the same Jacobian coordinates, without an NCCL call
 * or an extra launch on the critical path ("allreduce" of group elements = all-to-all of 128 bytes + local sum).
 *
 *   b200_peer_buffer_alloc   a zeroed exchange buffer on this device (cudaMalloc, so that it can be exported)
 *   b200_ipc_export / open / close   CUDA IPC handle (64 bytes) of a device allocation / its mapping in another
 *                            process; ranks exchange the handles out of band (torch.distributed, MPI, a pipe)
 *   b200_peer_group_create   bufs[r] = rank r's buffer as mapped HERE (bufs[rank] = the local one), world <= 8
 *   b200_msm_sharded_dev     all ranks must call it in the same order (the epoch counter lives in the group)
 *   b200_peer_group_status   B200_E_PEER if a wait ever timed out (~2 s) instead of hanging the GPU */
int b200_peer_buffer_alloc(void** dptr);
int b200_peer_buffer_free(void* dptr);
int b200_ipc_export(const void* dptr, void* handle64_out);
int b200_ipc_open(const void* handle64, void** dptr);
int b200_ipc_close(void* dptr);
int b200_peer_group_create(int rank, int world, void* const* bufs, uint64_t* group);
int b200_peer_group_release(uint64_t group);
int b200_peer_group_status(uint64_t group);
int b200_msm_sharded_dev(uint64_t ck_handle, size_t base_offset, const void* d_scalars_mont, size_t n,
                         uint64_t group, void* d_out_jacobian, void* stream);

/* ---- Poseidon random oracle on the device (SURVEY.md §8f-3) ----------------------------------------------------
 * `PoseidonRO::squeeze` (src/provider/poseidon.rs:93-127): the sponge over the vendored neptune permutation
 * (src/frontend/gadgets/poseidon/), IO pattern [Absorb(n), Squeeze(1)], Simplex mode -- the hash NIFS::prove draws the
 * folding challenge from (src/nova/nifs.rs:47-63).  The constants (PoseidonConstants::new_with_strength_and_type(
 * Standard, Sponge): R_F, R_P, Grain-LFSR round constants, Cauchy MDS) come from the host (nova_b200/poseidon.py mirrors
 * their generation) in Montgomery form: rc[(R_F + R_P) * (arity + 1)], mds[(arity + 1)^2] row-major.
 * out = three field elements: the full hash (Montgomery), the challenge = its low num_bits bits (bit num_bits - 1
 * forced when start_with_one; Montgomery, same field), and the challenge as a canonical integer -- which
 * b200_to_mont_dev turns into an element of the OTHER curve's field (base_as_scalar), so that
 * commit_T -> absorb -> r -> fold can be enqueued without a host round trip. */
int b200_poseidon_register(int field_id, int arity, int r_f, int r_p, const void* rc_mont, const void* mds_mont,
                           uint64_t* poseidon_handle);
int b200_poseidon_release(uint64_t poseidon_handle);
int b200_poseidon_ro(uint64_t poseidon_handle, const void* elems_mont, size_t n, int num_bits, int start_with_one,
                     void* out96);
int b200_poseidon_ro_dev(uint64_t poseidon_handle, const void* d_elems_mont, size_t n, int num_bits, int start_with_one,
                         void* d_out96, void* stream);
/* out[i] = in[i] as a Montgomery element of field_id, in[i] a canonical integer < p */
int b200_to_mont_dev(int field_id, const void* d_canonical, size_t n, void* d_out, void* stream);

/* ---- ONE process, N GPUs behind one call (SURVEY.md §8b: "b200_init(device_count) + a key sharded across GPUs") ----
 * A host that calls CommitmentEngine::commit / DlogGroupExt::vartime_multiscalar_mul once (traits.rs:77-117,
 * pedersen.rs:263-270) gets the whole node: the key is distributed block-cyclically over the devices (every prefix
 * ck[..n] stays balanced), each device receives its strided slice of the scalars with one 2-D copy, runs the
 * Pippenger pipeline on its own stream, and the partial sums are exchanged by peer stores over NVLink inside the
 * last reduction kernel.  devices_or_null = NULL selects devices 0 .. ndev-1 (ndev <= 8).  Thread-safe; calls are
 * serialised (one MSM occupies all devices).  out = sum_i scalars[i] * ck[i] (+ r * h), Jacobian, 96 bytes. */
int b200_mgpu_init(int ndev, const int* devices_or_null);
int b200_mgpu_ck_register(int curve_id, const void* bases_affine_mont, size_t n, const void* h_affine_mont_or_null,
                          int window_bits, uint64_t* mgpu_key);
int b200_mgpu_ck_release(uint64_t mgpu_key);
int b200_mgpu_commit(uint64_t mgpu_key, const void* scalars_mont, size_t n, const void* r_mont_or_null,
                     void* out_jacobian_mont);

/* ---- R1CS witness field arithmetic (host-pointer forms) ---------------------------------- */
/* t[i] = az[i]*bz[i] - u*cz[i] - e1[i] (- e2[i] if e2 != NULL)   (r1cs/mod.rs:614-620,650-657) */
int b200_cross_term(int field_id, const void* az, const void* bz, const void* cz, const void* e1,
                    const void* e2_or_null, const void* u, size_t n, void* t);
/* out[i] = a[i] + r*b[i]   (RelaxedR1CSWitness::fold, r1cs/mod.rs:1044-1073) */
int b200_axpy(int field_id, const void* a, const void* b, const void* r, size_t n, void* out);
/* out[i] = a[i] + b[i]     (Z = Z1 + Z2, r1cs/mod.rs:589-609) */
int b200_vec_add(int field_id, const void* a, const void* b, size_t n, void* out);
/* z[i] += r*(z[i + n/2] - z[i]) for i < n/2; caller truncates to n/2
 * (MultilinearPolynomial::bind_poly_var_top, spartan/polys/multilinear.rs:65-84) */
int b200_bind_top(int field_id, void* z_inout, size_t n, const void* r);

/* device-pointer forms of the same (asynchronous on `stream`) */
int b200_cross_term_dev(int field_id, const void* az, const void* bz, const void* cz,
                        const void* e1, const void* e2_or_null, const void* u, size_t n, void* t,
                        void* stream);
int b200_axpy_dev(int field_id, const void* a, const void* b, const void* r, size_t n, void* out,
                  void* stream);
int b200_vec_add_dev(int field_id, const void* a, const void* b, size_t n, void* out, void* stream);
int b200_bind_top_dev(int field_id, void* z_inout, size_t n, const void* r, void* stream);
/* the same for k tables of one length in one launch: the 16 binds of a batched sum-check round (ppsnark.rs:960-966) */
int b200_bind_top_multi_dev(int field_id, void* const* d_tables, size_t k, size_t n, const void* d_r, void* stream);
/* out[i] = a[i]*b[i]   (TS[i] * (T[i]+r)^-1, spartan/ppsnark.rs:446-449) */
int b200_vec_mul_dev(int field_id, const void* a, const void* b, size_t n, void* out, void* stream);
/* LogUp fingerprints with the shift folded in: out[i] = val[i]*gamma + addr[i] + r; addr == NULL
 * means the cell's own index i   (MemorySumcheckInstance::compute_oracles, ppsnark.rs:386-435) */
int b200_logup_hash_dev(int field_id, const void* val, const void* addr_or_null, const void* gamma,
                        const void* r, size_t n, void* out, void* stream);

/* ---- sum-check rounds (spartan/sumcheck.rs) ------------------------------------------------
 * One call computes the O(N) sums of one round; the host keeps the O(1) algebra (claim
 * derivation with its inversion, sumcheck.rs:680-747), UniPoly and the transcript.
 * `len` = current polynomial length (even); lo = P[i], hi = P[i + len/2].  Forms:
 *   0 quad_prod  (sum A_lo B_lo, sum dA dB)                          sumcheck.rs:165-186
 *   1 linear     (sum A_lo-B_lo, sum A(-1)-B(-1))                    sumcheck.rs:352-377
 *   2 quadratic  (sum A_lo B_lo, sum A(-1)B(-1))                     sumcheck.rs:379-405
 *   3 cubic      (sum ABC_lo, sum dA dB dC, sum A(-1)B(-1)C(-1))     sumcheck.rs:407-443
 *   4 eq_cubic3  (t0, tinf) of eq*(A*B - C)                          sumcheck.rs:900-966
 *   5 eq_cubic2  (t0, tinf) of eq*(A*B - 1)                          sumcheck.rs:972-1033
 *   6 eq_quad1   t0 of eq*A                                          sumcheck.rs:1039-1080
 *   7,8,9        t(-1) fall-backs of 4,5,6 (tau = 0)                 sumcheck.rs:1082-1213
 *   10 dot_eq    sum Z[i] * eq[i]  (len = number of terms)
 *   11 dot       sum A[i] * B[i]   (inner_product, provider/ipa_pc.rs:102-108)
 * eq factor of index id: eq_left[id >> shift] * eq_right[id & (2^shift - 1)], or eq_right[id] when
 * eq_left is NULL (sumcheck.rs:1233-1251).  out receives 2, 2, 2, 3, 2, 2, 1, 1, 1, 1, 1, 1 elements. */
int b200_sc_eval(int field_id, int form, const void* A, const void* B, const void* C, size_t len,
                 const void* eq_left, size_t eq_left_len, const void* eq_right, size_t eq_right_len,
                 int shift, void* out);
int b200_sc_eval_dev(int field_id, int form, const void* A, const void* B, const void* C, size_t len,
                     const void* eq_left, const void* eq_right, int shift, void* out, void* stream);
/* Multi-GPU form (SURVEY.md §8e): the polynomials are sharded CYCLICALLY over id_mul ranks (rank
 * id_add holds global entries id_add, id_add + id_mul, ...).  (i, i + len/2) pairs stay
 * co-resident, so bind_top needs no exchange; the local index j weighs with the eq factor of the
 * global index j*id_mul + id_add.  Each rank gets partial sums; the host all-gathers 2-3 field
 * elements per round and adds them. */
int b200_sc_eval_sharded_dev(int field_id, int form, const void* A, const void* B, const void* C,
                             size_t local_len, const void* eq_left, const void* eq_right, int shift,
                             size_t id_mul, size_t id_add, void* out, void* stream);
/* CommitmentKey::new's validation loop (provider/hyperkzg.rs:113-119: every G1 base and h must be on
 * the curve, else NovaError::InvalidCommitmentKey), run on the device while the key is on its way
 * to HBM anyway.  *first_bad = SIZE_MAX when all n points satisfy y^2 = x^3 + b (the identity
 * encoding (0,0) passes, as halo2curves' is_on_curve does), else the smallest offending index.  A coordinate
 * >= p also counts as offending (it cannot be an in-memory field element; read_raw refuses it, ptau.rs:381). */
int b200_ck_validate(int curve_id, const void* bases, size_t n, size_t* first_bad);

/* ---- streamed witness hand-off (SURVEY.md §8f-2) ----------------------------------------------
 * WitnessCS::alloc only appends to aux_assignment (frontend/util_cs/witness_cs.rs:93-103); the
 * finished vector becomes R1CSWitness::new(shape, aux) and is committed (frontend/r1cs.rs:40-50,
 * r1cs/mod.rs:869-871).  A witness stream lets the host push every finished prefix while synthesis
 * is still running: the chunk's host->device copy and its share of the MSM's first stage (signed
 * window digits + bucket histogram) run on a side stream; `finish` runs the remaining stages and
 * returns commit(ck, W, r_W).  Chunks must stay valid and unmodified until `finish` returns (use
 * b200_host_alloc memory for copies that really overlap).  A short assignment is zero-extended to
 * n as R1CSWitness::new_with_blind does (r1cs/mod.rs:847-848); appending past n is B200_E_RANGE.
 * After `finish`, *d_witness (optional) is the device-resident W (n scalars, valid until
 * `release`) for the folds / SpMVs that follow. */
int b200_witness_begin(uint64_t ck_handle, size_t n, uint64_t* stream_handle);
int b200_witness_append(uint64_t stream_handle, const void* scalars, size_t count);
int b200_witness_finish(uint64_t stream_handle, const void* r_or_null, void* out_jacobian,
                        void** d_witness_or_null);
/* re-arm for the next witness of the same length (one per prove_step): keeps the workspace */
int b200_witness_reset(uint64_t stream_handle);
int b200_witness_release(uint64_t stream_handle);

/* ---- sum-check round loops with the transcript on the device (SURVEY.md §8f-3) ----------------
 * The reference interleaves, per round, an O(N) reduction, O(1) host algebra (UniPoly from the
 * evaluation points, univariate.rs:89-154; claim derivation / bound of EqSumCheckInstance,
 * sumcheck.rs:680-747, 1226-1231), `transcript.absorb(b"p", &poly)`, `transcript.squeeze(b"c")`
 * (Keccak256Transcript, provider/keccak.rs:98-160, non-evm) and the binds.  These entry points put
 * the O(1) part on the device too, so all rounds are enqueued back to back and the host reads the
 * proof once.  Prover messages are byte-identical to the host path.
 *
 * b200_transcript = the serialisable part of Keccak256Transcript (keccak.rs:19-27) after the last
 * squeeze; bytes absorbed since then travel separately as `pending` (= `transcript_buffer`,
 * at most B200_SC_MAX_PENDING bytes -- squeeze on the host first if there are more). */
typedef struct b200_transcript {
  uint64_t round;         /* Keccak256Transcript::round */
  unsigned char state[64]; /* Keccak256Transcript::state */
} b200_transcript;
#define B200_SC_MAX_PENDING 1984
/* device-resident running state of one sum-check (144 bytes, 16-byte aligned) */
typedef struct b200_sc_state {
  unsigned char claim[32];  /* running claim, Montgomery */
  unsigned char q[32];      /* EqSumCheckInstance::eval_eq_left, Montgomery (1 for plain kinds) */
  uint64_t round;           /* transcript round counter */
  unsigned char tstate[64]; /* transcript state */
  uint64_t rounds_done;
} b200_sc_state;
enum { B200_SC_ROUND_QUAD_PROD = 0, B200_SC_ROUND_CUBIC3_EQ = 1, B200_SC_ROUND_CUBIC3_EQ_M1 = 2 };
/* One round of O(1) prover work, asynchronous on `stream`: reads the reduction results d_res
 * (QUAD_PROD: [sum A_lo B_lo, sum dA dB]; CUBIC3_EQ: [t(0), t(inf)]; CUBIC3_EQ_M1 (tau == 0):
 * [t(0), t(inf), t(-1)]), builds the round polynomial, absorbs its compressed coefficients under
 * `absorb_label`, squeezes under `squeeze_label`, updates claim / q / transcript in *d_state, and
 * writes the compressed coefficients (2 or 3 x 32 B canonical little-endian = the proof bytes,
 * univariate.rs:177-190) to d_poly_out and the challenge (Montgomery) to d_r_out, where the bind
 * kernels of the same round read it. */
int b200_sc_round_dev(int field_id, int kind, void* d_state, const void* d_res, const void* d_tau,
                      const void* d_tau_inv, const void* d_pending, size_t pending_len,
                      int absorb_label, int squeeze_label, void* d_poly_out, void* d_r_out, void* stream);
/* One round of a BATCHED sum-check -- RelaxedR1CSSNARK::prove_helper of the MicroSpartan prover
 * (spartan/ppsnark.rs:886-983): every claim's evaluation points [s(0), lead, s(-1)] (the eq-weighted
 * ones derived from (t(0), t(inf)) and the claim's own running claim, sumcheck.rs:680-747), their
 * combination with the fixed coefficients into one cubic, absorb / squeeze, update_claim for every
 * running claim (sumcheck.rs:68-75) and the eq instances' bound values.  The host fills the descriptor
 * per round (slots of the sums the reductions of this round wrote; third-sum slots for tau = 0 rounds)
 * and enqueues reductions -> this call -> binds without reading anything back. */
#define B200_SCB_MAX_CLAIMS 16
#define B200_SCB_MAX_EQ 4
enum { B200_SCB_RAW3 = 0, B200_SCB_LIN2 = 1, B200_SCB_EQ_DEG2 = 2, B200_SCB_EQ_DEG1 = 3 };
typedef struct b200_scb_desc {
  int32_t nclaims, neq;
  int32_t kind[B200_SCB_MAX_CLAIMS];    /* B200_SCB_* */
  int32_t slot[B200_SCB_MAX_CLAIMS];    /* element index (32-byte units) of the claim's sums; 3 elements readable */
  int32_t slot_m1[B200_SCB_MAX_CLAIMS]; /* element index of t(-1) in a tau = 0 round, else -1 */
  int32_t eq_of[B200_SCB_MAX_CLAIMS];   /* eq instance of an EQ claim */
  const void* tau[B200_SCB_MAX_EQ];     /* device: this round's tau per eq instance (Montgomery) */
  const void* tau_inv[B200_SCB_MAX_EQ]; /* device: its inverse (ignored when tau = 0) */
} b200_scb_desc;
typedef struct b200_scb_state {           /* device resident, 1296 bytes */
  b200_sc_state head;                     /* head.claim = combined running claim; transcript; head.q unused */
  unsigned char coeff[B200_SCB_MAX_CLAIMS][32]; /* batching coefficients (powers of s, ppsnark.rs:915-921) */
  unsigned char claim[B200_SCB_MAX_CLAIMS][32]; /* running claims of the EQ claims */
  unsigned char q[B200_SCB_MAX_EQ][32];         /* eval_eq_left per eq instance */
} b200_scb_state;
int b200_sc_round_batched_dev(int field_id, const b200_scb_desc* desc, const void* d_sums, void* d_state,
                              const void* d_pending, size_t pending_len, int absorb_label, int squeeze_label,
                              void* d_poly_out, void* d_r_out, void* stream);
/* A whole batched sum-check in one call: RelaxedR1CSSNARK::prove_helper (src/spartan/ppsnark.rs:886-983) -- per round
 * every engine's evaluation points, their combination with the powers of one challenge, the cubic, the transcript
 * (absorb b"p", squeeze b"c"), the claim updates and the binds -- for claims expressed as sum forms over a set of
 * device tables of 2^num_rounds elements (bound in place).  Per round: all sums in two launches, the round kernel, one
 * bind launch; the last NOVA_B200_SC_TAIL_BITS (default 8) variables run inside one kernel.
 *   kind[i]    B200_SCB_*: how claim i's sums become its evaluation points [s(0), lead, s(-1)]
 *   form[i]    sum form 0..9 of b200_sc_eval (the pair forms) over tables tab[i][0..2] (-1 = unused)
 *   form_m1[i] eq claims: the third-sum form (7..9) for rounds whose tau is 0 (sumcheck.rs:1082-1213)
 *   eq_of[i]   eq claims: the EqSumCheckInstance (sumcheck.rs:590-747) weighting the sum; taus[g]: its num_rounds taus
 * Host inputs (Montgomery): coeffs [nclaims] (powers of the batching challenge, ppsnark.rs:915-921), claim (their
 * combination with the initial claims), running [nclaims] (initial claims; used by the eq claims).
 * Host outputs: polys_out [num_rounds][3][32] canonical LE, r_out [num_rounds][32] Montgomery, finals_out
 * [ntables][32] Montgomery (element 0 of every table after the last bind); *tr advances as the reference's. */
#define B200_SCP_MAX_TABLES 24
typedef struct b200_scp_program {
  int32_t nclaims, neq, ntables, num_rounds;
  int32_t kind[B200_SCB_MAX_CLAIMS];
  int32_t form[B200_SCB_MAX_CLAIMS];
  int32_t form_m1[B200_SCB_MAX_CLAIMS];
  int32_t eq_of[B200_SCB_MAX_CLAIMS];
  int32_t tab[B200_SCB_MAX_CLAIMS][3];
  void* tables[B200_SCP_MAX_TABLES];     /* device */
  const void* taus[B200_SCB_MAX_EQ];     /* host, Montgomery */
} b200_scp_program;
/* tuning: how many trailing variables of b200_sumcheck_batched run inside one kernel (0 = none; default 8 or
 * NOVA_B200_SC_TAIL_BITS).  bits < 0 only queries.  Returns the previous value. */
#define B200_SC_TAIL_MAX_BITS 14
int b200_sumcheck_tail_bits(int bits);
int b200_sumcheck_batched(int field_id, const b200_scp_program* prog, const void* coeffs, const void* claim,
                          const void* running, b200_transcript* tr, const void* pending, size_t pending_len,
                          void* polys_out, void* r_out, void* finals_out);
/* SumcheckProof::prove_quad_prod (sumcheck.rs:199-242) in one call.  d_A, d_B: device polynomials
 * of 2^num_rounds elements, bound in place (element 0 holds the final evaluation afterwards).
 * Host outputs: polys_out [num_rounds][2][32] canonical LE, r_out [num_rounds][32] Montgomery,
 * finals_out [2][32] Montgomery; *tr is advanced as the reference's transcript would be. */
int b200_sumcheck_quad_prod(int field_id, const void* claim, int num_rounds, void* d_A, void* d_B,
                            b200_transcript* tr, const void* pending, size_t pending_len,
                            void* polys_out, void* r_out, void* finals_out);
/* SumcheckProof::prove_cubic_with_three_inputs (sumcheck.rs:446-507): sum_x eq(tau,x)(A B - C).
 * taus: num_rounds host scalars (Montgomery); polys_out [num_rounds][3][32]; finals_out [3][32]. */
int b200_sumcheck_cubic3(int field_id, const void* claim, const void* taus, int num_rounds, void* d_A,
                         void* d_B, void* d_C, b200_transcript* tr, const void* pending,
                         size_t pending_len, void* polys_out, void* r_out, void* finals_out);
/* EqPolynomial::evals_from_points (spartan/polys/eq.rs:54-73): out has 2^ell entries */
int b200_eq_table(int field_id, const void* r, int ell, void* out);
int b200_eq_table_dev(int field_id, const void* r, int ell, void* out, void* stream);
/* MultilinearPolynomial::evaluate_with (spartan/polys/multilinear.rs:98-127): out = Z(r) */
int b200_mle_eval(int field_id, const void* Z, int ell, const void* r, void* out);
int b200_mle_eval_dev(int field_id, const void* Z, int ell, const void* r, void* out, void* stream);
/* MultilinearPolynomial::multi_evaluate_with (multilinear.rs:129-180): k polynomials of 2^ell entries at the
 * same point; the two sqrt-sized eq tables are built once, out receives k values (device pointers). */
int b200_mle_eval_multi_dev(int field_id, const void* const* d_Zs, size_t k, int ell, const void* d_r,
                            void* d_out, void* stream);
/* batch_invert (spartan/mod.rs:54-145); B200_E_ZERO if an element is zero */
int b200_batch_invert(int field_id, const void* in, size_t n, void* out);
int b200_batch_invert_dev(int field_id, const void* in, size_t n, void* out, int* d_zero_flag,
                          void* stream);
/* out[i] = sum_k coeffs[k]*polys[k][i], polys zero-extended to n, k <= 32
 * (PolyEvalWitness::batch, spartan/mod.rs:232-277; kzg_compute_batch_polynomial hyperkzg.rs:1028-1040) */
int b200_rlc(int field_id, const void* const* polys, const size_t* lens, size_t k, const void* coeffs,
             size_t n, void* out);
int b200_rlc_dev(int field_id, const void* const* d_polys, const size_t* lens, size_t k,
                 const void* d_coeffs, size_t n, void* d_out, void* stream);

/* ---- HyperKZG prover pieces (provider/hyperkzg.rs:926-1116) -------------------------------- */
/* out[j] = x*(p[2j+1] - p[2j]) + p[2j], j < n/2   (hyperkzg.rs:1085-1095) */
int b200_kzg_fold(int field_id, const void* p, size_t n, const void* x, void* out);
int b200_kzg_fold_dev(int field_id, const void* p, size_t n, const void* x, void* out, void* stream);
/* evals[q] = f(us[q]), q < nu <= 8 (Horner, hyperkzg.rs:1011-1019) */
int b200_poly_eval(int field_id, const void* f, size_t n, const void* us, size_t nu, void* evals);
int b200_poly_eval_dev(int field_id, const void* f, size_t n, const void* us, size_t nu, void* evals,
                       void* stream);
/* the same for k polynomials at the same nu <= 3 points (the 3-point evaluations of the whole HyperKZG fold chain,
 * hyperkzg.rs:1048-1056): evals[i * nu + q] = polys[i](us[q]).  Polynomials of up to 2^12 coefficients share ONE
 * launch; d_polys / lens are host arrays of device pointers / lengths. */
int b200_poly_eval_many_dev(int field_id, const void* const* d_polys, const size_t* lens, size_t k, const void* d_us,
                            size_t nu, void* d_evals, void* stream);
/* h = f / (X - u): n-1 coefficients, h[i-1] = f[i] + u*h[i] (hyperkzg.rs:961-999) */
int b200_poly_div(int field_id, const void* f, size_t n, const void* u, void* out);
int b200_poly_div_dev(int field_id, const void* f, size_t n, const void* u, void* out, void* stream);

/* ---- Mercury prover pieces (provider/mercury.rs) ---------------------------------------------
 * f is the coefficient vector of a univariate polynomial read as a row-major rows x cols matrix. */
/* out[r] = sum_c f[r*cols + c] * v[c], r < rows  (compute_h_poly, mercury.rs:369-386) */
int b200_mat_vec_rows(int field_id, const void* f, size_t rows, size_t cols, const void* v, void* out);
int b200_mat_vec_rows_dev(int field_id, const void* f, size_t rows, size_t cols, const void* v, void* out,
                          void* stream);
/* f = (X^cols - alpha) q + g  (divide_by_binomial, mercury.rs:319-356): every column c of f, as a polynomial in
 * Y = X^cols, is divided by (Y - alpha).  q receives (rows-1)*cols coefficients in row-major order, q[r*cols + c]
 * (the reference's quotient after its transpose; may be NULL when rows == 1), g[c] = column c at alpha.
 * B200_E_ARG if rows or cols is 0. */
int b200_div_binomial(int field_id, const void* f, size_t rows, size_t cols, const void* alpha, void* q, void* g);
int b200_div_binomial_dev(int field_id, const void* f, size_t rows, size_t cols, const void* alpha, void* q,
                          void* g, void* stream);
/* the s polynomial of the inner-product step (make_s_polynomial, mercury.rs:391-475), b - 1 coefficients:
 *   out[k] = sum_j (a1[j+k+1] b1[j] + a1[j] b1[j+k+1]) + gamma * sum_j (a2[j+k+1] b2[j] + a2[j] b2[j+k+1]),
 * k < b-1, j <= b-k-2; a1, b1, a2, b2 have b entries.  Computed directly (about 2b^2 products), not by NTT. */
int b200_mercury_s_poly(int field_id, const void* a1, const void* b1, const void* a2, const void* b2, size_t b,
                        const void* gamma, void* out);
int b200_mercury_s_poly_dev(int field_id, const void* a1, const void* b1, const void* a2, const void* b2, size_t b,
                            const void* gamma, void* out, void* stream);

/* ---- NeutronNova folding prover pieces (neutron/nifs.rs, neutron/relation.rs) ------------------
 * A structure of n = left * right rows; row k = i * left + j.  e1, e2 hold left + right entries (the split
 * power polynomial: e = the first `left`, f = the last `right`); az*, bz*, cz* hold n entries. */
/* the five sums of NIFS::prove_helper (nifs.rs:29-186) BEFORE its rho factors: with V_t = V1 + t (V2 - V1),
 *   out[m] = sum_i f_t[i] * sum_j e_t[j] * (Az_t[k] Bz_t[k] - Cz_t[k]),   t = 0, 2, 3, 4, 5 for m = 0..4,
 * as Montgomery elements.  One pass over the six n-vectors; with the second instance equal to the first every
 * sum is the is_sat sum (relation.rs:71-116).  B200_E_ARG if left or right is 0. */
int b200_neutron_evals(int field_id, const void* e1, const void* az1, const void* bz1, const void* cz1,
                       const void* e2, const void* az2, const void* bz2, const void* cz2, size_t left, size_t right,
                       void* out);
int b200_neutron_evals_dev(int field_id, const void* e1, const void* az1, const void* bz1, const void* cz1,
                           const void* e2, const void* az2, const void* bz2, const void* cz2, size_t left,
                           size_t right, void* out, void* stream);
/* PowPolynomial::split_evals (spartan/polys/power.rs:62-86), left + right entries: out[j] = tau^j (j < left),
 * out[left + i] = tau^(left * i) (i < right).  tau: one element (a device pointer on the _dev form).
 * B200_E_ARG if left is 0 or right < 2 (the reference indexes right[1]). */
int b200_pow_split_evals(int field_id, const void* tau, size_t left, size_t right, void* out);
int b200_pow_split_evals_dev(int field_id, const void* tau, size_t left, size_t right, void* out, void* stream);
/* out[i] = a[i] + r * (b[i] - a[i]), i < n: the witness folds W1 + r_b (W2 - W1), E1 + r_b (E - E1)
 * (FoldedWitness::fold, relation.rs:131-156).  out may alias a. */
int b200_lerp(int field_id, const void* a, const void* b, const void* r, size_t n, void* out);
int b200_lerp_dev(int field_id, const void* a, const void* b, const void* r, size_t n, void* out, void* stream);

/* ---- inner-product argument (provider/ipa_pc.rs:174-285), "next" row (f)1 of SURVEY.md §8 ------
 * The reference folds the commitment key every round (ck.fold, pedersen.rs:484-497: n/2 two-point
 * MSMs) and commits over the folded key.  Equivalent and GPU-friendlier: keep the ORIGINAL key
 * (registered once, window tables) and put the fold weights into the scalars:
 *     L_k = MSM(key, sL) + (c_L r0) * ck_c,   sL[j] = [j & nk/2] a[j mod nk/2] w[j]
 *     R_k = MSM(key, sR) + (c_R r0) * ck_c,   sR[j] = [!(j & nk/2)] a[(j mod nk/2) + nk/2] w[j]
 * with w the running product of r / r^-1 per original index.  Group elements are canonical, so
 * L_vec, R_vec and a_hat are bit-identical to the reference's. */
/* out[i] = v[i]*x_lo + v[i + n/2]*x_hi, i < n/2  (a and b folds, ipa_pc.rs:244-254) */
int b200_fold_halves_dev(int field_id, const void* v, size_t n, const void* x_lo, const void* x_hi,
                         void* out, void* stream);
int b200_ipa_scalars_dev(int field_id, const void* a, const void* w, size_t n, size_t nk, void* sL,
                         void* sR, void* stream);
/* nk == 0: w := 1 ; else w[j] *= (j & nk/2) ? r : r_inv */
int b200_ipa_weights_dev(int field_id, void* w, size_t n, size_t nk, const void* r, const void* r_inv,
                         void* stream);
/* The verifier's tensor vector s of InnerProductArgument::verify (ipa_pc.rs:334-349), times a scale:
 *     out[i] = scale * prod_{j < L} (bit j of i, most significant first ? r[j] : r_inv[j]),   i < 2^L
 * (the reference's s[0] = prod r^-1, s[i] = s[i - 2^pos] * r^2[L-1-pos] is the same product).  r, r_inv: L
 * Montgomery elements each; d_scale_or_null: one element, or NULL for 1.  It is also the prover's weights w after
 * all L rounds of b200_ipa_weights_dev.  With scale = a_hat and the key registered with h = ck_c, the verifier's
 * a_hat * ck_hat + a_hat * b_hat * (r0 * ck_c) is one b200_commit_dev(key, out, 2^L, blind = a_hat * b_hat * r0).
 * B200_E_ARG for L outside 0 .. 31 or a null pointer; nothing is written then. */
int b200_ipa_s_dev(int field_id, const void* d_r, const void* d_r_inv, int L, const void* d_scale_or_null, void* d_out,
                   void* stream);

/* ---- sparse matrices (r1cs/sparse.rs:19-319) ------------------------------------------------
 * CSR as in SparseMatrix{data, indices, indptr, cols} (sparse.rs:235-247); registration uploads
 * the matrix once and classifies its coefficients (+-1, small +-2..7, general: sparse.rs:40-105). */
int b200_spmv_register(int field_id, const void* data_mont, const uint64_t* indices,
                       const uint64_t* indptr, size_t rows, size_t cols, uint64_t* m_handle);
int b200_spmv_release(uint64_t m_handle);
int b200_spmv_dev(uint64_t m_handle, const void* d_z1, const void* d_z2_or_null, void* d_out1,
                  void* d_out2_or_null, void* stream);
/* out[col] = sum over entries (row, col, val) of rx[row]*val, for col < out_len (zero beyond the
 * matrix' columns): compute_eval_table_sparse (spartan/mod.rs:497-534), one matrix per call */
int b200_spmv_t(uint64_t m_handle, const void* rx, size_t out_len, void* out);
int b200_spmv_t_dev(uint64_t m_handle, const void* d_rx, size_t out_len, void* d_out, void* stream);
/* out[i] = table[idx[i]]: the L_row / L_col oracles of ppsnark (spartan/ppsnark.rs:236-250) */
int b200_gather(const void* table, size_t table_len, const uint64_t* idx, size_t n, void* out);
int b200_gather_dev(const void* d_table, const uint32_t* d_idx, size_t n, void* d_out, void* stream);
/* R1CSShapeSparkRepr::new (spartan/ppsnark.rs:117-190) from the matrices behind three spmv handles (same field,
 * rows, cols).  N: the caller's next_pow2(max(nnz_A + nnz_B + nnz_C, 2 num_vars, num_cons)); checked to be a
 * power of two >= total nnz, >= rows, >= cols and < 2^32.  Writes N entries each: d_vecs[0..7) = row, col, val_A,
 * val_B, val_C, ts_row, ts_col as Montgomery field elements; d_row_idx / d_col_idx = row / col as u32 (the gather
 * indices).  Padding slots have row 0 and col N - 1.  d_vecs is a host array of device pointers.
 * Unknown handle: B200_E_HANDLE; mismatched matrices or N not a power of two below 2^32: B200_E_ARG; N too
 * small: B200_E_RANGE.  Nothing is written on an error. */
int b200_spark_repr_dev(uint64_t hA, uint64_t hB, uint64_t hC, size_t N, void* const* d_vecs, uint32_t* d_row_idx,
                        uint32_t* d_col_idx, void* stream);
/* The verifier's matrix evaluations, multi_evaluate of RelaxedR1CSSNARK::verify (spartan/snark.rs:325-355):
 *     out[y] = sum over the entries (row, col, val) of matrix y of T_x[row] * T_y[col] * val,   y < k
 * for the k <= 3 matrices behind m_handles (a host array), in one launch (partitioned by entry ranges, so long and
 * empty rows cost no imbalance).  d_Tx / d_Ty: tx_len / ty_len Montgomery elements; d_out: k elements.
 *   B200_E_HANDLE  an unknown handle
 *   B200_E_ARG     k = 0, k > 3, matrices of different fields, a null pointer
 *   B200_E_RANGE   rows > tx_len or cols > ty_len of some matrix (the reference would index out of bounds)
 * Checked before any launch; nothing is written on an error.  A matrix without entries gives 0. */
int b200_r1cs_eval_dev(const uint64_t* m_handles, size_t k, const void* d_Tx, size_t tx_len, const void* d_Ty,
                       size_t ty_len, void* d_out, void* stream);
/* The same from the points, as the reference's closure takes them: T_x = eq(r_x) (2^ell_x entries) and
 * T_y = eq(r_y) (2^ell_y) are built on the device; r_x, r_y, out are host Montgomery elements.  ell_x, ell_y <= 34. */
int b200_r1cs_eval(const uint64_t* m_handles, size_t k, const void* r_x, int ell_x, const void* r_y, int ell_y,
                   void* out);
/* R1CSShape::multiply_vec / multiply_vec_pair (r1cs/mod.rs:407-471): k matrices, one or two z */
int b200_spmv_multi(const uint64_t* m_handles, size_t k, const void* z1, const void* z2_or_null,
                    size_t z_len, void* const* out1, void* const* out2_or_null);

#ifdef __cplusplus
}
#endif
#endif /* NOVA_B200_H */
