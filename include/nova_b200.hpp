// nova_b200.hpp -- C++ host-side mirror of the reference's provider surface for the hot path,
// layered on the C ABI (include/nova_b200.h).  The reference is Rust; no Rust toolchain exists in
// this image, so this header is the compiled-language host layer: same names, argument meaning
// and error behaviour as the traits it stands under, so that the Rust shim of INTEGRATION.md is a
// transliteration of it.
//
//   nova::b200::DlogGroup<Curve>::vartime_multiscalar_mul / batch_...   provider/traits.rs:77-117
//   nova::b200::CommitmentEngine<Curve>::commit / batch_commit          pedersen.rs:263-270,
//                                                                       hyperkzg.rs:584-612
//   nova::b200::R1CSShape::multiply_vec / multiply_vec_pair / cross_term r1cs/mod.rs:407-471,578-664
//   nova::b200::fold_witness, bind_poly_var_top                         r1cs/mod.rs:1044-1107,
//                                                                       polys/multilinear.rs:65-84
//   nova::b200::sumcheck_eval                                           spartan/sumcheck.rs (round sums)
//   nova::b200::R1CSShape(Dev)::multi_evaluate, ipa_s                   spartan/snark.rs:325-355,
//                                                                       ipa_pc.rs:334-349 (verifiers)
//
// Conventions: `Scalar` / `Affine` / `Point` are the FFI layouts (32 / 64 / 96 bytes).  Infallible
// trait functions (MSM, commit) throw std::logic_error on length mismatch (the reference
// `assert!`s, msm.rs:226) and std::runtime_error("GpuError: ...") on device failure
// (NovaError::GpuError, errors.rs:84-86).  All calls are thread-safe (rayon workers call commits
// concurrently in the reference: r1cs/mod.rs:509-512).
#pragma once
#include <array>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <utility>
#include <string>
#include <vector>

#include "nova_b200.h"

namespace nova {
namespace b200 {

struct Scalar { std::array<uint64_t, 4> limbs; };           // Montgomery, R = 2^256
struct Affine { Scalar x, y; };                             // identity: all zero
struct Point { Scalar x, y, z; bool is_identity() const {   // Jacobian; identity: z = 0
  return (z.limbs[0] | z.limbs[1] | z.limbs[2] | z.limbs[3]) == 0; } };
static_assert(sizeof(Scalar) == 32 && sizeof(Affine) == 64 && sizeof(Point) == 96, "FFI layout");

struct BN254 { static constexpr int curve = B200_CURVE_BN254_G1, scalar_field = B200_FIELD_BN254_FR; };
struct Grumpkin { static constexpr int curve = B200_CURVE_GRUMPKIN, scalar_field = B200_FIELD_BN254_FQ; };
struct Pallas { static constexpr int curve = B200_CURVE_PALLAS, scalar_field = B200_FIELD_PALLAS_FQ; };
struct Vesta { static constexpr int curve = B200_CURVE_VESTA, scalar_field = B200_FIELD_PALLAS_FP; };

inline void check(int rc, const char* what) {
  if (rc == B200_OK) return;
  std::string msg = std::string(what) + ": " + b200_last_error();
  if (rc == B200_E_ARG || rc == B200_E_RANGE) throw std::logic_error(msg);
  throw std::runtime_error("GpuError: " + msg);
}

// CommitmentKey{ck, h} resident on the device (pedersen.rs:32-38, hyperkzg.rs:76-84)
template <class C>
class CommitmentKey {
 public:
  CommitmentKey(const std::vector<Affine>& ck, const Affine* h = nullptr, int window_bits = 0) : n_(ck.size()) {
    check(b200_ck_register(C::curve, ck.data(), ck.size(), h, window_bits, &handle_), "b200_ck_register");
  }
  // Points from outside the process (load_setup -> read_ptau, hyperkzg.rs:658-675, ptau.rs:372-438): validated in
  // HBM before the tables are built.  Throws InvalidCommitmentKey with the index of the first bad point.
  struct InvalidCommitmentKey : std::runtime_error {
    size_t index;
    explicit InvalidCommitmentKey(size_t i)
        : std::runtime_error("InvalidCommitmentKey: point " + std::to_string(i) + " is non-canonical or off the curve"),
          index(i) {}
  };
  struct Untrusted {};
  CommitmentKey(Untrusted, const std::vector<Affine>& ck, const Affine* h = nullptr, int window_bits = 0)
      : n_(ck.size()) {
    size_t bad = 0;
    int rc = b200_ck_register_checked(C::curve, ck.data(), ck.size(), h, window_bits, &handle_, &bad);
    if (rc == B200_E_POINT) throw InvalidCommitmentKey(bad);
    check(rc, "b200_ck_register_checked");
  }
  // ck_derive_by_address (traits/commitment.rs:177-194): an address outside the table (NovaError::InvalidIndex, with
  // the smallest offending position) and more addresses than bases (NovaError::InvalidCommitmentKeyLength)
  struct InvalidIndex : std::runtime_error {
    size_t position;
    explicit InvalidIndex(size_t i)
        : std::runtime_error("InvalidIndex: address at position " + std::to_string(i) + " is outside the table"),
          position(i) {}
  };
  struct InvalidCommitmentKeyLength : std::runtime_error {
    InvalidCommitmentKeyLength() : std::runtime_error("InvalidCommitmentKeyLength: more addresses than bases") {}
  };
  // takes ownership of a key the library has already registered (b200_ck_derive_by_address) of n bases
  struct Adopt {};
  CommitmentKey(Adopt, uint64_t handle, size_t n) : handle_(handle), n_(n) {}
  CommitmentKey(CommitmentKey&& o) noexcept : handle_(o.handle_), n_(o.n_) { o.handle_ = 0; }
  CommitmentKey(const CommitmentKey&) = delete;
  CommitmentKey& operator=(const CommitmentKey&) = delete;
  ~CommitmentKey() { if (handle_) b200_ck_release(handle_); }
  size_t len() const { return n_; }
  uint64_t handle() const { return handle_; }
 private:
  uint64_t handle_ = 0;
  size_t n_;
};

template <class C>
struct DlogGroup {
  // msm(scalars, &ck[..scalars.len()])  (provider/traits.rs:79, msm.rs:225)
  static Point vartime_multiscalar_mul(const std::vector<Scalar>& scalars, const CommitmentKey<C>& ck) {
    if (scalars.size() > ck.len()) throw std::logic_error("scalars and bases length mismatch");
    Point out{};
    check(b200_msm(ck.handle(), 0, scalars.data(), scalars.size(), &out), "b200_msm");
    return out;
  }
  // one-shot bases (pedersen.rs:418-420)
  static Point vartime_multiscalar_mul(const std::vector<Scalar>& scalars, const std::vector<Affine>& bases) {
    if (scalars.size() != bases.size()) throw std::logic_error("scalars and bases length mismatch");
    Point out{};
    check(b200_msm_adhoc(C::curve, bases.data(), scalars.data(), scalars.size(), &out), "b200_msm_adhoc");
    return out;
  }
  // traits.rs:82-90
  static std::vector<Point> batch_vartime_multiscalar_mul(const std::vector<std::vector<Scalar>>& scalars,
                                                          const CommitmentKey<C>& ck) {
    std::vector<const void*> ptrs(scalars.size());
    std::vector<size_t> lens(scalars.size());
    for (size_t j = 0; j < scalars.size(); j++) { ptrs[j] = scalars[j].data(); lens[j] = scalars[j].size(); }
    std::vector<Point> out(scalars.size());
    check(b200_msm_batch(ck.handle(), ptrs.data(), lens.data(), scalars.size(), out.data()), "b200_msm_batch");
    return out;
  }
  template <class T>  // msm_small (msm.rs:469-503)
  static Point vartime_multiscalar_mul_small(const std::vector<T>& scalars, const CommitmentKey<C>& ck,
                                             int max_num_bits = 0) {
    static_assert(sizeof(T) == 1 || sizeof(T) == 2 || sizeof(T) == 4 || sizeof(T) == 8, "integer scalars");
    if (scalars.size() > ck.len()) throw std::logic_error("scalars and bases length mismatch");
    Point out{};
    check(b200_msm_small(ck.handle(), 0, scalars.data(), (int)sizeof(T), scalars.size(), max_num_bits, &out),
          "b200_msm_small");
    return out;
  }
  static Point batch_add(const CommitmentKey<C>& ck, const std::vector<uint64_t>& one_indices) {  // msm.rs:689
    Point out{};
    check(b200_msm_indices(ck.handle(), one_indices.data(), one_indices.size(), &out), "b200_msm_indices");
    return out;
  }
};

template <class C>
struct CommitmentEngine {
  // commit(ck, v, r) = MSM(v, ck[..len]) + h*r   (pedersen.rs:263-270)
  static Point commit(const CommitmentKey<C>& ck, const std::vector<Scalar>& v, const Scalar* r = nullptr) {
    if (ck.len() < v.size()) throw std::logic_error("commitment key too short");  // pedersen.rs:264
    Point out{};
    check(b200_commit(ck.handle(), v.data(), v.size(), r, &out), "b200_commit");
    return out;
  }
  static std::vector<Point> batch_commit(const CommitmentKey<C>& ck, const std::vector<std::vector<Scalar>>& vs) {
    return DlogGroup<C>::batch_vartime_multiscalar_mul(vs, ck);
  }
  // ck_derive_by_address (traits/commitment.rs:177-194, pedersen.rs:360-382, hyperkzg.rs:731-749), on the device:
  // derived[j] = sum of ck[i] over the i with addresses[i] = j, j < table_size, so that
  // commit(derived, T) == commit(ck, T[addresses]).  The new key carries ck's h and outlives ck.  An identity
  // generator in ck (the reference's panic) throws std::logic_error; table_size = 0 throws std::logic_error too (the
  // reference returns an empty key for no addresses; a key of no bases cannot be registered).
  static CommitmentKey<C> ck_derive_by_address(const CommitmentKey<C>& ck, const std::vector<size_t>& addresses,
                                               size_t table_size, int window_bits = 0) {
    using Key = CommitmentKey<C>;
    std::vector<uint64_t> a(addresses.begin(), addresses.end());
    uint64_t h = 0;
    size_t bad = SIZE_MAX;
    int rc = b200_ck_derive_by_address(ck.handle(), a.data(), a.size(), table_size, window_bits, &h, &bad);
    if (rc == B200_E_INDEX) throw typename Key::InvalidIndex(bad);
    if (rc == B200_E_RANGE && a.size() > ck.len()) throw typename Key::InvalidCommitmentKeyLength();
    if (rc == B200_E_POINT)
      throw std::logic_error("ck_derive_by_address: generator " + std::to_string(bad) + " is the identity");
    check(rc, "b200_ck_derive_by_address");
    return Key(typename Key::Adopt{}, h, table_size);
  }
};

// CSR matrix + R1CS shape (r1cs/sparse.rs:235-247, r1cs/mod.rs:407-471)
class SparseMatrix {
 public:
  SparseMatrix(int field, const std::vector<Scalar>& data, const std::vector<uint64_t>& indices,
               const std::vector<uint64_t>& indptr, size_t cols)
      : rows_(indptr.size() - 1), cols_(cols) {
    check(b200_spmv_register(field, data.data(), indices.data(), indptr.data(), rows_, cols, &handle_),
          "b200_spmv_register");
  }
  SparseMatrix(const SparseMatrix&) = delete;
  ~SparseMatrix() { if (handle_) b200_spmv_release(handle_); }
  uint64_t handle() const { return handle_; }
  size_t rows() const { return rows_; }
  size_t cols() const { return cols_; }
 private:
  uint64_t handle_ = 0;
  size_t rows_, cols_;
};

struct R1CSShape {
  const SparseMatrix &A, &B, &C;
  int field;
  // (Az, Bz, Cz); throws std::invalid_argument("InvalidWitnessLength") like r1cs/mod.rs:411-413
  std::array<std::vector<Scalar>, 3> multiply_vec(const std::vector<Scalar>& z) const {
    if (z.size() != A.cols()) throw std::invalid_argument("InvalidWitnessLength");
    std::array<std::vector<Scalar>, 3> out{std::vector<Scalar>(A.rows()), std::vector<Scalar>(B.rows()),
                                           std::vector<Scalar>(C.rows())};
    uint64_t hs[3] = {A.handle(), B.handle(), C.handle()};
    void* o[3] = {out[0].data(), out[1].data(), out[2].data()};
    check(b200_spmv_multi(hs, 3, z.data(), nullptr, z.size(), o, nullptr), "b200_spmv_multi");
    return out;
  }
  // [A(r_x, r_y), B(r_x, r_y), C(r_x, r_y)] = sum over each matrix's entries of eq(r_x)[row] eq(r_y)[col] val: the
  // verifier's multi_evaluate (spartan/snark.rs:325-355); both eq tables are built on the device (b200_r1cs_eval)
  std::array<Scalar, 3> multi_evaluate(const std::vector<Scalar>& r_x, const std::vector<Scalar>& r_y) const {
    std::array<Scalar, 3> out{};
    uint64_t hs[3] = {A.handle(), B.handle(), C.handle()};
    check(b200_r1cs_eval(hs, 3, r_x.data(), (int)r_x.size(), r_y.data(), (int)r_y.size(), out.data()),
          "b200_r1cs_eval");
    return out;
  }
  // T = AZ o BZ - u*CZ - E1 (- E2)   (commit_T / commit_T_relaxed, r1cs/mod.rs:614-620, 650-657)
  std::vector<Scalar> cross_term(const std::vector<Scalar>& az, const std::vector<Scalar>& bz,
                                 const std::vector<Scalar>& cz, const std::vector<Scalar>& e1, const Scalar& u,
                                 const std::vector<Scalar>* e2 = nullptr) const {
    std::vector<Scalar> t(az.size());
    check(b200_cross_term(field, az.data(), bz.data(), cz.data(), e1.data(), e2 ? e2->data() : nullptr, &u,
                          az.size(), t.data()), "b200_cross_term");
    return t;
  }
};

// W1 + r*W2 (RelaxedR1CSWitness::fold, r1cs/mod.rs:1058-1069)
inline std::vector<Scalar> fold_witness(int field, const std::vector<Scalar>& a, const std::vector<Scalar>& b,
                                        const Scalar& r) {
  if (a.size() != b.size()) throw std::invalid_argument("InvalidWitnessLength");  // r1cs/mod.rs:1054
  std::vector<Scalar> out(a.size());
  check(b200_axpy(field, a.data(), b.data(), &r, a.size(), out.data()), "b200_axpy");
  return out;
}
// MultilinearPolynomial::bind_poly_var_top (polys/multilinear.rs:65-84): in place, truncates
inline void bind_poly_var_top(int field, std::vector<Scalar>& Z, const Scalar& r) {
  check(b200_bind_top(field, Z.data(), Z.size(), &r), "b200_bind_top");
  Z.resize(Z.size() / 2);
}
// one round's O(N) sums (see include/nova_b200.h for the form table); returns 1-3 field elements
inline std::vector<Scalar> sumcheck_eval(int field, int form, const std::vector<Scalar>& A,
                                         const std::vector<Scalar>* B, const std::vector<Scalar>* C,
                                         const std::vector<Scalar>* eq_left, const std::vector<Scalar>* eq_right,
                                         int shift) {
  Scalar out[3];
  check(b200_sc_eval(field, form, A.data(), B ? B->data() : nullptr, C ? C->data() : nullptr, A.size(),
                     eq_left ? eq_left->data() : nullptr, eq_left ? eq_left->size() : 0,
                     eq_right ? eq_right->data() : nullptr, eq_right ? eq_right->size() : 0, shift, out),
        "b200_sc_eval");
  int n = form == 3 ? 3 : (form == 6 || form >= 7) ? 1 : 2;
  return std::vector<Scalar>(out, out + n);
}


// ---- device-resident vectors and the folding step without host round trips (SURVEY.md §7 step 7) ----
// W, E and T stay in HBM between calls; only commitments (96 B) and challenges (32 B) cross the bus.
// The O(1) instance algebra of RelaxedR1CSInstance::fold (u, X, and comm_W1 + r*comm_W2: two or three
// commitment-sized scalar multiplications, r1cs/mod.rs:1237-1292) stays in the host's own curve library.
class DeviceVec {
 public:
  DeviceVec() = default;
  explicit DeviceVec(size_t n) : n_(n) { check(b200_dev_alloc(32 * (n ? n : 1), &p_), "b200_dev_alloc"); }
  explicit DeviceVec(const std::vector<Scalar>& v) : DeviceVec(v.size()) {
    if (!v.empty()) check(b200_memcpy_h2d(p_, v.data(), 32 * v.size()), "b200_memcpy_h2d");
  }
  DeviceVec(DeviceVec&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
  DeviceVec& operator=(DeviceVec&& o) noexcept {
    if (this != &o) { release(); p_ = o.p_; n_ = o.n_; o.p_ = nullptr; o.n_ = 0; }
    return *this;
  }
  DeviceVec(const DeviceVec&) = delete;
  DeviceVec& operator=(const DeviceVec&) = delete;
  ~DeviceVec() { release(); }
  void* ptr() const { return p_; }
  size_t len() const { return n_; }
  std::vector<Scalar> to_host() const {
    std::vector<Scalar> v(n_);
    if (n_) check(b200_memcpy_d2h(v.data(), p_, 32 * n_), "b200_memcpy_d2h");
    return v;
  }
  static DeviceVec zeros(size_t n) {
    DeviceVec v(n);
    if (n) { check(b200_memset_dev(v.p_, 0, 32 * n, nullptr), "b200_memset_dev"); check(b200_sync(), "b200_sync"); }
    return v;
  }
 private:
  void release() { if (p_) b200_dev_free(p_); p_ = nullptr; }
  void* p_ = nullptr;
  size_t n_ = 0;
};

// CE::commit(ck, v, r) of a resident vector (pedersen.rs:263-270)
template <class C>
inline Point commit_resident(const CommitmentKey<C>& ck, const DeviceVec& v, const Scalar* r = nullptr) {
  if (ck.len() < v.len()) throw std::logic_error("commitment key too short");  // pedersen.rs:264
  DeviceVec out(3), blind;
  if (r) blind = DeviceVec(std::vector<Scalar>{*r});
  check(b200_commit_dev(ck.handle(), v.ptr(), v.len(), r ? blind.ptr() : nullptr, out.ptr(), nullptr), "b200_commit_dev");
  Point P{};
  check(b200_memcpy_d2h(&P, out.ptr(), 96), "b200_memcpy_d2h");  // synchronises: `blind` may now go
  return P;
}

// The IPA verifier's tensor vector (ipa_pc.rs:334-349) on the device: s[i] = scale * prod_j (bit j of i, most
// significant first ? r[j] : r_inv[j]), 2^L entries for the L = r.len() round challenges (b200_ipa_s_dev).  With
// scale = a_hat, commit_resident(ck, s, &blind) is the verifier's a_hat <s, ck> + blind * ck_c in one MSM.
inline DeviceVec ipa_s(int field, const DeviceVec& r, const DeviceVec& r_inv, const Scalar* scale = nullptr) {
  if (r_inv.len() != r.len()) throw std::invalid_argument("InvalidInputLength");
  DeviceVec out((size_t)1 << r.len()), sc;
  if (scale) sc = DeviceVec(std::vector<Scalar>{*scale});
  check(b200_ipa_s_dev(field, r.ptr(), r_inv.ptr(), (int)r.len(), scale ? sc.ptr() : nullptr, out.ptr(), nullptr),
        "b200_ipa_s_dev");
  check(b200_sync(), "b200_sync");  // `sc` may now go
  return out;
}

// CommitmentKey::new's on-curve loop (hyperkzg.rs:113-119): index of the first off-curve base, or SIZE_MAX
template <class C>
inline size_t validate_key(const std::vector<Affine>& ck) {
  size_t bad = 0;
  check(b200_ck_validate(C::curve, ck.data(), ck.size(), &bad), "b200_ck_validate");
  return bad;
}

// Streamed witness hand-off (frontend/util_cs/witness_cs.rs:93-103 appends; frontend/r1cs.rs:40-50 commits)
template <class C>
class WitnessStream {
 public:
  WitnessStream(const CommitmentKey<C>& ck, size_t num_vars) : n_(num_vars) {
    check(b200_witness_begin(ck.handle(), num_vars, &h_), "b200_witness_begin");
  }
  WitnessStream(const WitnessStream&) = delete;
  ~WitnessStream() { if (h_) b200_witness_release(h_); }
  // `chunk` must stay valid and unmodified until finish() returns (aux_assignment is append-only)
  void append(const Scalar* chunk, size_t count) { check(b200_witness_append(h_, chunk, count), "b200_witness_append"); }
  // -> commit(ck, W, r_W); *d_W (optional) = the resident witness, valid until reset() / destruction
  Point finish(const Scalar* r_W = nullptr, void** d_W = nullptr) {
    Point P{};
    check(b200_witness_finish(h_, r_W, &P, d_W), "b200_witness_finish");
    return P;
  }
  void reset() { check(b200_witness_reset(h_), "b200_witness_reset"); }  // next prove_step, same num_vars
  size_t len() const { return n_; }
 private:
  uint64_t h_ = 0;
  size_t n_;
};

struct RelaxedR1CSWitnessDev {  // r1cs/mod.rs:69-76 with W, E resident
  DeviceVec W, E;
  Scalar r_W{}, r_E{};
};

// R1CSShape with the matrices behind spmv handles and every vector resident (r1cs/mod.rs:407-431, 578-664)
struct R1CSShapeDev {
  const SparseMatrix &A, &B, &C;
  int field;
  size_t num_cons, num_vars, num_io;

  // z = (W, u, X)
  DeviceVec z(const DeviceVec& W, const Scalar& u, const std::vector<Scalar>& X) const {
    if (W.len() != num_vars) throw std::invalid_argument("InvalidWitnessLength");  // r1cs/mod.rs:411-413
    if (X.size() != num_io) throw std::invalid_argument("InvalidInputLength");
    DeviceVec out(num_vars + 1 + num_io);
    check(b200_memcpy_d2d(out.ptr(), W.ptr(), 32 * num_vars, nullptr), "b200_memcpy_d2d");
    std::vector<Scalar> tail{u};
    tail.insert(tail.end(), X.begin(), X.end());
    check(b200_sync(), "b200_sync");
    check(b200_memcpy_h2d((char*)out.ptr() + 32 * num_vars, tail.data(), 32 * tail.size()), "b200_memcpy_h2d");
    return out;
  }
  // multi_evaluate (spartan/snark.rs:325-355) on resident eq tables T_x (>= num_cons entries) and T_y (>= the
  // matrices' columns): one b200_r1cs_eval_dev over A, B and C
  std::array<Scalar, 3> multi_evaluate(const DeviceVec& T_x, const DeviceVec& T_y) const {
    DeviceVec out(3);
    uint64_t hs[3] = {A.handle(), B.handle(), C.handle()};
    check(b200_r1cs_eval_dev(hs, 3, T_x.ptr(), T_x.len(), T_y.ptr(), T_y.len(), out.ptr(), nullptr),
          "b200_r1cs_eval_dev");
    std::array<Scalar, 3> r{};
    check(b200_memcpy_d2h(r.data(), out.ptr(), 96), "b200_memcpy_d2h");
    return r;
  }
  std::array<DeviceVec, 3> multiply_vec(const DeviceVec& zv) const {
    std::array<DeviceVec, 3> out{DeviceVec(num_cons), DeviceVec(num_cons), DeviceVec(num_cons)};
    const SparseMatrix* M[3] = {&A, &B, &C};
    for (int k = 0; k < 3; k++)
      check(b200_spmv_dev(M[k]->handle(), zv.ptr(), nullptr, out[k].ptr(), nullptr, nullptr), "b200_spmv_dev");
    return out;
  }
  // commit_T (E2 == nullptr, u2 = 1) / commit_T_relaxed: Z = Z1 + Z2, T = AZ o BZ - (u1+u2) CZ - E1 (- E2).
  // `u_sum` = u1 + u2 is supplied by the caller (host field arithmetic).  -> (T resident, comm_T)
  template <class Cv>
  std::pair<DeviceVec, Point> commit_T(const CommitmentKey<Cv>& ck, const DeviceVec& Z1, const DeviceVec& Z2,
                                       const Scalar& u_sum, const DeviceVec& E1, const DeviceVec* E2,
                                       const Scalar* r_T) const {
    const size_t zl = num_vars + 1 + num_io;
    if (Z1.len() != zl || Z2.len() != zl || E1.len() != num_cons || (E2 && E2->len() != num_cons))
      throw std::invalid_argument("InvalidWitnessLength");
    DeviceVec Z(zl), T(num_cons), ud(std::vector<Scalar>{u_sum});
    check(b200_vec_add_dev(field, Z1.ptr(), Z2.ptr(), zl, Z.ptr(), nullptr), "b200_vec_add_dev");
    auto abc = multiply_vec(Z);
    check(b200_cross_term_dev(field, abc[0].ptr(), abc[1].ptr(), abc[2].ptr(), E1.ptr(), E2 ? E2->ptr() : nullptr,
                              ud.ptr(), num_cons, T.ptr(), nullptr), "b200_cross_term_dev");
    Point cT = commit_resident(ck, T, r_T);  // its D2H synchronises: temporaries above may now go
    return {std::move(T), cT};
  }
};

// RelaxedR1CSWitness::fold / fold_relaxed on resident vectors (r1cs/mod.rs:1044-1107).  The blinds
// r_W, r_E are host scalars: the caller folds them with its own field arithmetic.
inline RelaxedR1CSWitnessDev fold_witness_resident(int field, const RelaxedR1CSWitnessDev& W1, const DeviceVec& W2,
                                                   const DeviceVec& T, const Scalar& r, const DeviceVec* E2 = nullptr,
                                                   const Scalar* r_squared = nullptr) {
  if (W1.W.len() != W2.len()) throw std::invalid_argument("InvalidWitnessLength");  // r1cs/mod.rs:1054-1056
  RelaxedR1CSWitnessDev out{DeviceVec(W1.W.len()), DeviceVec(W1.E.len())};
  DeviceVec rd(std::vector<Scalar>{r});
  check(b200_axpy_dev(field, W1.W.ptr(), W2.ptr(), rd.ptr(), W2.len(), out.W.ptr(), nullptr), "b200_axpy_dev");
  check(b200_axpy_dev(field, W1.E.ptr(), T.ptr(), rd.ptr(), T.len(), out.E.ptr(), nullptr), "b200_axpy_dev");
  if (E2) {  // + r^2 E2
    if (!r_squared) throw std::logic_error("fold_relaxed needs r^2");
    DeviceVec r2(std::vector<Scalar>{*r_squared}), tmp(W1.E.len());
    check(b200_axpy_dev(field, out.E.ptr(), E2->ptr(), r2.ptr(), E2->len(), tmp.ptr(), nullptr), "b200_axpy_dev");
    check(b200_sync(), "b200_sync");
    out.E = std::move(tmp);
  }
  check(b200_sync(), "b200_sync");  // rd must outlive the launches
  return out;
}

// ---- sum-check round loops with the transcript on the device (SURVEY.md §8f-3) ------------------
// The serialisable part of Keccak256Transcript (keccak.rs:19-27): `round`, `state`, and the bytes
// absorbed since the last squeeze (`transcript_buffer`).
struct TranscriptState {
  b200_transcript tr{};
  std::vector<unsigned char> pending;
};
struct SumcheckProofOut {
  std::vector<std::vector<Scalar>> compressed_polys;  // canonical little-endian (the proof bytes)
  std::vector<Scalar> r;                              // challenges (Montgomery)
  std::vector<Scalar> final_evals;                    // Montgomery
};
namespace detail {
template <class Call>
inline SumcheckProofOut device_loop(TranscriptState& t, int num_rounds, int ncoef, int nfinals, Call call,
                                    const char* what) {
  std::vector<Scalar> polys((size_t)num_rounds * ncoef), rs(num_rounds), fin(nfinals);
  check(call(&t.tr, t.pending.empty() ? nullptr : t.pending.data(), t.pending.size(), polys.data(), rs.data(),
             fin.data()), what);
  t.pending.clear();
  SumcheckProofOut out;
  for (int j = 0; j < num_rounds; j++)
    out.compressed_polys.emplace_back(polys.begin() + (size_t)j * ncoef, polys.begin() + (size_t)(j + 1) * ncoef);
  out.r = std::move(rs);
  out.final_evals = std::move(fin);
  return out;
}
}  // namespace detail
// SumcheckProof::prove_quad_prod (sumcheck.rs:199-242); d_A / d_B are device polynomials, bound in place
inline SumcheckProofOut prove_quad_prod(int field, const Scalar& claim, int num_rounds, void* d_A, void* d_B,
                                        TranscriptState& t) {
  return detail::device_loop(t, num_rounds, 2, 2, [&](b200_transcript* tr, const void* p, size_t n, void* polys,
                                                      void* rs, void* fin) {
    return b200_sumcheck_quad_prod(field, &claim, num_rounds, d_A, d_B, tr, p, n, polys, rs, fin);
  }, "b200_sumcheck_quad_prod");
}
// SumcheckProof::prove_cubic_with_three_inputs (sumcheck.rs:446-507)
inline SumcheckProofOut prove_cubic_with_three_inputs(int field, const Scalar& claim, const std::vector<Scalar>& taus,
                                                      void* d_A, void* d_B, void* d_C, TranscriptState& t) {
  return detail::device_loop(t, (int)taus.size(), 3, 3, [&](b200_transcript* tr, const void* p, size_t n,
                                                            void* polys, void* rs, void* fin) {
    return b200_sumcheck_cubic3(field, &claim, taus.data(), (int)taus.size(), d_A, d_B, d_C, tr, p, n, polys, rs, fin);
  }, "b200_sumcheck_cubic3");
}

// RelaxedR1CSSNARK::prove_helper (ppsnark.rs:886-983) in one call.  The claims of all engines as data: claim i reads
// the sums of `form[i]` over the device tables tab[i][0..2] (weighted by eq instance eq_of[i] for the eq kinds) and turns
// them into evaluation points as `kind[i]` says; `coeffs` are the powers of the batching challenge, `claim` their
// combination with the initial claims, `running` the initial claims.  final_evals: element 0 of every table, in
// program order.
struct BatchedSumcheck {
  b200_scp_program prog{};
  std::vector<std::vector<Scalar>> taus;  // per eq instance, num_rounds Montgomery scalars (kept alive for prog.taus)
  int add_table(void* d_table) {
    prog.tables[prog.ntables] = d_table;
    return prog.ntables++;
  }
  int add_eq(std::vector<Scalar> t) {
    taus.push_back(std::move(t));
    return prog.neq++;
  }
  // kind: B200_SCB_*; form / form_m1: sc_form ids (include/nova_b200.h); tables: indices from add_table, -1 = unused
  void add_claim(int kind, int form, int form_m1, int a, int b, int c, int eq) {
    const int i = prog.nclaims++;
    prog.kind[i] = kind;
    prog.form[i] = form;
    prog.form_m1[i] = form_m1;
    prog.eq_of[i] = eq;
    prog.tab[i][0] = a;
    prog.tab[i][1] = b;
    prog.tab[i][2] = c;
  }
  SumcheckProofOut prove(int field, int num_rounds, const std::vector<Scalar>& coeffs, const Scalar& claim,
                         const std::vector<Scalar>& running, TranscriptState& t) {
    prog.num_rounds = num_rounds;
    for (int g = 0; g < prog.neq; g++) prog.taus[g] = taus[g].data();
    return detail::device_loop(t, num_rounds, 3, prog.ntables, [&](b200_transcript* tr, const void* p, size_t n,
                                                                   void* polys, void* rs, void* fin) {
      return b200_sumcheck_batched(field, &prog, coeffs.data(), &claim, running.data(), tr, p, n, polys, rs, fin);
    }, "b200_sumcheck_batched");
  }
};

// ---- one process, all GPUs of the node (b200_mgpu_*): the single call a CommitmentEngine::commit makes ------------
// The key is distributed block-cyclically over the devices; every commit of a prefix ck[..n] is fanned out inside the
// library and the partial sums are exchanged over NVLink inside the reduction kernels (include/nova_b200.h).
template <class C>
class MultiGpuCommitmentKey {
 public:
  // devices: explicit device ids, or empty for 0 .. ndev-1
  MultiGpuCommitmentKey(const std::vector<Affine>& bases, const Affine* h, int ndev, const std::vector<int>& devices = {})
      : n_(bases.size()) {
    check(b200_mgpu_init(ndev, devices.empty() ? nullptr : devices.data()), "b200_mgpu_init");
    check(b200_mgpu_ck_register(C::curve, bases.data(), bases.size(), h, 0, &handle_), "b200_mgpu_ck_register");
  }
  ~MultiGpuCommitmentKey() {
    if (handle_) b200_mgpu_ck_release(handle_);
  }
  MultiGpuCommitmentKey(const MultiGpuCommitmentKey&) = delete;
  MultiGpuCommitmentKey& operator=(const MultiGpuCommitmentKey&) = delete;
  size_t len() const { return n_; }
  // CommitmentEngineTrait::commit (pedersen.rs:263-270); r = nullptr: vartime_multiscalar_mul over ck[..v.len()]
  Point commit(const std::vector<Scalar>& v, const Scalar* r = nullptr) const {
    if (v.size() > n_) throw std::logic_error("commit: vector longer than the key");  // pedersen.rs:264
    Point out;
    check(b200_mgpu_commit(handle_, v.data(), v.size(), r, &out), "b200_mgpu_commit");
    return out;
  }

 private:
  uint64_t handle_ = 0;
  size_t n_;
};

// ---- Poseidon random oracle with the squeeze on the device (ROTrait for PoseidonRO, provider/poseidon.rs:60-127) --------
// The constants (R_F, R_P, Grain-LFSR round constants, Cauchy MDS; Montgomery form) are the caller's: a Rust host passes
// its `PoseidonConstantsCircuit`, the Python mirror derives them (nova_b200/poseidon.py).
class PoseidonRO {
 public:
  PoseidonRO(int field, int arity, int r_f, int r_p, const std::vector<Scalar>& round_constants, const std::vector<Scalar>& mds)
      : field_(field) {
    check(b200_poseidon_register(field, arity, r_f, r_p, round_constants.data(), mds.data(), &handle_), "b200_poseidon_register");
  }
  ~PoseidonRO() {
    if (handle_) b200_poseidon_release(handle_);
  }
  PoseidonRO(const PoseidonRO&) = delete;
  PoseidonRO& operator=(const PoseidonRO&) = delete;
  void absorb(const Scalar& e) { state_.push_back(e); }
  // -> (challenge as a Montgomery element of `field`, challenge as a canonical integer); the state becomes [hash]
  std::pair<Scalar, Scalar> squeeze(int num_bits, bool start_with_one = false) {
    Scalar out[3];
    check(b200_poseidon_ro(handle_, state_.data(), state_.size(), num_bits, start_with_one ? 1 : 0, out), "b200_poseidon_ro");
    state_.assign(1, out[0]);
    return {out[1], out[2]};
  }

 private:
  int field_;
  uint64_t handle_ = 0;
  std::vector<Scalar> state_;
};

}  // namespace b200
}  // namespace nova
