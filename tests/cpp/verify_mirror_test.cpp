// C++ host-mirror test of the verifier wrappers R1CSShape::multi_evaluate, R1CSShapeDev::multi_evaluate and ipa_s
// (include/nova_b200.hpp).
//   verify_mirror_test --compile-check   (no GPU: instantiates the wrappers and links)
//   verify_mirror_test <case>            case = [nnz][data], [nnz][indices u64], [rows+1][indptr u64], [1][cols],
//                                        [lx][r_x], [ly][r_y], [L][r], [L][r_inv], [1][scale] (each blob: u64 count, then
//                                        the elements; the one matrix is used as A, B and C); writes <case>.out =
//                                        multi_evaluate from the points (3 scalars), from resident eq tables
//                                        (3 scalars), then ipa_s(r, r_inv) and ipa_s(r, r_inv, &scale) (2^L scalars each)
#include <cstdio>
#include <fstream>

#include "../../include/nova_b200.hpp"

using namespace nova::b200;

template <class T>
static std::vector<T> read_blob(std::ifstream& f) {
  uint64_t k = 0;
  f.read((char*)&k, 8);
  std::vector<T> v(k);
  f.read((char*)v.data(), (std::streamsize)(k * sizeof(T)));
  return v;
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  if (std::string(argv[1]) == "--compile-check") {
    auto host = &R1CSShape::multi_evaluate;  // instantiated: the symbols must link
    auto dev = &R1CSShapeDev::multi_evaluate;
    auto s = &ipa_s;
    std::printf("verify_mirror_test compiled against %s (%p %p %p)\n", b200_version(), (void*)&host, (void*)&dev,
                (void*)&s);
    return 0;
  }
  std::ifstream f(argv[1], std::ios::binary);
  auto data = read_blob<Scalar>(f);
  auto indices = read_blob<uint64_t>(f);
  auto indptr = read_blob<uint64_t>(f);
  auto cols = read_blob<uint64_t>(f);
  auto r_x = read_blob<Scalar>(f);
  auto r_y = read_blob<Scalar>(f);
  auto r = read_blob<Scalar>(f);
  auto r_inv = read_blob<Scalar>(f);
  auto scale = read_blob<Scalar>(f);
  check(b200_init(0), "b200_init");
  const int field = B200_FIELD_PALLAS_FP;  // Vesta's scalar field
  SparseMatrix M(field, data, indices, indptr, cols[0]);
  R1CSShape shape{M, M, M, field};
  std::array<Scalar, 3> from_points = shape.multi_evaluate(r_x, r_y);
  DeviceVec rx(r_x), ry(r_y), Tx((size_t)1 << r_x.size()), Ty((size_t)1 << r_y.size());
  check(b200_eq_table_dev(field, rx.ptr(), (int)r_x.size(), Tx.ptr(), nullptr), "b200_eq_table_dev");
  check(b200_eq_table_dev(field, ry.ptr(), (int)r_y.size(), Ty.ptr(), nullptr), "b200_eq_table_dev");
  R1CSShapeDev dshape{M, M, M, field, M.rows(), 0, 0};
  std::array<Scalar, 3> from_tables = dshape.multi_evaluate(Tx, Ty);
  DeviceVec rd(r), rid(r_inv);
  std::vector<Scalar> s1 = ipa_s(field, rd, rid).to_host();
  std::vector<Scalar> s2 = ipa_s(field, rd, rid, &scale[0]).to_host();
  std::ofstream o(std::string(argv[1]) + ".out", std::ios::binary);
  o.write((const char*)from_points.data(), 96);
  o.write((const char*)from_tables.data(), 96);
  o.write((const char*)s1.data(), (std::streamsize)(32 * s1.size()));
  o.write((const char*)s2.data(), (std::streamsize)(32 * s2.size()));
  std::printf("verify mirror ok\n");
  return 0;
}
