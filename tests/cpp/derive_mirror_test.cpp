// C++ host-mirror test of CommitmentEngine<C>::ck_derive_by_address (include/nova_b200.hpp).
//   derive_mirror_test --compile-check      (no GPU: instantiates the entry and links)
//   derive_mirror_test <case>               case = [n][bases], [1][h], [m][addresses u64], [1][table_size], [t][T], [1][r]
//                                           (each blob: u64 count, then the elements); writes <case>.out =
//                                           commit(derived, T, r), commit(derived, T), then the InvalidIndex position
//                                           and whether InvalidCommitmentKeyLength was thrown (u64 each)
#include <cstdio>
#include <fstream>
#include <memory>

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
    auto derive = &CommitmentEngine<BN254>::ck_derive_by_address;  // instantiated: the symbol must link
    std::printf("derive_mirror_test compiled against %s (%p)\n", b200_version(), (void*)&derive);
    return 0;
  }
  std::ifstream f(argv[1], std::ios::binary);
  auto bases = read_blob<Affine>(f);
  auto h = read_blob<Affine>(f);
  auto addr64 = read_blob<uint64_t>(f);
  auto ts = read_blob<uint64_t>(f);
  auto T = read_blob<Scalar>(f);
  auto r = read_blob<Scalar>(f);
  check(b200_init(0), "b200_init");
  std::vector<size_t> addresses(addr64.begin(), addr64.end());
  std::unique_ptr<CommitmentKey<BN254>> derived;
  uint64_t bad_position = UINT64_MAX, length_error = 0;
  {
    CommitmentKey<BN254> ck(bases, &h[0]);
    derived.reset(new CommitmentKey<BN254>(CommitmentEngine<BN254>::ck_derive_by_address(ck, addresses, ts[0])));
    std::vector<size_t> wrong = addresses;
    wrong.back() = ts[0];
    try {
      CommitmentEngine<BN254>::ck_derive_by_address(ck, wrong, ts[0]);
    } catch (const CommitmentKey<BN254>::InvalidIndex& e) {
      bad_position = e.position;
    }
    std::vector<size_t> longer(bases.size() + 1, 0);
    try {
      CommitmentEngine<BN254>::ck_derive_by_address(ck, longer, ts[0]);
    } catch (const CommitmentKey<BN254>::InvalidCommitmentKeyLength&) {
      length_error = 1;
    }
  }  // the source key is released here; the derived key stays usable
  Point blinded = CommitmentEngine<BN254>::commit(*derived, T, &r[0]);
  Point plain = CommitmentEngine<BN254>::commit(*derived, T);
  std::ofstream o(std::string(argv[1]) + ".out", std::ios::binary);
  o.write((const char*)&blinded, 96);
  o.write((const char*)&plain, 96);
  o.write((const char*)&bad_position, 8);
  o.write((const char*)&length_error, 8);
  std::printf("derive mirror ok\n");
  return 0;
}
