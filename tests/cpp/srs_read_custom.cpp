// ParamsKZG::read_custom through the C++ mirror (include/spectre_b200.hpp), on a GPU:
//   srs_read_custom VALID BAD WHERE
// VALID must read checked, with the same bases and G2 trailer as an unchecked read of it. BAD must read unchecked and be
// refused checked, with WHERE (e.g. "g_lagrange[511]") in the exception text. Prints "read_custom ok" on success.
#include <cstdio>
#include <cstring>

#include "../../include/spectre_b200.hpp"

using halo2::poly::kzg::ParamsKZG;

static bool same(const std::vector<halo2::G1Affine>& a, const std::vector<halo2::G1Affine>& b) {
  return a.size() == b.size() && std::memcmp(a.data(), b.data(), a.size() * sizeof(halo2::G1Affine)) == 0;
}

int main(int argc, char** argv) {
  if (argc != 4) { std::fprintf(stderr, "usage: %s VALID BAD WHERE\n", argv[0]); return 2; }
  try {
    halo2::Backend be;
    ParamsKZG checked = ParamsKZG::read_custom(be, argv[1], SPB_SERDE_RAW_BYTES);
    ParamsKZG plain = ParamsKZG::read_custom(be, argv[1], SPB_SERDE_RAW_BYTES_UNCHECKED);
    if (checked.k() != plain.k() || !same(checked.get_g(SPB_BASIS_G), plain.get_g(SPB_BASIS_G)) ||
        !same(checked.get_g(SPB_BASIS_G_LAGRANGE), plain.get_g(SPB_BASIS_G_LAGRANGE))) {
      std::printf("checked and unchecked reads of %s differ\n", argv[1]);
      return 1;
    }
    ParamsKZG bad_plain = ParamsKZG::read_custom(be, argv[2], SPB_SERDE_RAW_BYTES_UNCHECKED);
    try {
      ParamsKZG bad = ParamsKZG::read_custom(be, argv[2], SPB_SERDE_RAW_BYTES);
      std::printf("checked read of %s was accepted\n", argv[2]);
      return 1;
    } catch (const std::runtime_error& e) {
      if (!std::strstr(e.what(), argv[3])) { std::printf("refusal does not name %s: %s\n", argv[3], e.what()); return 1; }
      std::printf("refused: %s\n", e.what());
    }
    std::printf("read_custom ok k=%u\n", checked.k());
  } catch (const std::exception& e) {
    std::printf("error: %s\n", e.what());
    return 1;
  }
  return 0;
}
