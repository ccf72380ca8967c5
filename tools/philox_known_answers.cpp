// Known-answer vectors of Philox-4x32 from PyTorch's host engine (at::Philox4_32, ATen/core/PhiloxRNGEngine.h), for
// tests/test_philox_cpu.py.  Host only, no CUDA and no libtorch: the engine is header-only.
//
//   TORCH=$(python -c "import torch, os; print(os.path.dirname(torch.__file__))")
//   g++ -std=c++17 -O1 -I$TORCH/include tools/philox_known_answers.cpp -o /tmp/philox_kat && /tmp/philox_kat
//
// at::Philox4_32(seed, subsequence, offset) starts at counter (offset_lo, offset_hi, subsequence_lo, subsequence_hi)
// with key (seed_lo, seed_hi); every fourth call of operator()(rounds) encrypts the counter and returns its 4 words
// in order.  Prints one Python tuple per vector: (rounds, (c0, c1, c2, c3), (k0, k1), (x0, x1, x2, x3)).
#include <ATen/core/PhiloxRNGEngine.h>

#include <cstdint>
#include <cstdio>

int main() {
  struct Vec { uint32_t c[4]; uint32_t k[2]; };
  const Vec vecs[] = {
      {{0u, 0u, 0u, 0u}, {0u, 0u}},
      {{0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu}, {0xffffffffu, 0xffffffffu}},
      {{0x243f6a88u, 0x85a308d3u, 0x13198a2eu, 0x03707344u}, {0xa4093822u, 0x299f31d0u}},
      {{7u, 3u, 11u, 0x5a17u}, {0x9abcdef0u, 0x12345678u}},        // the sampler's counter layout (c, b, step, 0x5a17)
      {{4095u, 0u, 351u, 2u}, {12345u, 0u}},                       // the dropout layout (row_lo, row_hi, chunk, layer)
  };
  for (int rounds : {10, 7}) {
    for (const Vec& v : vecs) {
      const uint64_t seed = (static_cast<uint64_t>(v.k[1]) << 32) | v.k[0];
      const uint64_t subsequence = (static_cast<uint64_t>(v.c[3]) << 32) | v.c[2];
      const uint64_t offset = (static_cast<uint64_t>(v.c[1]) << 32) | v.c[0];
      at::Philox4_32 eng(seed, subsequence, offset);
      uint32_t x[4];
      for (uint32_t& w : x) w = eng(rounds);
      std::printf("(%d, (0x%08x, 0x%08x, 0x%08x, 0x%08x), (0x%08x, 0x%08x), (0x%08x, 0x%08x, 0x%08x, 0x%08x)),\n", rounds,
                  v.c[0], v.c[1], v.c[2], v.c[3], v.k[0], v.k[1], x[0], x[1], x[2], x[3]);
    }
  }
  return 0;
}
