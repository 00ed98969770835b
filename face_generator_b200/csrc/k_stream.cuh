// Counter-based random streams drawn inside kernels: element i of stream (root, kind), where root is the step seed a
// captured step reads from device memory (fg_ctx::seed_dev) and kind names what is drawn.
#pragma once
#include <cstdint>

__device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__device__ __forceinline__ uint64_t stream_bits(uint64_t root, uint64_t kind, int64_t i) {
  return mix64((root * 8 + kind) * 0x100000001B3ull + (uint64_t)i);
}
