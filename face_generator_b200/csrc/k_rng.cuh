// The counter-based uniform stream of fg_noise_uniform, shared by the kernels that draw it (dataset.cu's
// uniform_pm1_kernel, the refinement's in-kernel noise in nets_c2f.cu): element i of stream `seed` depends on
// (seed, i) only, so any slice of the stream can be drawn on its own.
#pragma once
#include <cstdint>

namespace {
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
// element i of the 24-bit uniform stream in [-1, 1) (NN_UTILS.createNoiseInputs' uniform(-1, 1))
__device__ __forceinline__ float uniform_pm1_at(uint64_t seed, uint64_t i) {
  const uint64_t r = splitmix64(seed * 0x100000001B3ull + i);
  return (float)(r >> 40) * (2.0f / 16777216.0f) - 1.0f;
}
}  // namespace
