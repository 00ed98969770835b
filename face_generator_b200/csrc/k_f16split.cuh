// Device helpers of the 3xFP16 operand split (shared by k_conv_tc.cu and k_misc.cu).
#pragma once
#include <cuda_fp16.h>

// 3xFP16 split: x ~= hi + lo * 2^-11 with hi = fp16(x), lo = fp16((x - hi) * 2^11): 22 significant bits like the TF32
// split, operands of f16 MMAs (2x the TF32 rate, 4 bytes per element for hi+lo instead of 8).  fp16 subnormals
// keep the ABSOLUTE error at 2^-36, so a tensor whose max is in [2^-13, 65504] is represented to 2^-23 of that max.
// Activations and gradients are first scaled by the power of two of their own max|x| (scale_for_amax); weights are
// used as they are.  NaN and +-Inf pass through unclamped (hi = x, lo = 0), so that the MMA propagates them as the
// fp32 path does; the clamp only bounds finite values.
__device__ __forceinline__ void split_f16(float x, __half& hi, __half& lo) {
  const bool fin = fabsf(x) <= 3.402823466e38f;  // false for NaN and +-Inf
  hi = __float2half_rn(fin ? fminf(fmaxf(x, -65504.f), 65504.f) : x);
  lo = __float2half_rn(fin ? fminf(fmaxf((x - __half2float(hi)) * 2048.f, -65504.f), 65504.f) : 0.f);
}
// |x| as the max|x| reductions that set a tensor's scale see it: NaN and +-Inf count as 0, so that one non-finite
// element does not take the scaling away from the rest of its tensor (split_f16 passes that element through as it is)
__device__ __forceinline__ float finite_abs(float x) {
  const float a = fabsf(x);
  return a <= 3.402823466e38f ? a : 0.f;
}
// power of two that brings amax into [2^14, 2^15) (1 for an all-zero tensor); exponent clamped so that s and 1/s are normal
__device__ __forceinline__ float scale_for_amax(float amax) {
  if (!(amax > 0.f) || !isfinite(amax)) return 1.f;
  int ex;
  frexpf(amax, &ex);  // amax = m * 2^ex, m in [0.5, 1)
  const int e = max(-100, min(100, 15 - ex));
  return ldexpf(1.f, e);
}

// max|output| over the finite outputs of an elementwise producer (finite_abs) into a device word (option mma_f16: the
// power-of-two scale of the FP16 split is derived from it, k_conv_tc.cu).  Non-negative floats order like their bit
// patterns, so atomicMax on the bits is exact and order-independent (replicas stay identical).  Must be reached by all
// 32 lanes.
__device__ __forceinline__ void amax_commit(unsigned* amax, float m) {
  if (!amax) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  // thousands of warps hit ONE word: an atomic per warp serialises at the L2 (measured 100+ us on the pooling kernels).
  // A plain load first: only a warp that would actually raise the maximum issues the atomic (a handful per launch).
  if ((threadIdx.x & 31) == 0 && m > 0.f) {
    const unsigned bits = __float_as_uint(m);
    if (bits > *reinterpret_cast<volatile unsigned*>(amax)) atomicMax(amax, bits);
  }
}
__device__ __forceinline__ float amax4(float m, float a, float b, float c, float d) {
  return fmaxf(fmaxf(m, fmaxf(finite_abs(a), finite_abs(b))), fmaxf(finite_abs(c), finite_abs(d)));
}
