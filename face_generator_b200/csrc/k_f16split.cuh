// Device helpers of the 3xFP16 operand split (shared by k_conv_tc.cu and k_misc.cu).
#pragma once
#include <cuda_fp16.h>

// 3xFP16 split: x ~= hi + lo * 2^-11 with hi = fp16(x), lo = fp16((x - hi) * 2^11): 22 significant bits like the TF32
// split, operands of f16 MMAs (2x the TF32 rate, 4 bytes per element for hi+lo instead of 8).  fp16 subnormals
// keep the ABSOLUTE error at 2^-36, so a tensor whose max is in [2^-13, 65504] is represented to 2^-23 of that max;
// activations and weights are used as they are, gradients are first scaled by a power of two (tc_amax).
__device__ __forceinline__ void split_f16(float x, __half& hi, __half& lo) {
  const float xc = fminf(fmaxf(x, -65504.f), 65504.f);
  hi = __float2half_rn(xc);
  lo = __float2half_rn(fminf(fmaxf((x - __half2float(hi)) * 2048.f, -65504.f), 65504.f));
}
// power of two that brings amax into [2^14, 2^15) (1 for an all-zero tensor); exponent clamped so that s and 1/s are normal
__device__ __forceinline__ float scale_for_amax(float amax) {
  if (!(amax > 0.f) || !isfinite(amax)) return 1.f;
  int ex;
  frexpf(amax, &ex);  // amax = m * 2^ex, m in [0.5, 1)
  const int e = max(-100, min(100, 15 - ex));
  return ldexpf(1.f, e);
}
