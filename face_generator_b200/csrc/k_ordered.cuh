// Run-to-run reproducible cross-block sums (replacing float / double atomicAdd, whose order varies between runs).
//
// The blocks of a launch write their partial sums to rows of a workspace, ws[row * n + j], every entry of every row
// written exactly once (a row may be shared by several blocks that own disjoint entries), then call
// ordered_last_block(ticket).  Exactly one block -- the last to arrive -- gets true, sums the rows in row order with
// ordered_sum() and resets the ticket with ordered_release(), so the same inputs give bit-identical results.
#pragma once
#include <cstdint>

// all threads of the block must call it, after their partial stores
__device__ __forceinline__ bool ordered_last_block(unsigned* ticket) {
  __shared__ bool last;
  __threadfence();  // this block's partials are visible device-wide before its ticket
  __syncthreads();
  if (threadIdx.x == 0 && threadIdx.y == 0 && threadIdx.z == 0)
    last = atomicAdd(ticket, 1u) == gridDim.x * gridDim.y * gridDim.z - 1;
  __syncthreads();
  if (last) __threadfence();
  return last;
}
__device__ __forceinline__ double ordered_sum(const double* ws, int rows, int64_t n, int64_t j) {
  double s = 0;
  for (int r = 0; r < rows; ++r) s += __ldcg(ws + (int64_t)r * n + j);  // L2: written by other blocks
  return s;
}
__device__ __forceinline__ void ordered_release(unsigned* ticket) {
  if (threadIdx.x == 0 && threadIdx.y == 0 && threadIdx.z == 0) *ticket = 0;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// block-wide sum (blockDim.x multiple of 32, <= 1024): a xor tree over the lanes, then over the warp partials; result
// valid in thread 0
__device__ __forceinline__ double block_sum(double v) {
  __shared__ double red[32];
  __syncthreads();
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = threadIdx.x < (blockDim.x + 31) / 32 ? red[threadIdx.x] : 0.0;
    v = warp_sum(v);
  }
  return v;
}
// sum over a block of 256 threads in a fixed order (lanes, then warps); valid in thread 0
__device__ __forceinline__ double block_sum256(double v) {
  __shared__ double red[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < 8; ++w) s += red[w];
  return s;
}
