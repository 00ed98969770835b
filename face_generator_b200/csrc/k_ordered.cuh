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
