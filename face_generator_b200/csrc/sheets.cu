// sample.lua's image sheets (fg_image_grid): toGrid / toNeighboursGrid (sample.lua:156-168, :228-230), i.e.
// image.toDisplayTensor{input=images, nrow=nrow} at its defaults (padding 0, scaleeach false, min / max / symmetric
// unset), and the byte conversion of image.save's JPEG writer (clampImage, *255, to unsigned char).  The JPEG file is
// fg_jpeg_encode's (jpeg_enc.cu).
//
// toDisplayTensor: xmaps = min(nrow, count) columns, ymaps = ceil(count / xmaps) rows of (H+padding) x (W+padding)
// cells, image k in cell (k / xmaps, k % xmaps) at offset padding/2, every other pixel filled with the largest value
// of the images; then image.minmax over the whole grid.  As the fill is that maximum, the grid's extremes are those of
// the selected images, so two launches on the ctx stream:
//   grid_minmax_kernel  the minimum and maximum of the selected images: ordered bit patterns, atomicMin / atomicMax
//                       (exact: the result does not depend on the order), NaN left out
//   grid_layout_kernel  one output byte per thread: the cell's image pixel or the fill, minmax, clampImage, byte
// The three rules of torch/image that no available source pins (DESIGN.md section 2.4) are each one function below:
// grid_scale, grid_rescales and grid_byte; tests/grid_ref.py mirrors each in one function.
#include "fg_internal.h"

namespace {

constexpr int kGridMax = 4096;  // largest Hg / Wg

// float -> unsigned key with the same order (-0 just below +0); NaN never reaches it
__device__ __forceinline__ unsigned ordered_key(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// assumption 1: minmax divides the shifted values by (max - min), in float32 (not a multiply by its reciprocal)
__device__ __forceinline__ float grid_scale(float shifted, float range) { return __fdiv_rn(shifted, range); }
// assumption 2: a constant grid (max - min == 0) is shifted by -min and not divided
__device__ __forceinline__ bool grid_rescales(float range) { return range != 0.f; }
// assumption 3: clampImage saturates to [0, 1], the writer multiplies by 255 in float32 and truncates (C's
// (unsigned char) cast); NaN gives 0 (this library's choice)
__device__ __forceinline__ uint8_t grid_byte(float x) {
  if (x != x) return 0;
  x = x < 0.f ? 0.f : (x > 1.f ? 1.f : x);
  return (uint8_t)__fmul_rn(x, 255.f);
}

__device__ __forceinline__ int64_t pick(const int32_t* order, int k, int64_t N) {
  if (!order) return k;
  const int64_t i = order[k];
  return i < 0 ? 0 : (i >= N ? N - 1 : i);
}

// keys[0] = min, keys[1] = max (ordered keys) over the selected images; keys start at (0xffffffff, 0)
__global__ void grid_minmax_kernel(const float* __restrict__ images, int64_t N, int per, const int32_t* __restrict__ order,
                                   int count, unsigned* __restrict__ keys) {
  unsigned lo = 0xffffffffu, hi = 0u;
  const int64_t n = (int64_t)count * per;
  GRID_STRIDE(i, n) {
    const int k = (int)(i / per);
    const float v = images[pick(order, k, N) * per + (i - (int64_t)k * per)];
    if (v != v) continue;
    const unsigned key = ordered_key(v);
    lo = min(lo, key);
    hi = max(hi, key);
  }
  for (int o = 16; o > 0; o >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((threadIdx.x & 31) == 0) {
    if (lo != 0xffffffffu) atomicMin(keys, lo);
    if (hi != 0u) atomicMax(keys + 1, hi);
  }
}

__global__ void grid_layout_kernel(const float* __restrict__ images, int64_t N, int C, int H, int W, const int32_t* __restrict__ order,
                                   int count, int xmaps, int padding, int Hg, int Wg, const unsigned* __restrict__ keys,
                                   uint8_t* __restrict__ out) {
  // every value NaN: no extremes; taken as 0, 0
  const bool any = keys[0] != 0xffffffffu;
  const float mn = any ? key_value(keys[0]) : 0.f, mx = any ? key_value(keys[1]) : 0.f;
  const float range = __fsub_rn(mx, mn);
  const int ch = H + padding, cw = W + padding, half = padding / 2;
  const int64_t n = (int64_t)C * Hg * Wg;
  GRID_STRIDE(i, n) {
    const int x = (int)(i % Wg);
    const int64_t r = i / Wg;
    const int y = (int)(r % Hg), c = (int)(r / Hg);
    const int cy = y / ch, cx = x / cw, iy = y - cy * ch - half, ix = x - cx * cw - half;
    const int k = cy * xmaps + cx;
    float v = mx;  // the fill
    if (k < count && iy >= 0 && iy < H && ix >= 0 && ix < W) v = images[((pick(order, k, N) * C + c) * H + iy) * W + ix];
    float t = __fsub_rn(v, mn);
    if (grid_rescales(range)) t = grid_scale(t, range);
    out[i] = grid_byte(t);
  }
}

}  // namespace

extern "C" int fg_image_grid(fg_ctx* c, const float* images, int64_t N, int C, int H, int W, const int32_t* order, int count,
                             int nrow, int padding, uint8_t* out, int* Hg_out, int* Wg_out) {
  if (!c) {
    fg_set_error("null fg_ctx");
    return FG_ERR_INVALID;
  }
  FG_REQUIRE(images && N >= 1 && count >= 1 && nrow >= 1, "fg_image_grid: need images, N >= 1, count >= 1, nrow >= 1");
  FG_REQUIRE(C >= 1 && C <= 3 && H >= 1 && W >= 1, "fg_image_grid: images [%lld][%d][%d][%d] (1 to 3 channels)", (long long)N, C,
             H, W);
  FG_REQUIRE(padding >= 0 && padding % 2 == 0, "fg_image_grid: padding %d is not even and >= 0", padding);
  FG_REQUIRE(order || count <= N, "fg_image_grid: %d images asked of %lld", count, (long long)N);
  const int xmaps = nrow < count ? nrow : count, ymaps = (count + xmaps - 1) / xmaps;
  const int64_t Hg = (int64_t)ymaps * (H + padding), Wg = (int64_t)xmaps * (W + padding);
  FG_REQUIRE(Hg <= kGridMax && Wg <= kGridMax, "fg_image_grid: the grid is %lldx%lld, above %dx%d", (long long)Hg, (long long)Wg,
             kGridMax, kGridMax);
  const bool order_dev = order && fg_is_dev(order);
  if (order && !order_dev)
    for (int k = 0; k < count; ++k)
      FG_REQUIRE(order[k] >= 0 && order[k] < N, "fg_image_grid: order[%d] = %d outside [0, %lld)", k, order[k], (long long)N);
  if (Hg_out) *Hg_out = (int)Hg;
  if (Wg_out) *Wg_out = (int)Wg;
  if (!out) return FG_OK;
  FG_CUDA(cudaSetDevice(c->device));
  const int64_t per = (int64_t)C * H * W, n_out = (int64_t)C * Hg * Wg;
  const bool img_dev = fg_is_dev(images), out_dev = fg_is_dev(out);
  // one stream-ordered temporary: keys, then a host order, images and output
  const size_t o_order = 16, o_img = (o_order + sizeof(int32_t) * (order_dev || !order ? 0 : count) + 15) & ~(size_t)15,
               o_out = o_img + (img_dev ? 0 : sizeof(float) * (size_t)(N * per)), bytes = o_out + (out_dev ? 0 : (size_t)n_out);
  uint8_t* tmp = nullptr;
  FG_CUDA(cudaMallocAsync((void**)&tmp, bytes, c->stream));
  unsigned* keys = reinterpret_cast<unsigned*>(tmp);
  const int32_t* ord = order_dev ? order : (order ? reinterpret_cast<const int32_t*>(tmp + o_order) : nullptr);
  const float* img = img_dev ? images : reinterpret_cast<const float*>(tmp + o_img);
  uint8_t* dst = out_dev ? out : tmp + o_out;
  const unsigned init[2] = {0xffffffffu, 0u};
  cudaError_t e = cudaMemcpyAsync(keys, init, sizeof(init), cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess && order && !order_dev)
    e = cudaMemcpyAsync(tmp + o_order, order, sizeof(int32_t) * count, cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess && !img_dev) e = cudaMemcpyAsync(tmp + o_img, images, sizeof(float) * (size_t)(N * per), cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess) {
    grid_minmax_kernel<<<grid_for((int64_t)count * per, 256, c->sm_count * 8), 256, 0, c->stream>>>(img, N, (int)per, ord, count, keys);
    c->launches++;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) {
    grid_layout_kernel<<<grid_for(n_out, 256, c->sm_count * 16), 256, 0, c->stream>>>(img, N, C, H, W, ord, count, xmaps, padding,
                                                                                      (int)Hg, (int)Wg, keys, dst);
    c->launches++;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess && !out_dev) e = cudaMemcpyAsync(out, dst, (size_t)n_out, cudaMemcpyDeviceToHost, c->stream);
  const cudaError_t ef = cudaFreeAsync(tmp, c->stream);
  if (e == cudaSuccess) e = ef;
  if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
  if (e != cudaSuccess) {
    fg_set_error("fg_image_grid: %s", cudaGetErrorString(e));
    return FG_ERR_CUDA;
  }
  return FG_OK;
}
