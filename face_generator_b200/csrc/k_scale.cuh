// image.scale(src, w, h) on the device: the one home of the scaling rule (dataset.cu's gather / pair kernels,
// fg_image_scale and the coarse-to-fine refinement of nets_c2f.cu).
//
// image.scale [third-party `image` rock, un-pinned; default mode 'bilinear'] is separable; along one axis
// (generic/image.c, Main_scaleLinear_rowcol) it
//   - shrinks by area averaging: output i covers source [i*s, (i+1)*s), s = src_len/dst_len (float), partial
//     coverage of the first/last source pixel weighted by the covered fraction, divided by the total weight;
//   - enlarges by linear interpolation with s = (src_len-1)/(dst_len-1), last output = last source pixel;
//   - copies when the sizes match.
// The oracle restates the same in numpy (oracle/oracle_data.py).  PARITY UNPINNED (no `image` rock here).
#pragma once

namespace {
// weight of source index si for output index di along one axis (see the file header); *norm = total weight
struct Span {
  int i0, i1;      // source range [i0, i1]
  float w0, w1;    // weights of i0 and i1 (everything strictly between weighs 1)
  float norm;
};
__device__ __forceinline__ Span axis_span(int di, int src_len, int dst_len) {
  Span s;
  if (dst_len < src_len) {
    const float scale = (float)src_len / (float)dst_len;
    float f0 = (float)di * scale;
    const int a = (int)f0;
    f0 -= (float)a;
    float f1 = (float)(di + 1) * scale;
    int b = (int)f1;
    f1 -= (float)b;
    s.i0 = a;
    s.w0 = 1.f - f0;
    s.norm = (1.f - f0) + (float)(b - a - 1);
    if (b < src_len) {
      s.i1 = b;
      s.w1 = f1;
      s.norm += f1;
    } else {
      s.i1 = b - 1;
      s.w1 = (b - 1 == a) ? s.w0 : 1.f;
    }
  } else if (dst_len > src_len) {
    if (src_len == 1 || di == dst_len - 1) {
      s.i0 = s.i1 = src_len - 1;
      s.w0 = s.w1 = 1.f;
      s.norm = 1.f;
      if (src_len == 1) s.i0 = s.i1 = 0;
    } else {
      const float scale = (float)(src_len - 1) / (float)(dst_len - 1);
      float f = (float)di * scale;
      const int a = (int)f;
      f -= (float)a;
      s.i0 = a;
      s.i1 = a + 1;
      s.w0 = 1.f - f;
      s.w1 = f;
      s.norm = 1.f;
    }
  } else {
    s.i0 = s.i1 = di;
    s.w0 = s.w1 = 1.f;
    s.norm = 1.f;
  }
  return s;
}
__device__ __forceinline__ float span_w(const Span& s, int i) { return i == s.i0 ? s.w0 : (i == s.i1 ? s.w1 : 1.f); }

// image.scale's output pixel (y, x) of an Ho x Wo image from an Hs x Ws source, src(yy, xx) = source value: pass 1
// (width) then pass 2 (height), like image.scale's two-pass implementation.  Equal sizes multiply and divide by 1 only,
// so they copy the source bit for bit.
template <class Src>
__device__ __forceinline__ float scale_pixel(const Src& src, int y, int x, int Hs, int Ws, int Ho, int Wo) {
  const Span sy = axis_span(y, Hs, Ho), sx = axis_span(x, Ws, Wo);
  float acc_y = 0.f;
  for (int yy = sy.i0; yy <= sy.i1; ++yy) {
    float acc_x = 0.f;
    for (int xx = sx.i0; xx <= sx.i1; ++xx) acc_x += span_w(sx, xx) * src(yy, xx);
    acc_y += span_w(sy, yy) * (acc_x / sx.norm);
  }
  return acc_y / sy.norm;
}
// one fp32 plane [H][W] (shared or global memory)
struct PlaneSrc {
  const float* p;
  int W;
  __device__ __forceinline__ float operator()(int yy, int xx) const { return p[yy * W + xx]; }
};
}  // namespace
