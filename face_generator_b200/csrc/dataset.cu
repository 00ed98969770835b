// Device-resident dataset + on-GPU batch assembly (SURVEY.md 8(f).2).
//
// Replaces, for the train step's input side:
//   dataset.lua:80-117  loadRandomImages: image.load(path, nbChannels, "float") then image.scale(img, 32, 32)
//   adversarial.lua:244-249 / :276  the per-sample Lua loop that copies math.random(dataset:size()) images into
//                       `inputs`, and NN_UTILS.createNoiseInputs (utils/nn_utils.lua:35-39: uniform(-1,1))
// Decoding stays on the host (it happens once, at load time); what is kept on the GPU is the DECODED uint8 image
// at its original scale (dataset.originalScale = 64, dataset.lua:10), 4x smaller than the float tensors the
// reference keeps.  fg_dataset_gather turns B indices into the normalised, down-scaled fp32 NCHW batch in one
// kernel; fg_train_step_dataset draws the indices and both noise tensors on the device too, so a train step
// needs no host->device traffic at all.
//
// image.scale(src, w, h) [third-party `image` rock, un-pinned; default mode 'bilinear'] is separable; along one
// axis (generic/image.c, Main_scaleLinear_rowcol) it
//   - shrinks by area averaging: output i covers source [i*s, (i+1)*s), s = src_len/dst_len (float), partial
//     coverage of the first/last source pixel weighted by the covered fraction, divided by the total weight;
//   - enlarges by linear interpolation with s = (src_len-1)/(dst_len-1), last output = last source pixel;
//   - copies when the sizes match.
// image.load(..., "float") is byte/255; nbChannels = 1 on a colour file is image.rgb2y: 0.299 R + 0.587 G + 0.114 B.
// The oracle restates the same in numpy (oracle/oracle_data.py).  PARITY UNPINNED (no `image` rock here).
#include <algorithm>

#include "fg_internal.h"

#define LAUNCH_CHECK(c)                 \
  do {                                  \
    (c)->launches++;                    \
    FG_CUDA(cudaGetLastError());        \
  } while (0)

struct fg_dataset {
  fg_ctx* c = nullptr;
  int64_t N = 0;
  int Cs = 3, Hs = 64, Ws = 64;
  uint8_t* data = nullptr;  // [N][Cs][Hs][Ws]
  int32_t* idx = nullptr;   // [maxB] staging for host index lists / drawn indices
};

namespace {
inline int grid_for(int64_t n, int block, int cap = 132 * 16) {
  int64_t g = (n + block - 1) / block;
  return (int)std::max<int64_t>(1, std::min<int64_t>(g, cap));
}
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
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

// out[b][c][y][x] (C channels, Ho x Wo) from u8 data[idx[b]][Cs][Hs][Ws]; gray = Cs==3 && C==1 (rgb2y)
__global__ void gather_kernel(const uint8_t* __restrict__ data, const int32_t* __restrict__ idx, float* __restrict__ out,
                              int B, int C, int Cs, int Hs, int Ws, int Ho, int Wo, int64_t N) {
  const int64_t n = (int64_t)B * C * Ho * Wo;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % Wo);
    int64_t r = i / Wo;
    const int y = (int)(r % Ho);
    r /= Ho;
    const int ch = (int)(r % C);
    const int b = (int)(r / C);
    int64_t img = idx[b];
    img = img < 0 ? 0 : (img >= N ? N - 1 : img);
    const Span sy = axis_span(y, Hs, Ho), sx = axis_span(x, Ws, Wo);
    const bool gray = Cs == 3 && C == 1;
    const uint8_t* base = data + img * (int64_t)Cs * Hs * Ws;
    // pass 1 (width) then pass 2 (height), like image.scale's two-pass implementation
    float acc_y = 0.f;
    for (int yy = sy.i0; yy <= sy.i1; ++yy) {
      float acc_x = 0.f;
      for (int xx = sx.i0; xx <= sx.i1; ++xx) {
        float v;
        if (gray) {
          const float rr = base[(0 * Hs + yy) * Ws + xx] * (1.f / 255.f), gg = base[(1 * Hs + yy) * Ws + xx] * (1.f / 255.f),
                      bb = base[(2 * Hs + yy) * Ws + xx] * (1.f / 255.f);
          v = 0.299f * rr + 0.587f * gg + 0.114f * bb;
        } else {
          v = base[((int64_t)ch * Hs + yy) * Ws + xx] * (1.f / 255.f);
        }
        acc_x += span_w(sx, xx) * v;
      }
      acc_y += span_w(sy, yy) * (acc_x / sx.norm);
    }
    out[i] = acc_y / sy.norm;
  }
}
__global__ void draw_indices_kernel(int32_t* __restrict__ idx, int B, uint64_t seed, int64_t N) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) idx[i] = (int32_t)(splitmix64(seed * 0x100000001B3ull + (uint64_t)i) % (uint64_t)N);
}
__global__ void uniform_pm1_kernel(float* __restrict__ out, int64_t n, uint64_t seed) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t r = splitmix64(seed * 0x100000001B3ull + (uint64_t)i);
    out[i] = (float)(r >> 40) * (2.0f / 16777216.0f) - 1.0f;  // 24-bit uniform in [-1, 1)
  }
}
// ---- nearest neighbour by torch.dist (2-norm), brute force, HBM-bound ------------------------------------
// sample.lua:141-159 findClosestNeighboursOf: for every query the training image with the smallest torch.dist;
// adversarial_c2f.lua:305-325 approxParzen: the smallest distance between one ground truth and K generations.
// One warp per candidate, kQG queries staged in shared memory per pass; best[q] = (dist^2 bits << 32 | index),
// reduced with 64-bit atomicMin: non-negative floats order like their bit patterns, ties go to the lowest index
// (the reference keeps the first strict minimum).
constexpr int kQG = 4;
template <bool U8>
__global__ void __launch_bounds__(256) nearest_kernel(const float* __restrict__ cands, const uint8_t* __restrict__ data, int64_t N,
                                                      int D, int C, int Cs, int Hs, int Ws, const float* __restrict__ queries, int Q,
                                                      unsigned long long* __restrict__ best) {
  extern __shared__ float qs[];  // [kQG][D]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const bool gray = Cs == 3 && C == 1;
  for (int q0 = 0; q0 < Q; q0 += kQG) {
    const int nq = min(kQG, Q - q0);
    __syncthreads();
    for (int i = threadIdx.x; i < nq * D; i += blockDim.x) qs[i] = queries[(int64_t)q0 * D + i];
    __syncthreads();
    for (int64_t cand = (int64_t)blockIdx.x * nwarps + warp; cand < N; cand += (int64_t)gridDim.x * nwarps) {
      float acc[kQG] = {0.f, 0.f, 0.f, 0.f};
      for (int i = lane; i < D; i += 32) {
        float v;
        if (!U8) {
          v = cands[cand * D + i];
        } else {  // the 32x32 view of the cached image, same arithmetic as gather_kernel
          const int x = i & 31, y = (i >> 5) & 31, ch = i >> 10;
          const Span sy = axis_span(y, Hs, 32), sx = axis_span(x, Ws, 32);
          const uint8_t* base = data + cand * (int64_t)Cs * Hs * Ws;
          float acc_y = 0.f;
          for (int yy = sy.i0; yy <= sy.i1; ++yy) {
            float acc_x = 0.f;
            for (int xx = sx.i0; xx <= sx.i1; ++xx) {
              float p;
              if (gray) {
                p = 0.299f * (base[(0 * Hs + yy) * Ws + xx] * (1.f / 255.f)) + 0.587f * (base[(1 * Hs + yy) * Ws + xx] * (1.f / 255.f)) +
                    0.114f * (base[(2 * Hs + yy) * Ws + xx] * (1.f / 255.f));
              } else {
                p = base[((int64_t)ch * Hs + yy) * Ws + xx] * (1.f / 255.f);
              }
              acc_x += span_w(sx, xx) * p;
            }
            acc_y += span_w(sy, yy) * (acc_x / sx.norm);
          }
          v = acc_y / sy.norm;
        }
#pragma unroll
        for (int g = 0; g < kQG; ++g) {
          if (g < nq) {
            const float d = v - qs[g * D + i];
            acc[g] += d * d;
          }
        }
      }
#pragma unroll
      for (int g = 0; g < kQG; ++g) {
        float s = acc[g];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0 && g < nq)
          atomicMin(best + q0 + g, ((unsigned long long)__float_as_uint(s) << 32) | (unsigned long long)(uint32_t)cand);
      }
    }
  }
}
__global__ void nearest_unpack_kernel(const unsigned long long* __restrict__ best, int Q, int32_t* __restrict__ idx,
                                      float* __restrict__ dist) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q < Q) {
    idx[q] = (int32_t)(uint32_t)(best[q] & 0xffffffffull);
    dist[q] = sqrtf(__uint_as_float((uint32_t)(best[q] >> 32)));
  }
}

bool is_dev(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}
int gather(fg_dataset* d, const int32_t* idx_dev, int B, float* out_dev) {
  fg_ctx* c = d->c;
  gather_kernel<<<grid_for((int64_t)B * c->C * 1024, 256), 256, 0, c->stream>>>(d->data, idx_dev, out_dev, B, c->C, d->Cs, d->Hs,
                                                                               d->Ws, 32, 32, d->N);
  LAUNCH_CHECK(c);
  return FG_OK;
}
// queries [Q][D] (host or device); candidates either fp32 [N][D] (host or device) or the dataset cache.
// idx_out / dist_out: host or device, Q entries each.
int nearest_run(fg_ctx* c, const float* cands, const fg_dataset* d, int64_t N, int D, const float* queries, int Q,
                int32_t* idx_out, float* dist_out) {
  FG_REQUIRE(queries && idx_out && dist_out && Q >= 1 && N >= 1 && D >= 1 && D <= 3072 && N < ((int64_t)1 << 32),
             "nearest: need 1 <= D <= 3072 (3x32x32), Q >= 1, 1 <= N < 2^32");
  float *q_dev = nullptr, *c_dev = nullptr, *dist_dev = nullptr;
  int32_t* idx_dev = nullptr;
  unsigned long long* best = nullptr;
  int rc = FG_OK;
  auto fail = [&](cudaError_t e, const char* what) {
    if (e != cudaSuccess && rc == FG_OK) {
      fg_set_error("nearest: %s -> %s", what, cudaGetErrorString(e));
      rc = FG_ERR_CUDA;
    }
    return e != cudaSuccess;
  };
  do {
    const float* qd = queries;
    if (!is_dev(queries)) {
      if (fail(cudaMalloc((void**)&q_dev, sizeof(float) * (size_t)Q * D), "cudaMalloc")) break;
      if (fail(cudaMemcpyAsync(q_dev, queries, sizeof(float) * (size_t)Q * D, cudaMemcpyHostToDevice, c->stream), "H2D")) break;
      qd = q_dev;
    }
    const float* cd = cands;
    if (cands && !is_dev(cands)) {
      if (fail(cudaMalloc((void**)&c_dev, sizeof(float) * (size_t)N * D), "cudaMalloc")) break;
      if (fail(cudaMemcpyAsync(c_dev, cands, sizeof(float) * (size_t)N * D, cudaMemcpyHostToDevice, c->stream), "H2D")) break;
      cd = c_dev;
    }
    if (fail(cudaMalloc((void**)&best, sizeof(unsigned long long) * Q), "cudaMalloc")) break;
    if (fail(cudaMalloc((void**)&idx_dev, sizeof(int32_t) * Q), "cudaMalloc")) break;
    if (fail(cudaMalloc((void**)&dist_dev, sizeof(float) * Q), "cudaMalloc")) break;
    if (fail(cudaMemsetAsync(best, 0xff, sizeof(unsigned long long) * Q, c->stream), "memset")) break;
    const int warps = 8;
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((N + warps - 1) / warps, (int64_t)c->sm_count * 4));
    const size_t smem = sizeof(float) * kQG * D;
    if (d)
      nearest_kernel<true><<<grid, 32 * warps, smem, c->stream>>>(nullptr, d->data, N, D, c->C, d->Cs, d->Hs, d->Ws, qd, Q, best);
    else
      nearest_kernel<false><<<grid, 32 * warps, smem, c->stream>>>(cd, nullptr, N, D, 0, 0, 0, 0, qd, Q, best);
    c->launches++;
    if (fail(cudaGetLastError(), "nearest_kernel")) break;
    nearest_unpack_kernel<<<(Q + 127) / 128, 128, 0, c->stream>>>(best, Q, idx_dev, dist_dev);
    c->launches++;
    if (fail(cudaMemcpyAsync(idx_out, idx_dev, sizeof(int32_t) * Q, cudaMemcpyDefault, c->stream), "copy")) break;
    if (fail(cudaMemcpyAsync(dist_out, dist_dev, sizeof(float) * Q, cudaMemcpyDefault, c->stream), "copy")) break;
    fail(cudaStreamSynchronize(c->stream), "sync");
  } while (0);
  cudaFree(q_dev);
  cudaFree(c_dev);
  cudaFree(best);
  cudaFree(idx_dev);
  cudaFree(dist_dev);
  return rc;
}
}  // namespace

#define ENTER(d)                                      \
  do {                                                   \
    if (!(d) || !(d)->c) {                               \
      fg_set_error("null fg_dataset");                   \
      return FG_ERR_INVALID;                             \
    }                                                    \
    FG_CUDA(cudaSetDevice((d)->c->device));              \
  } while (0)

extern "C" {

int fg_dataset_create(fg_ctx* ctx, int64_t N, int Cs, int Hs, int Ws, fg_dataset** out) {
  if (!ctx || !out) {
    fg_set_error("fg_dataset_create: null argument");
    return FG_ERR_INVALID;
  }
  *out = nullptr;
  FG_REQUIRE(N >= 1 && (Cs == 1 || Cs == 3) && Hs >= 1 && Ws >= 1 && Hs <= 4096 && Ws <= 4096,
             "fg_dataset_create: need N >= 1, 1 or 3 channels, sizes in [1,4096]");
  FG_REQUIRE(!(Cs == 1 && ctx->C == 3), "fg_dataset_create: a grayscale cache cannot feed a colour context");
  FG_CUDA(cudaSetDevice(ctx->device));
  fg_dataset* d = new fg_dataset();
  d->c = ctx;
  d->N = N;
  d->Cs = Cs;
  d->Hs = Hs;
  d->Ws = Ws;
  if (cudaMalloc((void**)&d->data, (size_t)N * Cs * Hs * Ws) != cudaSuccess ||
      cudaMalloc((void**)&d->idx, sizeof(int32_t) * (size_t)ctx->maxB) != cudaSuccess) {
    fg_set_error("fg_dataset_create: cudaMalloc of %lld images failed", (long long)N);
    cudaGetLastError();
    if (d->data) cudaFree(d->data);
    delete d;
    return FG_ERR_CUDA;
  }
  *out = d;
  return FG_OK;
}
int fg_dataset_destroy(fg_dataset* d) {
  if (!d) return FG_OK;
  if (d->c) {
    cudaSetDevice(d->c->device);
    cudaStreamSynchronize(d->c->stream);
  }
  cudaFree(d->data);
  cudaFree(d->idx);
  delete d;
  return FG_OK;
}
int64_t fg_dataset_size(fg_dataset* d) { return d ? d->N : 0; }

int fg_dataset_upload(fg_dataset* d, int64_t first, int64_t count, const uint8_t* images) {
  ENTER(d);
  FG_REQUIRE(images && first >= 0 && count >= 1 && first + count <= d->N, "fg_dataset_upload: range [%lld, %lld) outside [0, %lld)",
             (long long)first, (long long)(first + count), (long long)d->N);
  const size_t per = (size_t)d->Cs * d->Hs * d->Ws;
  FG_CUDA(cudaMemcpyAsync(d->data + (size_t)first * per, images, (size_t)count * per, cudaMemcpyDefault, d->c->stream));
  FG_CUDA(cudaStreamSynchronize(d->c->stream));  // the caller may reuse its (pageable) buffer
  return FG_OK;
}
// out [B][C][32][32] fp32 (host or device) = scale(load(image idx[b]));  idx: B int32 (host or device), 0-based
int fg_dataset_gather(fg_dataset* d, const int32_t* idx, int B, float* out) {
  ENTER(d);
  fg_ctx* c = d->c;
  FG_REQUIRE(idx && out && B >= 1 && B <= c->maxB, "fg_dataset_gather: bad arguments (B %d, max %d)", B, c->maxB);
  const int32_t* idx_dev = idx;
  if (!is_dev(idx)) {
    for (int i = 0; i < B; ++i)
      FG_REQUIRE(idx[i] >= 0 && idx[i] < d->N, "fg_dataset_gather: index %d out of range [0, %lld)", idx[i], (long long)d->N);
    FG_CUDA(cudaMemcpyAsync(d->idx, idx, sizeof(int32_t) * B, cudaMemcpyHostToDevice, c->stream));
    idx_dev = d->idx;
  }
  const size_t n = (size_t)B * c->C * 1024;
  if (is_dev(out)) return gather(d, idx_dev, B, out);
  FG_TRY(gather(d, idx_dev, B, c->io_dev));
  FG_CUDA(cudaMemcpyAsync(out, c->io_dev, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}
// the index stream fg_train_step_dataset uses: B draws of math.random(N)-1, counter-based (splitmix64)
int fg_dataset_draw(fg_dataset* d, uint64_t seed, int B, int32_t* idx_out) {
  ENTER(d);
  fg_ctx* c = d->c;
  FG_REQUIRE(idx_out && B >= 1 && B <= c->maxB, "fg_dataset_draw: bad arguments");
  int32_t* dst = is_dev(idx_out) ? idx_out : d->idx;
  draw_indices_kernel<<<(B + 127) / 128, 128, 0, c->stream>>>(dst, B, seed, d->N);
  LAUNCH_CHECK(c);
  if (dst != idx_out) {
    FG_CUDA(cudaMemcpyAsync(idx_out, dst, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, c->stream));
    FG_CUDA(cudaStreamSynchronize(c->stream));
  }
  return FG_OK;
}
// NN_UTILS.createNoiseInputs on the device: n floats ~ U[-1, 1) from a counter-based generator
int fg_noise_uniform(fg_ctx* c, uint64_t seed, int64_t n, float* out) {
  if (!c) {
    fg_set_error("null fg_ctx");
    return FG_ERR_INVALID;
  }
  FG_CUDA(cudaSetDevice(c->device));
  FG_REQUIRE(out && n >= 1, "fg_noise_uniform: bad arguments");
  if (is_dev(out)) {
    uniform_pm1_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(out, n, seed);
    LAUNCH_CHECK(c);
    return FG_OK;
  }
  float* tmp = nullptr;
  FG_CUDA(cudaMalloc((void**)&tmp, sizeof(float) * (size_t)n));
  uniform_pm1_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(tmp, n, seed);
  c->launches++;
  cudaError_t e = cudaMemcpyAsync(out, tmp, sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost, c->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
  cudaFree(tmp);
  if (e != cudaSuccess) {
    fg_set_error("fg_noise_uniform: %s", cudaGetErrorString(e));
    return FG_ERR_CUDA;
  }
  return FG_OK;
}
// ---- scoring helpers of sample.lua / adversarial_c2f.lua (SURVEY.md 8(f).3) ------------------------------------
// NN_UTILS.sortImagesByPrediction's device part (utils/nn_utils.lua:90-98): D's prediction for N images in chunks
// of `chunk` (OPT.batchSize).  sample.lua never calls evaluate(), so training = 1 reproduces its live dropout
// (masks drawn from seed + chunk start); training = 0 is the deterministic evaluate() score.
int fg_D_score(fg_ctx* c, const float* images, int64_t N, int chunk, int training, uint64_t seed, float* preds_out) {
  if (!c) {
    fg_set_error("null fg_ctx");
    return FG_ERR_INVALID;
  }
  FG_REQUIRE(images && preds_out && N >= 1 && chunk >= 1 && chunk <= c->maxB, "fg_D_score: bad arguments (chunk %d, max %d)", chunk,
             c->maxB);
  const size_t img = (size_t)c->C * 1024;
  for (int64_t s = 0; s < N; s += chunk) {
    const int b = (int)std::min<int64_t>(chunk, N - s);
    FG_TRY(fg_D_forward(c, images + (size_t)s * img, b, training, nullptr, seed + (uint64_t)s, preds_out + s));
  }
  return FG_OK;
}
// for each of Q queries [Q][D] the candidate [N][D] with the smallest torch.dist (2-norm) and that distance
int fg_nearest(fg_ctx* c, const float* queries, int Q, const float* cands, int64_t N, int D, int32_t* idx_out, float* dist_out) {
  if (!c) {
    fg_set_error("null fg_ctx");
    return FG_ERR_INVALID;
  }
  FG_CUDA(cudaSetDevice(c->device));
  FG_REQUIRE(cands, "fg_nearest: null candidates");
  return nearest_run(c, cands, nullptr, N, D, queries, Q, idx_out, dist_out);
}
// sample.lua:141-159 findClosestNeighboursOf against the device-resident training set (32x32 view of every image)
int fg_dataset_nearest(fg_dataset* d, const float* queries, int Q, int32_t* idx_out, float* dist_out) {
  ENTER(d);
  return nearest_run(d->c, nullptr, d, d->N, d->c->C * 1024, queries, Q, idx_out, dist_out);
}

// One adversarial.lua loop body fed entirely on the device: real half-batch = gather(draw(4*seed)), noise for the
// D step = uniform(4*seed+1), for the G step = uniform(4*seed+2), dropout masks from `seed` as in fg_train_step.
int fg_train_step_dataset(fg_ctx* c, fg_dataset* d, const fg_hyper* h, int B, uint64_t seed, fg_step_stats* stats) {
  ENTER(d);
  FG_REQUIRE(c == d->c, "fg_train_step_dataset: the dataset belongs to another context");
  FG_REQUIRE(h && B >= 4 && B % 2 == 0 && B <= c->maxB, "fg_train_step_dataset: batch %d must be even, >= 4 and <= max_batch %d", B,
             c->maxB);
  const int Bh = B / 2;
  draw_indices_kernel<<<(Bh + 127) / 128, 128, 0, c->stream>>>(d->idx, Bh, seed * 4, d->N);
  LAUNCH_CHECK(c);
  FG_TRY(gather(d, d->idx, Bh, c->in_real));
  uniform_pm1_kernel<<<grid_for((int64_t)Bh * kNoiseDim, 256), 256, 0, c->stream>>>(c->in_noiseD, (int64_t)Bh * kNoiseDim, seed * 4 + 1);
  LAUNCH_CHECK(c);
  uniform_pm1_kernel<<<grid_for((int64_t)B * kNoiseDim, 256), 256, 0, c->stream>>>(c->in_noiseG, (int64_t)B * kNoiseDim, seed * 4 + 2);
  LAUNCH_CHECK(c);
  FG_TRY(net_train_step(c, h, B, c->in_real, c->in_noiseD, c->in_noiseG, nullptr, nullptr, seed));
  if (stats) {
    FG_CUDA(cudaStreamSynchronize(c->stream));
    const DeviceStats& s = *c->hstats;
    stats->loss_D = s.loss_D;
    stats->loss_G = s.loss_G;
    for (int i = 0; i < 4; ++i) stats->conf[i] = s.conf[i];
    stats->trained_D = s.trained_D;
    stats->t_D = s.t_D;
    stats->t_G = s.t_G;
    stats->acc_D = s.acc_D;
  }
  return FG_OK;
}

}  // extern "C"
