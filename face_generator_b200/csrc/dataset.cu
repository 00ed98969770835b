// Device-resident dataset + on-GPU batch assembly (SURVEY.md 8(f).2).
//
// Replaces, for the train step's input side:
//   dataset.lua:80-117  loadRandomImages: image.load(path, nbChannels, "float") then image.scale(img, 32, 32)
//   adversarial.lua:244-249 / :276  the per-sample Lua loop that copies math.random(dataset:size()) images into
//                       `inputs`, and NN_UTILS.createNoiseInputs (utils/nn_utils.lua:35-39: uniform(-1,1))
// Decoding happens once, at load time (JPEG files on the GPU too, jpeg.cu); what is kept on the GPU is the DECODED uint8 image
// at its original scale (dataset.originalScale = 64, dataset.lua:10), 4x smaller than the float tensors the
// reference keeps.  fg_dataset_gather turns B indices into the normalised, down-scaled fp32 NCHW batch in one
// kernel; fg_train_step_dataset draws the indices and both noise tensors on the device too, so a train step
// needs no host->device traffic at all.
//
// image.scale(src, w, h) is scale_pixel of k_scale.cuh.  image.load(..., "float") is byte/255; nbChannels = 1 on a
// colour file is image.rgb2y: 0.299 R + 0.587 G + 0.114 B.  The oracle restates the same in numpy
// (oracle/oracle_data.py).  PARITY UNPINNED (no `image` rock here).
#include <algorithm>

#include "fg_internal.h"
#include "k_rng.cuh"
#include "k_scale.cuh"

namespace {
// image.load(..., "float") of channel ch of one cached image: byte/255, image.rgb2y when gray
struct U8Src {
  const uint8_t* base;
  int ch, Hs, Ws;
  bool gray;
  __device__ __forceinline__ float operator()(int yy, int xx) const {
    if (gray) {
      const float rr = base[(0 * Hs + yy) * Ws + xx] * (1.f / 255.f), gg = base[(1 * Hs + yy) * Ws + xx] * (1.f / 255.f),
                  bb = base[(2 * Hs + yy) * Ws + xx] * (1.f / 255.f);
      return 0.299f * rr + 0.587f * gg + 0.114f * bb;
    }
    return base[((int64_t)ch * Hs + yy) * Ws + xx] * (1.f / 255.f);
  }
};
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
    const U8Src src{data + img * (int64_t)Cs * Hs * Ws, ch, Hs, Ws, Cs == 3 && C == 1};
    out[i] = scale_pixel(src, y, x, Hs, Ws, Ho, Wo);
  }
}
// dataset_c2f.lua:49-62 _toResult at fineSize S, one cached image per CTA:
//   fine   = the S x S gather of the image (the per-pixel code of gather_kernel, so bit-identical to it), kept in
//            shared memory as fp32 (the reference holds it in a FloatTensor before scaling it again)
//   tmp    = image.scale(fine, cs, cs)            (shared memory)
//   coarse = image.scale(tmp, S, S)
//   diff   = fine - coarse                        (torch.add(fine, -1, coarse))
// Outputs are NCHW [B][C][S][S]; any may be null.  Per image: Cs*Hs*Ws bytes read, up to 3 * C * S*S * 4 bytes
// written.  Dynamic shared memory: C*S*S floats of fine, then C*cs*cs of tmp (c2f_pairs_smem; 96 KB at S = cs = 64).
constexpr int kPairThreads = 256;
size_t c2f_pairs_smem(int C, int S, int cs) { return sizeof(float) * ((size_t)C * S * S + (size_t)C * cs * cs); }
__global__ void __launch_bounds__(kPairThreads) c2f_pairs_kernel(const uint8_t* __restrict__ data, const int32_t* __restrict__ idx,
                                                                 float* __restrict__ fine, float* __restrict__ coarse,
                                                                 float* __restrict__ diff, int C, int Cs, int Hs, int Ws, int S,
                                                                 int cs, int64_t N) {
  extern __shared__ float pair_smem[];
  const int b = blockIdx.x, SS = S * S, n = C * SS, m = cs * cs;
  float* sfine = pair_smem;
  float* stmp = pair_smem + n;
  int64_t img = idx[b];
  img = img < 0 ? 0 : (img >= N ? N - 1 : img);
  const uint8_t* base = data + img * (int64_t)Cs * Hs * Ws;
  const bool gray = Cs == 3 && C == 1;
  const int64_t o = (int64_t)b * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int ch = i / SS, r = i - ch * SS, y = r / S, x = r - y * S;
    const float v = scale_pixel(U8Src{base, ch, Hs, Ws, gray}, y, x, Hs, Ws, S, S);
    sfine[i] = v;
    if (fine) fine[o + i] = v;
  }
  if (!coarse && !diff) return;
  __syncthreads();
  for (int i = threadIdx.x; i < C * m; i += blockDim.x) {
    const int ch = i / m, r = i - ch * m, y = r / cs, x = r - y * cs;
    stmp[i] = scale_pixel(PlaneSrc{sfine + ch * SS, S}, y, x, S, S, cs, cs);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int ch = i / SS, r = i - ch * SS, y = r / S, x = r - y * S;
    const float v = scale_pixel(PlaneSrc{stmp + ch * m, cs}, y, x, cs, cs, S, S);
    if (coarse) coarse[o + i] = v;
    if (diff) diff[o + i] = sfine[i] - v;
  }
}
// fg_image_scale: dst [NC][Ho][Wo] = image.scale of each plane of src [NC][Hs][Ws], one output pixel per thread
__global__ void image_scale_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t NC, int Hs, int Ws, int Ho,
                                   int Wo) {
  const int64_t n = NC * Ho * Wo;
  GRID_STRIDE(i, n) {
    const int x = (int)(i % Wo);
    const int64_t r = i / Wo;
    const int y = (int)(r % Ho);
    const int64_t plane = r / Ho;
    dst[i] = scale_pixel(PlaneSrc{src + plane * Hs * Ws, Ws}, y, x, Hs, Ws, Ho, Wo);
  }
}
// root (optional): the stream is *root * kinds + seed, read on the device (the per-iteration stream roots of a captured
// multi-iteration step, k_seed_roots)
__global__ void draw_indices_kernel(int32_t* __restrict__ idx, int B, uint64_t seed, int64_t N, const uint64_t* root = nullptr,
                                    uint64_t kinds = 0) {
  if (root) seed += *root * kinds;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) idx[i] = (int32_t)(splitmix64(seed * 0x100000001B3ull + (uint64_t)i) % (uint64_t)N);
}
__global__ void uniform_pm1_kernel(float* __restrict__ out, int64_t n, uint64_t seed, const uint64_t* root = nullptr,
                                   uint64_t kinds = 0) {
  if (root) seed += *root * kinds;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    out[i] = uniform_pm1_at(seed, (uint64_t)i);
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
                                                      int D, int C, int Cs, int Hs, int Ws, int S, const float* __restrict__ queries,
                                                      int Q, unsigned long long* __restrict__ best) {
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
        } else {  // the S x S view of the cached image, same arithmetic as gather_kernel
          const int x = i % S, y = (i / S) % S, ch = i / (S * S);
          const Span sy = axis_span(y, Hs, S), sx = axis_span(x, Ws, S);
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

int gather(fg_dataset* d, const int32_t* idx_dev, int B, float* out_dev, int size = 32) {
  fg_ctx* c = d->c;
  gather_kernel<<<grid_for((int64_t)B * c->C * size * size, 256), 256, 0, c->stream>>>(d->data, idx_dev, out_dev, B, c->C, d->Cs,
                                                                                       d->Hs, d->Ws, size, size, d->N);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int gather_c2f(fg_dataset* d, const int32_t* idx_dev, int B, int S, int cs, float* fine, float* coarse, float* diff) {
  fg_ctx* c = d->c;
  const size_t smem = c2f_pairs_smem(c->C, S, cs);
  if (smem > 48 * 1024) FG_CUDA(cudaFuncSetAttribute(c2f_pairs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  c2f_pairs_kernel<<<B, kPairThreads, smem, c->stream>>>(d->data, idx_dev, fine, coarse, diff, c->C, d->Cs, d->Hs, d->Ws, S, cs, d->N);
  LAUNCH_CHECK(c);
  return FG_OK;
}
// a host index list is range-checked and staged in d->idx; a device one is used as is (the kernels clamp it)
int stage_indices(fg_dataset* d, const int32_t* idx, int B, const char* what, const int32_t** idx_dev) {
  *idx_dev = idx;
  if (fg_is_dev(idx)) return FG_OK;
  for (int i = 0; i < B; ++i)
    FG_REQUIRE(idx[i] >= 0 && idx[i] < d->N, "%s: index %d out of range [0, %lld)", what, idx[i], (long long)d->N);
  FG_CUDA(cudaMemcpyAsync(d->idx, idx, sizeof(int32_t) * B, cudaMemcpyHostToDevice, d->c->stream));
  *idx_dev = d->idx;
  return FG_OK;
}
// queries [Q][D] (host or device); candidates either fp32 [N][D] (host or device) or the dataset cache at S x S
// (D = C*S*S).  idx_out / dist_out: host or device, Q entries each.
int nearest_run(fg_ctx* c, const float* cands, const fg_dataset* d, int S, int64_t N, int D, const float* queries, int Q,
                int32_t* idx_out, float* dist_out) {
  FG_REQUIRE(queries && idx_out && dist_out && Q >= 1 && N >= 1 && D >= 1 && D <= 12288 && N < ((int64_t)1 << 32),
             "nearest: need 1 <= D <= 12288 (3x64x64), Q >= 1, 1 <= N < 2^32");
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
    if (!fg_is_dev(queries)) {
      if (fail(cudaMalloc((void**)&q_dev, sizeof(float) * (size_t)Q * D), "cudaMalloc")) break;
      if (fail(cudaMemcpyAsync(q_dev, queries, sizeof(float) * (size_t)Q * D, cudaMemcpyHostToDevice, c->stream), "H2D")) break;
      qd = q_dev;
    }
    const float* cd = cands;
    if (cands && !fg_is_dev(cands)) {
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
    if (smem > 48 * 1024) {  // above 3x32x32: opt in to the larger dynamic shared memory
      auto fn = d ? nearest_kernel<true> : nearest_kernel<false>;
      if (fail(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute")) break;
    }
    if (d)
      nearest_kernel<true><<<grid, 32 * warps, smem, c->stream>>>(nullptr, d->data, N, D, c->C, d->Cs, d->Hs, d->Ws, S, qd, Q, best);
    else
      nearest_kernel<false><<<grid, 32 * warps, smem, c->stream>>>(cd, nullptr, N, D, 0, 0, 0, 0, 0, qd, Q, best);
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
    // the device-fed multi-iteration steps capture the draws and gathers, i.e. d->data, d->idx and d->N, into the
    // step graphs of this ctx (32x32, --scale 16 and c2f alike): none of them may be replayed once these are freed,
    // even if a later dataset is allocated at the same host address
    d->c->graph_epoch++;
  }
  jpeg_scratch_free(d->jpeg);
  jpeg_enc_scratch_free(d->jpeg_enc);
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
int fg_dataset_gather(fg_dataset* d, const int32_t* idx, int B, float* out) { return fg_dataset_gather_sized(d, idx, B, 32, out); }
// the same at any square size in [1, 32] (dataset.lua setScale(size)); out [B][C][size][size]
int fg_dataset_gather_sized(fg_dataset* d, const int32_t* idx, int B, int size, float* out) {
  ENTER(d);
  fg_ctx* c = d->c;
  FG_REQUIRE(idx && out && B >= 1 && B <= c->maxB, "fg_dataset_gather: bad arguments (B %d, max %d)", B, c->maxB);
  FG_REQUIRE(size >= 1 && size <= 32, "fg_dataset_gather_sized: size %d outside [1, 32]", size);
  const int32_t* idx_dev;
  FG_TRY(stage_indices(d, idx, B, "fg_dataset_gather", &idx_dev));
  const size_t n = (size_t)B * c->C * size * size;
  if (fg_is_dev(out)) return gather(d, idx_dev, B, out, size);
  FG_TRY(gather(d, idx_dev, B, c->io_dev, size));
  FG_CUDA(cudaMemcpyAsync(out, c->io_dev, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}
// dataset_c2f.lua:49-62 _toResult at fineSize 32 (fg_dataset_gather_c2f_sized at 32)
int fg_dataset_gather_c2f(fg_dataset* d, const int32_t* idx, int B, int coarse_size, float* fine, float* coarse, float* diff) {
  return fg_dataset_gather_c2f_sized(d, idx, B, 32, coarse_size, fine, coarse, diff);
}
// _toResult at fineSize S in {16, 32, 64} for B images: fine, coarse, diff [B][C][S][S] fp32, each host or device or
// NULL.  Host outputs go through one temporary device buffer (this entry is not on a train step's path).
int fg_dataset_gather_c2f_sized(fg_dataset* d, const int32_t* idx, int B, int fine_size, int coarse_size, float* fine,
                                float* coarse, float* diff) {
  ENTER(d);
  fg_ctx* c = d->c;
  FG_REQUIRE(idx && B >= 1 && B <= c->maxB, "fg_dataset_gather_c2f: bad arguments (B %d, max %d)", B, c->maxB);
  if (!(fine_size == 16 || fine_size == 32 || fine_size == 64)) {
    fg_set_error("fg_dataset_gather_c2f_sized: fine size %d is not supported (16, 32 or 64)", fine_size);
    return FG_ERR_UNSUPPORTED;
  }
  FG_REQUIRE(coarse_size >= 1 && coarse_size <= fine_size, "fg_dataset_gather_c2f: coarse size %d outside [1, %d]", coarse_size,
             fine_size);
  const int32_t* idx_dev;
  FG_TRY(stage_indices(d, idx, B, "fg_dataset_gather_c2f", &idx_dev));
  const size_t n = (size_t)B * c->C * fine_size * fine_size;
  float* user[3] = {fine, coarse, diff};
  float* dev[3] = {fine, coarse, diff};
  int n_host = 0;
  for (int k = 0; k < 3; ++k) n_host += user[k] && !fg_is_dev(user[k]);
  if (n_host == 0) return gather_c2f(d, idx_dev, B, fine_size, coarse_size, fine, coarse, diff);
  float* tmp = nullptr;
  FG_CUDA(cudaMalloc((void**)&tmp, sizeof(float) * n * n_host));
  for (int k = 0, j = 0; k < 3; ++k)
    if (user[k] && !fg_is_dev(user[k])) dev[k] = tmp + n * j++;
  int rc = gather_c2f(d, idx_dev, B, fine_size, coarse_size, dev[0], dev[1], dev[2]);
  cudaError_t e = cudaSuccess;
  for (int k = 0; k < 3 && rc == FG_OK && e == cudaSuccess; ++k)
    if (dev[k] != user[k]) e = cudaMemcpyAsync(user[k], dev[k], n * sizeof(float), cudaMemcpyDeviceToHost, c->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
  cudaFree(tmp);
  if (rc == FG_OK && e != cudaSuccess) {
    fg_set_error("fg_dataset_gather_c2f: %s", cudaGetErrorString(e));
    rc = FG_ERR_CUDA;
  }
  return rc;
}
// the index stream fg_train_step_dataset uses: B draws of math.random(N)-1, counter-based (splitmix64)
int fg_dataset_draw(fg_dataset* d, uint64_t seed, int B, int32_t* idx_out) {
  ENTER(d);
  fg_ctx* c = d->c;
  FG_REQUIRE(idx_out && B >= 1 && B <= c->maxB, "fg_dataset_draw: bad arguments");
  int32_t* dst = fg_is_dev(idx_out) ? idx_out : d->idx;
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
  if (fg_is_dev(out)) {
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
// image.scale(x, Wo, Ho) on fp32 NCHW images, host or device.  Host buffers go through temporary device memory (this
// entry is not on a hot path; fg_c2f_refine scales inside its own kernel).
int fg_image_scale(fg_ctx* c, const float* src, int64_t N, int C, int Hs, int Ws, int Ho, int Wo, float* dst) {
  if (!c) {
    fg_set_error("null fg_ctx");
    return FG_ERR_INVALID;
  }
  FG_REQUIRE(src && dst && N >= 1 && C >= 1, "fg_image_scale: bad arguments");
  FG_REQUIRE(Hs >= 1 && Ws >= 1 && Ho >= 1 && Wo >= 1 && Hs <= 256 && Ws <= 256 && Ho <= 256 && Wo <= 256,
             "fg_image_scale: sizes %dx%d -> %dx%d outside [1, 256]", Hs, Ws, Ho, Wo);
  FG_CUDA(cudaSetDevice(c->device));
  const int64_t NC = N * C;
  const size_t n_src = (size_t)NC * Hs * Ws, n_dst = (size_t)NC * Ho * Wo;
  const bool src_dev = fg_is_dev(src), dst_dev = fg_is_dev(dst);
  float* tmp = nullptr;
  if (!src_dev || !dst_dev) FG_CUDA(cudaMalloc((void**)&tmp, sizeof(float) * ((src_dev ? 0 : n_src) + (dst_dev ? 0 : n_dst))));
  const float* s = src_dev ? src : tmp;
  float* d = dst_dev ? dst : tmp + (src_dev ? 0 : n_src);
  cudaError_t e = src_dev ? cudaSuccess : cudaMemcpyAsync(tmp, src, sizeof(float) * n_src, cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess) {
    image_scale_kernel<<<grid_for((int64_t)n_dst, 256), 256, 0, c->stream>>>(s, d, NC, Hs, Ws, Ho, Wo);
    c->launches++;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess && !dst_dev) e = cudaMemcpyAsync(dst, d, sizeof(float) * n_dst, cudaMemcpyDeviceToHost, c->stream);
  if (e == cudaSuccess && tmp) e = cudaStreamSynchronize(c->stream);
  cudaFree(tmp);
  if (e != cudaSuccess) {
    fg_set_error("fg_image_scale: %s", cudaGetErrorString(e));
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
  return nearest_run(c, cands, nullptr, 0, N, D, queries, Q, idx_out, dist_out);
}
// sample.lua:141-159 findClosestNeighboursOf against the device-resident training set (32x32 view of every image)
int fg_dataset_nearest(fg_dataset* d, const float* queries, int Q, int32_t* idx_out, float* dist_out) {
  return fg_dataset_nearest_sized(d, 32, queries, Q, idx_out, dist_out);
}
// the same against the size x size view of every image (DATASET.setScale(OPT.scale), then loadImages): queries
// [Q][C][size][size]
int fg_dataset_nearest_sized(fg_dataset* d, int size, const float* queries, int Q, int32_t* idx_out, float* dist_out) {
  ENTER(d);
  FG_REQUIRE(size >= 1 && size <= 64, "fg_dataset_nearest_sized: size %d outside [1, 64]", size);
  return nearest_run(d->c, nullptr, d, size, d->N, d->c->C * size * size, queries, Q, idx_out, dist_out);
}

}  // extern "C"

// ---- batch assembly of the device-fed --scale 16 and coarse-to-fine steps (nets_s16.cu, nets_c2f.cu) ----------
// Eager launches on the ctx stream into device buffers: no allocation, no host synchronisation.
int dataset_check_feed(const fg_dataset* d, const fg_ctx* c, const char* what) {
  FG_REQUIRE(d && d->c == c, "%s: the dataset belongs to another context", what);
  FG_REQUIRE(!(d->Cs == 1 && c->C == 3), "%s: a grayscale cache cannot feed a colour context", what);
  return FG_OK;
}
int dataset_draw_gather(fg_dataset* d, uint64_t seed, int B, int size, float* out_dev, const uint64_t* root, uint64_t kinds) {
  fg_ctx* c = d->c;
  draw_indices_kernel<<<(B + 127) / 128, 128, 0, c->stream>>>(d->idx, B, seed, d->N, root, kinds);
  LAUNCH_CHECK(c);
  return gather(d, d->idx, B, out_dev, size);
}
int dataset_draw_gather_c2f(fg_dataset* d, uint64_t seed, int B, int fine_size, int coarse_size, float* fine, float* coarse,
                            float* diff, const uint64_t* root, uint64_t kinds) {
  fg_ctx* c = d->c;
  draw_indices_kernel<<<(B + 127) / 128, 128, 0, c->stream>>>(d->idx, B, seed, d->N, root, kinds);
  LAUNCH_CHECK(c);
  return gather_c2f(d, d->idx, B, fine_size, coarse_size, fine, coarse, diff);
}
int noise_uniform_dev(fg_ctx* c, uint64_t seed, int64_t n, float* out_dev, const uint64_t* root, uint64_t kinds) {
  uniform_pm1_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(out_dev, n, seed, root, kinds);
  LAUNCH_CHECK(c);
  return FG_OK;
}
