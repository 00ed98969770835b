// The denoising autoencoders of train_denoiser.lua and the batch step that trains them:
//   AE  = Sequential(ENCODER, DECODER), ENCODER = nn.WhiteNoise(0, noise_std) (dpnn)           train_denoiser.lua:83-113
//   DECODER = conv(C->8,3, no pad) SpatialBN(8) LeakyReLU(0.333) | conv(8->8,3, no pad) SpatialBN(8) LeakyReLU Dropout(p)
//             View(8(S-4)^2) Linear(8(S-4)^2, 2048) BatchNormalization(2048) LeakyReLU Dropout(p)
//             Linear(2048, C S S) Sigmoid View(C,S,S)
//   AE2 = DECODER:clone(), fed with AE's output (:117)
//   step = fevalAE + optim.adam, then fevalAE2 + optim.adam, both on ONE Adam state (OPTSTATE.adam, :335-336)
// Kernels: the valid 3x3 convolutions, the BatchNorm / LeakyReLU / Dropout layers, WhiteNoise and Sigmoid+BCE live here;
// the two Linear layers are ConvL layers on the wgmma kernels (convl.h); the optimizer is k_optim_update.
//
// LeakyReLU follows the waifu2x module the reference ships (LeakyReLU.lua): forward max(x,0) + a min(x,0), gradient
// slope 1 at x >= 0 (THNN's nn.LeakyReLU uses the negative slope at x == 0 exactly).
#include <algorithm>
#include <cmath>
#include <cstring>

#include "convl.h"
#include "fg_internal.h"
#include "k_ordered.cuh"
#include "k_stream.cuh"

namespace {
constexpr float kSlope = 0.333f;
constexpr int kHidden = 2048;
constexpr int kBnDn = 2 * (8 + 8 + kHidden);  // [rm1 8][rv1 8][rm2 8][rv2 8][rm3 2048][rv3 2048]
// random streams of a step (stream root = the step seed, *seed_dev): WhiteNoise of forward k (0: the AE step, 1: AE's
// forward inside the AE2 step) and the dropout keep flags of forward k (0, 1: AE; 2: AE2)
constexpr uint64_t kKindNoise = 0, kKindMask = 2;

// images NCHW -> x NHWC (+ WhiteNoise).  noise (NCHW, may be null) is added as given; else with seed_dev it is drawn:
// std * N(0,1) by Box-Muller on the stream (seed, kind); noise_out (may be null) receives what was added.
// t (may be null) receives the clean images in NHWC (the BCE targets).
__global__ void dn_input_kernel(const float* __restrict__ img, const float* __restrict__ noise,
                                const uint64_t* __restrict__ seed_dev, uint64_t kind, float std, float* __restrict__ noise_out,
                                float* __restrict__ x, float* __restrict__ t, int B, int C, int HW) {
  const int64_t n = (int64_t)B * C * HW;
  const uint64_t root = seed_dev ? *seed_dev : 0;
  GRID_STRIDE(i, n) {
    const int q = (int)(i % HW);
    const int64_t r = i / HW;
    const int ch = (int)(r % C);
    const int64_t b = r / C;
    const int64_t o = (b * HW + q) * C + ch;
    const float v = img[i];
    float e = 0.f;
    if (noise) {
      e = noise[i];
    } else if (seed_dev) {
      const uint64_t r1 = stream_bits(root, kind, i), r2 = mix64(r1 ^ 0xD1B54A32D192ED03ull);
      const float u1 = (float)((r1 >> 40) + 1) * (1.0f / 16777216.0f), u2 = (float)(r2 >> 40) * (1.0f / 16777216.0f);
      e = std * sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
    }
    if (noise_out) noise_out[i] = e;
    x[o] = v + e;
    if (t) t[o] = v;
  }
}
// dropout keep flags: 1 with probability 1 - p (u >= p) on the stream (seed, kind)
__global__ void dn_mask_kernel(float* __restrict__ m, int64_t n, float p, const uint64_t* __restrict__ seed_dev, uint64_t kind) {
  const uint64_t root = *seed_dev;
  GRID_STRIDE(i, n) m[i] = (float)(stream_bits(root, kind, i) >> 40) * (1.0f / 16777216.0f) >= p ? 1.f : 0.f;
}

// ---- valid (unpadded) 3x3 convolutions with 8 output channels, NHWC; W in the reference layout [8][CIN][3][3] ----
// out [B][H-2][H-2][8] = bias + conv(in [B][H][H][CIN])
template <int CIN>
__global__ void __launch_bounds__(256) vconv3_fwd_kernel(const float* __restrict__ in, const float* __restrict__ W,
                                                         const float* __restrict__ bias, float* __restrict__ out, int B, int H) {
  __shared__ float w[8 * CIN * 9];
  for (int i = threadIdx.x; i < 8 * CIN * 9; i += blockDim.x) w[i] = W[i];
  __syncthreads();
  const int Ho = H - 2;
  float bs[8];
#pragma unroll
  for (int o = 0; o < 8; ++o) bs[o] = bias[o];
  GRID_STRIDE(p, (int64_t)B * Ho * Ho) {
    const int xo = (int)(p % Ho);
    const int64_t r = p / Ho;
    const int yo = (int)(r % Ho);
    const int64_t b = r / Ho;
    float acc[8];
#pragma unroll
    for (int o = 0; o < 8; ++o) acc[o] = bs[o];
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const float* src = in + ((b * H + yo + k / 3) * H + xo + k % 3) * CIN;
#pragma unroll
      for (int c = 0; c < CIN; ++c) {
        const float v = src[c];
#pragma unroll
        for (int o = 0; o < 8; ++o) acc[o] = fmaf(v, w[(o * CIN + c) * 9 + k], acc[o]);
      }
    }
    float4* dst = reinterpret_cast<float4*>(out + p * 8);
    dst[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    dst[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
  }
}
// data gradient of the 8->8 layer: dx [B][H][H][8] from dy [B][H-2][H-2][8]
__global__ void __launch_bounds__(256) vconv3_dgrad8_kernel(const float* __restrict__ dy, const float* __restrict__ W,
                                                            float* __restrict__ dx, int B, int H) {
  __shared__ float w[8 * 8 * 9];
  for (int i = threadIdx.x; i < 8 * 8 * 9; i += blockDim.x) w[i] = W[i];
  __syncthreads();
  const int Ho = H - 2;
  GRID_STRIDE(p, (int64_t)B * H * H) {
    const int x = (int)(p % H);
    const int64_t r = p / H;
    const int y = (int)(r % H);
    const int64_t b = r / H;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const int yo = y - k / 3, xo = x - k % 3;
      if (yo < 0 || yo >= Ho || xo < 0 || xo >= Ho) continue;
      const float* src = dy + ((b * Ho + yo) * Ho + xo) * 8;
#pragma unroll
      for (int o = 0; o < 8; ++o) {
        const float d = src[o];
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[c] = fmaf(d, w[(o * 8 + c) * 9 + k], acc[c]);
      }
    }
    float4* dst = reinterpret_cast<float4*>(dx + p * 8);
    dst[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    dst[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
  }
}
// weight and bias gradient: dW[o][c][k] += sum_p dy[p][o] in[p + off(k)][c], db[o] += sum_p dy[p][o].  Each block sums a
// contiguous range of output pixels (tiles of 32 staged in shared memory, fp32 per tile, fp64 across tiles) into one
// row of partials; the last block adds the rows in block order (k_ordered.cuh).
template <int CIN>
__global__ void __launch_bounds__(256) vconv3_wgrad_kernel(const float* __restrict__ in, const float* __restrict__ dy, int B, int H,
                                                           int64_t ppb, double* __restrict__ ws, unsigned* __restrict__ ticket,
                                                           float* __restrict__ dW, float* __restrict__ db) {
  constexpr int NW = 8 * CIN * 9, NT = NW + 8, TP = 32, KC = 9 * CIN;
  static_assert(NT <= 3 * 256, "three outputs per thread");
  __shared__ float sdy[TP][8];
  __shared__ float sx[TP][KC];
  const int Ho = H - 2;
  const int64_t P = (int64_t)B * Ho * Ho;
  const int64_t p0 = blockIdx.x * ppb, p1 = min(P, p0 + ppb);
  double acc[3] = {0, 0, 0};
  for (int64_t t0 = p0; t0 < p1; t0 += TP) {
    const int np = (int)min((int64_t)TP, p1 - t0);
    for (int i = threadIdx.x; i < TP * 8; i += blockDim.x) {
      const int pp = i / 8;
      sdy[pp][i % 8] = pp < np ? dy[(t0 + pp) * 8 + i % 8] : 0.f;
    }
    for (int i = threadIdx.x; i < TP * KC; i += blockDim.x) {
      const int pp = i / KC, e = i % KC, k = e / CIN, c = e % CIN;
      float v = 0.f;
      if (pp < np) {
        const int64_t p = t0 + pp;
        const int xo = (int)(p % Ho);
        const int64_t r = p / Ho;
        const int yo = (int)(r % Ho);
        const int64_t b = r / Ho;
        v = in[((b * H + yo + k / 3) * H + xo + k % 3) * CIN + c];
      }
      sx[pp][e] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 3; ++kk) {
      const int j = threadIdx.x + 256 * kk;
      if (j >= NT) continue;
      float s = 0.f;
      if (j < NW) {
        const int o = j / KC, c = (j % KC) / 9, k = j % 9;
        for (int pp = 0; pp < TP; ++pp) s = fmaf(sdy[pp][o], sx[pp][k * CIN + c], s);
      } else {
        for (int pp = 0; pp < TP; ++pp) s += sdy[pp][j - NW];
      }
      acc[kk] += s;
    }
    __syncthreads();
  }
#pragma unroll
  for (int kk = 0; kk < 3; ++kk) {
    const int j = threadIdx.x + 256 * kk;
    if (j < NT) ws[(int64_t)blockIdx.x * NT + j] = acc[kk];
  }
  if (ordered_last_block(ticket)) {
    for (int j = threadIdx.x; j < NT; j += blockDim.x) {
      const float v = (float)ordered_sum(ws, gridDim.x, NT, j);
      if (j < NW) dW[j] += v;
      else db[j - NW] += v;
    }
    ordered_release(ticket);
  }
}

// ---- BatchNorm (spatial at C = 8 over B*HW rows, 1-D at C = 2048 over B rows) + LeakyReLU + Dropout ----
// Rows r = b*HW + q of z [P][C]; the dropout keep flag of (r, ch) is masks[b*mps + moff + ch*HW + q] (the reference's
// NCHW flattening).  The two reductions run on a (column groups x row chunks) grid: each block sums its columns over
// its rows in fp64 with a fixed lane order and writes one row of partials; the last block adds them in chunk order.
__device__ __forceinline__ int bn_cols(int C) { return C < 32 ? C : 32; }

// acc[0..C) = sum z, acc[C..2C) = sum z^2
__global__ void __launch_bounds__(256) dn_bn_stats_kernel(const float* __restrict__ z, int64_t P, int C, int64_t rpc,
                                                          double* __restrict__ ws, unsigned* __restrict__ ticket,
                                                          double* __restrict__ acc) {
  __shared__ double sm[2][256];
  const int cols = bn_cols(C), lanes = blockDim.x / cols;
  const int cl = threadIdx.x % cols, lane = threadIdx.x / cols, ch = blockIdx.x * cols + cl;
  const int64_t r0 = blockIdx.y * rpc, r1 = min(P, r0 + rpc);
  double s = 0, q = 0;
  if (lane < lanes && ch < C)
    for (int64_t r = r0 + lane; r < r1; r += lanes) {
      const double v = z[r * C + ch];
      s += v;
      q += v * v;
    }
  sm[0][threadIdx.x] = s;
  sm[1][threadIdx.x] = q;
  __syncthreads();
  if (lane == 0 && ch < C) {
    for (int l = 1; l < lanes; ++l) {
      s += sm[0][l * cols + cl];
      q += sm[1][l * cols + cl];
    }
    ws[(int64_t)blockIdx.y * 2 * C + ch] = s;
    ws[(int64_t)blockIdx.y * 2 * C + C + ch] = q;
  }
  if (ordered_last_block(ticket)) {
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) acc[i] = ordered_sum(ws, gridDim.y, 2 * C, i);
    ordered_release(ticket);
  }
}
// h = drop(lrelu(gamma (z - mean) istd + beta))
__global__ void dn_bn_act_kernel(const float* __restrict__ z, const float* __restrict__ mean, const float* __restrict__ istd,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ masks,
                                 int mps, int moff, int HW, float scale, float* __restrict__ h, int64_t P, int C) {
  GRID_STRIDE(i, P * C) {
    const int ch = (int)(i % C);
    const int64_t r = i / C;
    const float u = gamma[ch] * ((z[i] - mean[ch]) * istd[ch]) + beta[ch];
    float o = u > 0.f ? u : kSlope * u;
    if (masks) o *= masks[(r / HW) * mps + moff + (int64_t)ch * HW + r % HW] * scale;
    h[i] = o;
  }
}
__device__ __forceinline__ float bn_act_grad(const float* __restrict__ dh, const float* __restrict__ masks, int mps, int moff,
                                             int HW, float scale, int64_t i, int64_t r, int ch, float u) {
  float d = dh[i];
  if (masks) d *= masks[(r / HW) * mps + moff + (int64_t)ch * HW + r % HW] * scale;
  return u >= 0.f ? d : kSlope * d;  // waifu2x LeakyReLU: slope 1 at u == 0
}
// acc[0..C) = sum g, acc[C..2C) = sum g xhat, g = the gradient at the BatchNorm output
__global__ void __launch_bounds__(256) dn_bn_bwd_reduce_kernel(const float* __restrict__ dh, const float* __restrict__ z,
                                                               const float* __restrict__ mean, const float* __restrict__ istd,
                                                               const float* __restrict__ gamma, const float* __restrict__ beta,
                                                               const float* __restrict__ masks, int mps, int moff, int HW,
                                                               float scale, int64_t P, int C, int64_t rpc,
                                                               double* __restrict__ ws, unsigned* __restrict__ ticket,
                                                               double* __restrict__ acc) {
  __shared__ double sm[2][256];
  const int cols = bn_cols(C), lanes = blockDim.x / cols;
  const int cl = threadIdx.x % cols, lane = threadIdx.x / cols, ch = blockIdx.x * cols + cl;
  const int64_t r0 = blockIdx.y * rpc, r1 = min(P, r0 + rpc);
  double sg = 0, sgx = 0;
  if (lane < lanes && ch < C) {
    const float m = mean[ch], is = istd[ch], ga = gamma[ch], be = beta[ch];
    for (int64_t r = r0 + lane; r < r1; r += lanes) {
      const int64_t i = r * C + ch;
      const float xh = (z[i] - m) * is;
      const float g = bn_act_grad(dh, masks, mps, moff, HW, scale, i, r, ch, ga * xh + be);
      sg += g;
      sgx += (double)g * (double)xh;
    }
  }
  sm[0][threadIdx.x] = sg;
  sm[1][threadIdx.x] = sgx;
  __syncthreads();
  if (lane == 0 && ch < C) {
    for (int l = 1; l < lanes; ++l) {
      sg += sm[0][l * cols + cl];
      sgx += sm[1][l * cols + cl];
    }
    ws[(int64_t)blockIdx.y * 2 * C + ch] = sg;
    ws[(int64_t)blockIdx.y * 2 * C + C + ch] = sgx;
  }
  if (ordered_last_block(ticket)) {
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) acc[i] = ordered_sum(ws, gridDim.y, 2 * C, i);
    ordered_release(ticket);
  }
}
// dz = gamma istd (g - mean g - xhat mean(g xhat)) in training (mg: k_bn_bwd_finalize), gamma istd g in evaluation (mg null)
__global__ void dn_bn_bwd_apply_kernel(const float* __restrict__ dh, const float* __restrict__ z, const float* __restrict__ mean,
                                       const float* __restrict__ istd, const float* __restrict__ gamma,
                                       const float* __restrict__ beta, const float* __restrict__ masks, int mps, int moff, int HW,
                                       float scale, const float* __restrict__ mg, float* __restrict__ dz, int64_t P, int C) {
  GRID_STRIDE(i, P * C) {
    const int ch = (int)(i % C);
    const int64_t r = i / C;
    const float is = istd[ch], ga = gamma[ch];
    const float xh = (z[i] - mean[ch]) * is;
    const float g = bn_act_grad(dh, masks, mps, moff, HW, scale, i, r, ch, ga * xh + beta[ch]);
    dz[i] = mg ? ga * is * (g - mg[ch] - xh * mg[C + ch]) : ga * is * g;
  }
}

// ---- nn.Sigmoid + nn.BCECriterion against image targets: y, dlogit and the mean loss in one pass ----
// the 2015 Lua BCECriterion (eps = 1e-12, size-averaged), composed with Sigmoid.backward as k_sigmoid_bce does
__global__ void __launch_bounds__(256) dn_sigmoid_bce_kernel(const float* __restrict__ z, const float* __restrict__ t,
                                                             float* __restrict__ y, float* __restrict__ dz, int64_t n,
                                                             double* __restrict__ ws, unsigned* __restrict__ ticket,
                                                             float* __restrict__ loss) {
  const float eps = 1e-12f, invN = 1.0f / (float)n;
  double s = 0;
  GRID_STRIDE(i, n) {
    const float yy = 1.0f / (1.0f + expf(-z[i])), tt = t[i];
    y[i] = yy;
    s += (double)(tt * logf(yy + eps) + (1.0f - tt) * logf(1.0f - yy + eps));
    dz[i] = -(tt - yy) / (yy * (1.0f - yy + eps) + eps) * invN * yy * (1.0f - yy);
  }
  s = block_sum256(s);
  if (threadIdx.x == 0) ws[blockIdx.x] = s;
  if (ordered_last_block(ticket)) {
    if (threadIdx.x == 0) *loss = (float)(-ordered_sum(ws, gridDim.x, 1, 0) / (double)n);
    ordered_release(ticket);
  }
}

struct DnStats {  // device; mirrored to fg_dn_stats
  float loss[2];
  int t;
  float step;  // the Adam step size of the update that follows (k_adam_prep)
};
}  // namespace

// One decoder: its layers, activations (NHWC) and BatchNorm state
struct DnDec {
  ConvL L1, L2;
  int64_t c1W = 0, c1b = 0, g1 = 0, b1 = 0, c2W = 0, c2b = 0, g2 = 0, b2 = 0, g3 = 0, b3 = 0;
  float *x = nullptr, *z1 = nullptr, *h1 = nullptr, *z2 = nullptr, *h2 = nullptr, *z3 = nullptr, *h3 = nullptr,
        *z4 = nullptr, *y = nullptr;
  float *mean[3] = {}, *istd[3] = {};
  float* bn = nullptr;  // [kBnDn] running statistics
  const float* masks = nullptr;  // keep flags of the last training forward ([B][mps]); null: evaluation
  int B = 0;
  bool train = true, valid = false;
};

struct fg_dn {
  fg_ctx* c = nullptr;
  int S = 16, C = 3, maxB = 0, mps = 0;
  int grad_B = 0;       // batch of the gradients in dz4..dz1 (the last backward; 0: none yet)
  float p_drop = 0.2f;  // Dropout probability of the forwards that follow (kept as 1/(1-p) in training)
  NetPair net;  // PG / gG: AE1's decoder, PD / gD: AE2; mG == mD and vG == vD: the one shared Adam state
  DnDec dec[2];
  DnStats* dstats = nullptr;
  DnStats* hstats = nullptr;  // pinned mirror
  float *t = nullptr, *dz4 = nullptr, *dh3 = nullptr, *dz3 = nullptr, *dh2 = nullptr, *dz2 = nullptr, *dh1 = nullptr,
        *dz1 = nullptr, *mg = nullptr;
  double* acc = nullptr;
  float *noise[2] = {}, *masks[3] = {};  // what the last forwards added / kept (drawn or copied)
  float *in_img = nullptr, *in_noise = nullptr, *in_masks = nullptr, *io = nullptr;
  std::vector<void*> allocs;
  ConvLEnv env;
};

namespace {
int dalloc(fg_dn* n, float** p, size_t elems) { return fg_dalloc(n->c, n->allocs, p, elems); }

// getParameters() order of one decoder; L1 / L2 carry their own offsets
int64_t make_dn_layout(DnDec& d, int C, int S) {
  const int A = (S - 4) * (S - 4);
  int64_t o = 0;
  d.c1W = o; o += 8 * C * 9;
  d.c1b = o; o += 8;
  d.g1 = o; o += 8;
  d.b1 = o; o += 8;
  d.c2W = o; o += 8 * 8 * 9;
  d.c2b = o; o += 8;
  d.g2 = o; o += 8;
  d.b2 = o; o += 8;
  ConvL& L1 = d.L1;
  L1.Cin = 8 * A; L1.Cout = kHidden; L1.k = 1; L1.H = 1;
  L1.cA = 8; L1.cS = A;  // View(8(S-4)^2) flattens [8][S-4][S-4]; ours is [S-4][S-4][8]
  L1.w_off = o; o += (int64_t)kHidden * 8 * A;
  L1.b_off = o; o += kHidden;
  d.g3 = o; o += kHidden;
  d.b3 = o; o += kHidden;
  ConvL& L2 = d.L2;
  L2.Cin = kHidden; L2.Cout = C * S * S; L2.k = 1; L2.H = 1;
  L2.nA = C; L2.nS = S * S;  // View(C,S,S) of the output rows; ours is [S][S][C]
  L2.w_off = o; o += (int64_t)C * S * S * kHidden;
  L2.b_off = o; o += C * S * S;
  L1.tf = "dn.L1.fwd"; L1.td = "dn.L1.dgrad"; L1.tw = "dn.L1.wgrad";
  L2.tf = "dn.L2.fwd"; L2.td = "dn.L2.dgrad"; L2.tw = "dn.L2.wgrad";
  return o;
}

int dn_alloc(fg_dn* n) {
  fg_ctx* c = n->c;
  const size_t B = n->maxB, C = n->C, S = n->S, img = C * S * S;
  const size_t A1 = (S - 2) * (S - 2), A2 = (S - 4) * (S - 4);
  n->env.c = c;
  n->env.maxB = n->maxB;
  n->env.allocs = &n->allocs;
  const int64_t np = make_dn_layout(n->dec[0], n->C, n->S);
  make_dn_layout(n->dec[1], n->C, n->S);
  NetPair& p = n->net;
  p.nG = p.nD = np;
  FG_TRY(dalloc(n, &p.PG, np));
  FG_TRY(dalloc(n, &p.PD, np));
  FG_TRY(dalloc(n, &p.gG, np + kGradTail));
  FG_TRY(dalloc(n, &p.gD, np + kGradTail));
  p.tailG = p.gG + np;
  p.tailD = p.gD + np;
  FG_TRY(dalloc(n, &p.mG, np));
  FG_TRY(dalloc(n, &p.vG, np));
  p.mD = p.mG;
  p.vD = p.vG;
  float* tmp = nullptr;
  FG_TRY(dalloc(n, &tmp, (sizeof(DnStats) + 3) / 4));
  n->dstats = (DnStats*)tmp;
  FG_CUDA(cudaMallocHost((void**)&n->hstats, sizeof(DnStats)));
  memset(n->hstats, 0, sizeof(DnStats));
  float init[kBnDn];
  for (int i = 0; i < kBnDn; ++i) init[i] = (i >= 8 && i < 16) || (i >= 24 && i < 32) || i >= 32 + kHidden ? 1.f : 0.f;
  for (DnDec& d : n->dec) {
    FG_TRY(convl_alloc(n->env, d.L1));
    FG_TRY(convl_alloc(n->env, d.L2));
    FG_TRY(dalloc(n, &d.x, B * img));
    FG_TRY(dalloc(n, &d.z1, B * A1 * 8));
    FG_TRY(dalloc(n, &d.h1, B * A1 * 8));
    FG_TRY(dalloc(n, &d.z2, B * A2 * 8));
    FG_TRY(dalloc(n, &d.h2, B * A2 * 8));
    FG_TRY(dalloc(n, &d.z3, B * kHidden));
    FG_TRY(dalloc(n, &d.h3, B * kHidden));
    FG_TRY(dalloc(n, &d.z4, B * img));
    FG_TRY(dalloc(n, &d.y, B * img));
    for (int i = 0; i < 3; ++i) {
      FG_TRY(dalloc(n, &d.mean[i], i == 2 ? kHidden : 8));
      FG_TRY(dalloc(n, &d.istd[i], i == 2 ? kHidden : 8));
    }
    FG_TRY(dalloc(n, &d.bn, kBnDn));
    FG_CUDA(cudaMemcpyAsync(d.bn, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
  }
  FG_TRY(dalloc(n, &n->t, B * img));
  FG_TRY(dalloc(n, &n->dz4, B * img));
  FG_TRY(dalloc(n, &n->dh3, B * kHidden));
  FG_TRY(dalloc(n, &n->dz3, B * kHidden));
  FG_TRY(dalloc(n, &n->dh2, B * A2 * 8));
  FG_TRY(dalloc(n, &n->dz2, B * A2 * 8));
  FG_TRY(dalloc(n, &n->dh1, B * A1 * 8));
  FG_TRY(dalloc(n, &n->dz1, B * A1 * 8));
  FG_TRY(dalloc(n, &n->mg, 2 * kHidden));
  FG_TRY(dalloc(n, reinterpret_cast<float**>(&n->acc), 2 * 2 * kHidden));
  for (auto& q : n->noise) FG_TRY(dalloc(n, &q, B * img));
  for (auto& q : n->masks) FG_TRY(dalloc(n, &q, B * n->mps));
  FG_TRY(dalloc(n, &n->in_img, B * img));
  FG_TRY(dalloc(n, &n->in_noise, 2 * B * img));
  FG_TRY(dalloc(n, &n->in_masks, 3 * B * n->mps));
  FG_TRY(dalloc(n, &n->io, B * img));
  // the largest dY split (L2's output or L1's) and the packed weight gradient of the larger Linear
  const size_t dy = B * std::max<size_t>(img, kHidden);
  FG_TRY(dalloc(n, &n->env.dy.hi, dy));
  FG_TRY(dalloc(n, &n->env.dy.lo, dy));
  FG_TRY(dalloc(n, &n->env.ws, std::max<size_t>((size_t)kHidden * 8 * A2, img * kHidden)));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

int& pack_state(fg_dn* n, int net) { return net ? n->net.D_pack : n->net.G_pack; }
const float* params(fg_dn* n, int net) { return net ? n->net.PD : n->net.PG; }
float* grads(fg_dn* n, int net) { return net ? n->net.gD : n->net.gG; }

int pack(fg_dn* n, int net) {
  DnDec& d = n->dec[net];
  if (pack_state(n, net) == pack_key(n->c)) return FG_OK;
  FG_TRY(convl_pack(n->c, d.L1, params(n, net)));
  FG_TRY(convl_pack(n->c, d.L2, params(n, net)));
  pack_state(n, net) = pack_key(n->c);
  return FG_OK;
}

// a (column groups x row chunks) grid for the BatchNorm reductions: enough blocks to fill the GPU, >= 64 rows each
dim3 bn_grid(fg_ctx* c, int64_t P, int C, int64_t* rpc) {
  const int cols = C < 32 ? C : 32, groups = (C + cols - 1) / cols;
  int64_t chunks = std::min<int64_t>(std::max(1, c->sm_count * 4 / groups), (P + 63) / 64);
  if (chunks < 1) chunks = 1;
  *rpc = (P + chunks - 1) / chunks;
  return dim3(groups, (unsigned)((P + *rpc - 1) / *rpc));
}

// layer l (0, 1: spatial, 2: 1-D) of decoder d: BatchNorm (batch statistics + running update in training, running
// statistics in evaluation) -> LeakyReLU -> Dropout (masks: null = none)
int bn_fwd(fg_dn* n, DnDec& d, int l, const float* z, float* h, int64_t P, int C, const float* P0, int64_t g, int64_t b,
           const float* masks, int moff, int HW, float scale) {
  fg_ctx* c = n->c;
  float *rm = d.bn + (l == 2 ? 32 : 16 * l), *rv = rm + (l == 2 ? kHidden : 8);
  if (d.train) {
    int64_t rpc;
    const dim3 grid = bn_grid(c, P, C, &rpc);
    FG_TRY(red_check(c, grid.y, 2 * C));
    dn_bn_stats_kernel<<<grid, 256, 0, c->stream>>>(z, P, C, rpc, c->red_ws, c->red_ticket, n->acc);
    LAUNCH_CHECK(c);
    FG_TRY(k_bn_finalize(c, n->acc, d.mean[l], d.istd[l], rm, rv, P, C));
  } else {
    FG_TRY(k_bn_eval_prep(c, rm, rv, d.mean[l], d.istd[l], C));
  }
  dn_bn_act_kernel<<<grid_for(P * C, 256), 256, 0, c->stream>>>(z, d.mean[l], d.istd[l], P0 + g, P0 + b, masks, n->mps, moff, HW,
                                                                scale, h, P, C);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int bn_bwd(fg_dn* n, DnDec& d, int l, const float* dh, const float* z, float* dz, int64_t P, int C, const float* P0, float* G,
           int64_t g, int64_t b, const float* masks, int moff, int HW, float scale) {
  fg_ctx* c = n->c;
  int64_t rpc;
  const dim3 grid = bn_grid(c, P, C, &rpc);
  FG_TRY(red_check(c, grid.y, 2 * C));
  dn_bn_bwd_reduce_kernel<<<grid, 256, 0, c->stream>>>(dh, z, d.mean[l], d.istd[l], P0 + g, P0 + b, masks, n->mps, moff, HW, scale,
                                                       P, C, rpc, c->red_ws, c->red_ticket, n->acc);
  LAUNCH_CHECK(c);
  FG_TRY(k_bn_bwd_finalize(c, n->acc, n->mg, G + g, G + b, P, C));
  dn_bn_bwd_apply_kernel<<<grid_for(P * C, 256), 256, 0, c->stream>>>(dh, z, d.mean[l], d.istd[l], P0 + g, P0 + b, masks, n->mps,
                                                                      moff, HW, scale, d.train ? n->mg : nullptr, dz, P, C);
  LAUNCH_CHECK(c);
  return FG_OK;
}

int vconv_fwd(fg_dn* n, const float* in, const float* W, const float* bias, float* out, int B, int H, int Cin) {
  fg_ctx* c = n->c;
  const int64_t P = (int64_t)B * (H - 2) * (H - 2);
  if (Cin == 1) vconv3_fwd_kernel<1><<<grid_for(P, 256), 256, 0, c->stream>>>(in, W, bias, out, B, H);
  else if (Cin == 3) vconv3_fwd_kernel<3><<<grid_for(P, 256), 256, 0, c->stream>>>(in, W, bias, out, B, H);
  else vconv3_fwd_kernel<8><<<grid_for(P, 256), 256, 0, c->stream>>>(in, W, bias, out, B, H);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int vconv_wgrad(fg_dn* n, const float* in, const float* dy, float* dW, float* db, int B, int H, int Cin) {
  fg_ctx* c = n->c;
  const int64_t P = (int64_t)B * (H - 2) * (H - 2);
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(c->sm_count * 2, (P + 255) / 256));
  const int64_t ppb = (P + grid - 1) / grid;
  FG_TRY(red_check(c, grid, 8 * Cin * 9 + 8));
  if (Cin == 1) vconv3_wgrad_kernel<1><<<grid, 256, 0, c->stream>>>(in, dy, B, H, ppb, c->red_ws, c->red_ticket, dW, db);
  else if (Cin == 3) vconv3_wgrad_kernel<3><<<grid, 256, 0, c->stream>>>(in, dy, B, H, ppb, c->red_ws, c->red_ticket, dW, db);
  else vconv3_wgrad_kernel<8><<<grid, 256, 0, c->stream>>>(in, dy, B, H, ppb, c->red_ws, c->red_ticket, dW, db);
  LAUNCH_CHECK(c);
  return FG_OK;
}

// decoder `net` on d.x (NHWC [B][S][S][C]) -> d.z4 (logits, NHWC); masks: [B][mps] keep flags (training) or null
int dec_forward(fg_dn* n, int net, int B, bool training, const float* masks) {
  DnDec& d = n->dec[net];
  const int S = n->S, A2 = (S - 4) * (S - 4);
  const float* P = params(n, net);
  const float scale = 1.0f / (1.0f - n->p_drop);
  FG_TRY(pack(n, net));
  d.B = B;
  d.train = training;
  d.masks = training ? masks : nullptr;
  FG_TRY(vconv_fwd(n, d.x, P + d.c1W, P + d.c1b, d.z1, B, S, n->C));
  FG_TRY(bn_fwd(n, d, 0, d.z1, d.h1, (int64_t)B * (S - 2) * (S - 2), 8, P, d.g1, d.b1, nullptr, 0, 1, 1.f));
  FG_TRY(vconv_fwd(n, d.h1, P + d.c2W, P + d.c2b, d.z2, B, S - 2, 8));
  FG_TRY(bn_fwd(n, d, 1, d.z2, d.h2, (int64_t)B * A2, 8, P, d.g2, d.b2, d.masks, 0, A2, scale));
  FG_TRY(convl_fwd(n->env, d.L1, d.h2, P, d.z3, B));
  FG_TRY(bn_fwd(n, d, 2, d.z3, d.h3, B, kHidden, P, d.g3, d.b3, d.masks, 8 * A2, 1, scale));
  FG_TRY(convl_fwd(n->env, d.L2, d.h3, P, d.z4, B));
  d.valid = true;
  return FG_OK;
}
// from dz4 (gradient at the logits, NHWC) of the last forward of decoder `net`: += its parameter gradients
int dec_backward(fg_dn* n, int net) {
  DnDec& d = n->dec[net];
  if (!d.valid) {
    fg_set_error("denoiser backward needs a preceding forward of the same decoder");
    return FG_ERR_STATE;
  }
  const int S = n->S, A2 = (S - 4) * (S - 4), B = d.B;
  const float* P = params(n, net);
  float* G = grads(n, net);
  n->grad_B = B;
  const float scale = 1.0f / (1.0f - n->p_drop);
  FG_TRY(convl_bwd(n->env, d.L2, d.h3, n->dz4, G, n->dh3, B));
  FG_TRY(bn_bwd(n, d, 2, n->dh3, d.z3, n->dz3, B, kHidden, P, G, d.g3, d.b3, d.masks, 8 * A2, 1, scale));
  FG_TRY(convl_bwd(n->env, d.L1, d.h2, n->dz3, G, n->dh2, B));
  FG_TRY(bn_bwd(n, d, 1, n->dh2, d.z2, n->dz2, (int64_t)B * A2, 8, P, G, d.g2, d.b2, d.masks, 0, A2, scale));
  FG_TRY(vconv_wgrad(n, d.h1, n->dz2, G + d.c2W, G + d.c2b, B, S - 2, 8));
  vconv3_dgrad8_kernel<<<grid_for((int64_t)B * (S - 2) * (S - 2), 256), 256, 0, n->c->stream>>>(n->dz2, P + d.c2W, n->dh1, B,
                                                                                                  S - 2);
  LAUNCH_CHECK(n->c);
  FG_TRY(bn_bwd(n, d, 0, n->dh1, d.z1, n->dz1, (int64_t)B * (S - 2) * (S - 2), 8, P, G, d.g1, d.b1, nullptr, 0, 1, 1.f));
  return vconv_wgrad(n, d.x, n->dz1, G + d.c1W, G + d.c1b, B, S, n->C);
}

// d.x = images (device NCHW) + WhiteNoise: noise given (device NCHW), or drawn on stream kind (seed_dev != null), or none
int dn_input(fg_dn* n, int net, const float* img, int B, const float* noise, bool draw, int k, float std, bool targets) {
  fg_ctx* c = n->c;
  const int HW = n->S * n->S;
  const bool any = noise || draw;
  dn_input_kernel<<<grid_for((int64_t)B * n->C * HW, 256), 256, 0, c->stream>>>(
      img, noise, draw && !noise ? c->seed_dev : nullptr, kKindNoise + k, std, any ? n->noise[k] : nullptr, n->dec[net].x,
      targets ? n->t : nullptr, B, n->C, HW);
  LAUNCH_CHECK(c);
  return FG_OK;
}
// keep flags of forward k: given (device [B][mps]) or drawn into n->masks[k]
int dn_masks(fg_dn* n, const float* given, int B, int k, float p, const float** out) {
  fg_ctx* c = n->c;
  if (given) {
    *out = given;
    return FG_OK;
  }
  const int64_t cnt = (int64_t)B * n->mps;
  dn_mask_kernel<<<grid_for(cnt, 256), 256, 0, c->stream>>>(n->masks[k], cnt, p, c->seed_dev, kKindMask + k);
  LAUNCH_CHECK(c);
  *out = n->masks[k];
  return FG_OK;
}

int sigmoid_bce(fg_dn* n, int net, int B, float* loss) {
  fg_ctx* c = n->c;
  const int64_t cnt = (int64_t)B * n->C * n->S * n->S;
  const int grid = grid_for(cnt, 256, c->sm_count * 4);
  FG_TRY(red_check(c, grid, 1));
  dn_sigmoid_bce_kernel<<<grid, 256, 0, c->stream>>>(n->dec[net].z4, n->t, n->dec[net].y, n->dz4, cnt, c->red_ws, c->red_ticket,
                                                     loss);
  LAUNCH_CHECK(c);
  return FG_OK;
}

// penalty -> clamp -> Adam on the shared state (fevalAE / fevalAE2 + optim.adam, train_denoiser.lua:278-291, :335)
int dn_optim(fg_dn* n, int net, const fg_dn_hyper* h) {
  fg_ctx* c = n->c;
  FG_TRY(k_adam_prep(c, &n->dstats->t, &n->dstats->step, h->lr, h->beta1, h->beta2));
  NetPair& p = n->net;
  FG_TRY(k_optim_update(c, FG_OPT_ADAM, net ? p.PD : p.PG, grads(n, net), p.mG, p.vG, p.nG, h->beta1, h->beta2, h->eps, 0.f,
                        h->L1, h->L2, h->clamp, 1.0f, &n->dstats->step, nullptr, &n->dstats->t));
  pack_state(n, net) = -1;
  return FG_OK;
}

// the per-batch body of train_denoiser.lua:247-341 on device inputs (images NCHW [B]; noise [2][B] NCHW or null;
// masks [3][B][mps] or null); the draws read the step seed from c->seed_dev
int train_step(fg_dn* n, const fg_dn_hyper* h, int B, const float* img, const float* noise, const float* masks) {
  fg_ctx* c = n->c;
  const size_t im = (size_t)B * n->C * n->S * n->S, mk = (size_t)B * n->mps;
  const float* m;
  // ---- fevalAE + adam ----
  FG_TRY(pair_zero_grads(c, n->net, FG_NET_G));
  FG_TRY(dn_input(n, 0, img, B, noise, true, 0, h->noise_std, true));
  FG_TRY(dn_masks(n, masks, B, 0, h->p_drop, &m));
  FG_TRY(dec_forward(n, 0, B, true, m));
  FG_TRY(sigmoid_bce(n, 0, B, &n->dstats->loss[0]));
  FG_TRY(dec_backward(n, 0));
  FG_TRY(dn_optim(n, 0, h));
  // ---- fevalAE2 + adam: AE forward again (fresh noise and masks, updated parameters, running statistics updated) ----
  FG_TRY(pair_zero_grads(c, n->net, FG_NET_D));
  FG_TRY(dn_input(n, 0, img, B, noise ? noise + im : nullptr, true, 1, h->noise_std, false));
  FG_TRY(dn_masks(n, masks ? masks + mk : nullptr, B, 1, h->p_drop, &m));
  FG_TRY(dec_forward(n, 0, B, true, m));
  FG_TRY(k_sigmoid_fwd(c, n->dec[0].z4, n->dec[1].x, (int64_t)im));  // AE's output, NHWC, is AE2's input
  FG_TRY(dn_masks(n, masks ? masks + 2 * mk : nullptr, B, 2, h->p_drop, &m));
  FG_TRY(dec_forward(n, 1, B, true, m));
  FG_TRY(sigmoid_bce(n, 1, B, &n->dstats->loss[1]));
  FG_TRY(dec_backward(n, 1));
  FG_TRY(dn_optim(n, 1, h));
  FG_CUDA(cudaMemcpyAsync(n->hstats, n->dstats, sizeof(DnStats), cudaMemcpyDeviceToHost, c->stream));
  return FG_OK;
}
}  // namespace

#define ENTER(n)                                \
  do {                                          \
    if (!(n) || !(n)->c) {                      \
      fg_set_error("null fg_dn");               \
      return FG_ERR_INVALID;                    \
    }                                           \
    FG_CUDA(cudaSetDevice((n)->c->device));     \
  } while (0)
#define NET_OK(net, what) FG_REQUIRE((net) == 0 || (net) == 1, "%s: net %d must be 0 (AE1's decoder) or 1 (AE2)", what, net)

extern "C" {

void fg_dn_hyper_default(fg_dn_hyper* h) {
  if (!h) return;
  h->lr = 1e-3f;
  h->beta1 = 0.9f;
  h->beta2 = 0.999f;
  h->eps = 1e-8f;
  h->L1 = 0.f;
  h->L2 = 0.f;
  h->clamp = 1.f;
  h->p_drop = 0.2f;
  h->noise_std = 0.1f;
}

int64_t fg_dn_param_count(int channels, int size) {
  if ((channels != 1 && channels != 3) || (size != 16 && size != 32)) return -1;
  DnDec d;
  return make_dn_layout(d, channels, size);
}
int fg_dn_mask_per_sample(int size) {
  if (size != 16 && size != 32) return -1;
  return 8 * (size - 4) * (size - 4) + kHidden;
}

int fg_dn_create(fg_ctx* ctx, int size, fg_dn** out) {
  if (!ctx || !out) {
    fg_set_error("fg_dn_create: null argument");
    return FG_ERR_INVALID;
  }
  *out = nullptr;
  if (size != 16 && size != 32) {
    fg_set_error("fg_dn_create: image size %d; the denoiser supports 16 and 32", size);
    return FG_ERR_UNSUPPORTED;
  }
  if (ctx->world > 1) {
    fg_set_error("fg_dn_create: the denoiser runs on one GPU; this context is data parallel (%d ranks)", ctx->world);
    return FG_ERR_UNSUPPORTED;
  }
  FG_CUDA(cudaSetDevice(ctx->device));
  fg_dn* n = new fg_dn();
  n->c = ctx;
  n->S = size;
  n->C = ctx->C;
  n->maxB = ctx->maxB;
  n->mps = fg_dn_mask_per_sample(size);
  const int r = dn_alloc(n);
  if (r != FG_OK) {
    fg_dn_destroy(n);
    return r;
  }
  *out = n;
  return FG_OK;
}
int fg_dn_destroy(fg_dn* n) {
  if (!n) return FG_OK;
  if (n->c) {
    cudaSetDevice(n->c->device);
    cudaStreamSynchronize(n->c->stream);
  }
  pair_free(n->net);
  if (n->hstats) cudaFreeHost(n->hstats);
  for (void* p : n->allocs) cudaFree(p);
  delete n;
  return FG_OK;
}

int fg_dn_set_params(fg_dn* n, int net, const float* src) {
  ENTER(n);
  NET_OK(net, "fg_dn_set_params");
  FG_REQUIRE(src, "fg_dn_set_params: null source");
  return pair_set_params(n->c, n->net, net, src);
}
int fg_dn_get_params(fg_dn* n, int net, float* dst) {
  ENTER(n);
  NET_OK(net, "fg_dn_get_params");
  FG_REQUIRE(dst, "fg_dn_get_params: null destination");
  return pair_get_params(n->c, n->net, net, dst);
}
int fg_dn_get_grads(fg_dn* n, int net, float* dst) {
  ENTER(n);
  NET_OK(net, "fg_dn_get_grads");
  FG_REQUIRE(dst, "fg_dn_get_grads: null destination");
  return pair_get_grads(n->c, n->net, net, dst);
}
int fg_dn_zero_grads(fg_dn* n, int net) {
  ENTER(n);
  NET_OK(net, "fg_dn_zero_grads");
  return pair_zero_grads(n->c, n->net, net);
}
int fg_dn_set_bn_state(fg_dn* n, int net, const float* src) {
  ENTER(n);
  NET_OK(net, "fg_dn_set_bn_state");
  FG_REQUIRE(src, "fg_dn_set_bn_state: null source");
  FG_CUDA(cudaMemcpyAsync(n->dec[net].bn, src, kBnDn * sizeof(float), cudaMemcpyDefault, n->c->stream));
  FG_CUDA(cudaStreamSynchronize(n->c->stream));
  return FG_OK;
}
int fg_dn_get_bn_state(fg_dn* n, int net, float* dst) {
  ENTER(n);
  NET_OK(net, "fg_dn_get_bn_state");
  FG_REQUIRE(dst, "fg_dn_get_bn_state: null destination");
  return fg_to_user(n->c, dst, n->dec[net].bn, kBnDn);
}
int fg_dn_set_adam_state(fg_dn* n, const float* m, const float* v, int t) {
  ENTER(n);
  fg_ctx* c = n->c;
  const size_t bytes = n->net.nG * sizeof(float);
  if (m) FG_CUDA(cudaMemcpyAsync(n->net.mG, m, bytes, cudaMemcpyDefault, c->stream));
  if (v) FG_CUDA(cudaMemcpyAsync(n->net.vG, v, bytes, cudaMemcpyDefault, c->stream));
  FG_CUDA(cudaMemcpyAsync(&n->dstats->t, &t, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}
int fg_dn_get_adam_state(fg_dn* n, float* m, float* v, int* t) {
  ENTER(n);
  fg_ctx* c = n->c;
  if (m) FG_TRY(fg_to_user(c, m, n->net.mG, n->net.nG));
  if (v) FG_TRY(fg_to_user(c, v, n->net.vG, n->net.nG));
  if (t) {
    FG_CUDA(cudaMemcpyAsync(t, &n->dstats->t, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    FG_CUDA(cudaStreamSynchronize(c->stream));
  }
  return FG_OK;
}

int fg_dn_forward(fg_dn* n, int net, const float* x, int B, int training, const float* noise, const float* masks, uint64_t seed,
                  float* out) {
  ENTER(n);
  NET_OK(net, "fg_dn_forward");
  FG_REQUIRE(x && B >= 1 && B <= n->maxB && (!training || B >= 2), "fg_dn_forward: batch %d out of range [%d,%d]", B,
             training ? 2 : 1, n->maxB);
  fg_ctx* c = n->c;
  const size_t im = (size_t)B * n->C * n->S * n->S;
  fg_dn_hyper h;
  fg_dn_hyper_default(&h);
  n->p_drop = h.p_drop;
  FG_TRY(k_set_u64(c, c->seed_dev, seed));
  const float *xd, *nd = nullptr, *md = nullptr;
  FG_TRY(fg_to_dev(c, x, im, n->in_img, &xd));
  if (training && noise && net == 0) FG_TRY(fg_to_dev(c, noise, im, n->in_noise, &nd));
  if (training && masks) FG_TRY(fg_to_dev(c, masks, (size_t)B * n->mps, n->in_masks, &md));
  // WhiteNoise belongs to AE1 in training only (evaluate(): identity); AE2 has none
  FG_TRY(dn_input(n, net, xd, B, nd, training && net == 0, 0, h.noise_std, false));
  if (training) FG_TRY(dn_masks(n, md, B, 0, h.p_drop, &md));
  FG_TRY(dec_forward(n, net, B, training != 0, md));
  FG_TRY(k_sigmoid_fwd(c, n->dec[net].z4, n->dec[net].y, (int64_t)im));
  if (out) {
    FG_TRY(k_nhwc_to_nchw(c, n->dec[net].y, n->io, B, n->C, n->S * n->S));
    FG_TRY(fg_to_user(c, out, n->io, im));
  }
  return FG_OK;
}
int fg_dn_backward(fg_dn* n, int net, const float* dout) {
  ENTER(n);
  NET_OK(net, "fg_dn_backward");
  FG_REQUIRE(dout, "fg_dn_backward: null gradient");
  fg_ctx* c = n->c;
  DnDec& d = n->dec[net];
  FG_REQUIRE(d.valid, "fg_dn_backward: no forward of decoder %d to differentiate", net);
  const size_t im = (size_t)d.B * n->C * n->S * n->S;
  const float* dd;
  FG_TRY(fg_to_dev(c, dout, im, n->in_img, &dd));
  FG_TRY(k_nchw_to_nhwc(c, dd, n->io, d.B, n->C, n->S * n->S));
  FG_TRY(k_sigmoid_bwd(c, n->io, d.y, n->dz4, (int64_t)im));
  return dec_backward(n, net);
}

int fg_dn_train_step(fg_dn* n, const fg_dn_hyper* h, int B, const float* images, const float* noise, const float* masks,
                     uint64_t seed, fg_dn_stats* stats) {
  ENTER(n);
  FG_REQUIRE(h && images, "fg_dn_train_step: null input");
  FG_REQUIRE(B >= 2 && B <= n->maxB, "fg_dn_train_step: batch %d out of range [2,%d]", B, n->maxB);
  FG_REQUIRE(h->p_drop >= 0.f && h->p_drop < 1.f, "fg_dn_train_step: p_drop %g outside [0,1)", h->p_drop);
  fg_ctx* c = n->c;
  const size_t im = (size_t)B * n->C * n->S * n->S;
  const float *id, *nd = nullptr, *md = nullptr;
  FG_TRY(fg_to_dev(c, images, im, n->in_img, &id));
  if (noise) FG_TRY(fg_to_dev(c, noise, 2 * im, n->in_noise, &nd));
  if (masks) FG_TRY(fg_to_dev(c, masks, 3 * (size_t)B * n->mps, n->in_masks, &md));
  n->p_drop = h->p_drop;
  FG_TRY(net_graph_run(c, n->net, B, h, sizeof(*h), {id, nd, md}, seed, [&]() { return train_step(n, h, B, id, nd, md); }));
  // A replayed step does not run the host side of its body: set what it would have set.  The step leaves AE1's
  // activations of its second forward beside the sigmoid output of its first, so fg_dn_backward needs a new forward.
  for (DnDec& d : n->dec) {
    d.B = B;
    d.train = true;
    d.valid = false;
  }
  n->grad_B = B;
  if (stats) {
    FG_CUDA(cudaStreamSynchronize(c->stream));
    stats->loss_AE1 = n->hstats->loss[0];
    stats->loss_AE2 = n->hstats->loss[1];
    stats->t = n->hstats->t;
  }
  return FG_OK;
}

// AE1_DECODER:evaluate():forward(images) in chunks of at most `chunk` images (train.lua --denoise, nn_utils.lua:144-155)
int fg_dn_denoise(fg_dn* n, const float* images, int N, int chunk, float* out) {
  ENTER(n);
  FG_REQUIRE(images && out && N >= 1 && chunk >= 1 && chunk <= n->maxB, "fg_dn_denoise: bad arguments (chunk %d, max %d)", chunk,
             n->maxB);
  fg_ctx* c = n->c;
  const size_t img = (size_t)n->C * n->S * n->S;
  const bool out_dev = fg_is_dev(out);
  for (int s = 0; s < N; s += chunk) {
    const int b = std::min(chunk, N - s);
    const float* xd;
    FG_TRY(fg_to_dev(c, images + (size_t)s * img, b * img, n->in_img, &xd));
    FG_TRY(dn_input(n, 0, xd, b, nullptr, false, 0, 0.f, false));
    FG_TRY(dec_forward(n, 0, b, false, nullptr));
    FG_TRY(k_sigmoid_fwd(c, n->dec[0].z4, n->dec[0].y, (int64_t)b * img));
    float* dst = out_dev ? out + (size_t)s * img : n->io;
    FG_TRY(k_nhwc_to_nchw(c, n->dec[0].y, dst, b, n->C, n->S * n->S));
    if (!out_dev) {
      FG_CUDA(cudaMemcpyAsync(out + (size_t)s * img, n->io, b * img * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
      FG_CUDA(cudaStreamSynchronize(c->stream));  // io and in_img are reused by the next chunk
    }
  }
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

int64_t fg_dn_debug_tensor(fg_dn* n, const char* name, float* dst, int64_t max_elems) {
  if (!n || !n->c || !name) {
    fg_set_error("fg_dn_debug_tensor: null argument");
    return -1;
  }
  cudaSetDevice(n->c->device);
  const int64_t img = (int64_t)n->C * n->S * n->S, A1 = 8 * (n->S - 2) * (n->S - 2), A2 = 8 * (n->S - 4) * (n->S - 4);
  const int B = n->dec[0].B;
  std::vector<DebugTensor> ents = {{"noise0", n->noise[0], img, B}, {"noise1", n->noise[1], img, B},
                                   {"masks0", n->masks[0], n->mps, B}, {"masks1", n->masks[1], n->mps, B},
                                   {"masks2", n->masks[2], n->mps, n->dec[1].B}};
  // the activations of each decoder's last forward (NHWC) and the gradients of the last backward (shared scratch)
  static const char* names[2][15] = {
      {"AE1.x", "AE1.z1", "AE1.h1", "AE1.z2", "AE1.h2", "AE1.z3", "AE1.h3", "AE1.z4", "AE1.y", "AE1.mean1", "AE1.istd1",
       "AE1.mean2", "AE1.istd2", "AE1.mean3", "AE1.istd3"},
      {"AE2.x", "AE2.z1", "AE2.h1", "AE2.z2", "AE2.h2", "AE2.z3", "AE2.h3", "AE2.z4", "AE2.y", "AE2.mean1", "AE2.istd1",
       "AE2.mean2", "AE2.istd2", "AE2.mean3", "AE2.istd3"}};
  for (int k = 0; k < 2; ++k) {
    const DnDec& d = n->dec[k];
    const int b = d.B;
    const float* act[9] = {d.x, d.z1, d.h1, d.z2, d.h2, d.z3, d.h3, d.z4, d.y};
    const int64_t per[9] = {img, A1, A1, A2, A2, kHidden, kHidden, img, img};
    for (int i = 0; i < 9; ++i) ents.push_back({names[k][i], act[i], per[i], b});
    for (int l = 0; l < 3; ++l) {
      ents.push_back({names[k][9 + 2 * l], d.mean[l], l == 2 ? kHidden : 8, 1});
      ents.push_back({names[k][10 + 2 * l], d.istd[l], l == 2 ? kHidden : 8, 1});
    }
  }
  const int gb = n->grad_B;
  const float* gp[7] = {n->dz4, n->dh3, n->dz3, n->dh2, n->dz2, n->dh1, n->dz1};
  const int64_t gper[7] = {img, kHidden, kHidden, A2, A2, A1, A1};
  static const char* gnames[7] = {"dz4", "dh3", "dz3", "dh2", "dz2", "dh1", "dz1"};
  for (int i = 0; i < 7; ++i) ents.push_back({gnames[i], gb ? gp[i] : nullptr, gper[i], gb});
  return debug_tensor_copy(n->c, "fg_dn_debug_tensor", ents.data(), ents.size(), name, dst, max_elems);
}

}  // extern "C"
