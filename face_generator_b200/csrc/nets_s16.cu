// The `--scale 16` nets of train.lua (models.create_G / create_D pick them when dimensions[2] == 16, models.lua:87-104)
// and the adversarial.lua loop body on them:
//   G16 = models.lua:27-51   create_G_decoder_upsampling16: Linear(100, 128*4*4) View(128,4,4) PReLU | Up2 conv(128->256,5)
//         BN PReLU | Up2 conv(256->128,5) BN PReLU | conv(128->C,3) Sigmoid  -- the 32x32 generator with every size halved
//   D16 = models.lua:279-316 create_D16_d: ConcatTable{conv branch, dense branch} JoinTable(2) Linear(1152,1) Sigmoid
//         conv branch : conv(C->128,3) PReLU conv(128->128,3) PReLU AvgPool2 conv(128->512,3,STRIDE 2) PReLU
//                       conv(512->1024,3,STRIDE 2) PReLU SpatialDropout() View(4096) Linear(4096,1024) PReLU
//         dense branch: View(C*256) Linear(C*256,128) PReLU Dropout() Linear(128,128) PReLU
//   loop = adversarial.lua:83-288 (the same fevalD / fevalG_on_D / accuracy gate / interruptable optimizers as the 32x32 nets)
// Kernels: the two upsampled 5x5 layers use the phase-collapsed wgmma kernels of the 32x32 generator (forward with
// BatchNorm partials from the epilogue, wgrad, dgrad with the upsample backward folded in); every other layer is a ConvL
// (convl.h).  A stride-2 "same" 3x3 convolution is the stride-1 one sampled at the even pixels: forward = stride-1
// kernel + subsample, backward = the stride-1 dgrad / wgrad of dY with zeros inserted at the odd pixels.  That is exact
// (the inserted zeros contribute nothing) and keeps both layers on the tensor cores at 4x their minimal FLOPs, which
// is 0.2 ms at batch 256.
#include <algorithm>
#include <cstring>

#include "convl.h"
#include "fg_internal.h"
#include "k_conv_tc.h"
#include "k_misc.h"

#define LAUNCH_CHECK(c)                 \
  do {                                  \
    (c)->launches++;                    \
    FG_CUDA(cudaGetLastError());        \
  } while (0)

namespace {
constexpr int kS16Mask = 1024 + 128;  // nn.SpatialDropout() planes + nn.Dropout() of the dense branch, per sample
constexpr int kSide = 16;

inline int grid_for(int64_t n, int block, int cap = 132 * 16) {
  int64_t g = (n + block - 1) / block;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}
#define GRID_STRIDE(i, n) \
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < (n); i += (int64_t)gridDim.x * blockDim.x)

// nn.SpatialAveragePooling(2,2,2,2), NHWC.  x [B][H][W][C] -> y [B][H/2][W/2][C]
__global__ void avgpool2_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t n = (int64_t)B * Ho * Wo * C;
  GRID_STRIDE(i, n) {
    const int ch = (int)(i % C);
    int64_t r = i / C;
    const int xo = (int)(r % Wo); r /= Wo;
    const int yo = (int)(r % Ho);
    const int64_t b = r / Ho;
    const float* p = x + (((b * H + 2 * yo) * W + 2 * xo) * (int64_t)C + ch);
    y[i] = 0.25f * ((p[0] + p[C]) + (p[(int64_t)W * C] + p[(int64_t)W * C + C]));
  }
}
__global__ void avgpool2_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int B, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t n = (int64_t)B * H * W * C;
  GRID_STRIDE(i, n) {
    const int ch = (int)(i % C);
    int64_t r = i / C;
    const int xx = (int)(r % W); r /= W;
    const int yy = (int)(r % H);
    const int64_t b = r / H;
    dx[i] = 0.25f * dy[((b * Ho + yy / 2) * Wo + xx / 2) * (int64_t)C + ch];
  }
}
// stride-2 sampling of a stride-1 "same" convolution output: y[b][yo][xo][c] = x[b][2yo][2xo][c]
__global__ void subsample2_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t n = (int64_t)B * Ho * Wo * C;
  GRID_STRIDE(i, n) {
    const int ch = (int)(i % C);
    int64_t r = i / C;
    const int xo = (int)(r % Wo); r /= Wo;
    const int yo = (int)(r % Ho);
    const int64_t b = r / Ho;
    y[i] = x[((b * H + 2 * yo) * W + 2 * xo) * (int64_t)C + ch];
  }
}
// its adjoint: dx[b][y][x][c] = (y, x both even) ? dy[b][y/2][x/2][c] : 0
__global__ void zero_insert2_kernel(const float* __restrict__ dy, float* __restrict__ dx, int B, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t n = (int64_t)B * H * W * C;
  GRID_STRIDE(i, n) {
    const int ch = (int)(i % C);
    int64_t r = i / C;
    const int xx = (int)(r % W); r /= W;
    const int yy = (int)(r % H);
    const int64_t b = r / H;
    dx[i] = ((xx | yy) & 1) ? 0.f : dy[((b * Ho + yy / 2) * Wo + xx / 2) * (int64_t)C + ch];
  }
}
// nn.SpatialDropout() (p = 0.5): one keep flag per (sample, plane), NO rescale in training; evaluate() scales by 1-p.
// x, y: [B][HW][C]; masks[b*stride + moff + ch]; masks == nullptr: y = x * eval_scale.  Its own adjoint.
__global__ void plane_dropout_kernel(const float* __restrict__ x, const float* __restrict__ masks, int64_t stride, int moff,
                                     float eval_scale, float* __restrict__ y, int B, int HW, int C) {
  const int64_t n = (int64_t)B * HW * C;
  GRID_STRIDE(i, n) {
    const int ch = (int)(i % C);
    const int64_t b = i / ((int64_t)HW * C);
    y[i] = x[i] * (masks ? masks[b * stride + moff + ch] : eval_scale);
  }
}
// nn.JoinTable(2) of {a [B][Na], b [B][Nb]} -> [B][Na+Nb], and the split of its gradient
__global__ void join2_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int B, int Na,
                             int Nb) {
  const int N = Na + Nb;
  GRID_STRIDE(i, (int64_t)B * N) {
    const int j = (int)(i % N);
    const int64_t r = i / N;
    out[i] = j < Na ? a[r * Na + j] : b[r * Nb + (j - Na)];
  }
}
__global__ void split2_kernel(const float* __restrict__ in, float* __restrict__ a, float* __restrict__ b, int B, int Na, int Nb) {
  const int N = Na + Nb;
  GRID_STRIDE(i, (int64_t)B * N) {
    const int j = (int)(i % N);
    const int64_t r = i / N;
    if (j < Na) a[r * Na + j] = in[i]; else b[r * Nb + (j - Na)] = in[i];
  }
}

struct UpsL {  // nn.SpatialUpSamplingNearest(2) -> 5x5 "same" convolution; H = output side
  int Cin = 0, Cout = 0, H = 0;
  int64_t w_off = 0, b_off = 0;
  float *Wp = nullptr, *Wpd = nullptr;                                            // fp32 tap-major packs (FFMA path)
  float *Wf_hi = nullptr, *Wf_lo = nullptr, *Wd_hi = nullptr, *Wd_lo = nullptr;   // phase-collapsed TF32 packs [36][..][..]
  float *h_hi = nullptr, *h_lo = nullptr;                                         // split of the low-res input (fwd -> wgrad)
  float* sx = nullptr;                                                            // (max|h|, 1/scale) of its FP16 split
  const char *tf = "", *td = "", *tw = "";
  ConvGeom geom(int B) const { return ConvGeom{B, H, H, Cin, Cout, 5, 2}; }
};
}  // namespace

struct fg_s16 {
  fg_ctx* c = nullptr;
  int maxB = 0, C = 3;
  int64_t nG = 0, nD = 0;
  float *PG = nullptr, *PD = nullptr, *gG = nullptr, *gD = nullptr, *mG = nullptr, *vG = nullptr, *mD = nullptr,
        *vD = nullptr;
  float* bnG = nullptr;  // [768] running mean/var of the two BatchNorm layers (256 + 256 + 128 + 128)
  DeviceStats *dstats = nullptr, *hstats = nullptr;
  float* acc_hist = nullptr;
  // G
  ConvL GL1, GC3;
  UpsL GU[2];
  int64_t Ga[3] = {0, 0, 0}, Gg[2] = {0, 0}, Gbe[2] = {0, 0};
  float *G_x = nullptr, *G_z0 = nullptr, *G_h0 = nullptr, *G_z1 = nullptr, *G_h1 = nullptr, *G_z2 = nullptr, *G_h2 = nullptr,
        *G_z3 = nullptr, *G_y = nullptr;
  float *bn_mean[2] = {nullptr, nullptr}, *bn_istd[2] = {nullptr, nullptr}, *bn_mg = nullptr;
  float *G_dz3 = nullptr, *G_dfull = nullptr, *G_dz = nullptr, *G_dz0 = nullptr;
  // D
  ConvL Dc[4], DF1, DE1, DE2;
  int64_t Dca[4] = {0, 0, 0, 0}, Daf = 0, Dae1 = 0, Dae2 = 0, DJW = 0, DJb = 0;
  float *D_x = nullptr, *D_z[4] = {}, *D_h[4] = {}, *D_zfull = nullptr, *D_p1 = nullptr, *D_d3 = nullptr, *D_zf = nullptr,
        *D_hf = nullptr, *D_ze1 = nullptr, *D_he1 = nullptr, *D_de1 = nullptr, *D_ze2 = nullptr, *D_he2 = nullptr,
        *D_joint = nullptr, *D_logit = nullptr, *D_out = nullptr, *D_masks = nullptr, *D_dlogit = nullptr, *D_dx = nullptr,
        *D_dx2 = nullptr, *D_djoint = nullptr, *D_dhf = nullptr, *D_dhe2 = nullptr;
  // shared scratch
  float *ga = nullptr, *gb = nullptr, *dy_hi = nullptr, *dy_lo = nullptr, *ws = nullptr;
  float *in_a = nullptr, *in_b = nullptr, *in_c = nullptr, *in_m1 = nullptr, *in_m2 = nullptr, *io = nullptr;
  bool G_packed = false, D_packed = false;
  int G_pack_impl = -1, D_pack_impl = -1;
  int G_B = 0, D_B = 0;
  bool G_valid = false, G_train = true, D_valid = false, D_train = true;
  std::vector<void*> allocs;
  ConvLEnv env;
  std::vector<fg_ctx::StepGraph> graphs;  // captured train steps
};

namespace {
int dalloc(fg_s16* n, float** p, size_t elems) { return convl_dalloc(n->env, p, elems); }
inline bool use_tc(const fg_ctx* c, const ConvGeom& g) { return c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(g); }
inline bool use_tc_wgrad(const fg_ctx* c, const ConvGeom& g) { return use_tc(c, g) && g.Cout % 128 == 0 && g.Cin % 64 == 0; }
// option "mma_f16": the upsampled layers' hi/lo buffers hold the 3xFP16 split (see convl.cu)
inline bool f16_on(const fg_ctx* c) { return c->mma_f16 && c->conv_impl == FG_CONV_TC_COLLAPSED; }

void make_layouts(fg_s16* n) {
  const int C = n->C;
  {  // G16Layout: getParameters() order of models.lua:27-51
    int64_t o = 0;
    ConvL& L1 = n->GL1;
    L1.Cin = 100; L1.Cout = 2048; L1.k = 1; L1.H = 1;
    L1.nA = 128; L1.nS = 16;  // View(128,4,4): reference row c*16+s <-> our NHWC row s*128+c
    L1.w_off = o; o += 2048 * 100;
    L1.b_off = o; o += 2048;
    L1.tf = "s16.G.L1.fwd"; L1.td = "s16.G.L1.dgrad"; L1.tw = "s16.G.L1.wgrad";
    n->Ga[0] = o; o += 1;
    const int ci[2] = {128, 256}, co[2] = {256, 128}, hs[2] = {8, 16};
    static const char* tf[2] = {"s16.G.C1.fwd", "s16.G.C2.fwd"};
    static const char* td[2] = {"s16.G.C1.dgrad", "s16.G.C2.dgrad"};
    static const char* tw[2] = {"s16.G.C1.wgrad", "s16.G.C2.wgrad"};
    for (int i = 0; i < 2; ++i) {
      UpsL& U = n->GU[i];
      U.Cin = ci[i]; U.Cout = co[i]; U.H = hs[i];
      U.w_off = o; o += (int64_t)co[i] * ci[i] * 25;
      U.b_off = o; o += co[i];
      n->Gg[i] = o; o += co[i];
      n->Gbe[i] = o; o += co[i];
      n->Ga[i + 1] = o; o += 1;
      U.tf = tf[i]; U.td = td[i]; U.tw = tw[i];
    }
    ConvL& C3 = n->GC3;
    C3.Cin = 128; C3.Cout = C; C3.k = 3; C3.H = kSide;
    C3.w_off = o; o += (int64_t)C * 128 * 9;
    C3.b_off = o; o += C;
    C3.tf = "s16.G.C3.fwd"; C3.td = "s16.G.C3.dgrad"; C3.tw = "s16.G.C3.wgrad";
    n->nG = o;
  }
  {  // D16Layout: conv branch, dense branch, joint Linear (ConcatTable order, models.lua:306-313)
    const int ci[4] = {C, 128, 128, 512}, co[4] = {128, 128, 512, 1024}, hw[4] = {16, 16, 8, 4};  // stride-1 sides
    static const char* tf[4] = {"s16.D.c1.fwd", "s16.D.c2.fwd", "s16.D.c3.fwd", "s16.D.c4.fwd"};
    static const char* td[4] = {"s16.D.c1.dgrad", "s16.D.c2.dgrad", "s16.D.c3.dgrad", "s16.D.c4.dgrad"};
    static const char* tw[4] = {"s16.D.c1.wgrad", "s16.D.c2.wgrad", "s16.D.c3.wgrad", "s16.D.c4.wgrad"};
    int64_t o = 0;
    for (int i = 0; i < 4; ++i) {
      ConvL& L = n->Dc[i];
      L.Cin = ci[i]; L.Cout = co[i]; L.k = 3; L.H = hw[i];
      L.w_off = o; o += (int64_t)co[i] * ci[i] * 9;
      L.b_off = o; o += co[i];
      n->Dca[i] = o; o += 1;
      L.tf = tf[i]; L.td = td[i]; L.tw = tw[i];
    }
    ConvL& F1 = n->DF1;
    F1.Cin = 4096; F1.Cout = 1024; F1.k = 1; F1.H = 1;
    F1.cA = 1024; F1.cS = 4;  // View(4096) flattens [1024][2][2]; ours is [2][2][1024]
    F1.w_off = o; o += (int64_t)1024 * 4096;
    F1.b_off = o; o += 1024;
    F1.tf = "s16.D.F1.fwd"; F1.td = "s16.D.F1.dgrad"; F1.tw = "s16.D.F1.wgrad";
    n->Daf = o; o += 1;
    ConvL& E1 = n->DE1;
    E1.Cin = C * 256; E1.Cout = 128; E1.k = 1; E1.H = 1;
    E1.cA = C; E1.cS = 256;  // View(C*256) flattens the NCHW image; ours is [16][16][C]
    E1.w_off = o; o += (int64_t)128 * C * 256;
    E1.b_off = o; o += 128;
    E1.tf = "s16.D.E1.fwd"; E1.td = "s16.D.E1.dgrad"; E1.tw = "s16.D.E1.wgrad";
    n->Dae1 = o; o += 1;
    ConvL& E2 = n->DE2;
    E2.Cin = 128; E2.Cout = 128; E2.k = 1; E2.H = 1;
    E2.w_off = o; o += 128 * 128;
    E2.b_off = o; o += 128;
    E2.tf = "s16.D.E2.fwd"; E2.td = "s16.D.E2.dgrad"; E2.tw = "s16.D.E2.wgrad";
    n->Dae2 = o; o += 1;
    n->DJW = o; o += 1152;
    n->DJb = o; o += 1;
    n->nD = o;
  }
}

int s16_alloc(fg_s16* n) {
  const size_t B = n->maxB, C = n->C;
  make_layouts(n);
  n->env.c = n->c;
  n->env.maxB = n->maxB;
  n->env.allocs = &n->allocs;
  FG_TRY(dalloc(n, &n->PG, n->nG));
  FG_TRY(dalloc(n, &n->PD, n->nD));
  FG_TRY(dalloc(n, &n->gG, n->nG + kGradTail));
  FG_TRY(dalloc(n, &n->gD, n->nD + kGradTail));
  FG_TRY(dalloc(n, &n->mG, n->nG));
  FG_TRY(dalloc(n, &n->vG, n->nG));
  FG_TRY(dalloc(n, &n->mD, n->nD));
  FG_TRY(dalloc(n, &n->vD, n->nD));
  FG_TRY(dalloc(n, &n->bnG, 768));
  {  // nn.SpatialBatchNormalization: running_mean = 0, running_var = 1
    float init[768];
    for (int i = 0; i < 768; ++i) init[i] = (i >= 256 && i < 512) || i >= 640 ? 1.f : 0.f;
    FG_CUDA(cudaMemcpyAsync(n->bnG, init, sizeof(init), cudaMemcpyHostToDevice, n->c->stream));
    FG_CUDA(cudaStreamSynchronize(n->c->stream));
  }
  float* tmp = nullptr;
  FG_TRY(dalloc(n, &tmp, (sizeof(DeviceStats) + 3) / 4));
  n->dstats = (DeviceStats*)tmp;
  FG_TRY(dalloc(n, &n->acc_hist, kAccHistMax));
  FG_CUDA(cudaMallocHost((void**)&n->hstats, sizeof(DeviceStats)));
  memset(n->hstats, 0, sizeof(DeviceStats));
  // ---- G ----
  FG_TRY(convl_alloc(n->env, n->GL1));
  FG_TRY(convl_alloc(n->env, n->GC3));
  for (int i = 0; i < 2; ++i) {
    UpsL& U = n->GU[i];
    const size_t nw25 = (size_t)25 * U.Cout * U.Cin, nw36 = (size_t)36 * U.Cout * U.Cin;
    FG_TRY(dalloc(n, &U.Wp, nw25));
    FG_TRY(dalloc(n, &U.Wpd, nw25));
    FG_TRY(dalloc(n, &U.Wf_hi, nw36));
    FG_TRY(dalloc(n, &U.Wf_lo, nw36));
    FG_TRY(dalloc(n, &U.Wd_hi, nw36));
    FG_TRY(dalloc(n, &U.Wd_lo, nw36));
    const size_t nx = B * (U.H / 2) * (U.H / 2) * U.Cin;
    FG_TRY(dalloc(n, &U.h_hi, nx));
    FG_TRY(dalloc(n, &U.h_lo, nx));
    FG_TRY(dalloc(n, &U.sx, 2));
  }
  FG_TRY(dalloc(n, &n->G_x, B * 100));
  FG_TRY(dalloc(n, &n->G_z0, B * 2048));
  FG_TRY(dalloc(n, &n->G_h0, B * 2048));
  FG_TRY(dalloc(n, &n->G_z1, B * 64 * 256));
  FG_TRY(dalloc(n, &n->G_h1, B * 64 * 256));
  FG_TRY(dalloc(n, &n->G_z2, B * 256 * 128));
  FG_TRY(dalloc(n, &n->G_h2, B * 256 * 128));
  FG_TRY(dalloc(n, &n->G_z3, B * 256 * C));
  FG_TRY(dalloc(n, &n->G_y, B * 256 * C));
  for (int i = 0; i < 2; ++i) {
    FG_TRY(dalloc(n, &n->bn_mean[i], 256));
    FG_TRY(dalloc(n, &n->bn_istd[i], 256));
  }
  FG_TRY(dalloc(n, &n->bn_mg, 512));
  FG_TRY(dalloc(n, &n->G_dz3, B * 256 * C));
  FG_TRY(dalloc(n, &n->G_dfull, B * 256 * 256));  // full-resolution dgrad of C2 on the FFMA path: [B][16][16][256]
  FG_TRY(dalloc(n, &n->G_dz, B * 256 * 128));
  FG_TRY(dalloc(n, &n->G_dz0, B * 2048));
  // ---- D ----
  for (int i = 0; i < 4; ++i) FG_TRY(convl_alloc(n->env, n->Dc[i]));
  FG_TRY(convl_alloc(n->env, n->DF1));
  FG_TRY(convl_alloc(n->env, n->DE1));
  FG_TRY(convl_alloc(n->env, n->DE2));
  FG_TRY(dalloc(n, &n->D_x, B * 256 * C));
  const size_t zsz[4] = {B * 256 * 128, B * 256 * 128, B * 16 * 512, B * 4 * 1024};
  for (int i = 0; i < 4; ++i) {
    FG_TRY(dalloc(n, &n->D_z[i], zsz[i]));
    FG_TRY(dalloc(n, &n->D_h[i], zsz[i]));
  }
  FG_TRY(dalloc(n, &n->D_zfull, B * 64 * 512));  // stride-1 output of c3 ([B][8][8][512]) / c4 ([B][4][4][1024])
  FG_TRY(dalloc(n, &n->D_p1, B * 64 * 128));
  FG_TRY(dalloc(n, &n->D_d3, B * 4096));
  FG_TRY(dalloc(n, &n->D_zf, B * 1024));
  FG_TRY(dalloc(n, &n->D_hf, B * 1024));
  FG_TRY(dalloc(n, &n->D_ze1, B * 128));
  FG_TRY(dalloc(n, &n->D_he1, B * 128));
  FG_TRY(dalloc(n, &n->D_de1, B * 128));
  FG_TRY(dalloc(n, &n->D_ze2, B * 128));
  FG_TRY(dalloc(n, &n->D_he2, B * 128));
  FG_TRY(dalloc(n, &n->D_joint, B * 1152));
  FG_TRY(dalloc(n, &n->D_djoint, B * 1152));
  FG_TRY(dalloc(n, &n->D_dhf, B * 1024));
  FG_TRY(dalloc(n, &n->D_dhe2, B * 128));
  FG_TRY(dalloc(n, &n->D_logit, B));
  FG_TRY(dalloc(n, &n->D_out, B));
  FG_TRY(dalloc(n, &n->D_dlogit, B));
  FG_TRY(dalloc(n, &n->D_masks, B * kS16Mask));
  FG_TRY(dalloc(n, &n->D_dx, B * 256 * C));
  FG_TRY(dalloc(n, &n->D_dx2, B * 256 * C));
  // ---- shared scratch ----
  const size_t big = B * 256 * 128;  // largest activation: [B][16][16][128] = [B][8][8][512]
  FG_TRY(dalloc(n, &n->ga, big));
  FG_TRY(dalloc(n, &n->gb, big));
  FG_TRY(dalloc(n, &n->dy_hi, big));
  FG_TRY(dalloc(n, &n->dy_lo, big));
  FG_TRY(dalloc(n, &n->ws, (size_t)9 * 1024 * 512));  // largest weight tensor (c4); F1 is 4096*1024, the 5x5 packs 36*256*128
  n->env.ga = n->ga; n->env.dy_hi = n->dy_hi; n->env.dy_lo = n->dy_lo; n->env.ws = n->ws;
  FG_TRY(dalloc(n, &n->in_a, B * 256 * C));
  FG_TRY(dalloc(n, &n->in_b, B * 100));
  FG_TRY(dalloc(n, &n->in_c, B * 100));
  FG_TRY(dalloc(n, &n->in_m1, B * kS16Mask));
  FG_TRY(dalloc(n, &n->in_m2, B * kS16Mask));
  FG_TRY(dalloc(n, &n->io, B * 256 * C));
  FG_CUDA(cudaStreamSynchronize(n->c->stream));
  return FG_OK;
}

int pack_G(fg_s16* n) {
  fg_ctx* c = n->c;
  if (n->G_packed && n->G_pack_impl == pack_key(c)) return FG_OK;
  FG_TRY(convl_pack(c, n->GL1, n->PG));
  FG_TRY(convl_pack(c, n->GC3, n->PG));
  for (int i = 0; i < 2; ++i) {
    UpsL& U = n->GU[i];
    if (use_tc_wgrad(c, U.geom(n->maxB)) && f16_on(c))
      FG_TRY(tc_pack_collapsed_h(c, n->PG + U.w_off, U.Wf_hi, U.Wf_lo, U.Wd_hi, U.Wd_lo, U.Cout, U.Cin));
    else if (use_tc_wgrad(c, U.geom(n->maxB)))
      FG_TRY(tc_pack_collapsed(c, n->PG + U.w_off, U.Wf_hi, U.Wf_lo, U.Wd_hi, U.Wd_lo, U.Cout, U.Cin));
    else
      FG_TRY(k_pack_weights(c, n->PG + U.w_off, U.Wp, U.Wpd, U.Cout, U.Cin, 25, 0, 0, 0, 0));
  }
  n->G_packed = true;
  n->G_pack_impl = pack_key(c);
  return FG_OK;
}
int pack_D(fg_s16* n) {
  fg_ctx* c = n->c;
  if (n->D_packed && n->D_pack_impl == pack_key(c)) return FG_OK;
  for (int i = 0; i < 4; ++i) FG_TRY(convl_pack(c, n->Dc[i], n->PD));
  FG_TRY(convl_pack(c, n->DF1, n->PD));
  FG_TRY(convl_pack(c, n->DE1, n->PD));
  FG_TRY(convl_pack(c, n->DE2, n->PD));
  n->D_packed = true;
  n->D_pack_impl = pack_key(c);
  return FG_OK;
}

// ---------------------------------------------------------------------------------------------------
// G16
// ---------------------------------------------------------------------------------------------------
// *parts (in: want BatchNorm partials; out: how many tiles wrote one into c->bn_parts, 0 = none)
int ups_fwd(fg_s16* n, UpsL& U, const float* h, float* z, int B, int* parts) {
  fg_ctx* c = n->c;
  const ConvGeom g = U.geom(B);
  const bool want = *parts != 0;
  *parts = 0;
  if (!use_tc_wgrad(c, U.geom(n->maxB))) {
    ScopedTimer tm(c, U.tf);
    return k_conv_simt(c, h, U.Wp, n->PG + U.b_off, z, g);
  }
  const int64_t nh = (int64_t)B * (U.H / 2) * (U.H / 2) * U.Cin;
  const bool h16 = f16_on(c);
  if (h16) {
    FG_TRY(tc_amax(c, h, nh, U.sx));
    FG_TRY(tc_split_h(c, h, U.h_hi, U.h_lo, nh, U.sx));
  } else {
    FG_TRY(tc_split(c, h, U.h_hi, U.h_lo, nh));  // kept for the weight gradient
  }
  ScopedTimer tm(c, U.tf);
  float* st = want && c->bn_epilogue ? c->bn_parts : nullptr;
  return tc_conv_fwd(c, U.h_hi, U.h_lo, U.Wf_hi, U.Wf_lo, n->PG + U.b_off, z, g, 2, st, st ? parts : nullptr, h16,
                     h16 ? U.sx + 1 : nullptr);
}
// dW += wgrad; dh = dgrad.  *pooled: dh already is the gradient of the LOW-RES input (tensor-core path folds the 2x2 sum of
// the upsample backward into the dgrad GEMM); otherwise dh is the full-resolution gradient the consumer sums 2x2.
int ups_bwd(fg_s16* n, UpsL& U, const float* h, const float* dz, float* dh, int B, bool* pooled) {
  fg_ctx* c = n->c;
  const ConvGeom g = U.geom(B);
  if (!use_tc_wgrad(c, U.geom(n->maxB))) {
    {
      ScopedTimer tm(c, U.tw);
      FG_TRY(k_wgrad_simt(c, h, dz, n->ws, g));
    }
    FG_TRY(k_unpack_wgrad(c, n->ws, n->gG + U.w_off, U.Cout, U.Cin, 25, 0, 0, 0, 0));
    *pooled = false;
    ScopedTimer tm(c, U.td);
    return k_conv_simt(c, dz, U.Wpd, nullptr, dh, ConvGeom{B, U.H, U.H, U.Cout, U.Cin, 5, 1});
  }
  const int64_t ndz = (int64_t)B * U.H * U.H * U.Cout;
  const bool h16 = f16_on(c);
  float* sdy = n->env.sdy;
  if (h16) {
    FG_TRY(tc_amax(c, dz, ndz, sdy));
    FG_TRY(tc_split_h(c, dz, n->dy_hi, n->dy_lo, ndz, sdy));
  } else {
    FG_TRY(tc_split(c, dz, n->dy_hi, n->dy_lo, ndz));
  }
  {
    ScopedTimer tm(c, U.tw);
    FG_TRY(tc_conv_wgrad(c, U.h_hi, U.h_lo, n->dy_hi, n->dy_lo, n->ws, g, h16, h16 ? sdy + 1 : nullptr, h16 ? U.sx + 1 : nullptr));
  }
  FG_TRY(tc_combine_collapsed_wgrad(c, n->ws, n->gG + U.w_off, U.Cout, U.Cin));
  *pooled = true;
  ScopedTimer tm(c, U.td);
  return tc_conv_dgrad_ups(c, n->dy_hi, n->dy_lo, U.Wd_hi, U.Wd_lo, dh, g, h16, h16 ? sdy + 1 : nullptr);
}

// BatchNorm statistics of layer i (0: 256 channels at 8x8, 1: 128 channels at 16x16) -> bn_mean / bn_istd
int bn_stats(fg_s16* n, int i, const float* z, int B, bool training, int parts) {
  fg_ctx* c = n->c;
  const int Cc = i == 0 ? 256 : 128;
  const int64_t P = (int64_t)B * (i == 0 ? 64 : 256);
  float *rm = n->bnG + (i == 0 ? 0 : 512), *rv = rm + Cc;
  if (!training) return k_bn_eval_prep(c, rm, rv, n->bn_mean[i], n->bn_istd[i], Cc);
  if (parts) return k_bn_finalize_parts(c, c->bn_parts, parts, n->bn_mean[i], n->bn_istd[i], rm, rv, P, Cc);
  FG_TRY(k_bn_stats(c, z, c->bn_acc, P, Cc));
  return k_bn_finalize(c, c->bn_acc, n->bn_mean[i], n->bn_istd[i], rm, rv, P, Cc);
}

// noise: device [B][100]; the image lands in G_y (NHWC [B][16][16][C])
int G_forward(fg_s16* n, const float* noise, int B, bool training) {
  fg_ctx* c = n->c;
  FG_REQUIRE(B >= 1 && B <= n->maxB, "s16 G forward: batch %d out of range [1,%d]", B, n->maxB);
  FG_TRY(pack_G(n));
  const float* P = n->PG;
  if (noise != n->G_x) FG_CUDA(cudaMemcpyAsync(n->G_x, noise, sizeof(float) * B * 100, cudaMemcpyDeviceToDevice, c->stream));
  FG_TRY(convl_fwd(n->env, n->GL1, n->G_x, P, n->G_z0, B));
  FG_TRY(k_prelu_fwd(c, n->G_z0, P + n->Ga[0], n->G_h0, (int64_t)B * 2048));
  int parts = training ? 1 : 0;
  FG_TRY(ups_fwd(n, n->GU[0], n->G_h0, n->G_z1, B, &parts));
  FG_TRY(bn_stats(n, 0, n->G_z1, B, training, parts));
  FG_TRY(k_bn_prelu_apply(c, n->G_z1, n->bn_mean[0], n->bn_istd[0], P + n->Gg[0], P + n->Gbe[0], P + n->Ga[1], n->G_h1,
                          (int64_t)B * 64, 256));
  parts = training ? 1 : 0;
  FG_TRY(ups_fwd(n, n->GU[1], n->G_h1, n->G_z2, B, &parts));
  FG_TRY(bn_stats(n, 1, n->G_z2, B, training, parts));
  FG_TRY(k_bn_prelu_apply(c, n->G_z2, n->bn_mean[1], n->bn_istd[1], P + n->Gg[1], P + n->Gbe[1], P + n->Ga[2], n->G_h2,
                          (int64_t)B * 256, 128));
  FG_TRY(convl_fwd(n->env, n->GC3, n->G_h2, P, n->G_z3, B));
  FG_TRY(k_sigmoid_fwd(c, n->G_z3, n->G_y, (int64_t)B * 256 * n->C));
  n->G_B = B;
  n->G_train = training;
  n->G_valid = true;
  return FG_OK;
}
// dy: NHWC [B][16][16][C]; accumulates into gG; dnoise (device [B][100]) may be null
int G_backward(fg_s16* n, const float* dy, float* dnoise) {
  fg_ctx* c = n->c;
  if (!n->G_valid || !n->G_train) {
    fg_set_error("s16 G backward needs a preceding training-mode G forward");
    return FG_ERR_STATE;
  }
  const int B = n->G_B;
  const float* P = n->PG;
  float* G = n->gG;
  FG_TRY(k_sigmoid_bwd(c, dy, n->G_y, n->G_dz3, (int64_t)B * 256 * n->C));
  FG_TRY(convl_bwd(n->env, n->GC3, n->G_h2, n->G_dz3, G, n->G_dfull, B));
  bool pooled = false;
  // BN2 + PReLU, C2
  FG_TRY(k_bn_prelu_bwd_reduce(c, n->G_dfull, n->G_z2, n->bn_mean[1], n->bn_istd[1], P + n->Gg[1], P + n->Gbe[1], P + n->Ga[2],
                               c->bn_acc, G + n->Ga[2], B, 16, 16, 128, 0));
  FG_TRY(k_bn_bwd_finalize(c, c->bn_acc, n->bn_mg, G + n->Gg[1], G + n->Gbe[1], (int64_t)B * 256, 128));
  FG_TRY(k_bn_prelu_bwd_apply(c, n->G_dfull, n->G_z2, n->bn_mean[1], n->bn_istd[1], P + n->Gg[1], P + n->Gbe[1], P + n->Ga[2],
                              n->bn_mg, n->G_dz, B, 16, 16, 128, 0, nullptr, nullptr, G + n->GU[1].b_off));
  FG_TRY(ups_bwd(n, n->GU[1], n->G_h1, n->G_dz, n->G_dfull, B, &pooled));
  // BN1 + PReLU, C1 (the 2x2 sum = backward of the nearest upsample is folded into the loads when not pooled yet)
  FG_TRY(k_bn_prelu_bwd_reduce(c, n->G_dfull, n->G_z1, n->bn_mean[0], n->bn_istd[0], P + n->Gg[0], P + n->Gbe[0], P + n->Ga[1],
                               c->bn_acc, G + n->Ga[1], B, 8, 8, 256, pooled ? 0 : 1));
  FG_TRY(k_bn_bwd_finalize(c, c->bn_acc, n->bn_mg, G + n->Gg[0], G + n->Gbe[0], (int64_t)B * 64, 256));
  FG_TRY(k_bn_prelu_bwd_apply(c, n->G_dfull, n->G_z1, n->bn_mean[0], n->bn_istd[0], P + n->Gg[0], P + n->Gbe[0], P + n->Ga[1],
                              n->bn_mg, n->G_dz, B, 8, 8, 256, pooled ? 0 : 1, nullptr, nullptr, G + n->GU[0].b_off));
  FG_TRY(ups_bwd(n, n->GU[0], n->G_h0, n->G_dz, n->G_dfull, B, &pooled));
  FG_TRY(k_prelu_bwd(c, n->G_dfull, n->G_z0, P + n->Ga[0], n->G_dz0, G + n->Ga[0], B, 4, 4, 128, pooled ? 0 : 1));
  return convl_bwd(n->env, n->GL1, n->G_x, n->G_dz0, G, dnoise, B);
}

// ---------------------------------------------------------------------------------------------------
// D16
// ---------------------------------------------------------------------------------------------------
// x: NHWC device [B][16][16][C]; keep flags already in D_masks when training
int D_forward(fg_s16* n, const float* x, int B, bool training) {
  fg_ctx* c = n->c;
  FG_REQUIRE(B >= 1 && B <= n->maxB, "s16 D forward: batch %d out of range [1,%d]", B, n->maxB);
  FG_TRY(pack_D(n));
  const float* P = n->PD;
  if (x != n->D_x) FG_CUDA(cudaMemcpyAsync(n->D_x, x, sizeof(float) * (size_t)B * 256 * n->C, cudaMemcpyDeviceToDevice, c->stream));
  const float* masks = training ? n->D_masks : nullptr;
  // ---- conv branch ----
  FG_TRY(convl_fwd(n->env, n->Dc[0], n->D_x, P, n->D_z[0], B));
  FG_TRY(k_prelu_fwd(c, n->D_z[0], P + n->Dca[0], n->D_h[0], (int64_t)B * 256 * 128));
  FG_TRY(convl_fwd(n->env, n->Dc[1], n->D_h[0], P, n->D_z[1], B));
  FG_TRY(k_prelu_fwd(c, n->D_z[1], P + n->Dca[1], n->D_h[1], (int64_t)B * 256 * 128));
  avgpool2_fwd_kernel<<<grid_for((int64_t)B * 64 * 128, 256), 256, 0, c->stream>>>(n->D_h[1], n->D_p1, B, 16, 16, 128);
  LAUNCH_CHECK(c);
  FG_TRY(convl_fwd(n->env, n->Dc[2], n->D_p1, P, n->D_zfull, B));  // stride 1 at 8x8 ...
  subsample2_kernel<<<grid_for((int64_t)B * 16 * 512, 256), 256, 0, c->stream>>>(n->D_zfull, n->D_z[2], B, 8, 8, 512);  // ... -> 4x4
  LAUNCH_CHECK(c);
  FG_TRY(k_prelu_fwd(c, n->D_z[2], P + n->Dca[2], n->D_h[2], (int64_t)B * 16 * 512));
  FG_TRY(convl_fwd(n->env, n->Dc[3], n->D_h[2], P, n->D_zfull, B));  // stride 1 at 4x4 ...
  subsample2_kernel<<<grid_for((int64_t)B * 4 * 1024, 256), 256, 0, c->stream>>>(n->D_zfull, n->D_z[3], B, 4, 4, 1024);  // ... -> 2x2
  LAUNCH_CHECK(c);
  FG_TRY(k_prelu_fwd(c, n->D_z[3], P + n->Dca[3], n->D_h[3], (int64_t)B * 4096));
  plane_dropout_kernel<<<grid_for((int64_t)B * 4096, 256), 256, 0, c->stream>>>(n->D_h[3], masks, kS16Mask, 0, 0.5f, n->D_d3, B, 4,
                                                                                1024);
  LAUNCH_CHECK(c);
  FG_TRY(convl_fwd(n->env, n->DF1, n->D_d3, P, n->D_zf, B));
  FG_TRY(k_prelu_fwd(c, n->D_zf, P + n->Daf, n->D_hf, (int64_t)B * 1024));
  // ---- dense branch ----
  FG_TRY(convl_fwd(n->env, n->DE1, n->D_x, P, n->D_ze1, B));
  FG_TRY(k_prelu_fwd(c, n->D_ze1, P + n->Dae1, n->D_he1, (int64_t)B * 128));
  const float* de1 = n->D_he1;
  if (training) {  // nn.Dropout() (p = 0.5, v2): keep * 2 in training, identity in evaluation
    FG_TRY(k_dropout_nhwc(c, n->D_he1, n->D_masks, kS16Mask, 1024, 1, 128, 2.0f, n->D_de1, B));
    de1 = n->D_de1;
  }
  FG_TRY(convl_fwd(n->env, n->DE2, de1, P, n->D_ze2, B));
  FG_TRY(k_prelu_fwd(c, n->D_ze2, P + n->Dae2, n->D_he2, (int64_t)B * 128));
  // ---- JoinTable(2) -> Linear(1152, 1) ----
  join2_kernel<<<grid_for((int64_t)B * 1152, 256), 256, 0, c->stream>>>(n->D_hf, n->D_he2, n->D_joint, B, 1024, 128);
  LAUNCH_CHECK(c);
  FG_TRY(k_gemv_fwd(c, n->D_joint, P + n->DJW, P + n->DJb, n->D_logit, B, 1152));
  n->D_B = B;
  n->D_train = training;
  n->D_valid = true;
  return FG_OK;
}
// dlogit [B]; want_dx: the image gradient (sum over the two branches, nn.ConcatTable backward) into D_dx (NHWC)
int D_backward(fg_s16* n, const float* dlogit, bool want_wgrad, bool want_dx) {
  fg_ctx* c = n->c;
  if (!n->D_valid) {
    fg_set_error("s16 D backward needs a preceding D forward");
    return FG_ERR_STATE;
  }
  const int B = n->D_B;
  const float* P = n->PD;
  float* G = want_wgrad ? n->gD : nullptr;
  const bool tr = n->D_train;
  const float* masks = tr ? n->D_masks : nullptr;
  if (G) FG_TRY(k_gemv_wgrad_add(c, n->D_joint, dlogit, G + n->DJW, G + n->DJb, B, 1152));
  FG_TRY(k_gemv_dgrad(c, dlogit, P + n->DJW, n->D_djoint, B, 1152));
  split2_kernel<<<grid_for((int64_t)B * 1152, 256), 256, 0, c->stream>>>(n->D_djoint, n->D_dhf, n->D_dhe2, B, 1024, 128);
  LAUNCH_CHECK(c);
  float *cur = n->ga, *oth = n->gb;  // gradient ping-pong: every stage reads `cur`, writes `oth`, then they swap
  {  // dense branch
    FG_TRY(k_prelu_bwd(c, n->D_dhe2, n->D_ze2, P + n->Dae2, cur, G ? G + n->Dae2 : nullptr, B, 1, 1, 128, 0));
    FG_TRY(convl_bwd(n->env, n->DE2, tr ? n->D_de1 : n->D_he1, cur, G, oth, B));
    std::swap(cur, oth);
    if (tr) {
      FG_TRY(k_dropout_nhwc(c, cur, n->D_masks, kS16Mask, 1024, 1, 128, 2.0f, oth, B));
      std::swap(cur, oth);
    }
    FG_TRY(k_prelu_bwd(c, cur, n->D_ze1, P + n->Dae1, oth, G ? G + n->Dae1 : nullptr, B, 1, 1, 128, 0));
    std::swap(cur, oth);
    FG_TRY(convl_bwd(n->env, n->DE1, n->D_x, cur, G, want_dx ? n->D_dx2 : nullptr, B));
  }
  {  // conv branch
    FG_TRY(k_prelu_bwd(c, n->D_dhf, n->D_zf, P + n->Daf, cur, G ? G + n->Daf : nullptr, B, 1, 1, 1024, 0));
    FG_TRY(convl_bwd(n->env, n->DF1, n->D_d3, cur, G, oth, B));  // -> gradient of the View(4096) input, [B][2][2][1024]
    std::swap(cur, oth);
    plane_dropout_kernel<<<grid_for((int64_t)B * 4096, 256), 256, 0, c->stream>>>(cur, masks, kS16Mask, 0, 0.5f, oth, B, 4, 1024);
    LAUNCH_CHECK(c);
    std::swap(cur, oth);
    FG_TRY(k_prelu_bwd(c, cur, n->D_z[3], P + n->Dca[3], oth, G ? G + n->Dca[3] : nullptr, B, 2, 2, 1024, 0));
    std::swap(cur, oth);
    zero_insert2_kernel<<<grid_for((int64_t)B * 16 * 1024, 256), 256, 0, c->stream>>>(cur, oth, B, 4, 4, 1024);
    LAUNCH_CHECK(c);
    std::swap(cur, oth);
    FG_TRY(convl_bwd(n->env, n->Dc[3], n->D_h[2], cur, G, oth, B));  // -> [B][4][4][512]
    std::swap(cur, oth);
    FG_TRY(k_prelu_bwd(c, cur, n->D_z[2], P + n->Dca[2], oth, G ? G + n->Dca[2] : nullptr, B, 4, 4, 512, 0));
    std::swap(cur, oth);
    zero_insert2_kernel<<<grid_for((int64_t)B * 64 * 512, 256), 256, 0, c->stream>>>(cur, oth, B, 8, 8, 512);
    LAUNCH_CHECK(c);
    std::swap(cur, oth);
    FG_TRY(convl_bwd(n->env, n->Dc[2], n->D_p1, cur, G, oth, B));  // -> [B][8][8][128]
    std::swap(cur, oth);
    avgpool2_bwd_kernel<<<grid_for((int64_t)B * 256 * 128, 256), 256, 0, c->stream>>>(cur, oth, B, 16, 16, 128);
    LAUNCH_CHECK(c);
    std::swap(cur, oth);
    FG_TRY(k_prelu_bwd(c, cur, n->D_z[1], P + n->Dca[1], oth, G ? G + n->Dca[1] : nullptr, B, 16, 16, 128, 0));
    std::swap(cur, oth);
    FG_TRY(convl_bwd(n->env, n->Dc[1], n->D_h[0], cur, G, oth, B));
    std::swap(cur, oth);
    FG_TRY(k_prelu_bwd(c, cur, n->D_z[0], P + n->Dca[0], oth, G ? G + n->Dca[0] : nullptr, B, 16, 16, 128, 0));
    std::swap(cur, oth);
    FG_TRY(convl_bwd(n->env, n->Dc[0], n->D_x, cur, G, want_dx ? n->D_dx : nullptr, B));
  }
  if (want_dx) FG_TRY(k_add(c, n->D_dx, n->D_dx2, n->D_dx, (int64_t)B * 256 * n->C));
  return FG_OK;
}

// penalty -> clamp -> interruptable optimizer on the flat vectors (adversarial.lua:219-231, interruptable_optimizers.lua)
int optim(fg_s16* n, int net, const fg_hyper* h, float grad_scale) {
  fg_ctx* c = n->c;
  const bool isD = net == FG_NET_D;
  float *p = isD ? n->PD : n->PG, *g = isD ? n->gD : n->gG, *m = isD ? n->mD : n->mG, *v = isD ? n->vD : n->vG;
  const int64_t cnt = isD ? n->nD : n->nG;
  const float l1 = isD ? h->D_L1 : h->G_L1, l2 = isD ? h->D_L2 : h->G_L2;
  const bool pen = l1 != 0.f || l2 != 0.f;
  const float l1_grad = !pen ? 0.f : (isD ? l1 : l2);  // adversarial.lua:223 scales sign(p) by G_L2
  if (pen) FG_TRY(k_penalty_loss(c, p, cnt, l1, l2, isD ? &n->dstats->loss_D : &n->dstats->loss_G));
  FG_TRY(k_optim_update(c, isD ? c->opt_D : c->opt_G, p, g, m, v, cnt, h->beta1, h->beta2, h->eps,
                        isD ? c->sgd_mom_D : c->sgd_mom_G, l1_grad, pen ? l2 : 0.f, isD ? h->D_clamp : h->G_clamp, grad_scale,
                        isD ? &n->dstats->step_D : &n->dstats->step_G, isD ? &n->dstats->do_train_D : &n->dstats->do_train_G,
                        isD ? &n->dstats->t_D : &n->dstats->t_G));
  if (isD) n->D_packed = false; else n->G_packed = false;
  return FG_OK;
}
// the accuracy gate, t += 1 and the step size, on this net's own statistics block (kernel shared with the 32x32 loop)
int gate_prep(fg_s16* n, int net, const fg_hyper* h, const float* tail4, int B) {
  fg_ctx* c = n->c;
  DeviceStats* sd = c->dstats;
  float* sa = c->acc_hist;
  c->dstats = n->dstats;
  c->acc_hist = n->acc_hist;
  const int r = k_gate_and_prep(c, net, h, tail4, B, (float)c->world);
  c->dstats = sd;
  c->acc_hist = sa;
  return r;
}

// one iteration of the adversarial.lua loop body (D_iterations = G_iterations = 1) on the 16x16 nets
int train_step(fg_s16* n, const fg_hyper* h, int B, const float* real, const float* noiseD, const float* noiseG,
               const float* masksD, const float* masksG, uint64_t seed) {
  fg_ctx* c = n->c;
  const int Bh = B / 2, C = n->C;
  const size_t img = (size_t)C * 256;
  const float inv_world = 1.0f / (float)c->world;
  // ---- D step (adversarial.lua:240-268) ----
  FG_TRY(G_forward(n, noiseD, Bh, true));  // createImages: G in training mode (nn_utils.lua:52)
  FG_TRY(k_nchw_to_nhwc(c, real, n->D_x, Bh, C, 256));
  FG_CUDA(cudaMemcpyAsync(n->D_x + Bh * img, n->G_y, sizeof(float) * Bh * img, cudaMemcpyDeviceToDevice, c->stream));
  if (masksD)
    FG_CUDA(cudaMemcpyAsync(n->D_masks, masksD, sizeof(float) * (size_t)B * kS16Mask, cudaMemcpyDeviceToDevice, c->stream));
  else
    FG_TRY(k_bernoulli_keep(c, n->D_masks, (int64_t)B * kS16Mask, 1, 0.5f, c->seed_dev));
  FG_CUDA(cudaMemsetAsync(n->gD, 0, sizeof(float) * (n->nD + kGradTail), c->stream));
  FG_TRY(D_forward(n, n->D_x, B, true));
  FG_TRY(k_sigmoid_bce(c, n->D_logit, n->D_out, n->D_dlogit, &n->dstats->loss_D, n->gD + n->nD, B, Bh));
  FG_TRY(D_backward(n, n->D_dlogit, true, false));
  if (c->world > 1) FG_TRY(net_allreduce(c, n->gD, n->nD + kGradTail));
  FG_TRY(gate_prep(n, FG_NET_D, h, n->gD + n->nD, B));
  FG_TRY(optim(n, FG_NET_D, h, inv_world));
  // ---- G step (adversarial.lua:275-288) ----
  FG_CUDA(cudaMemsetAsync(n->gG, 0, sizeof(float) * (n->nG + kGradTail), c->stream));
  FG_TRY(G_forward(n, noiseG, B, true));
  if (masksG)
    FG_CUDA(cudaMemcpyAsync(n->D_masks, masksG, sizeof(float) * (size_t)B * kS16Mask, cudaMemcpyDeviceToDevice, c->stream));
  else
    FG_TRY(k_bernoulli_keep(c, n->D_masks, (int64_t)B * kS16Mask, 2, 0.5f, c->seed_dev));
  FG_TRY(D_forward(n, n->G_y, B, true));
  FG_TRY(k_sigmoid_bce(c, n->D_logit, n->D_out, n->D_dlogit, &n->dstats->loss_G, n->gG + n->nG, B, B));
  FG_TRY(D_backward(n, n->D_dlogit, false, true));  // D's weight grads are discarded by the reference (:209 vs :92)
  FG_TRY(G_backward(n, n->D_dx, nullptr));
  if (c->world > 1) FG_TRY(net_allreduce(c, n->gG, n->nG + kGradTail));
  FG_TRY(gate_prep(n, FG_NET_G, h, n->gG + n->nG, B));
  FG_TRY(optim(n, FG_NET_G, h, inv_world));
  FG_CUDA(cudaMemcpyAsync(n->hstats, n->dstats, sizeof(DeviceStats), cudaMemcpyDeviceToHost, c->stream));
  return FG_OK;
}
}  // namespace

#define ENTER(n)                                         \
  do {                                                   \
    if (!(n) || !(n)->c) {                               \
      fg_set_error("null fg_s16");                       \
      return FG_ERR_INVALID;                             \
    }                                                    \
    FG_CUDA(cudaSetDevice((n)->c->device));              \
  } while (0)

extern "C" {

int fg_s16_create(fg_ctx* ctx, fg_s16** out) {
  if (!ctx || !out) {
    fg_set_error("fg_s16_create: null argument");
    return FG_ERR_INVALID;
  }
  *out = nullptr;
  FG_CUDA(cudaSetDevice(ctx->device));
  fg_s16* n = new fg_s16();
  n->c = ctx;
  n->maxB = ctx->maxB;
  n->C = ctx->C;
  const int r = s16_alloc(n);
  if (r != FG_OK) {
    fg_s16_destroy(n);
    return r;
  }
  *out = n;
  return FG_OK;
}
int fg_s16_destroy(fg_s16* n) {
  if (!n) return FG_OK;
  if (n->c) {
    cudaSetDevice(n->c->device);
    cudaStreamSynchronize(n->c->stream);
  }
  for (auto& g : n->graphs)
    if (g.exec) cudaGraphExecDestroy(g.exec);
  for (void* p : n->allocs) cudaFree(p);
  if (n->hstats) cudaFreeHost(n->hstats);
  delete n;
  return FG_OK;
}
int64_t fg_s16_param_count(int net, int channels) {
  fg_s16 tmp;
  tmp.C = channels;
  make_layouts(&tmp);
  return net == FG_NET_D ? tmp.nD : tmp.nG;
}
int fg_s16_mask_per_sample(void) { return kS16Mask; }

int fg_s16_set_params(fg_s16* n, int net, const float* src) {
  ENTER(n);
  FG_REQUIRE(src && (net == FG_NET_G || net == FG_NET_D), "fg_s16_set_params: bad arguments");
  const bool isD = net == FG_NET_D;
  FG_CUDA(cudaMemcpyAsync(isD ? n->PD : n->PG, src, sizeof(float) * (isD ? n->nD : n->nG), cudaMemcpyDefault, n->c->stream));
  FG_CUDA(cudaStreamSynchronize(n->c->stream));
  if (isD) n->D_packed = false; else n->G_packed = false;
  return FG_OK;
}
int fg_s16_get_params(fg_s16* n, int net, float* dst) {
  ENTER(n);
  FG_REQUIRE(dst && (net == FG_NET_G || net == FG_NET_D), "fg_s16_get_params: bad arguments");
  const bool isD = net == FG_NET_D;
  return fg_to_user(n->c, dst, isD ? n->PD : n->PG, isD ? n->nD : n->nG);
}
int fg_s16_get_grads(fg_s16* n, int net, float* dst) {
  ENTER(n);
  FG_REQUIRE(dst && (net == FG_NET_G || net == FG_NET_D), "fg_s16_get_grads: bad arguments");
  const bool isD = net == FG_NET_D;
  return fg_to_user(n->c, dst, isD ? n->gD : n->gG, isD ? n->nD : n->nG);
}
int fg_s16_zero_grads(fg_s16* n, int net) {
  ENTER(n);
  const bool isD = net == FG_NET_D;
  FG_CUDA(cudaMemsetAsync(isD ? n->gD : n->gG, 0, sizeof(float) * ((isD ? n->nD : n->nG) + kGradTail), n->c->stream));
  return FG_OK;
}
float* fg_s16_params_ptr(fg_s16* n, int net) { return !n ? nullptr : (net == FG_NET_D ? n->PD : n->PG); }
float* fg_s16_grads_ptr(fg_s16* n, int net) { return !n ? nullptr : (net == FG_NET_D ? n->gD : n->gG); }

int fg_s16_set_adam_state(fg_s16* n, int net, const float* m, const float* v, int t) {
  ENTER(n);
  const bool isD = net == FG_NET_D;
  const size_t cnt = isD ? n->nD : n->nG;
  if (m) FG_CUDA(cudaMemcpyAsync(isD ? n->mD : n->mG, m, sizeof(float) * cnt, cudaMemcpyDefault, n->c->stream));
  if (v) FG_CUDA(cudaMemcpyAsync(isD ? n->vD : n->vG, v, sizeof(float) * cnt, cudaMemcpyDefault, n->c->stream));
  FG_CUDA(cudaMemcpyAsync(isD ? &n->dstats->t_D : &n->dstats->t_G, &t, sizeof(int), cudaMemcpyHostToDevice, n->c->stream));
  FG_CUDA(cudaStreamSynchronize(n->c->stream));
  return FG_OK;
}
int fg_s16_get_adam_state(fg_s16* n, int net, float* m, float* v, int* t) {
  ENTER(n);
  const bool isD = net == FG_NET_D;
  const size_t cnt = isD ? n->nD : n->nG;
  if (m) FG_TRY(fg_to_user(n->c, m, isD ? n->mD : n->mG, cnt));
  if (v) FG_TRY(fg_to_user(n->c, v, isD ? n->vD : n->vG, cnt));
  if (t) {
    FG_CUDA(cudaMemcpyAsync(t, isD ? &n->dstats->t_D : &n->dstats->t_G, sizeof(int), cudaMemcpyDeviceToHost, n->c->stream));
    FG_CUDA(cudaStreamSynchronize(n->c->stream));
  }
  return FG_OK;
}
// running_mean / running_var of G's two nn.SpatialBatchNormalization layers: [mean1 256][var1 256][mean2 128][var2 128]
int fg_s16_set_bn_state(fg_s16* n, const float* src768) {
  ENTER(n);
  FG_REQUIRE(src768, "fg_s16_set_bn_state: null source");
  FG_CUDA(cudaMemcpyAsync(n->bnG, src768, sizeof(float) * 768, cudaMemcpyDefault, n->c->stream));
  FG_CUDA(cudaStreamSynchronize(n->c->stream));
  return FG_OK;
}
int fg_s16_get_bn_state(fg_s16* n, float* dst768) {
  ENTER(n);
  FG_REQUIRE(dst768, "fg_s16_get_bn_state: null destination");
  return fg_to_user(n->c, dst768, n->bnG, 768);
}

// noise [B][100] -> images [B][C][16][16] (NCHW; host or device pointers).  training != 0: batch statistics + running
// stat update (nn_utils.lua:52 createImages leaves G in training mode); 0: evaluate() with the running statistics.
int fg_s16_G_forward(fg_s16* n, const float* noise, int B, int training, float* img_out) {
  ENTER(n);
  FG_REQUIRE(noise && B >= 1 && B <= n->maxB, "fg_s16_G_forward: bad arguments (batch %d, max %d)", B, n->maxB);
  const float* nd;
  FG_TRY(fg_to_dev(n->c, noise, (size_t)B * 100, n->in_b, &nd));
  FG_TRY(G_forward(n, nd, B, training != 0));
  if (img_out) {
    FG_TRY(k_nhwc_to_nchw(n->c, n->G_y, n->io, B, n->C, 256));
    FG_TRY(fg_to_user(n->c, img_out, n->io, (size_t)B * n->C * 256));
  }
  return FG_OK;
}
int fg_s16_G_backward(fg_s16* n, const float* d_img, float* d_noise) {
  ENTER(n);
  FG_REQUIRE(d_img, "fg_s16_G_backward: null gradient");
  const float* dd;
  FG_TRY(fg_to_dev(n->c, d_img, (size_t)n->G_B * n->C * 256, n->in_a, &dd));
  FG_TRY(k_nchw_to_nhwc(n->c, dd, n->io, n->G_B, n->C, 256));
  FG_TRY(G_backward(n, n->io, d_noise ? n->in_c : nullptr));
  if (d_noise) FG_TRY(fg_to_user(n->c, d_noise, n->in_c, (size_t)n->G_B * 100));
  return FG_OK;
}
int fg_s16_D_forward(fg_s16* n, const float* img, int B, int training, const float* masks, uint64_t seed, float* out) {
  ENTER(n);
  FG_REQUIRE(img && B >= 1 && B <= n->maxB, "fg_s16_D_forward: bad arguments (batch %d, max %d)", B, n->maxB);
  fg_ctx* c = n->c;
  const float* id;
  FG_TRY(fg_to_dev(c, img, (size_t)B * n->C * 256, n->in_a, &id));
  FG_TRY(k_nchw_to_nhwc(c, id, n->D_x, B, n->C, 256));
  if (training) {
    if (masks)
      FG_CUDA(cudaMemcpyAsync(n->D_masks, masks, sizeof(float) * (size_t)B * kS16Mask, cudaMemcpyDefault, c->stream));
    else
      FG_TRY(k_bernoulli_keep(c, n->D_masks, (int64_t)B * kS16Mask, seed, 0.5f));
  }
  FG_TRY(D_forward(n, n->D_x, B, training != 0));
  FG_TRY(k_sigmoid_fwd(c, n->D_logit, n->D_out, B));
  if (out) FG_TRY(fg_to_user(c, out, n->D_out, B));
  return FG_OK;
}
int fg_s16_D_backward(fg_s16* n, const float* d_out, int want_wgrad, float* d_img) {
  ENTER(n);
  FG_REQUIRE(d_out, "fg_s16_D_backward: null gradient");
  fg_ctx* c = n->c;
  const float* dd;
  FG_TRY(fg_to_dev(c, d_out, (size_t)n->D_B, n->in_b, &dd));
  FG_TRY(k_sigmoid_bwd(c, dd, n->D_out, n->D_dlogit, n->D_B));
  FG_TRY(D_backward(n, n->D_dlogit, want_wgrad != 0, d_img != nullptr));
  if (d_img) {
    FG_TRY(k_nhwc_to_nchw(c, n->D_dx, n->io, n->D_B, n->C, 256));
    FG_TRY(fg_to_user(c, d_img, n->io, (size_t)n->D_B * n->C * 256));
  }
  return FG_OK;
}

// data parallel: rank 0's parameters, optimizer moments, step counters and BatchNorm running statistics to every rank
int fg_s16_dp_broadcast_params(fg_s16* n) {
  ENTER(n);
  fg_ctx* c = n->c;
  if (c->world <= 1) return FG_OK;
  FG_TRY(net_group(true));
  const size_t bG = n->nG * sizeof(float), bD = n->nD * sizeof(float);
  FG_TRY(net_broadcast(c, n->PG, bG));
  FG_TRY(net_broadcast(c, n->PD, bD));
  FG_TRY(net_broadcast(c, n->mG, bG));
  FG_TRY(net_broadcast(c, n->vG, bG));
  FG_TRY(net_broadcast(c, n->mD, bD));
  FG_TRY(net_broadcast(c, n->vD, bD));
  FG_TRY(net_broadcast(c, n->bnG, 768 * sizeof(float)));
  FG_TRY(net_broadcast(c, n->dstats, sizeof(DeviceStats)));
  FG_TRY(net_broadcast(c, n->acc_hist, kAccHistMax * sizeof(float)));
  FG_TRY(net_group(false));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  n->G_packed = n->D_packed = false;
  return FG_OK;
}

int fg_s16_train_step(fg_s16* n, const fg_hyper* h, int B, const float* real, const float* noise_D, const float* noise_G,
                      const float* masks_D, const float* masks_G, uint64_t seed, fg_step_stats* stats) {
  ENTER(n);
  FG_REQUIRE(h && real && noise_D && noise_G, "fg_s16_train_step: null input");
  FG_REQUIRE(B >= 4 && B % 2 == 0 && B <= n->maxB, "fg_s16_train_step: batch %d must be even, >= 4 and <= max_batch %d", B,
             n->maxB);
  fg_ctx* c = n->c;
  const float *rd, *nd, *ng, *md = nullptr, *mg = nullptr;
  FG_TRY(fg_to_dev(c, real, (size_t)(B / 2) * n->C * 256, n->in_a, &rd));
  FG_TRY(fg_to_dev(c, noise_D, (size_t)(B / 2) * 100, n->in_b, &nd));
  FG_TRY(fg_to_dev(c, noise_G, (size_t)B * 100, n->in_c, &ng));
  if (masks_D) FG_TRY(fg_to_dev(c, masks_D, (size_t)B * kS16Mask, n->in_m1, &md));
  if (masks_G) FG_TRY(fg_to_dev(c, masks_G, (size_t)B * kS16Mask, n->in_m2, &mg));
  {  // eager the first time, then a captured CUDA graph of the step (nets.cu net_graph_run); the seed is read on the device
    std::vector<uint8_t> key;
    auto add = [&key](const void* p, size_t nb) { key.insert(key.end(), (const uint8_t*)p, (const uint8_t*)p + nb); };
    const void* ptrs[] = {rd, nd, ng, md, mg, (const void*)c->stream, c->nccl_comm};
    const int meta[3] = {c->graph_epoch, B, pack_key(c)};
    add(meta, sizeof(meta));
    add(h, sizeof(*h));
    add(ptrs, sizeof(ptrs));
    FG_TRY(net_graph_run(
        c, n->graphs, key, seed, [&]() { return train_step(n, h, B, rd, nd, ng, md, mg, 0); },
        [n]() { n->G_packed = n->D_packed = false; }, true));
  }
  if (stats) {
    FG_CUDA(cudaStreamSynchronize(c->stream));
    const DeviceStats& s = *n->hstats;
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
