// The `--scale 16` nets of train.lua (models.create_G / create_D pick them when dimensions[2] == 16, models.lua:87-104)
// and the adversarial.lua loop body on them:
//   G16 = models.lua:27-51   create_G_decoder_upsampling16: Linear(100, 128*4*4) View(128,4,4) PReLU | Up2 conv(128->256,5)
//         BN PReLU | Up2 conv(256->128,5) BN PReLU | conv(128->C,3) Sigmoid  -- the 32x32 generator with every size halved
//   D16 = models.lua:279-316 create_D16_d: ConcatTable{conv branch, dense branch} JoinTable(2) Linear(1152,1) Sigmoid
//         conv branch : conv(C->128,3) PReLU conv(128->128,3) PReLU AvgPool2 conv(128->512,3,STRIDE 2) PReLU
//                       conv(512->1024,3,STRIDE 2) PReLU SpatialDropout() View(4096) Linear(4096,1024) PReLU
//         dense branch: View(C*256) Linear(C*256,128) PReLU Dropout() Linear(128,128) PReLU
//   loop = adversarial.lua:83-288 (the same fevalD / fevalG_on_D / accuracy gate / interruptable optimizers as the 32x32 nets)
// Kernels: G16 is the 32x32 nets' generator type at side 16 (UpsGen, gen.cu); every layer of D16 is a ConvL (convl.h).  A
// stride-2 "same" 3x3 convolution is the stride-1 one sampled at the even pixels: forward = stride-1 kernel + subsample,
// backward = the stride-1 dgrad / wgrad of dY with zeros inserted at the odd pixels.  That is exact (the inserted zeros
// contribute nothing) and keeps both layers on the tensor cores at 4x their minimal FLOPs, which is 0.2 ms at batch 256.
#include <algorithm>

#include "convl.h"
#include "fg_internal.h"
#include "k_misc.h"

namespace {
constexpr int kS16Mask = 1024 + 128;  // nn.SpatialDropout() planes + nn.Dropout() of the dense branch, per sample
constexpr int kSide = 16;

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
}  // namespace

struct fg_s16 {
  fg_ctx* c = nullptr;
  int maxB = 0, C = 3;
  NetPair net;  // bnG: the running mean / var of G's two BatchNorm layers
  UpsGen G;
  // D
  ConvL Dc[4], DF1, DE1, DE2;
  int64_t Dca[4] = {0, 0, 0, 0}, Daf = 0, Dae1 = 0, Dae2 = 0, DJW = 0, DJb = 0;
  float *D_x = nullptr, *D_z[4] = {}, *D_h[4] = {}, *D_zfull = nullptr, *D_p1 = nullptr, *D_d3 = nullptr, *D_zf = nullptr,
        *D_hf = nullptr, *D_ze1 = nullptr, *D_he1 = nullptr, *D_de1 = nullptr, *D_ze2 = nullptr, *D_he2 = nullptr,
        *D_joint = nullptr, *D_logit = nullptr, *D_out = nullptr, *D_masks = nullptr, *D_dlogit = nullptr, *D_dx = nullptr,
        *D_dx2 = nullptr, *D_djoint = nullptr, *D_dhf = nullptr, *D_dhe2 = nullptr;
  // shared scratch
  float *ga = nullptr, *gb = nullptr, *ws = nullptr;
  float *in_a = nullptr, *in_b = nullptr, *in_c = nullptr, *io = nullptr;
  IterStage iter_stage;  // the inputs of the host-fed and device-fed train steps, stacked per iteration
  int D_B = 0;
  bool D_valid = false, D_train = true;
  std::vector<void*> allocs;
  ConvLEnv env;
};

namespace {
int dalloc(fg_s16* n, float** p, size_t elems) { return convl_dalloc(n->env, p, elems); }

void make_d16_layout(fg_s16* n) {
  const int C = n->C;
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
    n->net.nD = o;
  }
}

int s16_alloc(fg_s16* n) {
  const size_t B = n->maxB, C = n->C;
  make_d16_layout(n);
  n->env.c = n->c;
  n->env.maxB = n->maxB;
  n->env.allocs = &n->allocs;
  FG_TRY(pair_alloc(n->c, n->allocs, n->net, make_g_layout(n->C, kSide).total, n->net.nD, true));
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
  FG_TRY(dalloc(n, &n->env.dy.hi, big));
  FG_TRY(dalloc(n, &n->env.dy.lo, big));
  FG_TRY(dalloc(n, &n->ws, (size_t)9 * 1024 * 512));  // largest weight tensor (c4); F1 is 4096*1024, the 5x5 packs 36*256*128
  n->env.ga = n->ga; n->env.ws = n->ws;
  // G.L1 keeps K = 100 (on the FFMA kernels): padding it would change its bits.  Two backward launches per 5x5 layer.
  static const GenDesc g16{kSide, "s16.", 0, false};
  FG_TRY(gen_alloc(n->env, n->G, g16));
  FG_TRY(dalloc(n, &n->in_a, B * 256 * C));
  FG_TRY(dalloc(n, &n->in_b, B * 100));
  FG_TRY(dalloc(n, &n->in_c, B * 100));
  FG_TRY(dalloc(n, &n->io, B * 256 * C));
  n->net.keep = {{"Dstep.z1", n->D_z[0], 256 * 128}, {"Dstep.z2", n->D_z[1], 256 * 128}, {"Dstep.z3", n->D_z[2], 16 * 512},
                 {"Dstep.z4", n->D_z[3], 4 * 1024},  {"Dstep.zf", n->D_zf, 1024},        {"Dstep.ze1", n->D_ze1, 128},
                 {"Dstep.ze2", n->D_ze2, 128},       {"Dstep.logit", n->D_logit, 1},     {"Dstep.out", n->D_out, 1}};
  FG_CUDA(cudaStreamSynchronize(n->c->stream));
  return FG_OK;
}

int pack_D(fg_s16* n) {
  fg_ctx* c = n->c;
  if (n->net.D_pack == pack_key(c)) return FG_OK;
  for (int i = 0; i < 4; ++i) FG_TRY(convl_pack(c, n->Dc[i], n->net.PD));
  FG_TRY(convl_pack(c, n->DF1, n->net.PD));
  FG_TRY(convl_pack(c, n->DE1, n->net.PD));
  FG_TRY(convl_pack(c, n->DE2, n->net.PD));
  n->net.D_pack = pack_key(c);
  return FG_OK;
}

// ---------------------------------------------------------------------------------------------------
// D16
// ---------------------------------------------------------------------------------------------------
// x: NHWC device [B][16][16][C]; keep flags already in D_masks when training
int D_forward(fg_s16* n, const float* x, int B, bool training) {
  fg_ctx* c = n->c;
  FG_REQUIRE(B >= 1 && B <= n->maxB, "s16 D forward: batch %d out of range [1,%d]", B, n->maxB);
  FG_TRY(pack_D(n));
  const float* P = n->net.PD;
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
  const float* P = n->net.PD;
  float* G = want_wgrad ? n->net.gD : nullptr;
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

// the 16x16 nets in the loop body (pair_train_step, netpair.cu): real [B/2][C][16][16], noiseD [B/2][100] and noiseG
// [B][100] per iteration
struct S16Step final : StepNets {
  fg_s16* n;
  const float *real, *noiseD, *noiseG;
  S16Step(fg_s16* n, const fg_hyper* h, int B, const float* real, const float* noiseD, const float* noiseG)
      : StepNets(n->c, n->net, h, B, n->D_logit, n->D_out, n->D_dlogit, n->D_masks, kS16Mask, true, false), n(n), real(real),
        noiseD(noiseD), noiseG(noiseG) {}
  int g_forward(int j, bool d_iter) override {
    const int rows = d_iter ? B / 2 : B;
    return gen_forward(n->env, n->G, n->net, (d_iter ? noiseD : noiseG) + (size_t)j * rows * 100, rows, true);
  }
  int d_input(int j) override {
    const int Bh = B / 2;
    const size_t img = (size_t)n->C * 256;
    FG_TRY(k_nchw_to_nhwc(c, real + (size_t)j * Bh * img, n->D_x, Bh, n->C, 256));
    FG_CUDA(cudaMemcpyAsync(n->D_x + Bh * img, n->G.y, sizeof(float) * Bh * img, cudaMemcpyDeviceToDevice, c->stream));
    return FG_OK;
  }
  int draw_masks(int kind, const uint64_t* root) override {
    return k_bernoulli_keep(c, n->D_masks, (int64_t)B * kS16Mask, kind, 0.5f, root);
  }
  int d_forward(bool on_g) override { return D_forward(n, on_g ? n->G.y : n->D_x, B, true); }
  int d_backward(bool want_wgrad, bool want_dx) override { return D_backward(n, n->D_dlogit, want_wgrad, want_dx); }
  int g_backward() override { return gen_backward(n->env, n->G, n->net, n->D_dx, nullptr); }
};

}  // namespace

#define ENTER(n)                                         \
  do {                                                   \
    if (!(n) || !(n)->c) {                               \
      fg_set_error("null fg_s16");                       \
      return FG_ERR_INVALID;                             \
    }                                                    \
    FG_CUDA(cudaSetDevice((n)->c->device));              \
  } while (0)

namespace {
// d_iters D iterations + g_iters G iterations on inputs stacked per iteration (fg_train_step_iters at 16x16), for the
// entry `what`
int train_step_iters(fg_s16* n, const char* what, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real,
                     const float* noise_D, const float* noise_G, const float* masks_D, const float* masks_G, uint64_t seed,
                     fg_step_stats* stats) {
  ENTER(n);
  fg_ctx* c = n->c;
  FG_TRY(step_check(c, what, B, d_iters, g_iters, h && real && noise_D && noise_G));
  const size_t nd = d_iters, ng = g_iters, Bh = B / 2, M = n->maxB, img = (size_t)n->C * 256;
  IterStage& s = n->iter_stage;
  const float *rd, *zd, *zg, *md, *mg;
  FG_TRY(s.in(c, n->allocs, 0, real, nd * Bh * img, nd * M / 2 * img, &rd));
  FG_TRY(s.in(c, n->allocs, 1, noise_D, nd * Bh * 100, nd * M / 2 * 100, &zd));
  FG_TRY(s.in(c, n->allocs, 2, noise_G, ng * B * 100, ng * M * 100, &zg));
  FG_TRY(s.in(c, n->allocs, 3, masks_D, nd * B * kS16Mask, nd * M * kS16Mask, &md));
  FG_TRY(s.in(c, n->allocs, 4, masks_G, ng * B * kS16Mask, ng * M * kS16Mask, &mg));
  S16Step st(n, h, B, rd, zd, zg);
  return pair_train_step(st, d_iters, g_iters, md, mg, seed, {rd, zd, zg, md, mg, nullptr}, nullptr, stats);
}

// the same fed on the device: the streams of fg_train_step_dataset_iters, the real halves at 16x16; the draws run
// inside the step
int train_step_dataset_iters(fg_s16* n, fg_dataset* d, const char* what, const fg_hyper* h, int B, int d_iters, int g_iters,
                             uint64_t seed, fg_step_stats* stats) {
  ENTER(n);
  fg_ctx* c = n->c;
  FG_TRY(step_check(c, what, B, d_iters, g_iters, h, d, true));
  const int Bh = B / 2;
  const size_t M = n->maxB, img = (size_t)n->C * 256;
  IterStage& s = n->iter_stage;
  FG_TRY(s.reserve(c, n->allocs, 0, d_iters * M / 2 * img));
  FG_TRY(s.reserve(c, n->allocs, 1, d_iters * M / 2 * 100));
  FG_TRY(s.reserve(c, n->allocs, 2, g_iters * M * 100));
  float *real = s.p[0], *zd = s.p[1], *zg = s.p[2];
  const std::function<int()> feed = [&]() -> int {
    for (int j = 0; j < d_iters; ++j) {
      FG_TRY(dataset_draw_gather(d, 0, Bh, kSide, real + (size_t)j * Bh * img, c->seed_dev + j, 4));
      FG_TRY(noise_uniform_dev(c, 1, (int64_t)Bh * 100, zd + (size_t)j * Bh * 100, c->seed_dev + j, 4));
    }
    for (int j = 0; j < g_iters; ++j)
      FG_TRY(noise_uniform_dev(c, 2, (int64_t)B * 100, zg + (size_t)j * B * 100, c->seed_dev + j, 4));
    return FG_OK;
  };
  S16Step st(n, h, B, real, zd, zg);
  return pair_train_step(st, d_iters, g_iters, nullptr, nullptr, seed, {real, zd, zg, nullptr, nullptr, d}, &feed, stats);
}
}  // namespace

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
  pair_free(n->net);
  for (void* p : n->allocs) cudaFree(p);
  delete n;
  return FG_OK;
}
int64_t fg_s16_param_count(int net, int channels) {
  if (net != FG_NET_D) return make_g_layout(channels, kSide).total;
  fg_s16 tmp;
  tmp.C = channels;
  make_d16_layout(&tmp);
  return tmp.net.nD;
}
int fg_s16_mask_per_sample(void) { return kS16Mask; }

int fg_s16_set_params(fg_s16* n, int net, const float* src) {
  ENTER(n);
  FG_REQUIRE(src && (net == FG_NET_G || net == FG_NET_D), "fg_s16_set_params: bad arguments");
  return pair_set_params(n->c, n->net, net, src);
}
int fg_s16_get_params(fg_s16* n, int net, float* dst) {
  ENTER(n);
  FG_REQUIRE(dst && (net == FG_NET_G || net == FG_NET_D), "fg_s16_get_params: bad arguments");
  return pair_get_params(n->c, n->net, net, dst);
}
int fg_s16_get_grads(fg_s16* n, int net, float* dst) {
  ENTER(n);
  FG_REQUIRE(dst && (net == FG_NET_G || net == FG_NET_D), "fg_s16_get_grads: bad arguments");
  return pair_get_grads(n->c, n->net, net, dst);
}
int fg_s16_zero_grads(fg_s16* n, int net) {
  ENTER(n);
  return pair_zero_grads(n->c, n->net, net);
}
float* fg_s16_params_ptr(fg_s16* n, int net) { return !n ? nullptr : (net == FG_NET_D ? n->net.PD : n->net.PG); }
float* fg_s16_grads_ptr(fg_s16* n, int net) { return !n ? nullptr : (net == FG_NET_D ? n->net.gD : n->net.gG); }

int fg_s16_set_adam_state(fg_s16* n, int net, const float* m, const float* v, int t) {
  ENTER(n);
  return pair_set_adam_state(n->c, n->net, net, m, v, t);
}
int fg_s16_get_adam_state(fg_s16* n, int net, float* m, float* v, int* t) {
  ENTER(n);
  return pair_get_adam_state(n->c, n->net, net, m, v, t);
}
// running_mean / running_var of G's two nn.SpatialBatchNormalization layers: [mean1 256][var1 256][mean2 128][var2 128]
int fg_s16_set_bn_state(fg_s16* n, const float* src768) {
  ENTER(n);
  FG_REQUIRE(src768, "fg_s16_set_bn_state: null source");
  return pair_set_bn_state(n->c, n->net, src768);
}
int fg_s16_get_bn_state(fg_s16* n, float* dst768) {
  ENTER(n);
  FG_REQUIRE(dst768, "fg_s16_get_bn_state: null destination");
  return pair_get_bn_state(n->c, n->net, dst768);
}

// noise [B][100] -> images [B][C][16][16] (NCHW; host or device pointers).  training != 0: batch statistics + running
// stat update (nn_utils.lua:52 createImages leaves G in training mode); 0: evaluate() with the running statistics.
int fg_s16_G_forward(fg_s16* n, const float* noise, int B, int training, float* img_out) {
  ENTER(n);
  FG_REQUIRE(noise && B >= 1 && B <= n->maxB, "fg_s16_G_forward: bad arguments (batch %d, max %d)", B, n->maxB);
  const float* nd;
  FG_TRY(fg_to_dev(n->c, noise, (size_t)B * 100, n->in_b, &nd));
  FG_TRY(gen_forward(n->env, n->G, n->net, nd, B, training != 0));
  if (img_out) {
    FG_TRY(k_nhwc_to_nchw(n->c, n->G.y, n->io, B, n->C, 256));
    FG_TRY(fg_to_user(n->c, img_out, n->io, (size_t)B * n->C * 256));
  }
  return FG_OK;
}
int fg_s16_G_backward(fg_s16* n, const float* d_img, float* d_noise) {
  ENTER(n);
  FG_REQUIRE(d_img, "fg_s16_G_backward: null gradient");
  const float* dd;
  FG_TRY(fg_to_dev(n->c, d_img, (size_t)n->G.B * n->C * 256, n->in_a, &dd));
  FG_TRY(k_nchw_to_nhwc(n->c, dd, n->io, n->G.B, n->C, 256));
  FG_TRY(gen_backward(n->env, n->G, n->net, n->io, d_noise ? n->in_c : nullptr));
  if (d_noise) FG_TRY(fg_to_user(n->c, d_noise, n->in_c, (size_t)n->G.B * 100));
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
  return pair_broadcast(n->c, n->net);
}

int fg_s16_train_step(fg_s16* n, const fg_hyper* h, int B, const float* real, const float* noise_D, const float* noise_G,
                      const float* masks_D, const float* masks_G, uint64_t seed, fg_step_stats* stats) {
  return train_step_iters(n, "fg_s16_train_step", h, B, 1, 1, real, noise_D, noise_G, masks_D, masks_G, seed, stats);
}

// train.lua --scale 16 fed on the device: real = gather at 16x16 of draw(4*seed, B/2), noise_D = uniform(4*seed+1),
// noise_G = uniform(4*seed+2), dropout masks from `seed` (the streams of fg_train_step_dataset)
int fg_s16_train_step_dataset(fg_s16* n, fg_dataset* d, const fg_hyper* h, int B, uint64_t seed, fg_step_stats* stats) {
  return train_step_dataset_iters(n, d, "fg_s16_train_step_dataset", h, B, 1, 1, seed, stats);
}

// d_iters D iterations + g_iters G iterations on inputs stacked per iteration (fg_train_step_iters at 16x16)
int fg_s16_train_step_iters(fg_s16* n, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real,
                            const float* noise_D, const float* noise_G, const float* masks_D, const float* masks_G,
                            uint64_t seed, fg_step_stats* stats) {
  return train_step_iters(n, "fg_s16_train_step_iters", h, B, d_iters, g_iters, real, noise_D, noise_G, masks_D, masks_G, seed,
                          stats);
}

// fg_s16_train_step_iters fed on the device: the streams of fg_train_step_dataset_iters, the real halves at 16x16
int fg_s16_train_step_dataset_iters(fg_s16* n, fg_dataset* d, const fg_hyper* h, int B, int d_iters, int g_iters,
                                    uint64_t seed, fg_step_stats* stats) {
  return train_step_dataset_iters(n, d, "fg_s16_train_step_dataset_iters", h, B, d_iters, g_iters, seed, stats);
}

int64_t fg_s16_debug_tensor(fg_s16* n, const char* name, float* dst, int64_t max_elems) {
  if (!n || !n->c || !name) {
    fg_set_error("fg_s16_debug_tensor: null argument");
    return -1;
  }
  cudaSetDevice(n->c->device);
  const int db = n->D_B;
  auto d = [&](const float* p) { return n->D_valid ? p : nullptr; };
  std::vector<DebugTensor> ents = {
      {"D.z1", d(n->D_z[0]), 256 * 128, db}, {"D.z2", d(n->D_z[1]), 256 * 128, db}, {"D.z3", d(n->D_z[2]), 16 * 512, db},
      {"D.z4", d(n->D_z[3]), 4 * 1024, db}, {"D.p1", d(n->D_p1), 64 * 128, db}, {"D.zf", d(n->D_zf), 1024, db},
      {"D.ze1", d(n->D_ze1), 128, db}, {"D.ze2", d(n->D_ze2), 128, db}, {"D.logit", d(n->D_logit), 1, db},
      {"D.out", d(n->D_out), 1, db}};
  pair_keep_rows(n->net, ents);
  gen_debug_rows(n->G, ents);
  return debug_tensor_copy(n->c, "fg_s16_debug_tensor", ents.data(), ents.size(), name, dst, max_elems);
}

}  // extern "C"
