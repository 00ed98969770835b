// The `--scale 16` nets of train.lua (models.create_G / create_D pick them when dimensions[2] == 16, models.lua:87-104)
// and the adversarial.lua loop body on them:
//   G16 = models.lua:27-51   create_G_decoder_upsampling16: Linear(100, 128*4*4) View(128,4,4) PReLU | Up2 conv(128->256,5)
//         BN PReLU | Up2 conv(256->128,5) BN PReLU | conv(128->C,3) Sigmoid  -- the 32x32 generator with every size halved
//   D16 = models.lua:279-316 create_D16_d: ConcatTable{conv branch, dense branch} JoinTable(2) Linear(1152,1) Sigmoid
//         conv branch : conv(C->128,3) PReLU conv(128->128,3) PReLU AvgPool2 conv(128->512,3,STRIDE 2) PReLU
//                       conv(512->1024,3,STRIDE 2) PReLU SpatialDropout() View(4096) Linear(4096,1024) PReLU
//         dense branch: View(C*256) Linear(C*256,128) PReLU Dropout() Linear(128,128) PReLU
//   loop = adversarial.lua:83-288 (the same fevalD / fevalG_on_D / accuracy gate / interruptable optimizers as the 32x32 nets)
// Trainer: the 32x32 nets' trainer type at side 16 (UpsGan, ups_gan.cu); this file holds D16 and the C entry points.
// Kernels: G16 is the 32x32 nets' generator type at side 16 (UpsGen, gen.cu); every layer of D16 is a ConvL (convl.h).  A
// stride-2 "same" 3x3 convolution is the stride-1 one sampled at the even pixels: forward = stride-1 kernel + subsample,
// backward = the stride-1 dgrad / wgrad of dY with zeros inserted at the odd pixels.  That is exact (the inserted zeros
// contribute nothing) and keeps both layers on the tensor cores at 4x their minimal FLOPs, which is 0.2 ms at batch 256.
#include <algorithm>

#include "fg_internal.h"
#include "k_misc.h"
#include "ups_gan.h"

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

int k_subsample2(fg_ctx* c, const float* x, float* y, int B, int H, int W, int C) {
  subsample2_kernel<<<grid_for((int64_t)B * (H / 2) * (W / 2) * C, 256), 256, 0, c->stream>>>(x, y, B, H, W, C);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_zero_insert2(fg_ctx* c, const float* dy, float* dx, int B, int H, int W, int C) {
  zero_insert2_kernel<<<grid_for((int64_t)B * H * W * C, 256), 256, 0, c->stream>>>(dy, dx, B, H, W, C);
  LAUNCH_CHECK(c);
  return FG_OK;
}

namespace {
// D16: every layer a ConvL, activations NHWC
struct D16 final : GanD {
  ConvL Dc[4], DF1, DE1, DE2;
  int64_t Dca[4] = {0, 0, 0, 0}, Daf = 0, Dae1 = 0, Dae2 = 0, DJW = 0, DJb = 0;
  float *z[4] = {}, *h[4] = {}, *zfull = nullptr, *p1 = nullptr, *d3 = nullptr, *zf = nullptr, *hf = nullptr,
        *ze1 = nullptr, *he1 = nullptr, *de1 = nullptr, *ze2 = nullptr, *he2 = nullptr, *joint = nullptr, *dx2 = nullptr,
        *djoint = nullptr, *dhf = nullptr, *dhe2 = nullptr;
  float *ga = nullptr, *gb = nullptr;  // the backward's gradient ping-pong
  bool valid = false, train = true;

  int64_t layout(int C) override;
  int dalloc(float** q, size_t elems) { return convl_dalloc(n->env, q, elems); }
  int alloc() override;
  int forward(const float* x, int B, bool training, const fg_hyper* h) override;
  int backward(bool want_wgrad, bool want_dx) override;
  int draw_masks(int B, uint64_t seed, const fg_hyper*, const uint64_t* root) override {
    return k_bernoulli_keep(n->c, masks, (int64_t)B * kS16Mask, seed, 0.5f, root);
  }
  void debug_rows(std::vector<DebugTensor>& ents) const override;
};

// conv branch, dense branch, joint Linear (ConcatTable order, models.lua:306-313)
int64_t D16::layout(int C) {
  const int ci[4] = {C, 128, 128, 512}, co[4] = {128, 128, 512, 1024}, hw[4] = {16, 16, 8, 4};  // stride-1 sides
  static const char* tf[4] = {"s16.D.c1.fwd", "s16.D.c2.fwd", "s16.D.c3.fwd", "s16.D.c4.fwd"};
  static const char* td[4] = {"s16.D.c1.dgrad", "s16.D.c2.dgrad", "s16.D.c3.dgrad", "s16.D.c4.dgrad"};
  static const char* tw[4] = {"s16.D.c1.wgrad", "s16.D.c2.wgrad", "s16.D.c3.wgrad", "s16.D.c4.wgrad"};
  int64_t o = 0;
  for (int i = 0; i < 4; ++i) {
    ConvL& L = Dc[i];
    L.Cin = ci[i]; L.Cout = co[i]; L.k = 3; L.H = hw[i];
    L.w_off = o; o += (int64_t)co[i] * ci[i] * 9;
    L.b_off = o; o += co[i];
    Dca[i] = o; o += 1;
    L.tf = tf[i]; L.td = td[i]; L.tw = tw[i];
  }
  ConvL& F1 = DF1;
  F1.Cin = 4096; F1.Cout = 1024; F1.k = 1; F1.H = 1;
  F1.cA = 1024; F1.cS = 4;  // View(4096) flattens [1024][2][2]; ours is [2][2][1024]
  F1.w_off = o; o += (int64_t)1024 * 4096;
  F1.b_off = o; o += 1024;
  F1.tf = "s16.D.F1.fwd"; F1.td = "s16.D.F1.dgrad"; F1.tw = "s16.D.F1.wgrad";
  Daf = o; o += 1;
  ConvL& E1 = DE1;
  E1.Cin = C * 256; E1.Cout = 128; E1.k = 1; E1.H = 1;
  E1.cA = C; E1.cS = 256;  // View(C*256) flattens the NCHW image; ours is [16][16][C]
  E1.w_off = o; o += (int64_t)128 * C * 256;
  E1.b_off = o; o += 128;
  E1.tf = "s16.D.E1.fwd"; E1.td = "s16.D.E1.dgrad"; E1.tw = "s16.D.E1.wgrad";
  Dae1 = o; o += 1;
  ConvL& E2 = DE2;
  E2.Cin = 128; E2.Cout = 128; E2.k = 1; E2.H = 1;
  E2.w_off = o; o += 128 * 128;
  E2.b_off = o; o += 128;
  E2.tf = "s16.D.E2.fwd"; E2.td = "s16.D.E2.dgrad"; E2.tw = "s16.D.E2.wgrad";
  Dae2 = o; o += 1;
  DJW = o; o += 1152;
  DJb = o; o += 1;
  return o;
}

int D16::alloc() {
  ConvLEnv& e = n->env;
  const size_t B = e.maxB, C = n->c->C;
  for (int i = 0; i < 4; ++i) FG_TRY(convl_alloc(e, Dc[i]));
  FG_TRY(convl_alloc(e, DF1));
  FG_TRY(convl_alloc(e, DE1));
  FG_TRY(convl_alloc(e, DE2));
  FG_TRY(dalloc(&x, B * 256 * C));
  const size_t zsz[4] = {B * 256 * 128, B * 256 * 128, B * 16 * 512, B * 4 * 1024};
  for (int i = 0; i < 4; ++i) {
    FG_TRY(dalloc(&z[i], zsz[i]));
    FG_TRY(dalloc(&h[i], zsz[i]));
  }
  FG_TRY(dalloc(&zfull, B * 64 * 512));  // stride-1 output of c3 ([B][8][8][512]) / c4 ([B][4][4][1024])
  FG_TRY(dalloc(&p1, B * 64 * 128));
  FG_TRY(dalloc(&d3, B * 4096));
  FG_TRY(dalloc(&zf, B * 1024));
  FG_TRY(dalloc(&hf, B * 1024));
  FG_TRY(dalloc(&ze1, B * 128));
  FG_TRY(dalloc(&he1, B * 128));
  FG_TRY(dalloc(&de1, B * 128));
  FG_TRY(dalloc(&ze2, B * 128));
  FG_TRY(dalloc(&he2, B * 128));
  FG_TRY(dalloc(&joint, B * 1152));
  FG_TRY(dalloc(&djoint, B * 1152));
  FG_TRY(dalloc(&dhf, B * 1024));
  FG_TRY(dalloc(&dhe2, B * 128));
  FG_TRY(dalloc(&logit, B));
  FG_TRY(dalloc(&out, B));
  FG_TRY(dalloc(&dlogit, B));
  FG_TRY(dalloc(&masks, B * kS16Mask));
  FG_TRY(dalloc(&dx, B * 256 * C));
  FG_TRY(dalloc(&dx2, B * 256 * C));
  // ---- the layer scratch both nets share ----
  const size_t big = B * 256 * 128;  // largest activation: [B][16][16][128] = [B][8][8][512]
  FG_TRY(dalloc(&ga, big));
  FG_TRY(dalloc(&gb, big));
  FG_TRY(dalloc(&e.dy.hi, big));
  FG_TRY(dalloc(&e.dy.lo, big));
  FG_TRY(dalloc(&e.ws, (size_t)9 * 1024 * 512));  // largest weight tensor (c4); F1 is 4096*1024, the 5x5 packs 36*256*128
  e.ga = ga;
  n->net.keep = {{"Dstep.z1", z[0], 256 * 128}, {"Dstep.z2", z[1], 256 * 128}, {"Dstep.z3", z[2], 16 * 512},
                 {"Dstep.z4", z[3], 4 * 1024},  {"Dstep.zf", zf, 1024},        {"Dstep.ze1", ze1, 128},
                 {"Dstep.ze2", ze2, 128},       {"Dstep.logit", logit, 1},     {"Dstep.out", out, 1}};
  return FG_OK;
}

int D16::forward(const float* xin, int Bn, bool training, const fg_hyper*) {
  fg_ctx* c = n->c;
  ConvLEnv& e = n->env;
  FG_REQUIRE(Bn >= 1 && Bn <= e.maxB, "s16 D forward: batch %d out of range [1,%d]", Bn, e.maxB);
  FG_TRY(gan_pack_D(*n, {&Dc[0], &Dc[1], &Dc[2], &Dc[3], &DF1, &DE1, &DE2}));
  const float* P = n->net.PD;
  const int B = Bn;
  if (xin != x) FG_CUDA(cudaMemcpyAsync(x, xin, sizeof(float) * (size_t)B * 256 * c->C, cudaMemcpyDeviceToDevice, c->stream));
  const float* m = training ? masks : nullptr;
  // ---- conv branch ----
  FG_TRY(convl_fwd(e, Dc[0], x, P, z[0], B));
  FG_TRY(k_prelu_fwd(c, z[0], P + Dca[0], h[0], (int64_t)B * 256 * 128));
  FG_TRY(convl_fwd(e, Dc[1], h[0], P, z[1], B));
  FG_TRY(k_prelu_fwd(c, z[1], P + Dca[1], h[1], (int64_t)B * 256 * 128));
  avgpool2_fwd_kernel<<<grid_for((int64_t)B * 64 * 128, 256), 256, 0, c->stream>>>(h[1], p1, B, 16, 16, 128);
  LAUNCH_CHECK(c);
  FG_TRY(convl_fwd(e, Dc[2], p1, P, zfull, B));  // stride 1 at 8x8 ...
  subsample2_kernel<<<grid_for((int64_t)B * 16 * 512, 256), 256, 0, c->stream>>>(zfull, z[2], B, 8, 8, 512);  // ... -> 4x4
  LAUNCH_CHECK(c);
  FG_TRY(k_prelu_fwd(c, z[2], P + Dca[2], h[2], (int64_t)B * 16 * 512));
  FG_TRY(convl_fwd(e, Dc[3], h[2], P, zfull, B));  // stride 1 at 4x4 ...
  subsample2_kernel<<<grid_for((int64_t)B * 4 * 1024, 256), 256, 0, c->stream>>>(zfull, z[3], B, 4, 4, 1024);  // ... -> 2x2
  LAUNCH_CHECK(c);
  FG_TRY(k_prelu_fwd(c, z[3], P + Dca[3], h[3], (int64_t)B * 4096));
  plane_dropout_kernel<<<grid_for((int64_t)B * 4096, 256), 256, 0, c->stream>>>(h[3], m, kS16Mask, 0, 0.5f, d3, B, 4, 1024);
  LAUNCH_CHECK(c);
  FG_TRY(convl_fwd(e, DF1, d3, P, zf, B));
  FG_TRY(k_prelu_fwd(c, zf, P + Daf, hf, (int64_t)B * 1024));
  // ---- dense branch ----
  FG_TRY(convl_fwd(e, DE1, x, P, ze1, B));
  FG_TRY(k_prelu_fwd(c, ze1, P + Dae1, he1, (int64_t)B * 128));
  const float* e1 = he1;
  if (training) {  // nn.Dropout() (p = 0.5, v2): keep * 2 in training, identity in evaluation
    FG_TRY(k_dropout_nhwc(c, he1, masks, kS16Mask, 1024, 1, 128, 2.0f, de1, B));
    e1 = de1;
  }
  FG_TRY(convl_fwd(e, DE2, e1, P, ze2, B));
  FG_TRY(k_prelu_fwd(c, ze2, P + Dae2, he2, (int64_t)B * 128));
  // ---- JoinTable(2) -> Linear(1152, 1) ----
  join2_kernel<<<grid_for((int64_t)B * 1152, 256), 256, 0, c->stream>>>(hf, he2, joint, B, 1024, 128);
  LAUNCH_CHECK(c);
  FG_TRY(k_gemv_fwd(c, joint, P + DJW, P + DJb, logit, B, 1152));
  GanD::B = B;
  train = training;
  valid = true;
  return FG_OK;
}

// want_dx: the image gradient is the sum over the two branches (nn.ConcatTable backward)
int D16::backward(bool want_wgrad, bool want_dx) {
  fg_ctx* c = n->c;
  ConvLEnv& e = n->env;
  if (!valid) {
    fg_set_error("s16 D backward needs a preceding D forward");
    return FG_ERR_STATE;
  }
  const float* P = n->net.PD;
  float* G = want_wgrad ? n->net.gD : nullptr;
  const bool tr = train;
  const float* m = tr ? masks : nullptr;
  if (G) FG_TRY(k_gemv_wgrad_add(c, joint, dlogit, G + DJW, G + DJb, B, 1152));
  FG_TRY(k_gemv_dgrad(c, dlogit, P + DJW, djoint, B, 1152));
  split2_kernel<<<grid_for((int64_t)B * 1152, 256), 256, 0, c->stream>>>(djoint, dhf, dhe2, B, 1024, 128);
  LAUNCH_CHECK(c);
  float *cur = ga, *oth = gb;  // gradient ping-pong: every stage reads `cur`, writes `oth`, then they swap
  {  // dense branch
    FG_TRY(k_prelu_bwd(c, dhe2, ze2, P + Dae2, cur, G ? G + Dae2 : nullptr, B, 1, 1, 128, 0));
    FG_TRY(convl_bwd(e, DE2, tr ? de1 : he1, cur, G, oth, B));
    std::swap(cur, oth);
    if (tr) {
      FG_TRY(k_dropout_nhwc(c, cur, masks, kS16Mask, 1024, 1, 128, 2.0f, oth, B));
      std::swap(cur, oth);
    }
    FG_TRY(k_prelu_bwd(c, cur, ze1, P + Dae1, oth, G ? G + Dae1 : nullptr, B, 1, 1, 128, 0));
    std::swap(cur, oth);
    FG_TRY(convl_bwd(e, DE1, x, cur, G, want_dx ? dx2 : nullptr, B));
  }
  {  // conv branch
    FG_TRY(k_prelu_bwd(c, dhf, zf, P + Daf, cur, G ? G + Daf : nullptr, B, 1, 1, 1024, 0));
    FG_TRY(convl_bwd(e, DF1, d3, cur, G, oth, B));  // -> gradient of the View(4096) input, [B][2][2][1024]
    std::swap(cur, oth);
    plane_dropout_kernel<<<grid_for((int64_t)B * 4096, 256), 256, 0, c->stream>>>(cur, m, kS16Mask, 0, 0.5f, oth, B, 4, 1024);
    LAUNCH_CHECK(c);
    std::swap(cur, oth);
    FG_TRY(k_prelu_bwd(c, cur, z[3], P + Dca[3], oth, G ? G + Dca[3] : nullptr, B, 2, 2, 1024, 0));
    std::swap(cur, oth);
    zero_insert2_kernel<<<grid_for((int64_t)B * 16 * 1024, 256), 256, 0, c->stream>>>(cur, oth, B, 4, 4, 1024);
    LAUNCH_CHECK(c);
    std::swap(cur, oth);
    FG_TRY(convl_bwd(e, Dc[3], h[2], cur, G, oth, B));  // -> [B][4][4][512]
    std::swap(cur, oth);
    FG_TRY(k_prelu_bwd(c, cur, z[2], P + Dca[2], oth, G ? G + Dca[2] : nullptr, B, 4, 4, 512, 0));
    std::swap(cur, oth);
    zero_insert2_kernel<<<grid_for((int64_t)B * 64 * 512, 256), 256, 0, c->stream>>>(cur, oth, B, 8, 8, 512);
    LAUNCH_CHECK(c);
    std::swap(cur, oth);
    FG_TRY(convl_bwd(e, Dc[2], p1, cur, G, oth, B));  // -> [B][8][8][128]
    std::swap(cur, oth);
    avgpool2_bwd_kernel<<<grid_for((int64_t)B * 256 * 128, 256), 256, 0, c->stream>>>(cur, oth, B, 16, 16, 128);
    LAUNCH_CHECK(c);
    std::swap(cur, oth);
    FG_TRY(k_prelu_bwd(c, cur, z[1], P + Dca[1], oth, G ? G + Dca[1] : nullptr, B, 16, 16, 128, 0));
    std::swap(cur, oth);
    FG_TRY(convl_bwd(e, Dc[1], h[0], cur, G, oth, B));
    std::swap(cur, oth);
    FG_TRY(k_prelu_bwd(c, cur, z[0], P + Dca[0], oth, G ? G + Dca[0] : nullptr, B, 16, 16, 128, 0));
    std::swap(cur, oth);
    FG_TRY(convl_bwd(e, Dc[0], x, cur, G, want_dx ? dx : nullptr, B));
  }
  if (want_dx) FG_TRY(k_add(c, dx, dx2, dx, (int64_t)B * 256 * c->C));
  return FG_OK;
}

void D16::debug_rows(std::vector<DebugTensor>& ents) const {
  const int db = B;
  auto d = [&](const float* q) { return valid ? q : nullptr; };
  ents.insert(ents.end(), {{"D.z1", d(z[0]), 256 * 128, db}, {"D.z2", d(z[1]), 256 * 128, db}, {"D.z3", d(z[2]), 16 * 512, db},
                           {"D.z4", d(z[3]), 4 * 1024, db}, {"D.p1", d(p1), 64 * 128, db}, {"D.zf", d(zf), 1024, db},
                           {"D.ze1", d(ze1), 128, db}, {"D.ze2", d(ze2), 128, db}, {"D.logit", d(logit), 1, db},
                           {"D.out", d(out), 1, db}});
}
}  // namespace

struct fg_s16 : UpsGan {};

#define ENTER(n)                                         \
  do {                                                   \
    if (!(n) || !(n)->c) {                               \
      fg_set_error("null fg_s16");                       \
      return FG_ERR_INVALID;                             \
    }                                                    \
    FG_CUDA(cudaSetDevice((n)->c->device));              \
  } while (0)

extern "C" {

int fg_s16_create(fg_ctx* ctx, fg_s16** out) { return fg_s16_create_disc(ctx, FG_DISC_D16_D, out); }

int fg_s16_create_disc(fg_ctx* ctx, int disc, fg_s16** out) {
  if (!ctx || !out) {
    fg_set_error("fg_s16_create: null argument");
    return FG_ERR_INVALID;
  }
  *out = nullptr;
  if (disc == FG_DISC_DEFAULT) disc = FG_DISC_D16_D;
  FG_REQUIRE(fg_disc_side(disc), "fg_s16_create_disc: unknown discriminator %d", disc);
  if (fg_disc_side(disc) != kSide) {
    fg_set_error("fg_s16_create_disc: discriminator %d is a 32x32 net; the --scale 16 nets take FG_DISC_D16_D, "
                 "FG_DISC_D16, FG_DISC_D16_B or FG_DISC_D16_C", disc);
    return FG_ERR_UNSUPPORTED;
  }
  FG_CUDA(cudaSetDevice(ctx->device));
  fg_s16* n = new fg_s16();
  n->disc = disc;
  // G.L1 keeps K = 100 (on the FFMA kernels): padding it would change its bits.  Two backward launches per 5x5 layer.
  const bool d = disc == FG_DISC_D16_D;
  const GanDesc k16{{kSide, "s16.", 0, false}, d ? kS16Mask : dbr_mask_per_sample(disc), false};
  const int r = gan_alloc(*n, ctx, k16, d ? std::make_unique<D16>() : dbr_make(disc), nullptr);
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
  gan_free(*n);
  delete n;
  return FG_OK;
}
int64_t fg_s16_param_count(int net, int channels) {
  if (net != FG_NET_D) return make_g_layout(channels, kSide).total;
  return D16().layout(channels);
}
int fg_s16_mask_per_sample(void) { return kS16Mask; }
int fg_s16_get_disc(fg_s16* n) {
  ENTER(n);
  return n->disc;
}

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
  FG_REQUIRE(noise && B >= 1 && B <= n->c->maxB, "fg_s16_G_forward: bad arguments (batch %d, max %d)", B, n->c->maxB);
  return gan_G_forward(*n, noise, B, training != 0, img_out);
}
int fg_s16_G_backward(fg_s16* n, const float* d_img, float* d_noise) {
  ENTER(n);
  FG_REQUIRE(d_img, "fg_s16_G_backward: null gradient");
  return gan_G_backward(*n, d_img, d_noise);
}
int fg_s16_D_forward(fg_s16* n, const float* img, int B, int training, const float* masks, uint64_t seed, float* out) {
  ENTER(n);
  FG_REQUIRE(img && B >= 1 && B <= n->c->maxB, "fg_s16_D_forward: bad arguments (batch %d, max %d)", B, n->c->maxB);
  return gan_D_forward(*n, img, B, training != 0, masks, seed, out);
}
// fg_D_score on D16_d: predictions for N 16x16 images in chunks of `chunk`, dropout masks of chunk s drawn from
// seed + s when training (sample.lua --scale 16 never calls evaluate())
int fg_s16_D_score(fg_s16* n, const float* images, int64_t N, int chunk, int training, uint64_t seed, float* preds_out) {
  ENTER(n);
  FG_REQUIRE(images && preds_out && N >= 1 && chunk >= 1 && chunk <= n->c->maxB, "fg_s16_D_score: bad arguments (chunk %d, max %d)",
             chunk, n->c->maxB);
  const size_t img = (size_t)n->c->C * 256;
  for (int64_t s = 0; s < N; s += chunk) {
    const int b = (int)std::min<int64_t>(chunk, N - s);
    FG_TRY(fg_s16_D_forward(n, images + (size_t)s * img, b, training, nullptr, seed + (uint64_t)s, preds_out + s));
  }
  return FG_OK;
}
int fg_s16_D_backward(fg_s16* n, const float* d_out, int want_wgrad, float* d_img) {
  ENTER(n);
  FG_REQUIRE(d_out, "fg_s16_D_backward: null gradient");
  return gan_D_backward(*n, d_out, want_wgrad != 0, d_img);
}

// data parallel: rank 0's parameters, optimizer moments, step counters and BatchNorm running statistics to every rank
int fg_s16_dp_broadcast_params(fg_s16* n) {
  ENTER(n);
  return pair_broadcast(n->c, n->net);
}

int fg_s16_train_step(fg_s16* n, const fg_hyper* h, int B, const float* real, const float* noise_D, const float* noise_G,
                      const float* masks_D, const float* masks_G, uint64_t seed, fg_step_stats* stats) {
  ENTER(n);
  return gan_train_step_iters(*n, "fg_s16_train_step", h, B, 1, 1, real, noise_D, noise_G, masks_D, masks_G, seed, stats);
}

// train.lua --scale 16 fed on the device: real = gather at 16x16 of draw(4*seed, B/2), noise_D = uniform(4*seed+1),
// noise_G = uniform(4*seed+2), dropout masks from `seed` (the streams of fg_train_step_dataset)
int fg_s16_train_step_dataset(fg_s16* n, fg_dataset* d, const fg_hyper* h, int B, uint64_t seed, fg_step_stats* stats) {
  ENTER(n);
  return gan_train_step_dataset_iters(*n, d, "fg_s16_train_step_dataset", h, B, 1, 1, seed, stats);
}

// d_iters D iterations + g_iters G iterations on inputs stacked per iteration (fg_train_step_iters at 16x16)
int fg_s16_train_step_iters(fg_s16* n, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real,
                            const float* noise_D, const float* noise_G, const float* masks_D, const float* masks_G,
                            uint64_t seed, fg_step_stats* stats) {
  ENTER(n);
  return gan_train_step_iters(*n, "fg_s16_train_step_iters", h, B, d_iters, g_iters, real, noise_D, noise_G, masks_D,
                              masks_G, seed, stats);
}

// fg_s16_train_step_iters fed on the device: the streams of fg_train_step_dataset_iters, the real halves at 16x16
int fg_s16_train_step_dataset_iters(fg_s16* n, fg_dataset* d, const fg_hyper* h, int B, int d_iters, int g_iters,
                                    uint64_t seed, fg_step_stats* stats) {
  ENTER(n);
  return gan_train_step_dataset_iters(*n, d, "fg_s16_train_step_dataset_iters", h, B, d_iters, g_iters, seed, stats);
}

int64_t fg_s16_debug_tensor(fg_s16* n, const char* name, float* dst, int64_t max_elems) {
  if (!n || !n->c || !name) {
    fg_set_error("fg_s16_debug_tensor: null argument");
    return -1;
  }
  return gan_debug_tensor(*n, "fg_s16_debug_tensor", name, dst, max_elems);
}

}  // extern "C"
