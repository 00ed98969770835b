// Orchestration of G (models.lua:57-81), D (models.lua:382-416) and the adversarial.lua loop body
// (adversarial.lua:54-300) on one stream.  Kernels live in k_elem.cu / k_conv_simt.cu / k_conv_tc.cu.
#include <algorithm>

#include "fg_internal.h"
#include "k_conv_tc.h"

GLayout make_g_layout(int C) {
  GLayout L;
  int64_t o = 0;
  L.L1W = o; o += 8192 * 100;
  L.L1b = o; o += 8192;
  L.a1 = o; o += 1;
  L.C1W = o; o += 256 * 128 * 25;
  L.C1b = o; o += 256;
  L.g1 = o; o += 256;
  L.be1 = o; o += 256;
  L.a2 = o; o += 1;
  L.C2W = o; o += 128 * 256 * 25;
  L.C2b = o; o += 128;
  L.g2 = o; o += 128;
  L.be2 = o; o += 128;
  L.a3 = o; o += 1;
  L.C3W = o; o += (int64_t)C * 128 * 9;
  L.C3b = o; o += C;
  L.total = o;
  return L;
}
DLayout make_d_layout(int C) {
  DLayout L;
  const int cin[4] = {C, 64, 128, 256}, cout[4] = {64, 128, 256, 512};
  int64_t o = 0;
  for (int i = 0; i < 4; ++i) {
    L.cW[i] = o; o += (int64_t)cout[i] * cin[i] * 9;
    L.cb[i] = o; o += cout[i];
    L.ca[i] = o; o += 1;
  }
  L.L1W = o; o += 512 * 2048;
  L.L1b = o; o += 512;
  L.a5 = o; o += 1;
  L.L2W = o; o += 512 * 512;
  L.L2b = o; o += 512;
  L.a6 = o; o += 1;
  L.L3W = o; o += 512;
  L.L3b = o; o += 1;
  L.total = o;
  return L;
}

namespace {
const int kDcin[4] = {0 /*C*/, 64, 128, 256}, kDcout[4] = {64, 128, 256, 512}, kDhw[4] = {32, 16, 8, 4};
const int kDmoff[4] = {0, 64, 192, 448};
inline int dcin(const fg_ctx* c, int i) { return i == 0 ? c->C : kDcin[i]; }

inline std::vector<void*>& allocs(fg_ctx* c) { return c->allocs; }  // owned by the context: no process-wide state

int dalloc(fg_ctx* c, float** p, size_t n) {
  void* q = nullptr;
  FG_CUDA(cudaMalloc(&q, std::max<size_t>(n, 1) * sizeof(float)));
  FG_CUDA(cudaMemsetAsync(q, 0, std::max<size_t>(n, 1) * sizeof(float), c->stream));
  allocs(c).push_back(q);
  *p = (float*)q;
  return FG_OK;
}
}  // namespace

int net_alloc(fg_ctx* c) {
  const size_t B = c->maxB, C = c->C;
  c->gl = make_g_layout(c->C);
  c->dl = make_d_layout(c->C);
  const size_t nG = c->gl.total, nD = c->dl.total;
  FG_TRY(dalloc(c, &c->PG, nG));
  FG_TRY(dalloc(c, &c->PD, nD));
  FG_TRY(dalloc(c, &c->gG, nG + kGradTail));
  FG_TRY(dalloc(c, &c->gD, nD + kGradTail));
  c->ownPG = c->PG; c->ownPD = c->PD; c->ownGG = c->gG; c->ownGD = c->gD;
  c->tailG = c->gG + nG; c->tailD = c->gD + nD;
  FG_TRY(dalloc(c, &c->tail_sep, 2 * kGradTail));
  FG_TRY(dalloc(c, &c->mG, nG));
  FG_TRY(dalloc(c, &c->vG, nG));
  FG_TRY(dalloc(c, &c->mD, nD));
  FG_TRY(dalloc(c, &c->vD, nD));
  FG_TRY(dalloc(c, &c->bnG, 768));
  {  // running_mean = 0, running_var = 1 (nn.SpatialBatchNormalization init)
    std::vector<float> init(768, 0.f);
    for (int i = 256; i < 512; ++i) init[i] = 1.f;
    for (int i = 640; i < 768; ++i) init[i] = 1.f;
    FG_CUDA(cudaMemcpyAsync(c->bnG, init.data(), 768 * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    FG_CUDA(cudaStreamSynchronize(c->stream));
  }
  float* tmp = nullptr;
  FG_TRY(dalloc(c, &tmp, (sizeof(DeviceStats) + 3) / 4));
  c->dstats = (DeviceStats*)tmp;
  FG_TRY(dalloc(c, &c->acc_hist, kAccHistMax));
  FG_CUDA(cudaMallocHost((void**)&c->hstats, sizeof(DeviceStats)));
  memset(c->hstats, 0, sizeof(DeviceStats));
  FG_TRY(dalloc(c, &c->amax_slot, 64));
  {
    float* sd = nullptr;
    FG_TRY(dalloc(c, &sd, 2));
    c->seed_dev = reinterpret_cast<uint64_t*>(sd);
  }
  // packs
  FG_TRY(dalloc(c, &c->G_L1p, 8192 * 100 + 8192));  // + permuted bias behind the weights
  FG_TRY(dalloc(c, &c->G_L1pd, 8192 * 100));
  FG_TRY(dalloc(c, &c->G_C1p, 25 * 256 * 128));
  FG_TRY(dalloc(c, &c->G_C1pd, 25 * 256 * 128));
  FG_TRY(dalloc(c, &c->G_C2p, 25 * 256 * 128));
  FG_TRY(dalloc(c, &c->G_C2pd, 25 * 256 * 128));
  FG_TRY(dalloc(c, &c->G_C3p, 9 * C * 128));
  FG_TRY(dalloc(c, &c->G_C3pd, 9 * C * 128));
  for (int i = 0; i < 4; ++i) {
    const size_t n = (size_t)9 * kDcout[i] * dcin(c, i);
    FG_TRY(dalloc(c, &c->D_cp[i], n));
    FG_TRY(dalloc(c, &c->D_cpd[i], n));
  }
  FG_TRY(dalloc(c, &c->D_L1p, 512 * 2048));
  FG_TRY(dalloc(c, &c->D_L1pd, 512 * 2048));
  FG_TRY(dalloc(c, &c->D_L2pd, 512 * 512));
  c->wgrad_ws_elems = 9 * 512 * 256;
  FG_TRY(dalloc(c, &c->wgrad_ws, c->wgrad_ws_elems));
  c->splitk_ws_elems = (size_t)c->sm_count * 4 * 128 * 128;  // >= splits x output of every split-K weight gradient
  FG_TRY(dalloc(c, &c->splitk_ws, c->splitk_ws_elems));
  c->red_ws_elems = (size_t)4 << 20;  // >= blocks x partials of every ordered reduction (checked at each launch)
  FG_TRY(dalloc(c, reinterpret_cast<float**>(&c->red_ws), 2 * c->red_ws_elems));
  FG_TRY(dalloc(c, reinterpret_cast<float**>(&c->red_ws_opt), 2 * kOptRedRows));
  FG_TRY(dalloc(c, reinterpret_cast<float**>(&c->red_ticket), 2));  // zeroed; every ordered reduction resets its ticket
  FG_TRY(dalloc(c, &c->small_ws, (size_t)kSmallMaxParts * 9 * 4 * 128));
  // G activations
  FG_TRY(dalloc(c, &c->G_noise, B * kNoiseDim));
  FG_TRY(dalloc(c, &c->G_z0, B * 8192));
  FG_TRY(dalloc(c, &c->G_h0, B * 8192));
  FG_TRY(dalloc(c, &c->G_z1, B * 65536));
  FG_TRY(dalloc(c, &c->G_h1, B * 65536));
  FG_TRY(dalloc(c, &c->G_z2, B * 131072));
  FG_TRY(dalloc(c, &c->G_h2, B * 131072));
  FG_TRY(dalloc(c, &c->G_z3, B * 1024 * C));
  FG_TRY(dalloc(c, &c->G_y, B * 1024 * C));
  FG_TRY(dalloc(c, &tmp, 4 * 256 * 2));  // doubles
  c->bn_acc = (double*)tmp;
  FG_TRY(dalloc(c, &tmp, 32 * 2 * 256 * 2 + 64));  // doubles + tickets (zero-initialised)
  c->bn_slice_acc = (double*)tmp;
  FG_TRY(dalloc(c, &c->bn_parts, B * 2048));  // G.C2: 8 tiles/image x 2 x 128 ch; G.C1: 2 tiles/image x 2 x 256 ch
  FG_TRY(dalloc(c, &c->bn_mean1, 256));
  FG_TRY(dalloc(c, &c->bn_istd1, 256));
  FG_TRY(dalloc(c, &c->bn_mean2, 128));
  FG_TRY(dalloc(c, &c->bn_istd2, 128));
  FG_TRY(dalloc(c, &c->bn_mg, 512));
  FG_TRY(dalloc(c, &c->G_dz3, B * 1024 * C));
  FG_TRY(dalloc(c, &c->G_dfull, B * 262144));
  FG_TRY(dalloc(c, &c->G_dz2, B * 131072));
  FG_TRY(dalloc(c, &c->G_dz1, B * 65536));
  FG_TRY(dalloc(c, &c->G_dz0, B * 8192));
  // D activations
  FG_TRY(dalloc(c, &c->D_x, B * 1024 * C));
  for (int i = 0; i < 4; ++i) {
    const size_t n = B * (size_t)kDhw[i] * kDhw[i] * kDcout[i];
    FG_TRY(dalloc(c, &c->D_z[i], n));
    FG_TRY(dalloc(c, &c->D_p[i], n / 4));
  }
  FG_TRY(dalloc(c, &c->D_zl1, B * 512));
  FG_TRY(dalloc(c, &c->D_hl1, B * 512));
  FG_TRY(dalloc(c, &c->D_zl2, B * 512));
  FG_TRY(dalloc(c, &c->D_hl2, B * 512));
  FG_TRY(dalloc(c, &c->D_logit, B));
  FG_TRY(dalloc(c, &c->D_out, B));
  FG_TRY(dalloc(c, &c->D_masks, B * kMaskPerSample));
  FG_TRY(dalloc(c, &c->D_dlogit, B));
  FG_TRY(dalloc(c, &c->D_dh, B * 512));
  FG_TRY(dalloc(c, &c->D_dzl, B * 512));
  FG_TRY(dalloc(c, &c->D_dz, B * 65536));
  FG_TRY(dalloc(c, &c->D_dp, B * 16384));
  FG_TRY(dalloc(c, &c->D_dx, B * 1024 * C));
  FG_TRY(dalloc(c, &c->D_targets, B));
  c->io_dev_elems = std::max<size_t>(B * 1024 * C, B * kMaskPerSample);
  FG_TRY(dalloc(c, &c->io_dev, c->io_dev_elems));
  FG_TRY(dalloc(c, &c->io_dev2, c->io_dev_elems));
  {  // tensor-core path buffers
    fg_ctx::TcBufs& t = c->tcb;
    FG_TRY(dalloc(c, &t.G_h0_hi, B * 8192));
    FG_TRY(dalloc(c, &t.G_h0_lo, B * 8192));
    FG_TRY(dalloc(c, &t.G_xpad, B * 128));  // dalloc zero-fills: the 28 pad columns stay zero
    FG_TRY(dalloc(c, &t.G_x_hi, B * 128));
    FG_TRY(dalloc(c, &t.G_x_lo, B * 128));
    FG_TRY(dalloc(c, &t.G_L1pad, 8192 * 128));
    FG_TRY(dalloc(c, &t.G_L1w_hi, 8192 * 128));
    FG_TRY(dalloc(c, &t.G_L1w_lo, 8192 * 128));
    FG_TRY(dalloc(c, &t.G_h1_hi, B * 65536));
    FG_TRY(dalloc(c, &t.G_h1_lo, B * 65536));
    FG_TRY(dalloc(c, &t.dy_hi, B * 131072));
    FG_TRY(dalloc(c, &t.dy_lo, B * 131072));
    for (int i = 0; i < 2; ++i) {
      FG_TRY(dalloc(c, &t.G_Wf_hi[i], 36 * 256 * 128));
      FG_TRY(dalloc(c, &t.G_Wf_lo[i], 36 * 256 * 128));
      FG_TRY(dalloc(c, &t.G_Wd_hi[i], 36 * 256 * 128));
      FG_TRY(dalloc(c, &t.G_Wd_lo[i], 36 * 256 * 128));
      FG_TRY(dalloc(c, &t.G_Wx_hi[i], 25 * 256 * 128));
      FG_TRY(dalloc(c, &t.G_Wx_lo[i], 25 * 256 * 128));
    }
    for (int i = 0; i < 3; ++i) {
      const size_t n = B * (size_t)kDhw[i + 1] * kDhw[i + 1] * kDcout[i];
      FG_TRY(dalloc(c, &t.D_p_hi[i], n));
      FG_TRY(dalloc(c, &t.D_p_lo[i], n));
    }
    for (int i = 0; i < 2; ++i) {
      FG_TRY(dalloc(c, &t.D_lin_hi[i], B * (i == 0 ? 2048 : 512)));
      FG_TRY(dalloc(c, &t.D_lin_lo[i], B * (i == 0 ? 2048 : 512)));
    }
    for (int i = 0; i < 4; ++i) {
      FG_TRY(dalloc(c, &t.D_Lw_hi[i], i < 2 ? 512 * 2048 : 512 * 512));
      FG_TRY(dalloc(c, &t.D_Lw_lo[i], i < 2 ? 512 * 2048 : 512 * 512));
    }
    for (int i = 1; i < 4; ++i) {
      const size_t n = (size_t)9 * kDcout[i] * kDcin[i];
      FG_TRY(dalloc(c, &t.D_Wf_hi[i], n));
      FG_TRY(dalloc(c, &t.D_Wf_lo[i], n));
      FG_TRY(dalloc(c, &t.D_Wd_hi[i], n));
      FG_TRY(dalloc(c, &t.D_Wd_lo[i], n));
      FG_TRY(dalloc(c, &t.D_Wf_hh[i], n / 2));
      FG_TRY(dalloc(c, &t.D_Wf_hl[i], n / 2));
      FG_TRY(dalloc(c, &t.D_Wd_hh[i], n / 2));
      FG_TRY(dalloc(c, &t.D_Wd_hl[i], n / 2));
    }
    // FP16 split twins (halves: half the floats)
    FG_TRY(dalloc(c, &t.G_h0_hh, B * 4096));
    FG_TRY(dalloc(c, &t.G_h0_hl, B * 4096));
    FG_TRY(dalloc(c, &t.G_h1_hh, B * 32768));
    FG_TRY(dalloc(c, &t.G_h1_hl, B * 32768));
    FG_TRY(dalloc(c, &t.dy_hh, B * 65536));
    FG_TRY(dalloc(c, &t.dy_hl, B * 65536));
    for (int i = 0; i < 2; ++i) {
      FG_TRY(dalloc(c, &t.G_Wf_hh[i], 18 * 256 * 128));
      FG_TRY(dalloc(c, &t.G_Wf_hl[i], 18 * 256 * 128));
      FG_TRY(dalloc(c, &t.G_Wd_hh[i], 18 * 256 * 128));
      FG_TRY(dalloc(c, &t.G_Wd_hl[i], 18 * 256 * 128));
    }
    for (int i = 0; i < 3; ++i) {
      const size_t n = B * (size_t)kDhw[i + 1] * kDhw[i + 1] * kDcout[i];
      FG_TRY(dalloc(c, &t.D_p_hh[i], n / 2));
      FG_TRY(dalloc(c, &t.D_p_hl[i], n / 2));
    }
    FG_TRY(dalloc(c, &t.G_x_hh, B * 64));
    FG_TRY(dalloc(c, &t.G_x_hl, B * 64));
    FG_TRY(dalloc(c, &t.G_L1w_hh, 8192 * 64));
    FG_TRY(dalloc(c, &t.G_L1w_hl, 8192 * 64));
    for (int i = 0; i < 2; ++i) {
      FG_TRY(dalloc(c, &t.D_lin_hh[i], B * (i == 0 ? 1024 : 256)));
      FG_TRY(dalloc(c, &t.D_lin_hl[i], B * (i == 0 ? 1024 : 256)));
    }
    for (int i = 0; i < 4; ++i) {
      FG_TRY(dalloc(c, &t.D_Lw_hh[i], i < 2 ? 512 * 1024 : 512 * 256));
      FG_TRY(dalloc(c, &t.D_Lw_hl[i], i < 2 ? 512 * 1024 : 512 * 256));
    }
  }
  FG_TRY(dalloc(c, &c->in_real, B * 1024 * C));
  FG_TRY(dalloc(c, &c->in_noiseD, B * kNoiseDim));
  FG_TRY(dalloc(c, &c->in_noiseG, B * kNoiseDim));
  FG_TRY(dalloc(c, &c->in_masksD, B * kMaskPerSample));
  FG_TRY(dalloc(c, &c->in_masksG, B * kMaskPerSample));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

void net_free(fg_ctx* c) {
  for (void* p : allocs(c)) cudaFree(p);
  c->allocs.clear();
  if (c->hstats) cudaFreeHost(c->hstats);
  if (c->stage_pinned) cudaFreeHost(c->stage_pinned);
  for (int i = 0; i < 8; ++i)
    if (c->scratch[i]) cudaFree(c->scratch[i]);
}

int net_pack_G(fg_ctx* c) {
  if (c->G_packed) return FG_OK;
  const GLayout& L = c->gl;
  FG_TRY(k_pack_weights(c, c->PG + L.L1W, c->G_L1p, c->G_L1pd, 8192, 100, 1, 128, 64, 0, 0));
  FG_TRY(k_pack_weights(c, c->PG + L.L1b, c->G_L1p + 8192 * 100, nullptr, 8192, 1, 1, 128, 64, 0, 0));
  // the tap-major fp32 packs of the two 5x5 layers only feed the SIMT kernels (fallback / cross-check path)
  const bool tc_g = c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(ConvGeom{c->maxB, 16, 16, 128, 256, 5, 2}) &&
                    tc_conv_eligible(ConvGeom{c->maxB, 32, 32, 256, 128, 5, 2});
  if (!tc_g) {
    FG_TRY(k_pack_weights(c, c->PG + L.C1W, c->G_C1p, c->G_C1pd, 256, 128, 25, 0, 0, 0, 0));
    FG_TRY(k_pack_weights(c, c->PG + L.C2W, c->G_C2p, c->G_C2pd, 128, 256, 25, 0, 0, 0, 0));
  }
  FG_TRY(k_pack_weights(c, c->PG + L.C3W, c->G_C3p, c->G_C3pd, c->C, 128, 9, 0, 0, 0, 0));
  if (c->conv_impl != FG_CONV_SIMT) {
    fg_ctx::TcBufs& t = c->tcb;
    // G.L1 on the tensor cores: [8192'][100] -> [8192'][128] (pad columns stay zero), then the TF32 split
    FG_CUDA(cudaMemcpy2DAsync(t.G_L1pad, 128 * sizeof(float), c->G_L1p, 100 * sizeof(float), 100 * sizeof(float), 8192,
                              cudaMemcpyDeviceToDevice, c->stream));
    if (c->mma_f16 && c->conv_impl == FG_CONV_TC_COLLAPSED) FG_TRY(tc_split_h(c, t.G_L1pad, t.G_L1w_hh, t.G_L1w_hl, 8192 * 128));
    else FG_TRY(tc_split(c, t.G_L1pad, t.G_L1w_hi, t.G_L1w_lo, 8192 * 128));
    if (c->mma_f16 && c->conv_impl == FG_CONV_TC_COLLAPSED) {  // forward and dgrad read the FP16 split; wgrad needs no weights
      FG_TRY(tc_pack_collapsed_h(c, c->PG + L.C1W, t.G_Wf_hh[0], t.G_Wf_hl[0], t.G_Wd_hh[0], t.G_Wd_hl[0], 256, 128));
      FG_TRY(tc_pack_collapsed_h(c, c->PG + L.C2W, t.G_Wf_hh[1], t.G_Wf_hl[1], t.G_Wd_hh[1], t.G_Wd_hl[1], 128, 256));
    } else {
      FG_TRY(tc_pack_collapsed(c, c->PG + L.C1W, t.G_Wf_hi[0], t.G_Wf_lo[0], t.G_Wd_hi[0], t.G_Wd_lo[0], 256, 128));
      FG_TRY(tc_pack_collapsed(c, c->PG + L.C2W, t.G_Wf_hi[1], t.G_Wf_lo[1], t.G_Wd_hi[1], t.G_Wd_lo[1], 128, 256));
    }
    if (c->conv_impl == FG_CONV_TC_DENSE) {
      FG_TRY(tc_pack_split(c, c->PG + L.C1W, t.G_Wx_hi[0], t.G_Wx_lo[0], nullptr, nullptr, 256, 128, 25));
      FG_TRY(tc_pack_split(c, c->PG + L.C2W, t.G_Wx_hi[1], t.G_Wx_lo[1], nullptr, nullptr, 128, 256, 25));
    }
  }
  c->G_packed = true;
  return FG_OK;
}
int net_pack_D(fg_ctx* c) {
  if (c->D_packed) return FG_OK;
  const DLayout& L = c->dl;
  for (int i = 0; i < 4; ++i) {  // c2..c4 run on the tensor cores from their own TF32 packs (below) unless conv_impl = SIMT
    const ConvGeom gf{c->maxB, kDhw[i], kDhw[i], dcin(c, i), kDcout[i], 3, 1}, gd{c->maxB, kDhw[i], kDhw[i], kDcout[i], dcin(c, i), 3, 1};
    if (i > 0 && c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(gf) && tc_conv_eligible(gd)) continue;
    FG_TRY(k_pack_weights(c, c->PD + L.cW[i], c->D_cp[i], c->D_cpd[i], kDcout[i], dcin(c, i), 9, 0, 0, 0, 0));
  }
  // View(2048) flattens [512][2][2] in (c,h,w) order; ours is NHWC (h,w,c): permute the columns
  FG_TRY(k_pack_weights(c, c->PD + L.L1W, c->D_L1p, c->D_L1pd, 512, 2048, 1, 0, 0, 512, 4));
  FG_TRY(k_pack_weights(c, c->PD + L.L2W, nullptr, c->D_L2pd, 512, 512, 1, 0, 0, 0, 0));
  if (c->conv_impl != FG_CONV_SIMT) {
    fg_ctx::TcBufs& t = c->tcb;
    for (int i = 1; i < 4; ++i) {
      if (c->mma_f16 && c->conv_impl == FG_CONV_TC_COLLAPSED)
        FG_TRY(tc_pack_split_h(c, c->PD + L.cW[i], t.D_Wf_hh[i], t.D_Wf_hl[i], t.D_Wd_hh[i], t.D_Wd_hl[i], kDcout[i], kDcin[i], 9));
      else
        FG_TRY(tc_pack_split(c, c->PD + L.cW[i], t.D_Wf_hi[i], t.D_Wf_lo[i], t.D_Wd_hi[i], t.D_Wd_lo[i], kDcout[i], kDcin[i], 9));
    }
    if (c->mma_f16 && c->conv_impl == FG_CONV_TC_COLLAPSED) {
      FG_TRY(tc_split_h(c, c->D_L1p, t.D_Lw_hh[0], t.D_Lw_hl[0], 512 * 2048));
      FG_TRY(tc_split_h(c, c->D_L1pd, t.D_Lw_hh[1], t.D_Lw_hl[1], 512 * 2048));
      FG_TRY(tc_split_h(c, c->PD + L.L2W, t.D_Lw_hh[2], t.D_Lw_hl[2], 512 * 512));
      FG_TRY(tc_split_h(c, c->D_L2pd, t.D_Lw_hh[3], t.D_Lw_hl[3], 512 * 512));
    } else {
      FG_TRY(tc_split(c, c->D_L1p, t.D_Lw_hi[0], t.D_Lw_lo[0], 512 * 2048));
      FG_TRY(tc_split(c, c->D_L1pd, t.D_Lw_hi[1], t.D_Lw_lo[1], 512 * 2048));
      FG_TRY(tc_split(c, c->PD + L.L2W, t.D_Lw_hi[2], t.D_Lw_lo[2], 512 * 512));
      FG_TRY(tc_split(c, c->D_L2pd, t.D_Lw_hi[3], t.D_Lw_lo[3], 512 * 512));
    }
  }
  c->D_packed = true;
  return FG_OK;
}

// ---------------------------------------------------------------------------------------------------
// conv dispatch (SIMT now; tensor-core variants are selected in k_conv_tc.cu)
// ---------------------------------------------------------------------------------------------------
static int conv_fwd(fg_ctx* c, const char* tag, const float* in, const float* Wp, const float* bias, float* out,
                    ConvGeom g) {
  ScopedTimer t(c, tag);
  // 3-channel-side 3x3 convolutions get bandwidth-shaped kernels (k_conv_edge.cu; k_conv_small.cu for other widths)
  if (c->edge_impl && k_edge_eligible(g)) return k_conv_edge(c, in, Wp, bias, out, g);
  return k_small_eligible(g) ? k_conv_small(c, in, Wp, bias, out, g) : k_conv_simt(c, in, Wp, bias, out, g);
}
static int conv_wgrad(fg_ctx* c, const char* tag, const float* in, const float* dY, ConvGeom g, float* dW, int nA, int nS,
                      int cA, int cS) {
  {
    ScopedTimer t(c, tag);
    FG_TRY(k_small_eligible(g) ? k_wgrad_small(c, in, dY, c->wgrad_ws, g) : k_wgrad_simt(c, in, dY, c->wgrad_ws, g));
  }
  return k_unpack_wgrad(c, c->wgrad_ws, dW, g.Cout, g.Cin, g.k * g.k, nA, nS, cA, cS);
}

static inline bool use_tc(const fg_ctx* c, const ConvGeom& g) {
  return c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(g);
}
static inline bool use_tc_wgrad(const fg_ctx* c, const ConvGeom& g) {
  return use_tc(c, g) && g.Cout % 128 == 0 && g.Cin % 64 == 0;
}

// ---- option "mma_f16": every tensor-core operand in the 3xFP16 split (k_conv_tc.cu), f16 MMAs -----------------------
// Activations and gradients are scaled into fp16's range by a power of two found on the device (tc_amax): slot i of
// c->amax_slot holds (max|x|, 1/scale) of one tensor; the consuming kernels multiply their result by the inverse scales.
// One slot per tensor and pass, so that a producer can reduce max|output| while it writes the tensor (AmaxInto) instead of
// a separate read pass; amax_reset() zeroes the max words (not the inverse scales, which the weight-gradient kernels of
// a later pass still need) at the start of every forward / backward pass.
enum { kSlotDy = 0, kSlotH0 = 1, kSlotH1 = 2, kSlotDp = 3 /* +0..2 */, kSlotLin = 6 /* +0..1 */, kSlotX = 8,
       kSlotGdz = 9 /* +0..2: dz0, dz1, dz2 */, kSlotDdz = 12 /* +1..3 */, kSlotDzl = 16 /* +0..1 */, kNumSlots = 32 };
static inline bool f16_on(const fg_ctx* c) { return c->mma_f16 && c->conv_impl == FG_CONV_TC_COLLAPSED; }
static inline const float* inv_scale(const fg_ctx* c, int slot) { return c->amax_slot + 2 * slot + 1; }
static int amax_reset(fg_ctx* c) {
  if (!f16_on(c)) return FG_OK;
  for (int i = 0; i < kNumSlots; ++i) c->amax_valid[i] = false;
  FG_CUDA(cudaMemset2DAsync(c->amax_slot, 2 * sizeof(float), 0, sizeof(float), kNumSlots, c->stream));
  return FG_OK;
}
struct AmaxInto {  // the ONE elementwise producer launched inside the scope reports max|output| into `slot`
  fg_ctx* c;
  AmaxInto(fg_ctx* c_, int slot) : c(c_) {
    if (f16_on(c)) {
      c->amax_out = reinterpret_cast<unsigned*>(c->amax_slot + 2 * slot);
      c->amax_id = slot;
    }
  }
  ~AmaxInto() { c->amax_out = nullptr; }
};
// slot: where the inverse scale goes (what the consumers read); amax_from: the slot a producer reduced max|x| into (-1: slot)
static int split_h_scaled(fg_ctx* c, const float* x, float* hh, float* hl, int64_t n, int slot, int amax_from = -1) {
  const int src = amax_from >= 0 && c->amax_valid[amax_from] ? amax_from : slot;
  if (c->amax_valid[src]) c->amax_valid[src] = false;  // the producer already reduced max|x| into the slot
  else FG_TRY(tc_amax(c, x, n, c->amax_slot + 2 * src));
  return tc_split_h(c, x, hh, hl, n, c->amax_slot + 2 * src, c->amax_slot + 2 * slot + 1);
}

// nn.Linear as a 1x1 convolution on a 1x1 image.  With only B rows the fp32 SIMT tiling leaves the GPU
// idle (8 CTAs at B=256); the tensor-core path splits the input on the fly and uses the pre-split weights.
// f16 mode: `in16` is the fp32 input (always given), split into keep16_h/l (or the dY scratch) under amax slot `slot`
static int lin_fwd(fg_ctx* c, const char* tag, const float* in, const float* Wp, int wi, const float* bias, float* out,
                   ConvGeom g, float* keep_hi = nullptr, float* keep_lo = nullptr, const float* in16 = nullptr,
                   float* keep16_h = nullptr, float* keep16_l = nullptr, int slot = kSlotDy, int amax_from = -1) {
  if (!use_tc(c, g)) return conv_fwd(c, tag, in, Wp, bias, out, g);
  fg_ctx::TcBufs& t = c->tcb;
  if (f16_on(c) && in16) {
    float *hh = keep16_h ? keep16_h : t.dy_hh, *hl = keep16_l ? keep16_l : t.dy_hl;
    FG_TRY(split_h_scaled(c, in16, hh, hl, (int64_t)g.B * g.Cin, slot, amax_from));
    ScopedTimer tm(c, tag);
    return tc_conv_fwd(c, hh, hl, t.D_Lw_hh[wi], t.D_Lw_hl[wi], bias, out, g, 0, nullptr, nullptr, 1, inv_scale(c, slot));
  }
  float* hi = keep_hi ? keep_hi : t.dy_hi;  // forward keeps the split of its input for the tensor-core wgrad
  float* lo = keep_lo ? keep_lo : t.dy_lo;
  if (in) FG_TRY(tc_split(c, in, hi, lo, (int64_t)g.B * g.Cin));  // nullptr: the producer already wrote keep_hi / keep_lo
  ScopedTimer tm(c, tag);
  return tc_conv_fwd(c, hi, lo, t.D_Lw_hi[wi], t.D_Lw_lo[wi], bias, out, g, 0);
}
// weight gradient of a Linear layer on the tensor cores: x split kept by the forward, dY split left in
// tcb.dy_* by the dgrad call that must precede this one
// f16 mode (xslot >= 0): x16_h/l = the FP16 split the forward kept (amax slot xslot), dY in t.dy_hh/hl (slot kSlotDy)
static int lin_wgrad_tc(fg_ctx* c, const char* tag, const float* x_hi, const float* x_lo, ConvGeom g, float* dW, int cA,
                        int cS, const float* x16_h = nullptr, const float* x16_l = nullptr, int xslot = -1) {
  fg_ctx::TcBufs& t = c->tcb;
  {
    ScopedTimer tm(c, tag);
    if (f16_on(c) && xslot >= 0)
      FG_TRY(tc_conv_wgrad(c, x16_h, x16_l, t.dy_hh, t.dy_hl, c->wgrad_ws, g, 1, inv_scale(c, kSlotDy), inv_scale(c, xslot)));
    else
      FG_TRY(tc_conv_wgrad(c, x_hi, x_lo, t.dy_hi, t.dy_lo, c->wgrad_ws, g));
  }
  return k_unpack_wgrad(c, c->wgrad_ws, dW, g.Cout, g.Cin, 1, 0, 0, cA, cS);
}

// G's two nn.SpatialUpSamplingNearest(2) -> 5x5 convolutions (li = 0: C1, li = 1: C2), forward.
// tensor-core path: split the low-res input into TF32 hi/lo once (kept for wgrad), then the phase conv.
// *stat_parts (optional, in: want BatchNorm partials; out: how many tiles wrote one into c->bn_parts, 0 = none)
static int g_ups_fwd(fg_ctx* c, int li, const char* tag, const float* h, float* h_hi, float* h_lo, const float* Wp,
                     const float* bias, float* z, ConvGeom g, int* stat_parts = nullptr) {
  const bool want = stat_parts && *stat_parts;
  if (stat_parts) *stat_parts = 0;
  if (!use_tc(c, g)) return conv_fwd(c, tag, h, Wp, bias, z, g);
  fg_ctx::TcBufs& t = c->tcb;
  float* st = want && c->bn_epilogue ? c->bn_parts : nullptr;
  if (f16_on(c)) {  // 3xFP16 split of the fp32 activation (h0 / h1 always exist), kept for the weight gradient
    float *hh = li == 0 ? t.G_h0_hh : t.G_h1_hh, *hl = li == 0 ? t.G_h0_hl : t.G_h1_hl;
    const int slot = li == 0 ? kSlotH0 : kSlotH1;
    FG_TRY(split_h_scaled(c, li == 0 ? c->G_h0 : c->G_h1, hh, hl, (int64_t)g.B * (g.H / 2) * (g.W / 2) * g.Cin, slot));
    ScopedTimer tm(c, tag);
    return tc_conv_fwd(c, hh, hl, t.G_Wf_hh[li], t.G_Wf_hl[li], bias, z, g, 2, st, st ? stat_parts : nullptr, 1, inv_scale(c, slot));
  }
  if (h) FG_TRY(tc_split(c, h, h_hi, h_lo, (int64_t)g.B * (g.H / 2) * (g.W / 2) * g.Cin));  // nullptr: producer wrote hi/lo
  ScopedTimer tm(c, tag);
  if (c->conv_impl == FG_CONV_TC_DENSE)
    return tc_conv_fwd(c, h_hi, h_lo, t.G_Wx_hi[li], t.G_Wx_lo[li], bias, z, g, 1, st, st ? stat_parts : nullptr);
  return tc_conv_fwd(c, h_hi, h_lo, t.G_Wf_hi[li], t.G_Wf_lo[li], bias, z, g, 2, st, st ? stat_parts : nullptr);
}
// backward of the same layer: dW += wgrad, dh = dgrad.  *pooled tells whether `dh` already is the gradient of
// the LOW-RES input (tensor-core path: the 2x2 sum of the upsample backward is folded into the dgrad GEMM) or the
// full-resolution gradient that the consumer still has to sum 2x2 (SIMT path).
static int g_ups_bwd(fg_ctx* c, int li, const char* wtag, const char* dtag, const float* h, const float* h_hi,
                     const float* h_lo, const float* dz, const float* Wpd, ConvGeom g, float* dW, float* dh, bool* pooled,
                     const float* dz_f32 = nullptr, int dz_amax = -1) {
  if (!use_tc_wgrad(c, g)) {
    FG_TRY(conv_wgrad(c, wtag, h, dz, g, dW, 0, 0, 0, 0));
    *pooled = false;
    return conv_fwd(c, dtag, dz, Wpd, nullptr, dh, ConvGeom{g.B, g.H, g.W, g.Cout, g.Cin, g.k, 1});
  }
  fg_ctx::TcBufs& t = c->tcb;
  if (f16_on(c) && dz_f32) {  // weight and data gradient on the FP16 split of the (scaled) gradient
    FG_TRY(split_h_scaled(c, dz_f32, t.dy_hh, t.dy_hl, (int64_t)g.B * g.H * g.W * g.Cout, kSlotDy, dz_amax));
    {
      ScopedTimer tm(c, wtag);
      FG_TRY(tc_conv_wgrad(c, li == 0 ? t.G_h0_hh : t.G_h1_hh, li == 0 ? t.G_h0_hl : t.G_h1_hl, t.dy_hh, t.dy_hl, c->wgrad_ws, g, 1,
                           inv_scale(c, kSlotDy), inv_scale(c, li == 0 ? kSlotH0 : kSlotH1)));
    }
    FG_TRY(tc_combine_collapsed_wgrad(c, c->wgrad_ws, dW, g.Cout, g.Cin));
    *pooled = true;
    ScopedTimer tm(c, dtag);
    return tc_conv_dgrad_ups(c, t.dy_hh, t.dy_hl, t.G_Wd_hh[li], t.G_Wd_hl[li], dh, g, 1, inv_scale(c, kSlotDy));
  }
  if (dz) FG_TRY(tc_split(c, dz, t.dy_hi, t.dy_lo, (int64_t)g.B * g.H * g.W * g.Cout));  // nullptr: producer wrote hi/lo
  {
    ScopedTimer tm(c, wtag);
    FG_TRY(tc_conv_wgrad(c, h_hi, h_lo, t.dy_hi, t.dy_lo, c->wgrad_ws, g));
  }
  FG_TRY(tc_combine_collapsed_wgrad(c, c->wgrad_ws, dW, g.Cout, g.Cin));
  *pooled = true;
  ScopedTimer tm(c, dtag);
  return tc_conv_dgrad_ups(c, t.dy_hi, t.dy_lo, t.G_Wd_hi[li], t.G_Wd_lo[li], dh, g);
}

// ---------------------------------------------------------------------------------------------------
// G
// ---------------------------------------------------------------------------------------------------
int net_G_forward(fg_ctx* c, const float* noise, int B, bool training) {
  FG_REQUIRE(B >= 1 && B <= c->maxB, "G forward: batch %d out of range [1,%d]", B, c->maxB);
  FG_TRY(net_pack_G(c));
  const GLayout& L = c->gl;
  float* P = c->PG;
  if (noise != c->G_noise)
    FG_CUDA(cudaMemcpyAsync(c->G_noise, noise, sizeof(float) * B * kNoiseDim, cudaMemcpyDeviceToDevice, c->stream));
  c->G_B = B;
  c->G_train = training;
  FG_TRY(amax_reset(c));
  const ConvGeom gL1{B, 1, 1, 128, 8192, 1, 1};  // K padded 100 -> 128 for the tensor-core path
  if (use_tc(c, gL1)) {
    fg_ctx::TcBufs& t = c->tcb;
    FG_CUDA(cudaMemcpy2DAsync(t.G_xpad, 128 * sizeof(float), c->G_noise, kNoiseDim * sizeof(float), kNoiseDim * sizeof(float), B,
                              cudaMemcpyDeviceToDevice, c->stream));
    if (f16_on(c)) {
      FG_TRY(split_h_scaled(c, t.G_xpad, t.G_x_hh, t.G_x_hl, (int64_t)B * 128, kSlotX));  // kept for the weight gradient
      ScopedTimer tm(c, "G.L1.fwd");
      FG_TRY(tc_conv_fwd(c, t.G_x_hh, t.G_x_hl, t.G_L1w_hh, t.G_L1w_hl, c->G_L1p + 8192 * 100, c->G_z0, gL1, 0, nullptr, nullptr, 1,
                         inv_scale(c, kSlotX)));
    } else {
      FG_TRY(tc_split(c, t.G_xpad, t.G_x_hi, t.G_x_lo, (int64_t)B * 128));  // kept for the weight gradient
      ScopedTimer tm(c, "G.L1.fwd");
      FG_TRY(tc_conv_fwd(c, t.G_x_hi, t.G_x_lo, t.G_L1w_hi, t.G_L1w_lo, c->G_L1p + 8192 * 100, c->G_z0, gL1, 0));
    }
  } else {
    FG_TRY(conv_fwd(c, "G.L1.fwd", c->G_noise, c->G_L1p, c->G_L1p + 8192 * 100, c->G_z0, ConvGeom{B, 1, 1, 100, 8192, 1, 1}));
  }
  {
    AmaxInto am(c, kSlotH0);
    FG_TRY(k_prelu_fwd(c, c->G_z0, P + L.a1, c->G_h0, (int64_t)B * 8192));
  }
  // training: the BatchNorm statistics come out of the convolution's epilogue (per-tile partials) when it ran on
  // the tensor cores; otherwise a separate pass over z computes them
  int parts = training ? 1 : 0;
  FG_TRY(g_ups_fwd(c, 0, "G.C1.fwd", c->G_h0, c->tcb.G_h0_hi, c->tcb.G_h0_lo, c->G_C1p, P + L.C1b, c->G_z1,
                   ConvGeom{B, 16, 16, 128, 256, 5, 2}, &parts));
  if (training) {
    if (parts) {
      FG_TRY(k_bn_finalize_parts(c, c->bn_parts, parts, c->bn_mean1, c->bn_istd1, c->bnG, c->bnG + 256, (int64_t)B * 256, 256));
    } else {
      FG_TRY(k_bn_stats(c, c->G_z1, c->bn_acc, (int64_t)B * 256, 256));
      FG_TRY(k_bn_finalize(c, c->bn_acc, c->bn_mean1, c->bn_istd1, c->bnG, c->bnG + 256, (int64_t)B * 256, 256));
    }
  } else {
    FG_TRY(k_bn_eval_prep(c, c->bnG, c->bnG + 256, c->bn_mean1, c->bn_istd1, 256));
  }
  const ConvGeom gC2{B, 32, 32, 256, 128, 5, 2};
  const bool h1_split = training && use_tc(c, gC2) && !f16_on(c);  // TF32 tensor-core path consumes h1 only as TF32 hi/lo
  {
    AmaxInto am(c, kSlotH1);
    FG_TRY(k_bn_prelu_apply(c, c->G_z1, c->bn_mean1, c->bn_istd1, P + L.g1, P + L.be1, P + L.a2,
                            c->G_h1, (int64_t)B * 256, 256, h1_split ? c->tcb.G_h1_hi : nullptr,
                            h1_split ? c->tcb.G_h1_lo : nullptr));
  }
  parts = training ? 1 : 0;
  FG_TRY(g_ups_fwd(c, 1, "G.C2.fwd", h1_split ? nullptr : c->G_h1, c->tcb.G_h1_hi, c->tcb.G_h1_lo, c->G_C2p, P + L.C2b,
                   c->G_z2, gC2, &parts));
  // "hbm.*" timers: the bandwidth-bound kernels bench.py reports against the measured HBM peak
  if (training) {
    if (parts) {
      ScopedTimer tm(c, "G.bn2.finalize");
      FG_TRY(k_bn_finalize_parts(c, c->bn_parts, parts, c->bn_mean2, c->bn_istd2, c->bnG + 512, c->bnG + 640, (int64_t)B * 1024, 128));
    } else {
      {
        ScopedTimer tm(c, "hbm.G.bn2.stats");
        FG_TRY(k_bn_stats(c, c->G_z2, c->bn_acc, (int64_t)B * 1024, 128));
      }
      FG_TRY(k_bn_finalize(c, c->bn_acc, c->bn_mean2, c->bn_istd2, c->bnG + 512, c->bnG + 640, (int64_t)B * 1024, 128));
    }
  } else {
    FG_TRY(k_bn_eval_prep(c, c->bnG + 512, c->bnG + 640, c->bn_mean2, c->bn_istd2, 128));
  }
  {
    ScopedTimer tm(c, "hbm.G.bn2.apply");
    FG_TRY(k_bn_prelu_apply(c, c->G_z2, c->bn_mean2, c->bn_istd2, P + L.g2, P + L.be2, P + L.a3, c->G_h2, (int64_t)B * 1024,
                            128));
  }
  FG_TRY(conv_fwd(c, "G.C3.fwd", c->G_h2, c->G_C3p, P + L.C3b, c->G_z3, ConvGeom{B, 32, 32, 128, c->C, 3, 1}));
  FG_TRY(k_sigmoid_fwd(c, c->G_z3, c->G_y, (int64_t)B * 1024 * c->C));
  c->G_fwd_valid = true;
  return FG_OK;
}

int net_G_backward(fg_ctx* c, const float* dy, float* dnoise) {
  if (!c->G_fwd_valid || !c->G_train) {
    fg_set_error("G backward needs a preceding training-mode G forward");
    return FG_ERR_STATE;
  }
  const GLayout& L = c->gl;
  float *P = c->PG, *G = c->gG;
  const int B = c->G_B, C = c->C;
  FG_TRY(amax_reset(c));
  FG_TRY(k_sigmoid_bwd(c, dy, c->G_y, c->G_dz3, (int64_t)B * 1024 * C));
  // C3
  FG_TRY(conv_wgrad(c, "G.C3.wgrad", c->G_h2, c->G_dz3, ConvGeom{B, 32, 32, 128, C, 3, 1}, G + L.C3W, 0, 0, 0, 0));
  FG_TRY(k_colsum_add(c, c->G_dz3, G + L.C3b, (int64_t)B * 1024, C, 0, 0));
  FG_TRY(conv_fwd(c, "G.C3.dgrad", c->G_dz3, c->G_C3pd, nullptr, c->G_dfull, ConvGeom{B, 32, 32, C, 128, 3, 1}));
  // BN2 + PReLU
  {
    ScopedTimer tm(c, "hbm.G.bn2.bwd_reduce");
    FG_TRY(k_bn_prelu_bwd_reduce(c, c->G_dfull, c->G_z2, c->bn_mean2, c->bn_istd2, P + L.g2, P + L.be2, P + L.a3, c->bn_acc,
                                 G + L.a3, B, 32, 32, 128, 0));
  }
  FG_TRY(k_bn_bwd_finalize(c, c->bn_acc, c->bn_mg, G + L.g2, G + L.be2, (int64_t)B * 1024, 128));
  // in tensor-core mode the BN-backward kernels also emit the TF32 hi/lo split of dz (no separate split pass)
  const ConvGeom gC2{B, 32, 32, 256, 128, 5, 2}, gC1{B, 16, 16, 128, 256, 5, 2};
  const bool tc2 = use_tc_wgrad(c, gC2) && !f16_on(c), tc1 = use_tc_wgrad(c, gC1) && !f16_on(c);  // fused TF32 hi/lo of dz
  {
    ScopedTimer tm(c, "hbm.G.bn2.bwd_apply");
    AmaxInto am(c, kSlotGdz + 2);
    FG_TRY(k_bn_prelu_bwd_apply(c, c->G_dfull, c->G_z2, c->bn_mean2, c->bn_istd2, P + L.g2, P + L.be2, P + L.a3, c->bn_mg,
                                c->G_dz2, B, 32, 32, 128, 0, tc2 ? c->tcb.dy_hi : nullptr, tc2 ? c->tcb.dy_lo : nullptr,
                                G + L.C2b));  // + the bias gradient of C2 (column sums of dz2) in the same pass
  }
  // C2
  bool pooled = false;
  FG_TRY(g_ups_bwd(c, 1, "G.C2.wgrad", "G.C2.dgrad", c->G_h1, c->tcb.G_h1_hi, c->tcb.G_h1_lo, tc2 ? nullptr : c->G_dz2,
                   c->G_C2pd, gC2, G + L.C2W, c->G_dfull, &pooled, c->G_dz2, kSlotGdz + 2));
  // BN1 + PReLU (the 2x2 sum = backward of the nearest upsample is folded into the loads)
  FG_TRY(k_bn_prelu_bwd_reduce(c, c->G_dfull, c->G_z1, c->bn_mean1, c->bn_istd1, P + L.g1, P + L.be1, P + L.a2, c->bn_acc,
                               G + L.a2, B, 16, 16, 256, pooled ? 0 : 1));
  FG_TRY(k_bn_bwd_finalize(c, c->bn_acc, c->bn_mg, G + L.g1, G + L.be1, (int64_t)B * 256, 256));
  const bool split1 = tc1 && pooled;
  {
    AmaxInto am(c, kSlotGdz + 1);
    FG_TRY(k_bn_prelu_bwd_apply(c, c->G_dfull, c->G_z1, c->bn_mean1, c->bn_istd1, P + L.g1, P + L.be1, P + L.a2, c->bn_mg,
                                c->G_dz1, B, 16, 16, 256, pooled ? 0 : 1, split1 ? c->tcb.dy_hi : nullptr,
                                split1 ? c->tcb.dy_lo : nullptr, G + L.C1b));
  }
  // C1
  FG_TRY(g_ups_bwd(c, 0, "G.C1.wgrad", "G.C1.dgrad", c->G_h0, c->tcb.G_h0_hi, c->tcb.G_h0_lo, split1 ? nullptr : c->G_dz1,
                   c->G_C1pd,
                   ConvGeom{B, 16, 16, 128, 256, 5, 2}, G + L.C1W, c->G_dfull, &pooled, c->G_dz1, kSlotGdz + 1));
  {
    AmaxInto am(c, kSlotGdz);
    FG_TRY(k_prelu_bwd(c, c->G_dfull, c->G_z0, P + L.a1, c->G_dz0, G + L.a1, B, 8, 8, 128, pooled ? 0 : 1));
  }
  // L1
  const ConvGeom gL1{B, 1, 1, 128, 8192, 1, 1};
  if (use_tc_wgrad(c, gL1)) {  // dW[8192'][128 (100 used)] = dz0^T x on the tensor cores (K = batch), pad columns dropped
    fg_ctx::TcBufs& t = c->tcb;
    if (f16_on(c)) {
      FG_TRY(split_h_scaled(c, c->G_dz0, t.dy_hh, t.dy_hl, (int64_t)B * 8192, kSlotDy, kSlotGdz));
      ScopedTimer tm(c, "G.L1.wgrad");
      FG_TRY(tc_conv_wgrad(c, t.G_x_hh, t.G_x_hl, t.dy_hh, t.dy_hl, t.G_L1pad, gL1, 1, inv_scale(c, kSlotDy), inv_scale(c, kSlotX)));
    } else {
      FG_TRY(tc_split(c, c->G_dz0, t.dy_hi, t.dy_lo, (int64_t)B * 8192));
      ScopedTimer tm(c, "G.L1.wgrad");
      FG_TRY(tc_conv_wgrad(c, t.G_x_hi, t.G_x_lo, t.dy_hi, t.dy_lo, t.G_L1pad, gL1));
    }
    FG_CUDA(cudaMemcpy2DAsync(c->wgrad_ws, 100 * sizeof(float), t.G_L1pad, 128 * sizeof(float), 100 * sizeof(float), 8192,
                              cudaMemcpyDeviceToDevice, c->stream));
    FG_TRY(k_unpack_wgrad(c, c->wgrad_ws, G + L.L1W, 8192, 100, 1, 128, 64, 0, 0));
    c->G_packed = false;  // G_L1pad was used as scratch: the next forward re-packs (it does anyway after the optimizer step)
  } else {
    FG_TRY(conv_wgrad(c, "G.L1.wgrad", c->G_noise, c->G_dz0, ConvGeom{B, 1, 1, 100, 8192, 1, 1}, G + L.L1W, 128, 64, 0, 0));
  }
  FG_TRY(k_colsum_add(c, c->G_dz0, G + L.L1b, B, 8192, 128, 64));
  if (dnoise)
    FG_TRY(conv_fwd(c, "G.L1.dgrad", c->G_dz0, c->G_L1pd, nullptr, dnoise, ConvGeom{B, 1, 1, 8192, 100, 1, 1}));
  return FG_OK;
}

// ---------------------------------------------------------------------------------------------------
// D
// ---------------------------------------------------------------------------------------------------
int net_D_forward(fg_ctx* c, const float* x, int B, bool training, const fg_hyper* h) {
  FG_REQUIRE(B >= 1 && B <= c->maxB, "D forward: batch %d out of range [1,%d]", B, c->maxB);
  FG_TRY(net_pack_D(c));
  FG_TRY(amax_reset(c));
  const DLayout& L = c->dl;
  float* P = c->PD;
  if (x != c->D_x)
    FG_CUDA(cudaMemcpyAsync(c->D_x, x, sizeof(float) * (size_t)B * 1024 * c->C, cudaMemcpyDeviceToDevice, c->stream));
  c->D_B = B;
  c->D_train = training;
  const float* masks = training ? c->D_masks : nullptr;
  const float* cur = c->D_x;
  static const char* tags[4] = {"D.C1.fwd", "D.C2.fwd", "D.C3.fwd", "D.C4.fwd"};
  const ConvGeom gL1d{B, 1, 1, 2048, 512, 1, 1};
  bool have_split = false;  // tcb.D_p_hi/lo[i-1] (resp. D_lin_hi/lo[0]) already written by the previous pooling kernel
  for (int i = 0; i < 4; ++i) {
    const int H = kDhw[i];
    const ConvGeom g{B, H, H, dcin(c, i), kDcout[i], 3, 1};
    fg_ctx::TcBufs& t = c->tcb;
    if (i > 0 && use_tc(c, g)) {
      if (f16_on(c)) {  // FP16 split of the pooled activation, kept for the weight gradient
        FG_TRY(split_h_scaled(c, cur, t.D_p_hh[i - 1], t.D_p_hl[i - 1], (int64_t)B * H * H * g.Cin, kSlotDp + i - 1));
        ScopedTimer tm(c, tags[i]);
        FG_TRY(tc_conv_fwd(c, t.D_p_hh[i - 1], t.D_p_hl[i - 1], t.D_Wf_hh[i], t.D_Wf_hl[i], P + L.cb[i], c->D_z[i], g, 0, nullptr,
                           nullptr, 1, inv_scale(c, kSlotDp + i - 1)));
      } else {
        if (!have_split) FG_TRY(tc_split(c, cur, t.D_p_hi[i - 1], t.D_p_lo[i - 1], (int64_t)B * H * H * g.Cin));
        ScopedTimer tm(c, tags[i]);
        FG_TRY(tc_conv_fwd(c, t.D_p_hi[i - 1], t.D_p_lo[i - 1], t.D_Wf_hi[i], t.D_Wf_lo[i], P + L.cb[i], c->D_z[i], g, 0));
      }
    } else {
      FG_TRY(conv_fwd(c, tags[i], cur, c->D_cp[i], P + L.cb[i], c->D_z[i], g));
    }
    // the pooled activation is the next tensor-core operand: its TF32 split comes out of the same kernel
    float *nhi = nullptr, *nlo = nullptr;
    if (i < 3) {
      const ConvGeom gn{B, kDhw[i + 1], kDhw[i + 1], kDcout[i], kDcout[i + 1], 3, 1};
      if (use_tc(c, gn)) { nhi = t.D_p_hi[i]; nlo = t.D_p_lo[i]; }
    } else if (use_tc(c, gL1d)) {
      nhi = t.D_lin_hi[0]; nlo = t.D_lin_lo[0];
    }
    if (f16_on(c)) nhi = nlo = nullptr;  // the FP16 split is made from the fp32 tensor (split_h_scaled)
    have_split = nhi != nullptr;
    {
      AmaxInto am(c, i < 3 ? kSlotDp + i : kSlotLin);  // p[0..2] feed c2..c4, p[3] the first Linear
      FG_TRY(k_d_act_pool_fwd(c, c->D_z[i], P + L.ca[i], masks, kDmoff[i], 1.0f - h->p_spatial, c->D_p[i], B, H, H,
                              kDcout[i], nhi, nlo));
    }
    cur = c->D_p[i];
  }
  const float scale = 1.0f / (1.0f - h->p_drop);
  c->D_drop_scale = scale;
  c->D_spatial_eval = 1.0f - h->p_spatial;
  FG_TRY(lin_fwd(c, "D.L1.fwd", have_split ? nullptr : c->D_p[3], c->D_L1p, 0, P + L.L1b, c->D_zl1, gL1d,
                 c->tcb.D_lin_hi[0], c->tcb.D_lin_lo[0], c->D_p[3], c->tcb.D_lin_hh[0], c->tcb.D_lin_hl[0], kSlotLin));
  {
    AmaxInto am(c, kSlotLin + 1);
    FG_TRY(k_lin_act_drop_fwd(c, c->D_zl1, P + L.a5, masks, 960, scale, c->D_hl1, B, 512));
  }
  FG_TRY(lin_fwd(c, "D.L2.fwd", c->D_hl1, P + L.L2W, 2, P + L.L2b, c->D_zl2, ConvGeom{B, 1, 1, 512, 512, 1, 1},
                 c->tcb.D_lin_hi[1], c->tcb.D_lin_lo[1], c->D_hl1, c->tcb.D_lin_hh[1], c->tcb.D_lin_hl[1], kSlotLin + 1));
  FG_TRY(k_lin_act_drop_fwd(c, c->D_zl2, P + L.a6, masks, 1472, scale, c->D_hl2, B, 512));
  {
    ScopedTimer tm(c, "D.L3.fwd");
    FG_TRY(k_gemv_fwd(c, c->D_hl2, P + L.L3W, P + L.L3b, c->D_logit, B, 512));
  }
  c->D_fwd_valid = true;
  return FG_OK;
}

int net_D_backward(fg_ctx* c, const float* dlogit, bool want_wgrad, bool want_dx) {
  if (!c->D_fwd_valid) {
    fg_set_error("D backward needs a preceding D forward");
    return FG_ERR_STATE;
  }
  const DLayout& L = c->dl;
  float *P = c->PD, *G = c->gD;
  const int B = c->D_B;
  const float* masks = c->D_train ? c->D_masks : nullptr;
  const float scale = c->D_drop_scale, eval_scale = c->D_spatial_eval;
  FG_TRY(amax_reset(c));
  // L3
  if (want_wgrad) {
    ScopedTimer tm(c, "D.L3.wgrad");
    FG_TRY(k_gemv_wgrad_add(c, c->D_hl2, dlogit, G + L.L3W, G + L.L3b, B, 512));
  }
  {
    ScopedTimer tm(c, "D.L3.dgrad");
    FG_TRY(k_gemv_dgrad(c, dlogit, P + L.L3W, c->D_dh, B, 512));
  }
  {
    AmaxInto am(c, kSlotDzl + 1);
    FG_TRY(k_lin_act_drop_bwd(c, c->D_dh, c->D_zl2, P + L.a6, masks, 1472, scale, c->D_dzl, want_wgrad ? G + L.a6 : nullptr, B,
                              512));
  }
  // L2
  const ConvGeom gL2{B, 1, 1, 512, 512, 1, 1}, gL1{B, 1, 1, 2048, 512, 1, 1};
  const bool tcw2 = want_wgrad && use_tc_wgrad(c, gL2), tcw1 = want_wgrad && use_tc_wgrad(c, gL1);
  if (want_wgrad) {
    if (!tcw2) FG_TRY(conv_wgrad(c, "D.L2.wgrad", c->D_hl1, c->D_dzl, gL2, G + L.L2W, 0, 0, 0, 0));
    FG_TRY(k_colsum_add(c, c->D_dzl, G + L.L2b, B, 512, 0, 0));
  }
  FG_TRY(lin_fwd(c, "D.L2.dgrad", c->D_dzl, c->D_L2pd, 3, nullptr, c->D_dh, ConvGeom{B, 1, 1, 512, 512, 1, 1}, nullptr, nullptr,
                 c->D_dzl, nullptr, nullptr, kSlotDy, kSlotDzl + 1));
  if (tcw2)
    FG_TRY(lin_wgrad_tc(c, "D.L2.wgrad", c->tcb.D_lin_hi[1], c->tcb.D_lin_lo[1], gL2, G + L.L2W, 0, 0, c->tcb.D_lin_hh[1],
                        c->tcb.D_lin_hl[1], kSlotLin + 1));
  {
    AmaxInto am(c, kSlotDzl);
    FG_TRY(k_lin_act_drop_bwd(c, c->D_dh, c->D_zl1, P + L.a5, masks, 960, scale, c->D_dzl, want_wgrad ? G + L.a5 : nullptr, B,
                              512));
  }
  // L1
  if (want_wgrad) {
    if (!tcw1) FG_TRY(conv_wgrad(c, "D.L1.wgrad", c->D_p[3], c->D_dzl, gL1, G + L.L1W, 0, 0, 512, 4));
    FG_TRY(k_colsum_add(c, c->D_dzl, G + L.L1b, B, 512, 0, 0));
  }
  FG_TRY(lin_fwd(c, "D.L1.dgrad", c->D_dzl, c->D_L1pd, 1, nullptr, c->D_dp, ConvGeom{B, 1, 1, 512, 2048, 1, 1}, nullptr, nullptr,
                 c->D_dzl, nullptr, nullptr, kSlotDy, kSlotDzl));
  if (tcw1)
    FG_TRY(lin_wgrad_tc(c, "D.L1.wgrad", c->tcb.D_lin_hi[0], c->tcb.D_lin_lo[0], gL1, G + L.L1W, 512, 4, c->tcb.D_lin_hh[0],
                        c->tcb.D_lin_hl[0], kSlotLin));
  static const char* wt[4] = {"D.C1.wgrad", "D.C2.wgrad", "D.C3.wgrad", "D.C4.wgrad"};
  static const char* dt[4] = {"D.C1.dgrad", "D.C2.dgrad", "D.C3.dgrad", "D.C4.dgrad"};
  for (int i = 3; i >= 0; --i) {
    const int H = kDhw[i], cin = dcin(c, i), cout = kDcout[i];
    const float* in = i == 0 ? c->D_x : c->D_p[i - 1];
    const ConvGeom gf{B, H, H, cin, cout, 3, 1}, gd{B, H, H, cout, cin, 3, 1};
    const bool tc = i > 0 && use_tc(c, gf) && use_tc(c, gd);
    const bool tc32 = tc && !f16_on(c);  // TF32 path: dz's hi/lo split comes out of the pooling-backward kernel
    fg_ctx::TcBufs& t = c->tcb;
    // dz and, for the tensor-core layers, its TF32 split in one pass
    {
      AmaxInto am(c, kSlotDdz + i);
      FG_TRY(k_d_act_pool_bwd(c, c->D_dp, c->D_z[i], P + L.ca[i], masks, kDmoff[i], eval_scale, c->D_dz,
                              want_wgrad ? G + L.ca[i] : nullptr, B, H, H, cout, tc32 ? t.dy_hi : nullptr, tc32 ? t.dy_lo : nullptr,
                              want_wgrad ? G + L.cb[i] : nullptr));  // + the conv bias gradient (column sums of dz)
    }
    if (tc && f16_on(c)) FG_TRY(split_h_scaled(c, c->D_dz, t.dy_hh, t.dy_hl, (int64_t)B * H * H * cout, kSlotDy, kSlotDdz + i));
    if (want_wgrad) {
      if (tc && use_tc_wgrad(c, gf)) {
        {
          ScopedTimer tm(c, wt[i]);
          if (f16_on(c))
            FG_TRY(tc_conv_wgrad(c, t.D_p_hh[i - 1], t.D_p_hl[i - 1], t.dy_hh, t.dy_hl, c->wgrad_ws, gf, 1, inv_scale(c, kSlotDy),
                                 inv_scale(c, kSlotDp + i - 1)));
          else
            FG_TRY(tc_conv_wgrad(c, t.D_p_hi[i - 1], t.D_p_lo[i - 1], t.dy_hi, t.dy_lo, c->wgrad_ws, gf));
        }
        FG_TRY(k_unpack_wgrad(c, c->wgrad_ws, G + L.cW[i], cout, cin, 9, 0, 0, 0, 0));
      } else {
        FG_TRY(conv_wgrad(c, wt[i], in, c->D_dz, gf, G + L.cW[i], 0, 0, 0, 0));
      }
    }
    if (i > 0 || want_dx) {
      if (tc && f16_on(c)) {
        ScopedTimer tm(c, dt[i]);
        FG_TRY(tc_conv_fwd(c, t.dy_hh, t.dy_hl, t.D_Wd_hh[i], t.D_Wd_hl[i], nullptr, c->D_dp, gd, 0, nullptr, nullptr, 1,
                           inv_scale(c, kSlotDy)));
      } else if (tc) {
        ScopedTimer tm(c, dt[i]);
        FG_TRY(tc_conv_fwd(c, t.dy_hi, t.dy_lo, t.D_Wd_hi[i], t.D_Wd_lo[i], nullptr, c->D_dp, gd, 0));
      } else {
        FG_TRY(conv_fwd(c, dt[i], c->D_dz, c->D_cpd[i], nullptr, i == 0 ? c->D_dx : c->D_dp, gd));
      }
    }
  }
  return FG_OK;
}

// ---------------------------------------------------------------------------------------------------
// optimizer: penalty -> clamp -> interruptableAdam, all on device
// ---------------------------------------------------------------------------------------------------
int net_optim(fg_ctx* c, int net, const fg_hyper* h, float grad_scale, bool gate) {
  (void)gate;
  const bool isD = net == FG_NET_D;
  float *p = isD ? c->PD : c->PG, *g = isD ? c->gD : c->gG, *m = isD ? c->mD : c->mG, *v = isD ? c->vD : c->vG;
  const int64_t n = isD ? c->dl.total : c->gl.total;
  const float l1 = isD ? h->D_L1 : h->G_L1, l2 = isD ? h->D_L2 : h->G_L2;
  const bool pen = l1 != 0.f || l2 != 0.f;
  // G quirk: the L1 gradient term is multiplied by G_L2 (adversarial.lua:223)
  const float l1_grad = !pen ? 0.f : (isD ? l1 : l2);
  if (pen) FG_TRY(k_penalty_loss(c, p, n, l1, l2, isD ? &c->dstats->loss_D : &c->dstats->loss_G));
  ScopedTimer tm(c, isD ? "hbm.optim.D" : "hbm.optim.G");
  FG_TRY(k_optim_update(c, isD ? c->opt_D : c->opt_G, p, g, m, v, n, h->beta1, h->beta2, h->eps,
                        isD ? c->sgd_mom_D : c->sgd_mom_G, l1_grad, pen ? l2 : 0.f, isD ? h->D_clamp : h->G_clamp, grad_scale,
                        isD ? &c->dstats->step_D : &c->dstats->step_G, isD ? &c->dstats->do_train_D : &c->dstats->do_train_G,
                        isD ? &c->dstats->t_D : &c->dstats->t_G));
  if (isD) c->D_packed = false; else c->G_packed = false;
  return FG_OK;
}

// GRAD_PARAMETERS_x:zero() incl. the DP tail scalars
int net_zero_grads(fg_ctx* c, int net) {
  const bool d = net == FG_NET_D;
  float *g = d ? c->gD : c->gG, *tail = d ? c->tailD : c->tailG;
  const int64_t n = d ? c->dl.total : c->gl.total;
  if (tail == g + n) {
    FG_CUDA(cudaMemsetAsync(g, 0, sizeof(float) * (n + kGradTail), c->stream));
  } else {  // caller-owned gradient buffer (fg_bind_params): the tail lives in the library
    FG_CUDA(cudaMemsetAsync(g, 0, sizeof(float) * n, c->stream));
    FG_CUDA(cudaMemsetAsync(tail, 0, sizeof(float) * kGradTail, c->stream));
  }
  return FG_OK;
}
int net_allreduce_grads(fg_ctx* c, int net) {
  const bool d = net == FG_NET_D;
  float *g = d ? c->gD : c->gG, *tail = d ? c->tailD : c->tailG;
  const int64_t n = d ? c->dl.total : c->gl.total;
  if (tail == g + n) return net_allreduce(c, g, n + kGradTail);
  FG_TRY(net_group(true));
  FG_TRY(net_allreduce(c, g, n));
  FG_TRY(net_allreduce(c, tail, kGradTail));
  return net_group(false);
}

// ---------------------------------------------------------------------------------------------------
// one iteration of the adversarial.lua loop body (D_iterations = G_iterations = 1)
// ---------------------------------------------------------------------------------------------------
// the step proper; the seed of the device-drawn dropout masks is read from c->seed_dev
static int train_step_body(fg_ctx* c, const fg_hyper* h, int B, const float* real, const float* noiseD, const float* noiseG,
                           const float* masksD, const float* masksG) {
  const uint64_t seed = 0;
  const uint64_t* seed_dev = c->seed_dev;
  const int Bh = B / 2, C = c->C;
  const size_t img = (size_t)C * 1024;
  const float world = (float)c->world;
  // ---- D step (adversarial.lua:240-268) ----
  FG_TRY(net_G_forward(c, noiseD, Bh, true));  // createImages: G in training mode (nn_utils.lua:52)
  FG_TRY(k_nchw_to_nhwc(c, real, c->D_x, Bh, C, 1024));
  FG_CUDA(cudaMemcpyAsync(c->D_x + Bh * img, c->G_y, sizeof(float) * Bh * img, cudaMemcpyDeviceToDevice, c->stream));
  if (masksD)
    FG_CUDA(cudaMemcpyAsync(c->D_masks, masksD, sizeof(float) * (size_t)B * kMaskPerSample, cudaMemcpyDeviceToDevice,
                            c->stream));
  else
    FG_TRY(k_masks_generate(c, c->D_masks, B, seed * 2 + 1, h->p_spatial, h->p_drop, seed_dev));
  FG_TRY(net_zero_grads(c, FG_NET_D));
  FG_TRY(net_D_forward(c, c->D_x, B, true, h));
  FG_TRY(k_sigmoid_bce(c, c->D_logit, c->D_out, c->D_dlogit, &c->dstats->loss_D, c->tailD, B, Bh));
  if (c->debug_keep) {  // tests: the G step's D forward overwrites these
    const float* src[8] = {c->D_z[0], c->D_z[1], c->D_z[2], c->D_z[3], c->D_zl1, c->D_zl2, c->D_logit, c->D_out};
    const size_t per[8] = {65536, 32768, 16384, 8192, 512, 512, 1, 1};
    for (int i = 0; i < 8; ++i) {
      if (!c->keep_D[i]) FG_TRY(dalloc(c, &c->keep_D[i], (size_t)c->maxB * per[i]));
      FG_CUDA(cudaMemcpyAsync(c->keep_D[i], src[i], sizeof(float) * B * per[i], cudaMemcpyDeviceToDevice, c->stream));
    }
    c->keep_B = B;
  }
  FG_TRY(net_D_backward(c, c->D_dlogit, true, false));
  const bool overlap = c->world > 1 && c->dp_overlap && !c->timing;
  if (overlap) {
    // D's gradient all-reduce, gate and optimizer on the communication stream; the G step's G forward (it depends on G's
    // parameters only) proceeds on the compute stream and D is joined before its next forward.  The replicas stay
    // bit-identical: the same reductions in the same order, only on another stream.
    if (!c->comm_stream) {
      FG_CUDA(cudaStreamCreateWithFlags(&c->comm_stream, cudaStreamNonBlocking));
      FG_CUDA(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
      FG_CUDA(cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
    }
    FG_CUDA(cudaEventRecord(c->ev_fork, c->stream));
    FG_CUDA(cudaStreamWaitEvent(c->comm_stream, c->ev_fork, 0));
    cudaStream_t compute = c->stream;
    c->stream = c->comm_stream;
    int r = net_allreduce_grads(c, FG_NET_D);
    if (r == FG_OK) r = k_gate_and_prep(c, FG_NET_D, h, c->tailD, B, world);
    if (r == FG_OK) r = net_optim(c, FG_NET_D, h, 1.0f / world, true);
    if (r == FG_OK && cudaEventRecord(c->ev_join, c->comm_stream) != cudaSuccess) r = FG_ERR_CUDA;
    c->stream = compute;
    FG_TRY(r);
  } else {
    if (c->world > 1) FG_TRY(net_allreduce_grads(c, FG_NET_D));
    FG_TRY(k_gate_and_prep(c, FG_NET_D, h, c->tailD, B, world));
    FG_TRY(net_optim(c, FG_NET_D, h, 1.0f / world, true));
  }
  // ---- G step (adversarial.lua:275-288) ----
  FG_TRY(net_zero_grads(c, FG_NET_G));
  {
    // while the collective is in flight the persistent convolution kernels leave a few SMs to it (FG_DP_RESERVE_SMS)
    static const int reserve = getenv("FG_DP_RESERVE_SMS") ? atoi(getenv("FG_DP_RESERVE_SMS")) : 0;
    c->reserve_sms = overlap ? reserve : 0;
    const int r = net_G_forward(c, noiseG, B, true);
    c->reserve_sms = 0;
    FG_TRY(r);
  }
  if (overlap) FG_CUDA(cudaStreamWaitEvent(c->stream, c->ev_join, 0));
  if (masksG)
    FG_CUDA(cudaMemcpyAsync(c->D_masks, masksG, sizeof(float) * (size_t)B * kMaskPerSample, cudaMemcpyDeviceToDevice,
                            c->stream));
  else
    FG_TRY(k_masks_generate(c, c->D_masks, B, seed * 2 + 2, h->p_spatial, h->p_drop, seed_dev));
  FG_TRY(net_D_forward(c, c->G_y, B, true, h));
  FG_TRY(k_sigmoid_bce(c, c->D_logit, c->D_out, c->D_dlogit, &c->dstats->loss_G, c->tailG, B, B));
  FG_TRY(net_D_backward(c, c->D_dlogit, false, true));  // D's weight grads are discarded by the reference (:209 vs :92)
  FG_TRY(net_G_backward(c, c->D_dx, nullptr));
  if (c->world > 1) FG_TRY(net_allreduce_grads(c, FG_NET_G));
  FG_TRY(k_gate_and_prep(c, FG_NET_G, h, c->tailG, B, world));
  FG_TRY(net_optim(c, FG_NET_G, h, 1.0f / world, false));
  FG_CUDA(cudaMemcpyAsync(c->hstats, c->dstats, sizeof(DeviceStats), cudaMemcpyDeviceToHost, c->stream));
  return FG_OK;
}

// ---------------------------------------------------------------------------------------------------
// CUDA-graph replay of the step.  A step is ~200 launches of mostly short kernels; replaying a captured graph removes
// the launch gaps (measured 4.19 -> 3.87 ms at batch 256).  A graph bakes in every kernel argument, so it is keyed on all
// of them: batch, hyper-parameters, input / parameter pointers, option epoch.  The first step with a new key runs
// eagerly (it also performs the lazy allocations), the second is captured, later ones are replayed.
// ---------------------------------------------------------------------------------------------------
void net_graphs_clear(fg_ctx* c) {
  for (auto& g : c->graphs)
    if (g.exec) cudaGraphExecDestroy(g.exec);
  c->graphs.clear();
}
namespace {
template <class T>
void key_add(std::vector<uint8_t>& k, const T& v) {
  const uint8_t* p = reinterpret_cast<const uint8_t*>(&v);
  k.insert(k.end(), p, p + sizeof(T));
}
}  // namespace

// Runs `body` (a sequence of launches on c->stream that reads its seed from c->seed_dev) eagerly the first time a key
// is seen, captures it the second time and replays the captured graph afterwards.  `repack` is called before the
// capture and after every replay: it must mark the weight packs stale (the captured sequence has to contain the pack
// kernels whatever the flags said at capture time, and a replayed optimizer step invalidates them again).
int net_graph_run(fg_ctx* c, std::vector<fg_ctx::StepGraph>& cache, const std::vector<uint8_t>& key, uint64_t seed,
                  const std::function<int()>& body, const std::function<void()>& repack, bool allow_graph) {
  FG_TRY(k_set_u64(c, c->seed_dev, seed));
  static const bool env_off = getenv("FG_GRAPH") && atoi(getenv("FG_GRAPH")) == 0;
  if (!allow_graph || !c->use_graph || env_off || c->timing || c->debug_keep) return body();
  fg_ctx::StepGraph* e = nullptr;
  for (auto& g : cache)
    if (g.key == key) e = &g;
  if (!e) {
    if (cache.size() >= 8) {  // oldest out
      if (cache.front().exec) cudaGraphExecDestroy(cache.front().exec);
      cache.erase(cache.begin());
    }
    cache.emplace_back();
    cache.back().key = key;
    return body();  // eager: warms every lazy allocation
  }
  if (e->failed) return body();
  if (!e->exec) {
    repack();
    const int64_t l0 = c->launches;
    FG_CUDA(cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeRelaxed));
    const int r = body();
    cudaGraph_t g = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(c->stream, &g);
    cudaGraphExec_t ex = nullptr;
    if (r == FG_OK && ce == cudaSuccess && g && cudaGraphInstantiate(&ex, g, 0) == cudaSuccess) {
      e->exec = ex;
      e->launches = c->launches - l0;
      c->launches = l0;
    } else {
      cudaGetLastError();
      e->failed = true;
    }
    if (g) cudaGraphDestroy(g);
    FG_TRY(r);
    if (e->failed) {  // nothing ran during the failed capture
      FG_TRY(k_set_u64(c, c->seed_dev, seed));
      return body();
    }
  }
  FG_CUDA(cudaGraphLaunch(e->exec, c->stream));
  c->launches += e->launches;
  repack();
  return FG_OK;
}

int net_train_step(fg_ctx* c, const fg_hyper* h, int B, const float* real, const float* noiseD, const float* noiseG,
                   const float* masksD, const float* masksG, uint64_t seed, bool allow_graph) {
  FG_REQUIRE(B >= 4 && B % 2 == 0 && B <= c->maxB, "train step: batch %d must be even, >=4 and <= %d", B, c->maxB);
  std::vector<uint8_t> key;
  key_add(key, c->graph_epoch);
  key_add(key, B);
  key_add(key, *h);
  const void* ptrs[] = {real, noiseD, noiseG, masksD, masksG, c->PG, c->PD, c->gG, c->gD, (const void*)c->stream, c->nccl_comm};
  key_add(key, ptrs);
  return net_graph_run(
      c, c->graphs, key, seed, [&]() { return train_step_body(c, h, B, real, noiseD, noiseG, masksD, masksG); },
      [c]() { c->G_packed = c->D_packed = false; }, allow_graph);
}
