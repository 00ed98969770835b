// TEST INFRASTRUCTURE (see fg_oracle.cpp header): the coarse-to-fine nets and loop of fg_oracle_c2f.h at a runtime fine
// size S = train_c2f.lua --fineSize (16, 32 or 64; models_c2f.lua:113-145 and :237-278 size everything from
// `dimensions`): G runs at S x S, D's convolutions at S and S/2, and its Linear reads View(256*(S/4)^2).
// PARITY UNPINNED, as for the 32x32 restatement.  Built into its own library, libfg_oracle_c2f_sized.so, by
// __graft_entry__.build(): this translation unit is fg_oracle.cpp (every op of the oracle) plus the sized nets and
// their exports fgo_c2fs_*.  At S = 32 the sized restatement equals the fixed-size one (tests/test_c2f_sizes.py).
#include "fg_oracle.cpp"

namespace {
// getParameters() order of create_D_c (models_c2f.lua:247-265); G's layout does not depend on S (C2fGLayout)
struct C2fDLayoutSized {  // models_c2f.lua:247-265
  int64_t cW[4], cb[4], ca[4], L1W, L1b, a5, L2W, L2b, total;
  int cin[4], cout[4];
  int flat;  // View(256*(S/4)^2)
  C2fDLayoutSized(int C, int S) {
    flat = 256 * (S / 4) * (S / 4);
    const int ci[4] = {C, 64, 64, 128}, co[4] = {64, 64, 128, 256};
    int64_t o = 0;
    for (int i = 0; i < 4; ++i) {
      cin[i] = ci[i]; cout[i] = co[i];
      cW[i] = o; o += (int64_t)co[i] * ci[i] * 9;
      cb[i] = o; o += co[i];
      ca[i] = o; o += 1;
    }
    L1W = o; o += (int64_t)512 * flat;
    L1b = o; o += 512;
    a5 = o; o += 1;
    L2W = o; o += 512;
    L2b = o; o += 1;
    total = o;
  }
};
inline int c2f_mask_per_sample(int S) { return 256 * (S / 4) * (S / 4) + 512; }  // [256][S/4][S/4] then [512]

template <class T>
struct C2fGNetSized {
  int B = 0, C = 3, S = 32;
  std::vector<T> x;              // JoinTable(2,2): [B][1+C][S][S], noise plane first (models_c2f.lua:116)
  std::vector<T> z[5], h[4];     // conv outputs, PReLU outputs; z[4] is the generated diff
  void forward(const T* P, const T* noise, const T* cond, int B_, int C_) {
    B = B_; C = C_;
    C2fGLayout L(C);
    const size_t HW = (size_t)S * S;
    x.resize((size_t)B * (C + 1) * HW);
    for (int b = 0; b < B; ++b) {
      std::copy(noise + (size_t)b * HW, noise + (size_t)(b + 1) * HW, x.begin() + (size_t)b * (C + 1) * HW);
      std::copy(cond + (size_t)b * C * HW, cond + (size_t)(b + 1) * C * HW, x.begin() + (size_t)b * (C + 1) * HW + HW);
    }
    const T* cur = x.data();
    for (int i = 0; i < 5; ++i) {
      const size_t n = (size_t)B * L.cout[i] * HW;
      z[i].resize(n);
      conv_fwd(B, L.cin[i], S, S, L.cout[i], L.k[i], cur, P + L.cW[i], P + L.cb[i], z[i].data());
      if (i < 4) {
        h[i].resize(n);
        prelu_fwd(n, z[i].data(), P[L.ca[i]], h[i].data());
        cur = h[i].data();
      }
    }
  }
  // dout [B][C][S][S]; accumulates into dP; the gradient w.r.t. {noise, coarse} is not needed by the loop
  void backward(const T* P, const T* dout, T* dP) {
    C2fGLayout L(C);
    const size_t HW = (size_t)S * S;
    std::vector<T> dz(dout, dout + (size_t)B * C * HW), dh;
    for (int i = 4; i >= 0; --i) {
      const T* in = i == 0 ? x.data() : h[i - 1].data();
      const bool need_dx = i > 0;
      if (need_dx) dh.assign((size_t)B * L.cin[i] * HW, T(0));
      conv_bwd(B, L.cin[i], S, S, L.cout[i], L.k[i], in, P + L.cW[i], dz.data(), need_dx ? dh.data() : nullptr,
               dP + L.cW[i], dP + L.cb[i]);
      if (i > 0) {
        dz.resize(dh.size());
        prelu_bwd(dh.size(), z[i - 1].data(), P[L.ca[i - 1]], dh.data(), dz.data(), dP + L.ca[i - 1]);
      }
    }
  }
};

template <class T>
struct C2fDNetSized {
  int B = 0, C = 3, S = 32;
  bool training = true;
  std::vector<T> x;                    // CAddTable: diff + coarse (models_c2f.lua:240)
  std::vector<T> z[4], h[4], p2, p4, d4;
  std::vector<unsigned char> arg2, arg4;
  std::vector<T> zl1, al1, hl1, logit, out, mask;
  void forward(const T* P, const T* diff, const T* cond, int B_, int C_, bool training_, const T* masks) {
    B = B_; C = C_; training = training_;
    C2fDLayoutSized L(C, S);
    const int hw[4] = {S, S, S / 2, S / 2}, F = L.flat, M = c2f_mask_per_sample(S);
    x.resize((size_t)B * C * S * S);
    for (size_t i = 0; i < x.size(); ++i) x[i] = diff[i] + cond[i];
    if (training) mask.assign(masks, masks + (size_t)B * M);
    const T* cur = x.data();
    for (int i = 0; i < 4; ++i) {
      const int H = hw[i];
      const size_t n = (size_t)B * L.cout[i] * H * H;
      z[i].resize(n); h[i].resize(n);
      conv_fwd(B, L.cin[i], H, H, L.cout[i], 3, cur, P + L.cW[i], P + L.cb[i], z[i].data());
      prelu_fwd(n, z[i].data(), P[L.ca[i]], h[i].data());
      cur = h[i].data();
      if (i == 1) {
        p2.resize(n / 4); arg2.resize(n / 4);
        maxpool2_fwd(B * 64, S, S, h[1].data(), p2.data(), arg2.data());
        cur = p2.data();
      } else if (i == 3) {
        p4.resize(n / 4); arg4.resize(n / 4);
        maxpool2_fwd(B * 256, S / 2, S / 2, h[3].data(), p4.data(), arg4.data());
      }
    }
    // nn.Dropout() p=0.5 (v2): train y = x*mask/(1-p), eval identity; then View(256*(S/4)^2) in (c,h,w) order
    d4.resize(p4.size());
    for (int b = 0; b < B; ++b)
      for (int j = 0; j < F; ++j)
        d4[(size_t)b * F + j] = training ? p4[(size_t)b * F + j] * mask[(size_t)b * M + j] * T(2) : p4[(size_t)b * F + j];
    zl1.resize((size_t)B * 512); al1.resize(zl1.size()); hl1.resize(zl1.size());
    linear_fwd(B, F, 512, d4.data(), P + L.L1W, P + L.L1b, zl1.data());
    prelu_fwd(zl1.size(), zl1.data(), P[L.a5], al1.data());
    for (int b = 0; b < B; ++b)
      for (int j = 0; j < 512; ++j)
        hl1[(size_t)b * 512 + j] = training ? al1[(size_t)b * 512 + j] * mask[(size_t)b * M + F + j] * T(2)
                                           : al1[(size_t)b * 512 + j];
    logit.resize(B); out.resize(B);
    linear_fwd(B, 512, 1, hl1.data(), P + L.L2W, P + L.L2b, logit.data());
    for (int b = 0; b < B; ++b) out[b] = d_output(sigmoid(logit[b]));  // fp32 at the criterion boundary (fg_oracle.cpp)
  }
  // dout [B] = dLoss/d(sigmoid output); dP may be null (weight grads skipped); ddiff = MODEL_D.gradInput[1]
  void backward(const T* P, const T* dout, T* dP, T* ddiff) {
    C2fDLayoutSized L(C, S);
    const int hw[4] = {S, S, S / 2, S / 2}, F = L.flat, M = c2f_mask_per_sample(S);
    T dummy = 0;
    auto gw = [&](int64_t off) { return dP ? dP + off : (T*)nullptr; };   // weight/bias grads (skipped if null)
    auto ga = [&](int64_t off) { return dP ? dP + off : &dummy; };        // PReLU slope grads
    std::vector<T> dlogit(B);
    for (int b = 0; b < B; ++b) dlogit[b] = dout[b] * out[b] * (T(1) - out[b]);
    std::vector<T> dhl1((size_t)B * 512), dal1(dhl1.size()), dzl1(dhl1.size());
    linear_bwd(B, 512, 1, hl1.data(), P + L.L2W, dlogit.data(), dhl1.data(), gw(L.L2W), gw(L.L2b));
    for (int b = 0; b < B; ++b)
      for (int j = 0; j < 512; ++j)
        dal1[(size_t)b * 512 + j] = training ? dhl1[(size_t)b * 512 + j] * mask[(size_t)b * M + F + j] * T(2)
                                            : dhl1[(size_t)b * 512 + j];
    prelu_bwd(dzl1.size(), zl1.data(), P[L.a5], dal1.data(), dzl1.data(), ga(L.a5));
    std::vector<T> dd4((size_t)B * F), dp4(dd4.size());
    linear_bwd(B, F, 512, d4.data(), P + L.L1W, dzl1.data(), dd4.data(), gw(L.L1W), gw(L.L1b));
    for (int b = 0; b < B; ++b)
      for (int j = 0; j < F; ++j)
        dp4[(size_t)b * F + j] = training ? dd4[(size_t)b * F + j] * mask[(size_t)b * M + j] * T(2) : dd4[(size_t)b * F + j];
    std::vector<T> dh, dz, dx;
    for (int i = 3; i >= 0; --i) {
      const int H = hw[i];
      const size_t n = (size_t)B * L.cout[i] * H * H;
      if (i == 3) {
        dh.resize(n);
        maxpool2_bwd(B * 256, S / 2, S / 2, dp4.data(), arg4.data(), dh.data());
      } else if (i == 1) {
        dh.resize(n);
        maxpool2_bwd(B * 64, S, S, dx.data(), arg2.data(), dh.data());
      } else {
        dh.swap(dx);
      }
      dz.resize(n);
      prelu_bwd(n, z[i].data(), P[L.ca[i]], dh.data(), dz.data(), ga(L.ca[i]));
      const T* in = i == 0 ? x.data() : (i == 2 ? p2.data() : h[i - 1].data());
      const bool need_dx = i > 0 || ddiff != nullptr;
      if (need_dx) dx.assign((size_t)B * L.cin[i] * H * H, T(0));
      conv_bwd(B, L.cin[i], H, H, L.cout[i], 3, in, P + L.cW[i], dz.data(), need_dx ? dx.data() : nullptr, gw(L.cW[i]),
               gw(L.cb[i]));
    }
    if (ddiff) std::copy(dx.begin(), dx.end(), ddiff);  // CAddTable backward: identity to both addends
  }
};

// One iteration of the adversarial_c2f.lua loop body (D_iterations = G_iterations = 1, adam for both) at fine size S.
//   real_diff[B/2,C,S,S]    fine-minus-coarse of the real half            (:127-130)
//   condD[B,C,S,S]          coarse images: rows < B/2 belong to the real samples, the rest to the fakes (:129,:137-141)
//   noiseD[B/2,1,S,S]       U(-1,1) for the generated half                (:135, :145)
//   condG[B,C,S,S], noiseG[B,1,S,S]  redrawn for the G step               (:168-174)
//   masksD/masksG[B,c2f_mask_per_sample(S)]  nn.Dropout keep flags of the two D forwards (16896 at S = 32)
// `optim.adam` (un-pinned third-party, 2015) is the routine interruptable_optimizers.lua:49-94 was copied from;
// the restatement uses the same update.
template <class T>
void c2f_train_iteration_sized(int B, int C, const Hyper& hp, const T* real_diff, const T* condD, const T* noiseD,
                         const T* condG, const T* noiseG, const T* masksD, const T* masksG, T* PD, T* PG, T* mD, T* vD,
                         T* mG, T* vG, int* tD, int* tG, double* stats, T* gradD_out, T* gradG_out, T* fake_out,
                         T* outD_out, int S) {
  C2fGLayout LG(C);
  C2fDLayoutSized LD(C, S);
  const int Bh = B / 2;
  const size_t img = (size_t)C * S * S;
  C2fGNetSized<T> G;
  C2fDNetSized<T> D;
  G.S = D.S = S;
  // ---- D step ----
  G.forward(PG, noiseD, condD + Bh * img, Bh, C);
  if (fake_out) std::copy(G.z[4].begin(), G.z[4].end(), fake_out);
  std::vector<T> inputs((size_t)B * img), targets(B);
  std::copy(real_diff, real_diff + Bh * img, inputs.begin());
  std::copy(G.z[4].begin(), G.z[4].end(), inputs.begin() + Bh * img);
  for (int i = 0; i < B; ++i) targets[i] = i < Bh ? T(1) : T(0);
  std::vector<T> gD(LD.total, T(0));
  D.forward(PD, inputs.data(), condD, B, C, true, masksD);
  if (outD_out) std::copy(D.out.begin(), D.out.end(), outD_out);
  T fD = bce_fwd(B, D.out.data(), targets.data());
  std::vector<T> df(B);
  bce_bwd(B, D.out.data(), targets.data(), df.data());
  D.backward(PD, df.data(), gD.data(), nullptr);
  fD += penalty_clamp(LD.total, PD, gD.data(), T(hp.D_L1), T(hp.D_L1), T(hp.D_L2), T(hp.D_clamp));  // :56-63, :74-76
  double conf[4] = {0, 0, 0, 0};
  for (int i = 0; i < B; ++i) {
    const bool pred1 = D.out[i] > T(0.5);
    const bool t1 = i < Bh;
    conf[(pred1 ? 0 : 1) + (t1 ? 0 : 2)] += 1;
  }
  if (gradD_out) std::copy(gD.begin(), gD.end(), gradD_out);
  *tD += 1;
  adam(LD.total, PD, gD.data(), mD, vD, *tD, hp.lr_D, hp.beta1, hp.beta2, hp.eps);
  // ---- G step ----
  std::vector<T> gG(LG.total, T(0));
  G.forward(PG, noiseG, condG, B, C);
  for (int i = 0; i < B; ++i) targets[i] = T(1);
  D.forward(PD, G.z[4].data(), condG, B, C, true, masksG);
  T fG = bce_fwd(B, D.out.data(), targets.data());
  bce_bwd(B, D.out.data(), targets.data(), df.data());
  std::vector<T> ddiff((size_t)B * img);
  D.backward(PD, df.data(), nullptr, ddiff.data());
  G.backward(PG, ddiff.data(), gG.data());
  // same quirk as adversarial.lua:223: sign(p) is scaled by G_L2 (adversarial_c2f.lua:108)
  fG += penalty_clamp(LG.total, PG, gG.data(), T(hp.G_L1), T(hp.G_L2), T(hp.G_L2), T(hp.G_clamp));
  if (gradG_out) std::copy(gG.begin(), gG.end(), gradG_out);
  *tG += 1;
  adam(LG.total, PG, gG.data(), mG, vG, *tG, hp.lr_G, hp.beta1, hp.beta2, hp.eps);
  stats[0] = (double)fD; stats[1] = (double)fG;
  stats[2] = conf[0]; stats[3] = conf[1]; stats[4] = conf[2]; stats[5] = conf[3];
  stats[6] = 0; stats[7] = 0;
}
}  // namespace

#define FG_C2FS_EXPORTS(SFX, T)                                                                                  \
  extern "C" {                                                                                                   \
  void* fgo_c2fs_G_new_##SFX(int S) {                                                                            \
    C2fGNetSized<T>* g = new C2fGNetSized<T>();                                                                  \
    g->S = S;                                                                                                    \
    return g;                                                                                                    \
  }                                                                                                              \
  void fgo_c2fs_G_free_##SFX(void* h) { delete (C2fGNetSized<T>*)h; }                                            \
  void fgo_c2fs_G_forward_##SFX(void* h, const T* P, const T* noise, const T* cond, int B, int C, T* out) {      \
    C2fGNetSized<T>* g = (C2fGNetSized<T>*)h;                                                                    \
    g->forward(P, noise, cond, B, C);                                                                            \
    std::copy(g->z[4].begin(), g->z[4].end(), out);                                                              \
  }                                                                                                              \
  void fgo_c2fs_G_backward_##SFX(void* h, const T* P, const T* dout, T* dP) {                                    \
    ((C2fGNetSized<T>*)h)->backward(P, dout, dP);                                                                \
  }                                                                                                              \
  void* fgo_c2fs_D_new_##SFX(int S) {                                                                            \
    C2fDNetSized<T>* d = new C2fDNetSized<T>();                                                                  \
    d->S = S;                                                                                                    \
    return d;                                                                                                    \
  }                                                                                                              \
  void fgo_c2fs_D_free_##SFX(void* h) { delete (C2fDNetSized<T>*)h; }                                            \
  void fgo_c2fs_D_forward_##SFX(void* h, const T* P, const T* diff, const T* cond, int B, int C, int training,   \
                                const T* masks, T* out) {                                                        \
    C2fDNetSized<T>* d = (C2fDNetSized<T>*)h;                                                                    \
    d->forward(P, diff, cond, B, C, training != 0, masks);                                                       \
    std::copy(d->out.begin(), d->out.end(), out);                                                                \
  }                                                                                                              \
  void fgo_c2fs_D_backward_##SFX(void* h, const T* P, const T* dout, T* dP, T* ddiff) {                          \
    ((C2fDNetSized<T>*)h)->backward(P, dout, dP, ddiff);                                                         \
  }                                                                                                              \
  void fgo_c2fs_train_iteration_##SFX(int S, int B, int C, const double* hp11, const T* real_diff,               \
                                      const T* condD, const T* noiseD, const T* condG, const T* noiseG,          \
                                      const T* masksD, const T* masksG, T* PD, T* PG, T* mD, T* vD, T* mG,       \
                                      T* vG, int* tD, int* tG, double* stats, T* gradD_out, T* gradG_out,        \
                                      T* fake_out, T* outD_out) {                                                \
    Hyper hp{hp11[0], hp11[1], hp11[2], hp11[3], hp11[4], hp11[5], hp11[6], hp11[7], hp11[8], hp11[9],           \
             hp11[10]};                                                                                          \
    c2f_train_iteration_sized<T>(B, C, hp, real_diff, condD, noiseD, condG, noiseG, masksD, masksG, PD, PG, mD,  \
                                 vD, mG, vG, tD, tG, stats, gradD_out, gradG_out, fake_out, outD_out, S);        \
  }                                                                                                              \
  }

FG_C2FS_EXPORTS(f64, double)
FG_C2FS_EXPORTS(f32, float)

extern "C" {
long fgo_c2fs_D_param_count(int C, int S) { return (long)C2fDLayoutSized(C, S).total; }
int fgo_c2fs_mask_per_sample(int S) { return c2f_mask_per_sample(S); }
}
