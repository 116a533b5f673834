// avc_neus.cu -- host orchestration + C ABI of the NeuS render forward / backward.
//
// Kernel sequence (one chunk of rays; see oracle/neus_manual.py for the same steps on the CPU):
//   pack            k_pack_linear per linear (weight-norm folded once per call)
//   placement       k_coarse_z -> [k_encode_samples -> value chain -> k_thin_nt(sdf)] -> k_upsample
//                   -> ... -> k_merge                      (renderer.py:336-352)
//   fine forward    k_encode_fine -> value chain (gemm_nt + EpiValue, stash z) -> sdf / feature heads
//                   -> k_chain_start -> gradient chain (gemm_nt + EpiChain) -> k_normal
//                   -> colour net (gemm_nt + EpiColor0/EpiRelu, k_thin_nt heads) -> k_composite_fwd
//   backward        k_composite_bwd -> colour backward -> k_dge -> second-order sweep (gemm_nt +
//                   EpiChainBwd, gemm_tn) -> value backward (gemm_nt + EpiDgrad, gemm_tn) -> k_wn_backward
#include <cstdio>
#include <cstring>

#include "avc_chain.h"
#include "avc_common.cuh"
#include "avc_gemm_simt.cuh"
#include "avc_gemm_tc.cuh"
#include "avc_neus_kernels.cuh"
#include "avc_neus_plan.cuh"

using namespace avc;

namespace {

inline int blocks_for(int64_t n, int threads) { return (int)((n + threads - 1) / threads); }

// -------------------------------------------------------------------------------- engine dispatch
// engine 0: fp32 FFMA tiles on the fp32 buffers; engine 1: wgmma tiles on the two-term bf16 copies.
// B operands are addressed by their offset in the packed-weight buffer (same offset in the bf16 split).
inline Split16 with_ld(Split16 s, int ld) { s.ld = ld; return s; }

// NP: MMAs per product on the wgmma engine: 3 = two-term split operands, 1 = the hi halves only (single-pass bf16).
template <int NP = 3, typename Epi>
int gemm_nt(const NeusPlan& pl, const NeusWs& w, cudaStream_t st, int64_t M, int N, int K, const float* A, int lda,
            const Split16& A16, int64_t pk_off, int ldb, const Epi& epi) {
  if (pl.cfg.engine == 1) {
    tc::SplitPtr a{A16.hi, A16.lo, lda}, b{w.pk_hi + pk_off, w.pk_lo + pk_off, ldb};
    return tc::launch_gemm_tc_nt<NP, Epi>(st, M, N, K, a, b, epi, /*b_const: the packed weights*/ true);
  }
  return launch_gemm_nt(st, M, N, (int)round_up(K, 4), A, lda, w.pack + pk_off, ldb, epi);
}
// The colour net (SURVEY Appendix C: it tolerates single-pass bf16) runs with cfg.color_products MMAs per product.
// (Single-pass forward / dgrad with split weight gradients was measured too: same gradient error as all-single -- the
// error enters through the rounded activations -- at half the gain; not kept.)
inline bool color_single(const NeusPlan& pl) { return pl.cfg.engine == 1 && pl.cfg.color_products == 1; }
template <typename Epi>
int gemm_nt_color(const NeusPlan& pl, const NeusWs& w, cudaStream_t st, int64_t M, int N, int K, const float* A, int lda,
                  const Split16& A16, int64_t pk_off, int ldb, const Epi& epi) {
  return color_single(pl) ? gemm_nt<1>(pl, w, st, M, N, K, A, lda, A16, pk_off, ldb, epi)
                          : gemm_nt<3>(pl, w, st, M, N, K, A, lda, A16, pk_off, ldb, epi);
}

int colsum(cudaStream_t st, const float* X, int ld, int NC, int64_t P, float scale, float* out);

// C[N1][ldc] += A^T B ; optionally bias_out[i] += sum_p A[p,i] (the bias gradient of the same linear): fused into the
// wgmma kernel as one extra 8-wide MMA against a tile of ones, a separate column-sum kernel for the fp32 engine.
inline int gemm_tn(const NeusPlan& pl, const NeusWs& w, cudaStream_t st, int64_t P, int N1, int N2, const float* A,
                   int lda, const Split16& A16, const float* B, int ldb, const Split16& B16, float* C, int ldc,
                   float* bias_out = nullptr, bool single = false) {
  (void)w;
  if (pl.cfg.engine == 1) {
    tc::SplitPtr a{A16.hi, A16.lo, lda}, b{B16.hi, B16.lo, ldb};
    if (single || pl.cfg.wgrad_products == 1) return tc::launch_gemm_tc_tn<1>(st, P, N1, N2, a, b, C, ldc, bias_out);
    return tc::launch_gemm_tc_tn<3>(st, P, N1, N2, a, b, C, ldc, bias_out);
  }
  AVC_TRY(launch_gemm_tn(st, P, N1, N2, A, lda, B, ldb, C, ldc));
  if (bias_out) AVC_TRY(colsum(st, A, lda, N1, P, 1.f, bias_out));
  return 0;
}

// -------------------------------------------------------------------------------- packing
int pack_weights(const NeusPlan& pl, const float* params, float* pack, cudaStream_t st) {
  static_assert(kMaxJobs >= 2 * kMaxLin + 4, "job table too small");
  PackJobs jobs;
  jobs.n = 0;
  int maxN = 1;
  auto add = [&](const PackJob& j) { jobs.j[jobs.n++] = j; if (j.N > maxN) maxN = j.N; };
  for (int l = 0; l <= pl.L; ++l) {
    const LinDim& d = pl.sdf[l];
    PackJob j;
    memset(&j, 0, sizeof(j));
    j.v = params + d.off_v; j.g = params + d.off_g; j.b = params + d.off_b;
    j.N = d.N; j.K = d.K;
    j.c0[0] = 0; j.c1[0] = d.K;
    j.W[0] = pack + d.pk_W; j.ldw[0] = d.Kp;
    j.WT[0] = pack + d.pk_WT;
    j.bias = pack + d.pk_b;
    if (l < pl.L) {
      j.ldwt[0] = d.Np;
    } else {
      j.ldwt[0] = pl.Fp;
      j.row_shift = 1; j.bias_shift = 1;
      j.row0 = pack + pl.pk_wsdf; j.row0_b = pack + pl.pk_bsdf;
    }
    add(j);
  }
  for (int l = 0; l < pl.Lc; ++l) {
    const LinDim& d = pl.col[l];
    PackJob j;
    memset(&j, 0, sizeof(j));
    j.v = params + d.off_v; j.g = params + d.off_g; j.b = params + d.off_b;
    j.N = d.N; j.K = d.K;
    if (l == 0) {
      j.c0[0] = 6; j.c1[0] = d.K;                 // feature columns
      j.W[0] = pack + d.pk_W; j.ldw[0] = pl.Fp;
      j.WT[0] = pack + d.pk_WT; j.ldwt[0] = pl.Hc;
      j.c0[1] = 0; j.c1[1] = 6;                   // points + normals columns
      j.W[1] = pack + pl.pk_c0x; j.ldw[1] = 8;
      j.WT[1] = pack + pl.pk_c0xT; j.ldwt[1] = pl.Hc;
    } else {
      j.c0[0] = 0; j.c1[0] = d.K;
      j.W[0] = pack + d.pk_W; j.ldw[0] = pl.Hc;
      j.WT[0] = pack + d.pk_WT; j.ldwt[0] = pl.Hc;
    }
    j.bias = pack + d.pk_b;
    add(j);
  }
  for (int h = 0; h < 2; ++h) {   // colour head lin{Lc} -> rows 0..2, extra_lin -> rows 3..5 of W6
    const LinDim& d = h == 0 ? pl.col[pl.Lc] : pl.extra;
    PackJob j;
    memset(&j, 0, sizeof(j));
    j.v = params + d.off_v; j.g = params + d.off_g; j.b = params + d.off_b;
    j.N = 3; j.K = pl.Hc;
    j.c0[0] = 0; j.c1[0] = pl.Hc;
    j.W[0] = pack + pl.pk_W6; j.ldw[0] = pl.Hc;
    j.bias = pack + pl.pk_b6;
    j.dst_row_off = 3 * h;
    add(j);
  }
  k_pack_linear<<<dim3(maxN, jobs.n), 128, 0, st>>>(jobs);
  AVC_LAUNCH_TRY();
  return 0;
}

// zero the padding of the packed buffer once per call (padding rows/cols must be exactly zero)
int zero_pack(const NeusPlan& pl, float* pack, cudaStream_t st) {
  AVC_CUDA_TRY(cudaMemsetAsync(pack, 0, sizeof(float) * (size_t)pl.pack_floats, st));
  return 0;
}

// zero + pack (+ bf16 split for the wgmma engine)
int prepare_weights(const NeusPlan& pl, const NeusWs& w, const float* params, cudaStream_t st) {
  AVC_TRY(zero_pack(pl, w.pack, st));
  AVC_TRY(pack_weights(pl, params, w.pack, st));
  if (pl.cfg.engine == 1) {
    tc::k_split_bf16<<<blocks_for(pl.pack_floats, 256), 256, 0, st>>>(w.pack, 1, (int)pl.pack_floats,
                                                                      (int)pl.pack_floats, w.pk_hi, w.pk_lo,
                                                                      (int)pl.pack_floats);
    AVC_LAUNCH_TRY();
  }
  return 0;
}

EncodeTargets make_targets(const NeusPlan& pl, const NeusWs& w) {
  EncodeTargets t;
  memset(&t, 0, sizeof(t));
  const bool tc1 = pl.cfg.engine == 1;      // wgmma engine: every consumer of the encoding reads the bf16 pairs ...
  t.in0 = tc1 ? nullptr : w.in[0]; t.ld0 = pl.sdf[0].Kp;
  t.in0_16 = w.in16[0];
  for (int l = 1; l <= pl.L; ++l) {
    if (!pl.sdf[l].skip) continue;
    if (t.n_skip >= 4) break;
    t.skip_ptr[t.n_skip] = (tc1 && l != pl.L) ? nullptr : w.in[l];      // ... except the thin sdf head (fp32 in[L])
    t.skip_ld[t.n_skip] = pl.sdf[l].Kp;
    t.skip_col[t.n_skip] = pl.sdf[l].K - pl.E;
    t.skip16[t.n_skip] = w.in16[l];
    ++t.n_skip;
  }
  return t;
}

// -------------------------------------------------------------------------------- per-point kernels and thin heads
// The launches below are shared by the render and the kernel self-test (avc_neus_kernel_test).
int encode_samples(const float* rays_o, const float* rays_d, const float* z, int nz, int pitch, int Rc, float scale,
                   int multires, int E, int EP, const EncodeTargets& t, cudaStream_t st) {
  k_encode_samples<<<blocks_for((int64_t)nz * Rc * 8, 256), 256, 0, st>>>(rays_o, rays_d, z, nz, pitch, Rc, scale,
                                                                         multires, E, EP, t);
  AVC_LAUNCH_TRY();
  return 0;
}

int encode_points(const float* pts, int64_t P, float scale, int multires, int E, int EP, const EncodeTargets& t,
                  cudaStream_t st) {
  k_encode_points<<<blocks_for(P * 8, 256), 256, 0, st>>>(pts, P, scale, multires, E, EP, t);
  AVC_LAUNCH_TRY();
  return 0;
}

int encode_fine(const float* rays_o, const float* rays_d, const float* z_vals, int S, int64_t Rc, float sample_dist,
                float scale, int multires, int E, int EP, float* cin, float* mid_z, float* inside, const EncodeTargets& t,
                cudaStream_t st) {
  k_encode_fine<<<blocks_for(Rc * S * 8, 256), 256, 0, st>>>(rays_o, rays_d, z_vals, S, Rc, sample_dist, scale, multires,
                                                            E, EP, cin, mid_z, inside, t);
  AVC_LAUNCH_TRY();
  return 0;
}

// sdf = (in[L] . W_L[0] + b_L[0]) / scale over the K inputs of the last linear only: the columns [K, Kp) of in[L]
// (K = 4 mod 8) are padding nothing writes, and a NaN there times the zero padded weight would still be NaN.  K is a
// multiple of 4, as the float4 loop needs.  Point p = r * nz + j is stored at sdf_out[r * pitch + j] (nz = 0: at p).
int sdf_head(const NeusPlan& pl, const float* inL, const float* pack, int64_t P, float* sdf_out, int nz, int pitch,
             cudaStream_t st) {
  const LinDim& dl = pl.sdf[pl.L];
  OutSdf os{sdf_out, 1.0f / pl.cfg.sdf_scale, nz, pitch};
  k_thin_nt<1, OutSdf><<<blocks_for(P, 8 * kThinPPW), 256, 0, st>>>(inL, dl.Kp, dl.K, pack + pl.pk_wsdf, dl.Kp,
                                                                    pack + pl.pk_bsdf, P, os);
  AVC_LAUNCH_TRY();
  return 0;
}

// rgb6 = sigmoid of both colour heads on the last hidden colour activation ch[Lc]
int color_heads(const NeusPlan& pl, const float* chL, const float* pack, int64_t P, float* rgb6, cudaStream_t st) {
  OutHeads oh{rgb6};
  k_thin_nt<6, OutHeads><<<blocks_for(P, 8 * kThinPPW), 256, 0, st>>>(chL, pl.Hc, pl.Hc, pack + pl.pk_W6, pl.Hc,
                                                                      pack + pl.pk_b6, P, oh);
  AVC_LAUNCH_TRY();
  return 0;
}

// nbar += cbar_0 . W0[:, 3:6]   (the normal columns of colour lin0)
int nbar_add_color(const NeusPlan& pl, const float* cbar0, const float* pack, int64_t P, float* nbar, cudaStream_t st) {
  OutNbarAdd on{nbar};
  k_thin_nt<6, OutNbarAdd><<<blocks_for(P, 8 * kThinPPW), 256, 0, st>>>(cbar0, pl.Hc, pl.Hc, pack + pl.pk_c0xT, pl.Hc,
                                                                        nullptr, P, on);
  AVC_LAUNCH_TRY();
  return 0;
}

// cbar_Lc = (y6bar . W6) * [ch[Lc] > 0]; the fp32 copy may be NULL
int heads_dgrad(const NeusPlan& pl, const float* y6bar, const float* pack, const float* chL, int64_t P, float* cbar,
                const Split16& c16, cudaStream_t st) {
  k_heads_dgrad<<<blocks_for(P * pl.Hc / 4, 256), 256, 0, st>>>(y6bar, pack + pl.pk_W6, pl.Hc, chL, P, cbar, c16);
  AVC_LAUNCH_TRY();
  return 0;
}

// start of the reverse sweep: qt[L-1] (fp32 copy may be NULL) and ge from the stash softplus'(z[L-1])
int chain_start(const NeusPlan& pl, const float* pack, const float* zprev, int64_t P, float* qt, float* ge,
                const Split16& qt16, cudaStream_t st) {
  const LinDim& dL = pl.sdf[pl.L];
  const LinDim& dp = pl.sdf[pl.L - 1];
  int64_t tot = P * (int64_t)(dp.Np / 4 > pl.EP ? dp.Np / 4 : pl.EP);   // threads: 4 qt columns each, 1 ge entry each
  k_chain_start<<<blocks_for(tot, 256), 256, 0, st>>>(pack + pl.pk_wsdf, dL.K, dL.skip ? 1 : 0, pl.E, pl.EP, zprev, dp.N,
                                                      dp.Np, P, qt, ge, qt16);
  AVC_LAUNCH_TRY();
  return 0;
}

// n = D(y)^T ge -> cin[p][3:6] and grad_out (or NULL)
int normals(const NeusPlan& pl, const float* ge, int64_t P, float* cin, float* grad_out, cudaStream_t st) {
  k_normal<<<blocks_for(P, 128), 128, 0, st>>>(ge, pl.EP, pl.cfg.sdf_multires, pl.cfg.sdf_scale, P, cin, grad_out);
  AVC_LAUNCH_TRY();
  return 0;
}

// gebar = D(y) nbar -> gebar and ubar_0 (fp32 copy or NULL, its split u16), pitch Kp_0
int dge(const NeusPlan& pl, const float* cin, const float* nbar, int64_t P, float* ubar0, float* gebar, const Split16& u16,
        cudaStream_t st) {
  k_dge<<<blocks_for(P * 8, 256), 256, 0, st>>>(cin, nbar, pl.EP, pl.E, pl.cfg.sdf_multires, pl.cfg.sdf_scale, P, ubar0,
                                                pl.sdf[0].Kp, gebar, u16);
  AVC_LAUNCH_TRY();
  return 0;
}

// the encoding half of skip layer l's input adjoint: ubar_l[p][K_l - E + e] = gebar[p][e] / sqrt(2)
int fill_gebar(const NeusPlan& pl, int l, const float* gebar, int64_t P, float* ubar, const Split16& u16, cudaStream_t st) {
  const LinDim& d = pl.sdf[l];
  k_fill_gebar<<<blocks_for(P * pl.E, 256), 256, 0, st>>>(gebar, pl.EP, pl.E, P, ubar, d.Kp, d.K - pl.E, u16);
  AVC_LAUNCH_TRY();
  return 0;
}

// SDFNetwork evaluators (avc_neus_sdf_eval): cin[p] = (x, 0, 0, 0, 0, 0) and out[p] = [sdf, feat]
__global__ void k_points_to_cin(const float* __restrict__ pts, int64_t P, float* __restrict__ cin) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  float4* c = reinterpret_cast<float4*>(cin + (size_t)p * 8);
  c[0] = make_float4(pts[p * 3], pts[p * 3 + 1], pts[p * 3 + 2], 0.f);
  c[1] = make_float4(0.f, 0.f, 0.f, 0.f);
}
__global__ void k_assemble_sdf_feat(const float* __restrict__ sdf, const float* __restrict__ feat, int Fp, int F, int64_t P,
                                    float* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P * (F + 1)) return;
  int64_t p = i / (F + 1);
  int c = (int)(i - p * (F + 1));
  out[i] = c == 0 ? sdf[p] : feat[(size_t)p * Fp + (c - 1)];
}

int points_to_cin(const float* pts, int64_t P, float* cin, cudaStream_t st) {
  k_points_to_cin<<<blocks_for(P, 256), 256, 0, st>>>(pts, P, cin);
  AVC_LAUNCH_TRY();
  return 0;
}

int assemble_sdf_feat(const NeusPlan& pl, const float* sdf, const float* feat, int64_t P, float* out, cudaStream_t st) {
  k_assemble_sdf_feat<<<blocks_for(P * (pl.F + 1), 256), 256, 0, st>>>(sdf, feat, pl.Fp, pl.F, P, out);
  AVC_LAUNCH_TRY();
  return 0;
}

// -------------------------------------------------------------------------------- value chain
// in[0] (and the skip columns) must hold the encoding of Pn points.  stash: keep z[l].
// Leaves in[L] ready; writes sdf[Pn] (thin) and, when want_feat, feat[Pn][Fp].
// wgmma engine, no stash, no features (sample placement, sdf queries): the whole chain of a 128-point tile in ONE
// kernel (avc_chain.cu), activations resident in shared memory.  Returns 1 when the fused kernel does not cover this
// network shape (the caller then runs the layer-by-layer launches), 0 on success.
int value_chain_fused(const NeusPlan& pl, const NeusWs& w, int64_t Pn, float* sdf_out, cudaStream_t st, int sdf_nz,
                      int sdf_pitch) {
  const char* env = getenv("AVC_FUSED_CHAIN");      // 0: layer-by-layer launches (A-B knob, read on every call)
  if ((env && atoi(env) == 0) || pl.L > chain::kMaxHidden) return 1;
  chain::Args a;
  memset(&a, 0, sizeof(a));
  a.L = pl.L;
  int n_skip = 0, ls = -1;
  for (int l = 1; l <= pl.L; ++l)
    if (pl.sdf[l].skip) { ++n_skip; ls = l; }
  if (n_skip > 1) return 1;
  for (int l = 0; l < pl.L; ++l) {
    const LinDim& d = pl.sdf[l];
    chain::Layer& y = a.lay[l];
    y.w_hi = w.pk_hi + d.pk_W; y.w_lo = w.pk_lo + d.pk_W; y.ldw = d.Kp; y.N = d.N; y.K = d.K;
    y.bias = w.pack + d.pk_b;
    y.oscale = pl.sdf[l + 1].skip ? kSqrtHalf : 1.f;
    y.next_skip_cols = (l + 1 < pl.L && pl.sdf[l + 1].skip) ? pl.E : 0;
  }
  a.a0_hi = w.in16[0].hi; a.a0_lo = w.in16[0].lo; a.ld0 = pl.sdf[0].Kp;
  if (ls >= 0) {
    a.skip_hi = w.in16[ls].hi; a.skip_lo = w.in16[ls].lo; a.skip_ld = pl.sdf[ls].Kp; a.skip_col0 = pl.sdf[ls].K - pl.E;
  }
  a.w_sdf = w.pack + pl.pk_wsdf; a.b_sdf = w.pack + pl.pk_bsdf; a.K_head = pl.sdf[pl.L].K;
  a.head_skip_cols = pl.sdf[pl.L].skip ? pl.E : 0;
  a.inv_scale = 1.0f / pl.cfg.sdf_scale;
  a.sdf_out = sdf_out; a.nz = sdf_nz; a.pitch = sdf_pitch; a.P = Pn;
  if (!chain::supported(a)) return 1;
  return chain::launch(a, st);
}

int value_chain(const NeusPlan& pl, const NeusWs& w, int64_t Pn, bool stash, bool want_feat, float* sdf_out,
                cudaStream_t st, int sdf_nz = 0, int sdf_pitch = 0) {
  if (pl.cfg.engine == 1 && !stash && !want_feat) {
    int r = value_chain_fused(pl, w, Pn, sdf_out, st, sdf_nz, sdf_pitch);
    if (r != 1) return r;
  }
  const float* pack = w.pack;
  for (int l = 0; l < pl.L; ++l) {
    const LinDim& d = pl.sdf[l];
    const bool fast = pl.cfg.engine == 1;
    EpiValue<false> e;
    e.bias = pack + d.pk_b;
    e.D1 = stash ? w.z[l] : nullptr; e.ldz = d.Np;     // w.z[l] holds softplus'(z_l), see EpiValue
    // wgmma engine: the fp32 copy of a hidden activation is only read by the thin sdf head (layer L)
    e.OUT = (pl.cfg.engine == 1 && l + 1 < pl.L) ? nullptr : w.in[l + 1]; e.ldo = pl.sdf[l + 1].Kp;
    e.oscale = pl.sdf[l + 1].skip ? kSqrtHalf : 1.f;
    e.N = d.N;
    e.o16 = w.in16[l + 1];
    if (fast) {
      EpiValue<true> ef{e.bias, e.D1, e.ldz, e.OUT, e.ldo, e.oscale, e.N, e.o16};
      AVC_TRY(gemm_nt(pl, w, st, Pn, d.N, d.K, w.in[l], d.Kp, w.in16[l], d.pk_W, d.Kp, ef));
    } else {
      AVC_TRY(gemm_nt(pl, w, st, Pn, d.N, d.K, w.in[l], d.Kp, w.in16[l], d.pk_W, d.Kp, e));
    }
  }
  const LinDim& dl = pl.sdf[pl.L];
  AVC_TRY(sdf_head(pl, w.in[pl.L], pack, Pn, sdf_out, sdf_nz, sdf_pitch, st));
  if (want_feat) {
    // wgmma engine: every consumer of the features reads the split (colour lin0 A operand, its weight gradient)
    EpiBias e{pack + dl.pk_b, pl.cfg.engine == 1 ? nullptr : w.feat, pl.Fp, pl.F, w.feat16};
    AVC_TRY(gemm_nt(pl, w, st, Pn, pl.F, dl.K, w.in[pl.L], dl.Kp, w.in16[pl.L], dl.pk_W, dl.Kp, e));
  }
  return 0;
}

// -------------------------------------------------------------------------------- gradient chain
// d sdf / d x by the reverse sweep of Appendix B (no second forward): needs the sp' stash of value_chain(stash = true)
// and cin[p][0:3] = x.  Writes the raw gradient into cin[p][3:6] and, optionally, grad_out [P][3].
int gradient_chain(const NeusPlan& pl, const NeusWs& w, int64_t P, float* grad_out, cudaStream_t st) {
  // wgmma engine: qt_l is only ever consumed as a split operand (gradient chain, second-order sweep, dW)
  const bool tc1 = pl.cfg.engine == 1;
  AVC_TRY(chain_start(pl, w.pack, w.z[pl.L - 1], P, tc1 ? nullptr : w.qt[pl.L - 1], w.ge, w.qt16[pl.L - 1], st));
  for (int l = pl.L - 1; l >= 1; --l) {
    const LinDim& d = pl.sdf[l];
    const LinDim& dq = pl.sdf[l - 1];
    EpiChain e;
    e.Nprev = dq.N; e.Npp = dq.Np; e.s = d.skip ? kSqrtHalf : 1.f;
    e.D1prev = w.z[l - 1]; e.QTprev = tc1 ? nullptr : w.qt[l - 1]; e.GE = w.ge; e.EP = pl.EP; e.E = pl.E;
    e.q16 = w.qt16[l - 1];
    AVC_TRY(gemm_nt(pl, w, st, P, d.K, d.N, w.qt[l], d.Np, w.qt16[l], d.pk_WT, d.Np, e));
  }
  const LinDim& d0 = pl.sdf[0];
  EpiGe eg{w.ge, pl.EP, pl.E};
  AVC_TRY(gemm_nt(pl, w, st, P, pl.E, d0.N, w.qt[0], d0.Np, w.qt16[0], d0.pk_WT, d0.Np, eg));
  return normals(pl, w.ge, P, w.cin, grad_out, st);
}

// -------------------------------------------------------------------------------- placement
// The per-kernel launches are shared by the render and the kernel self-test (avc_neus_kernel_test).
int coarse_z(const float* near, const float* far, const float* jitter, int n, int pitch, int Rc, float* z,
             cudaStream_t st) {
  k_coarse_z<<<blocks_for((int64_t)Rc * n, 256), 256, 0, st>>>(near, far, jitter, n, pitch, Rc, z);
  AVC_LAUNCH_TRY();
  return 0;
}

int upsample(const float* rays_o, const float* rays_d, const float* z, const float* sdf, int n, int pitch, int Rc,
             float inv_s, int per, float* newz, cudaStream_t st) {
  k_upsample<<<blocks_for(Rc, 8), 256, 0, st>>>(rays_o, rays_d, z, sdf, n, pitch, Rc, inv_s, per, newz);
  AVC_LAUNCH_TRY();
  return 0;
}

int merge(const float* z, const float* sdf, int n, int pitch, const float* newz, const float* news, int per, int Rc,
          float* zo, float* so, int pitch_o, cudaStream_t st) {
  k_merge<<<blocks_for(Rc, 8), 256, 0, st>>>(z, sdf, n, pitch, newz, news, per, Rc, zo, so, pitch_o);
  AVC_LAUNCH_TRY();
  return 0;
}

int place_samples(const NeusPlan& pl, const NeusWs& w, const float* rays_o, const float* rays_d, const float* near,
                  const float* far, const float* jitter, int Rc, float* z_out_raymajor, cudaStream_t st) {
  // ray-major buffers [Rc][S]; one warp per ray in the per-ray kernels
  const int S = pl.S;
  if (S > kPlaceMaxN || pl.per > kPlaceMaxNew) return AVC_E_BADCFG;
  float* z0 = (pl.cfg.n_importance == 0) ? z_out_raymajor : w.zA;
  AVC_TRY(coarse_z(near, far, jitter, pl.n0, S, Rc, z0, st));
  if (pl.cfg.n_importance == 0) return 0;
  EncodeTargets t = make_targets(pl, w);
  int64_t Pn = (int64_t)pl.n0 * Rc;
  AVC_TRY(encode_samples(rays_o, rays_d, w.zA, pl.n0, S, Rc, pl.cfg.sdf_scale, pl.cfg.sdf_multires, pl.E, pl.EP, t, st));
  AVC_TRY(value_chain(pl, w, Pn, false, false, w.sA, st, pl.n0, S));
  float *zc = w.zA, *sc = w.sA, *zn = w.zB, *sn = w.sB;
  int n = pl.n0;
  for (int i = 0; i < pl.steps; ++i) {
    const bool last = (i + 1 == pl.steps);
    float inv_s = 64.0f * (float)(1 << i);                                     // renderer.py:346
    AVC_TRY(upsample(rays_o, rays_d, zc, sc, n, S, Rc, inv_s, pl.per, w.newZ, st));
    if (!last) {
      Pn = (int64_t)pl.per * Rc;
      AVC_TRY(encode_samples(rays_o, rays_d, w.newZ, pl.per, pl.per, Rc, pl.cfg.sdf_scale, pl.cfg.sdf_multires, pl.E,
                             pl.EP, t, st));
      AVC_TRY(value_chain(pl, w, Pn, false, false, w.newS, st, 0, 0));   // newS is [Rc][per]: identity mapping
    }
    // the last round writes the merged depths straight into the caller's z_vals [Rc][S]
    AVC_TRY(merge(zc, sc, n, S, w.newZ, last ? nullptr : w.newS, pl.per, Rc, last ? z_out_raymajor : zn, sn, S, st));
    float* tz = zc; zc = zn; zn = tz;
    float* ts = sc; sc = sn; sn = ts;
    n += pl.per;
  }
  return 0;
}

// -------------------------------------------------------------------------------- fine forward
struct ChunkIO {
  const float *rays_o, *rays_d, *background;   // already offset to the chunk
  int bg_kind;
  float cos_anneal;
  int64_t Rc;
  avc_neus_outputs out;                        // already offset to the chunk (gradient_error not offset)
};

CompositeArgs make_composite_args(const NeusPlan& pl, const NeusWs& w, const ChunkIO& io) {
  CompositeArgs A;
  A.rays_d = io.rays_d; A.z_vals = io.out.z_vals; A.sdf = w.sdf; A.cin = w.cin; A.rgb6 = w.rgb6;
  A.background = io.background; A.bg_kind = io.bg_kind; A.ctx = w.ctx; A.cos_anneal = io.cos_anneal;
  A.sample_dist = 2.0f / (float)pl.n0;                                         // renderer.py:304
  A.S = pl.S; A.Rc = io.Rc;
  return A;
}

// Compositing forward of one chunk; adds the chunk's eikonal sums into ctx.  Only the per-ray outputs of `out` are used.
int composite_forward(const CompositeArgs& A, const avc_neus_outputs& out, float* ray_part, float* ctx,
                      cudaStream_t st) {
  k_composite_fwd<<<blocks_for(A.Rc, 8), 256, 0, st>>>(A, out.color_fine, out.extra_color_fine, out.s_val, out.cdf_fine,
                                                       out.weight_sum, out.weight_max, out.weights, ray_part);
  AVC_LAUNCH_TRY();
  k_reduce_ray_part<<<1, 1024, 0, st>>>(ray_part, A.Rc, 0, ctx + CTX_EIK_NUM);
  k_reduce_ray_part<<<1, 1024, 0, st>>>(ray_part, A.Rc, 1, ctx + CTX_EIK_DEN);
  AVC_LAUNCH_TRY();
  return 0;
}

// Compositing backward of one chunk; adds the chunk's inv_s adjoint into ctx.
int composite_backward(const CompositeArgs& A, const CompositeBwdArgs& G, float* ctx, cudaStream_t st) {
  k_composite_bwd<<<blocks_for(A.Rc, 8), 256, 0, st>>>(A, G);
  AVC_LAUNCH_TRY();
  k_reduce_ray_part<<<1, 1024, 0, st>>>(G.ray_part, A.Rc, 2, ctx + CTX_INVS_BAR);
  AVC_LAUNCH_TRY();
  return 0;
}

// Eikonal normaliser of one chunk, added into ctx (k_relax_count writes ray_part[r][1]).
int relax_count(const float* rays_o, const float* rays_d, const float* z_vals, int S, int64_t Rc, float sample_dist,
                float* ray_part, float* ctx, cudaStream_t st) {
  k_relax_count<<<blocks_for(Rc, 8), 256, 0, st>>>(rays_o, rays_d, z_vals, S, Rc, sample_dist, ray_part);
  k_reduce_ray_part<<<1, 1024, 0, st>>>(ray_part, Rc, 1, ctx + CTX_EIK_DEN);
  AVC_LAUNCH_TRY();
  return 0;
}

int ctx_init(const float* params, int64_t off_var, float* ctx, int zero_sums, cudaStream_t st) {
  k_ctx_init<<<1, 32, 0, st>>>(params, off_var, ctx, zero_sums);
  AVC_LAUNCH_TRY();
  return 0;
}

int finalize_fwd(const float* ctx, float* gerr_out, cudaStream_t st) {
  k_finalize_fwd<<<1, 32, 0, st>>>(ctx, gerr_out);
  AVC_LAUNCH_TRY();
  return 0;
}

int variance_grad(const float* params, int64_t off_var, const float* ctx, const float* g_sval, int64_t R,
                  float* grad_var, cudaStream_t st) {
  k_variance_grad<<<1, 256, 0, st>>>(params, off_var, ctx, g_sval, R, grad_var);
  AVC_LAUNCH_TRY();
  return 0;
}

// Runs the fine pass on io.out.z_vals; with write_outputs=false only the stash is (re)built.
int fine_forward(const NeusPlan& pl, const NeusWs& w, const ChunkIO& io, bool write_outputs, cudaStream_t st) {
  const int64_t P = io.Rc * pl.S;
  const float* pack = w.pack;
  EncodeTargets t = make_targets(pl, w);
  AVC_TRY(encode_fine(io.rays_o, io.rays_d, io.out.z_vals, pl.S, io.Rc, 2.0f / (float)pl.n0, pl.cfg.sdf_scale,
                      pl.cfg.sdf_multires, pl.E, pl.EP, w.cin, write_outputs ? io.out.mid_z_vals : nullptr,
                      write_outputs ? io.out.inside_sphere : nullptr, t, st));
  AVC_TRY(value_chain(pl, w, P, true, true, w.sdf, st));
  AVC_TRY(gradient_chain(pl, w, P, write_outputs ? io.out.gradients : nullptr, st));
  // ---- colour net
  {
    const LinDim& c0 = pl.col[0];
    // wgmma engine: the fp32 copy of a hidden colour activation is only read by the heads (layer Lc)
    const bool tc1 = pl.cfg.engine == 1;
    // ... and the split of the LAST hidden activation has no reader at all (the heads and their backward are thin fp32 ops)
    const Split16 none16{nullptr, nullptr, 0};
    EpiColor0 e0{pack + c0.pk_b, w.cin, pack + pl.pk_c0xT, pl.Hc, (tc1 && 1 < pl.Lc) ? nullptr : w.ch[1], pl.Hc,
                 (tc1 && 1 == pl.Lc) ? none16 : w.ch16[1]};
    AVC_TRY(gemm_nt_color(pl, w, st, P, pl.Hc, pl.F, w.feat, pl.Fp, w.feat16, c0.pk_W, pl.Fp, e0));
    for (int l = 1; l < pl.Lc; ++l) {
      const LinDim& c = pl.col[l];
      EpiRelu e{pack + c.pk_b, (tc1 && l + 1 < pl.Lc) ? nullptr : w.ch[l + 1], pl.Hc,
                (tc1 && l + 1 == pl.Lc) ? none16 : w.ch16[l + 1]};
      AVC_TRY(gemm_nt_color(pl, w, st, P, pl.Hc, pl.Hc, w.ch[l], pl.Hc, w.ch16[l], c.pk_W, pl.Hc, e));
    }
    AVC_TRY(color_heads(pl, w.ch[pl.Lc], pack, P, w.rgb6, st));
  }
  if (write_outputs) AVC_TRY(composite_forward(make_composite_args(pl, w, io), io.out, w.ray_part, w.ctx, st));
  return 0;
}

// (Measured and removed, r2: setting 32 / 48 / 64 MB of L2 aside for persisting accesses and making the operand pair a
// backward kernel writes -- zbar_{l-1}, ubar_{l+1}: read again by the next TN and the next NT -- the stream's access-policy
// window cost 1.5 / 4 / 14 % of the step: the carve-out takes L2 from the A-tile and epilogue-operand prefetches.)
// -------------------------------------------------------------------------------- backward
template <int NI>
int thin_tn(cudaStream_t st, const float* S, int lds, float s_scale, const float* Hm, int ldh, int NC, int64_t P,
            float* out, int si, int sc, float* bout, int split = NI, float* out2 = nullptr, float* bout2 = nullptr) {
  const int rows = 128;
  k_thin_tn<NI><<<blocks_for(P, rows), 256, 0, st>>>(S, lds, s_scale, Hm, ldh, NC, P, rows, out, si, sc, bout, split,
                                                     out2, bout2);
  AVC_LAUNCH_TRY();
  return 0;
}

int colsum(cudaStream_t st, const float* X, int ld, int NC, int64_t P, float scale, float* out) {
  const int rows = 64;
  k_colsum<<<blocks_for(P, rows), 256, 0, st>>>(X, ld, NC, P, rows, scale, out);
  AVC_LAUNCH_TRY();
  return 0;
}

// Accumulates dense dW / db of every linear into w.wbar (v / b slots of the flat layout) and the
// inv_s adjoint into ctx[CTX_INVS_BAR].  Requires the forward stash of this chunk in `w`.
int fine_backward(const NeusPlan& pl, const NeusWs& w, const ChunkIO& io, const avc_neus_cotangents& cot,
                  cudaStream_t st) {
  const int64_t P = io.Rc * pl.S;
  const float* pack = w.pack;
  float* wbar = w.wbar;
  // ---- compositing
  CompositeArgs A = make_composite_args(pl, w, io);
  CompositeBwdArgs G;
  G.g_color = cot.color_fine; G.g_extra = cot.extra_color_fine; G.g_wsum = cot.weight_sum; G.g_wmax = cot.weight_max;
  G.g_w = cot.weights; G.g_cdf = cot.cdf_fine; G.g_n = cot.gradients; G.g_gerr = cot.gradient_error;
  G.weights = io.out.weights;
  G.y6bar = w.y6bar; G.sdfbar = w.sdfbar; G.nbar = w.nbar; G.ray_part = w.ray_part;
  AVC_TRY(composite_backward(A, G, w.ctx, st));

  // ---- colour heads: lin{Lc} <- y6bar[:,0:3], extra_lin <- y6bar[:,3:6]   (models/fields.py:172-181)
  {
    const LinDim& dh = pl.col[pl.Lc];
    const LinDim& dx = pl.extra;
    // both heads read the same activation: one pass, rows 0..2 -> lin{Lc}, rows 3..5 -> extra_lin
    AVC_TRY(thin_tn<6>(st, w.y6bar, 8, 1.f, w.ch[pl.Lc], pl.Hc, pl.Hc, P, wbar + dh.off_v, pl.Hc, 1, wbar + dh.off_b, 3,
                       wbar + dx.off_v, wbar + dx.off_b));
    // wgmma engine: the hidden linears consume cbar as a split operand; its fp32 copy is only read at layer 0
    AVC_TRY(heads_dgrad(pl, w.y6bar, pack, w.ch[pl.Lc], P, (pl.cfg.engine == 1 && pl.Lc > 1) ? nullptr : w.cbar[0],
                        w.cbar16[0], st));
  }
  // ---- colour hidden linears l = Lc-1 .. 0 ; cbar_l lives in w.cbar[cur]
  int cur = 0;
  for (int l = pl.Lc - 1; l >= 0; --l) {
    const LinDim& c = pl.col[l];
    float* cb = w.cbar[cur];
    if (l > 0) {
      AVC_TRY(gemm_tn(pl, w, st, P, pl.Hc, pl.Hc, cb, pl.Hc, w.cbar16[cur], w.ch[l], pl.Hc, w.ch16[l], wbar + c.off_v, c.K,
                      wbar + c.off_b, color_single(pl)));
      // wgmma engine: ReLU mask from the split of ch[l]; the fp32 copy of cbar is only read at layer 0 (thin ops)
      const bool tc1 = pl.cfg.engine == 1;
      EpiDgradRelu e{tc1 ? nullptr : w.ch[l], w.ch16[l].hi, (tc1 && l > 1) ? nullptr : w.cbar[cur ^ 1], pl.Hc,
                     w.cbar16[cur ^ 1]};
      AVC_TRY(gemm_nt_color(pl, w, st, P, pl.Hc, pl.Hc, cb, pl.Hc, w.cbar16[cur], c.pk_WT, pl.Hc, e));
      cur ^= 1;
    } else {
      // lin0 input = [x(3), n(3), feat(F)]: dW[:, 6:] += cbar^T feat ; dW[:, :6] += cbar^T cin6
      AVC_TRY(gemm_tn(pl, w, st, P, pl.Hc, pl.F, cb, pl.Hc, w.cbar16[cur], w.feat, pl.Fp, w.feat16, wbar + c.off_v + 6, c.K,
                      wbar + c.off_b, color_single(pl)));
      AVC_TRY(thin_tn<6>(st, w.cin, 8, 1.f, cb, pl.Hc, pl.Hc, P, wbar + c.off_v, 1, c.K, nullptr));
      // featbar = cbar . W0[:, 6:]
      EpiStore es{pl.cfg.engine == 1 ? nullptr : w.featbar, pl.Fp, pl.F, w.featbar16};
      AVC_TRY(gemm_nt_color(pl, w, st, P, pl.F, pl.Hc, cb, pl.Hc, w.cbar16[cur], c.pk_WT, pl.Hc, es));
      // nbar += cbar . W0[:, 3:6]   (d/d points is discarded: pts is a leaf, models/fields.py:97)
      AVC_TRY(nbar_add_color(pl, cb, pack, P, w.nbar, st));
    }
  }

  // ---- SDF: second-order sweep in forward layer order
  int ucur = 0;
  {
    // wgmma engine: ubar_0 is only consumed as a split operand
    AVC_TRY(dge(pl, w.cin, w.nbar, P, pl.cfg.engine == 1 ? nullptr : w.ubar[0], w.gebar,
                with_ld(w.ubar16[0], pl.sdf[0].Kp), st));
  }
  for (int l = 0; l <= pl.L; ++l) {
    const LinDim& d = pl.sdf[l];
    float* ub = w.ubar[ucur];            // ubar_l : [P][Kp_l]
    if (l == pl.L) {
      // qt_L = e_0: only row 0 of W_L receives  sum_p ubar_L
      AVC_TRY(colsum(st, ub, d.Kp, d.K, P, 1.f, wbar + d.off_v));
      break;
    }
    const Split16 ub16 = with_ld(w.ubar16[ucur], d.Kp);
    AVC_TRY(gemm_tn(pl, w, st, P, d.N, d.K, w.qt[l], d.Np, w.qt16[l], ub, d.Kp, ub16, wbar + d.off_v, d.K));
    const LinDim& dn = pl.sdf[l + 1];
    EpiChainBwd e;
    e.N = d.N; e.Np = d.Np; e.D1 = w.z[l]; e.QT = pl.cfg.engine == 1 ? nullptr : w.qt[l]; e.qt16 = w.qt16[l];
    e.ZBAR = w.zbar[l];
    // wgmma engine: the fp32 copy of ubar_{l+1} is only read by the column sum at the last linear
    e.UNEXT = (pl.cfg.engine == 1 && l + 1 < pl.L) ? nullptr : w.ubar[ucur ^ 1];
    e.ldu = dn.Kp; e.s_next = dn.skip ? kSqrtHalf : 1.f;
    // the pair of ubar_L has no reader (the last linear only needs the column sum of the fp32 copy)
    const Split16 unext16 = (pl.cfg.engine == 1 && l + 1 == pl.L) ? Split16{nullptr, nullptr, 0} : with_ld(w.ubar16[ucur ^ 1], dn.Kp);
    e.u16 = unext16;
    AVC_TRY(gemm_nt(pl, w, st, P, d.N, d.K, ub, d.Kp, ub16, d.pk_W, d.Kp, e));
    if (dn.skip) {
      AVC_TRY(fill_gebar(pl, l + 1, w.gebar, P, w.ubar[ucur ^ 1], unext16, st));
    }
    ucur ^= 1;
  }

  // ---- SDF: value backward in reverse layer order
  {
    const LinDim& dL = pl.sdf[pl.L];
    const float inv_scale = 1.0f / pl.cfg.sdf_scale;
    // last linear: row 0 (sdf) via thin ops, rows 1.. (features) via the GEMM tiles
    AVC_TRY(thin_tn<1>(st, w.sdfbar, 1, inv_scale, w.in[pl.L], dL.Kp, dL.K, P, wbar + dL.off_v, 0, 1, wbar + dL.off_b));
    AVC_TRY(gemm_tn(pl, w, st, P, pl.F, dL.K, w.featbar, pl.Fp, w.featbar16, w.in[pl.L], dL.Kp, w.in16[pl.L],
                    wbar + dL.off_v + dL.K, dL.K, wbar + dL.off_b + 1));
    const LinDim& dp = pl.sdf[pl.L - 1];
    EpiDgrad e;
    e.Nprev = dp.N; e.Npp = dp.Np; e.s = dL.skip ? kSqrtHalf : 1.f;
    e.D1prev = w.z[pl.L - 1]; e.ZBARprev = w.zbar[pl.L - 1];
    e.sdfbar = w.sdfbar; e.wsdf = pack + pl.pk_wsdf; e.sdf_inv_scale = inv_scale;
    e.z16 = w.zbar16[pl.L - 1]; e.store_f32 = pl.cfg.engine != 1;
    AVC_TRY(gemm_nt(pl, w, st, P, dp.N, pl.F, w.featbar, pl.Fp, w.featbar16, dL.pk_WT, pl.Fp, e));
  }
  for (int l = pl.L - 1; l >= 0; --l) {
    const LinDim& d = pl.sdf[l];
    AVC_TRY(gemm_tn(pl, w, st, P, d.N, d.K, w.zbar[l], d.Np, w.zbar16[l], w.in[l], d.Kp, w.in16[l], wbar + d.off_v, d.K,
                    wbar + d.off_b));
    if (l == 0) break;
    const LinDim& dp = pl.sdf[l - 1];
    EpiDgrad e;
    e.Nprev = dp.N; e.Npp = dp.Np; e.s = d.skip ? kSqrtHalf : 1.f;
    e.D1prev = w.z[l - 1]; e.ZBARprev = w.zbar[l - 1];
    e.sdfbar = nullptr; e.wsdf = nullptr; e.sdf_inv_scale = 1.f;
    e.z16 = w.zbar16[l - 1]; e.store_f32 = pl.cfg.engine != 1;
    AVC_TRY(gemm_nt(pl, w, st, P, dp.N, d.N, w.zbar[l], d.Np, w.zbar16[l], d.pk_WT, d.Np, e));
  }
  return 0;
}

int weight_norm_backward_all(const NeusPlan& pl, const float* params, const float* wbar, float* grads,
                             cudaStream_t st) {
  WnJobs jobs;
  jobs.n = 0;
  int maxN = 1;
  auto one = [&](const LinDim& d) {
    jobs.j[jobs.n++] = WnJob{params + d.off_v, params + d.off_g, wbar + d.off_v, wbar + d.off_b, d.N, d.K,
                             grads + d.off_g, grads + d.off_v, grads + d.off_b};
    if (d.N > maxN) maxN = d.N;
  };
  for (int l = 0; l <= pl.L; ++l) one(pl.sdf[l]);
  for (int l = 0; l <= pl.Lc; ++l) one(pl.col[l]);
  one(pl.extra);
  k_wn_backward<<<dim3(maxN, jobs.n), 128, 0, st>>>(jobs);
  AVC_LAUNCH_TRY();
  return 0;
}

int check_ptr16(const void* p) { return ((uintptr_t)p & 15u) ? AVC_E_ALIGN : 0; }

avc_neus_outputs offset_outputs(const avc_neus_outputs& o, int64_t r0, int S) {
  avc_neus_outputs q = o;
  q.color_fine += r0 * 3; q.extra_color_fine += r0 * 3; q.s_val += r0; q.cdf_fine += r0 * S;
  q.weight_sum += r0; q.weight_max += r0; q.gradients += r0 * S * 3; q.weights += r0 * S;
  q.mid_z_vals += r0 * S; q.inside_sphere += r0 * S; q.z_vals += r0 * S;
  return q;
}

avc_neus_cotangents offset_cot(const avc_neus_cotangents& c, int64_t r0, int S) {
  avc_neus_cotangents q = c;
  if (q.color_fine) q.color_fine += r0 * 3;
  if (q.extra_color_fine) q.extra_color_fine += r0 * 3;
  if (q.s_val) q.s_val += r0;
  if (q.cdf_fine) q.cdf_fine += r0 * S;
  if (q.weight_sum) q.weight_sum += r0;
  if (q.weight_max) q.weight_max += r0;
  if (q.gradients) q.gradients += r0 * S * 3;
  if (q.weights) q.weights += r0 * S;
  return q;
}

}  // namespace

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" {

int avc_abi_version(void) { return AVC_ABI_VERSION; }

// Stall probe of the wgmma NT tiles (diagnostic builds only: -DAVC_NT_PROBE=1).  out[16][9]: per functor the summed
// cycles of the slots listed in avc_gemm_tc.cuh (AVC_NT_PROBE).  Returns AVC_E_BADCFG in a regular build.
int avc_nt_probe_read(unsigned long long* host_out, int reset) {
#ifdef AVC_NT_PROBE
  if (!host_out) return AVC_E_NULL;
  AVC_CUDA_TRY(cudaDeviceSynchronize());
  AVC_CUDA_TRY(cudaMemcpyFromSymbol(host_out, tc::g_nt_probe, sizeof(unsigned long long) * 16 * tc::kNtProbeSlots));
  if (reset) {
    static unsigned long long zeros[16 * tc::kNtProbeSlots];
    AVC_CUDA_TRY(cudaMemcpyToSymbol(tc::g_nt_probe, zeros, sizeof(zeros)));
  }
  return 0;
#else
  (void)host_out; (void)reset;
  return AVC_E_BADCFG;
#endif
}
const char* avc_build_arch(void) { return "sm_90a"; }

// Self-test of the backward epilogue functors through the wgmma NT tiles (tests/test_nt_epilogue_gpu.py):
// acc = A[M][K] . B[N][K]^T on the two-term split, then
//   kind 0  EpiChainBwd  D1 = X, qt = split of Y (both [M][ldx]), s_next = s -> ZBAR = OUT [M][ldx], ubar = OUT2 [M][ld2]
//   kind 1  EpiDgrad     D1prev = X, zbar_prev = Y (updated in place, fp32), s
//   kind 2  EpiDgrad     as 1 with the sdf term: sdfbar = v1 [M], wsdf = v2 [ldx], sdf_inv_scale = s2
//   kind 3  EpiChain     Nprev = Nv, D1prev = X, s -> qt_prev = OUT [M][ldx]; ge = OUT2 [M][ld2] += the columns >= Nv
//   kind 4  EpiDgradRelu mask from the bf16 hi half of X -> OUT [M][ldx]
//   kind 5  EpiGe        ge = OUT2 [M][ld2] += acc
// The functors below write an fp32 copy to OUT [M][ldx] and the bf16 split of it into OUT2, read as a bf16 array
// [M][2 ld2]: hi in columns [0, ld2), lo in columns [ld2, 2 ld2) of each row.
//   kind 6  EpiValue<true>  bias = v1 [N], oscale = s -> sp' stash D1 = Y [M][ldx] (padding written), OUT, split
//   kind 7  EpiBias         bias = v1 -> OUT, split
//   kind 8  EpiColor0       bias = v1, cin = X [M][8], WxT = v2 [6][ldx] -> OUT, split
//   kind 9  EpiRelu         bias = v1 -> OUT, split
//   kind 10 EpiStore        -> OUT, split
//   kind 11 EpiDgradRelu    as kind 4, and the split (the mask is read at the split's pitch, 2 ld2)
//   kinds 108..111          kinds 8..11 with one bf16 product on the hi halves (NPROD = 1)
// The staged functors with the output sets the renderer launches them with (kind 0 is the second-order sweep's last
// linear: zbar and the fp32 copy of ubar_next), the split into OUT2 as above:
//   kind 12 EpiChainBwd  as 0, but ubar_next = the split only (its extent is ldx)
//   kind 13 EpiDgrad     as 1, but zbar_prev = Y is only read: the new zbar_prev = the split only
//   kind 14 EpiDgrad     as 13 with the sdf term of kind 2
//   kind 15 EpiChain     as 3, but qt_prev = the split only; ge = OUT [M][ldx] += the columns >= Nv
// workspace >= 4 * (M + N) * round_up(K, 8) + 4 * M * ldx bytes (kind 11: + 8 * M * ld2 instead of 4 * M * ldx).
int avc_tc_epi_test(int32_t kind, const float* A, const float* B, int64_t M, int32_t N, int32_t K, int32_t Nv,
                    const float* X, float* Y, int32_t ldx, const float* v1, const float* v2, float s, float s2, float* OUT,
                    float* OUT2, int32_t ld2, void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!A || !B || !X || !workspace) return AVC_E_NULL;
  if (M <= 0 || N <= 0 || K <= 0 || ldx % 8 || ld2 % 8) return AVC_E_SIZE;
  const int ld = (int)round_up(K, 8);
  Carver cv(workspace);
  __nv_bfloat16* ah = cv.take<__nv_bfloat16>(M * ld);
  __nv_bfloat16* al = cv.take<__nv_bfloat16>(M * ld);
  __nv_bfloat16* bh = cv.take<__nv_bfloat16>((int64_t)N * ld);
  __nv_bfloat16* bl = cv.take<__nv_bfloat16>((int64_t)N * ld);
  const int ldm = kind % 100 == 11 ? 2 * ld2 : ldx;      // EpiDgradRelu reads its mask at the pitch of its split output
  __nv_bfloat16* xh = cv.take<__nv_bfloat16>(M * ldm);
  __nv_bfloat16* xl = cv.take<__nv_bfloat16>(M * ldm);
  if (cv.used() > workspace_bytes) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  tc::k_split_bf16<<<blocks_for(M * ld, 256), 256, 0, st>>>(A, M, K, K, ah, al, ld);
  tc::k_split_bf16<<<blocks_for((int64_t)N * ld, 256), 256, 0, st>>>(B, N, K, K, bh, bl, ld);
  const float* xs = (kind == 0 || kind == 12) ? Y : X;      // the operand that is read as a bf16 pair
  if (kind == 0 || kind == 12 || kind == 4 || kind % 100 == 11)
    tc::k_split_bf16<<<blocks_for(M * ldm, 256), 256, 0, st>>>(xs, M, ldx, ldx, xh, xl, ldm);
  AVC_LAUNCH_TRY();
  const tc::SplitPtr a{ah, al, ld}, b{bh, bl, ld};
  const Split16 none{nullptr, nullptr, ldx};
  switch (kind) {
    case 0: {
      EpiChainBwd e;
      e.N = N; e.Np = ldx; e.D1 = X; e.QT = nullptr; e.qt16 = Split16{xh, xl, ldx}; e.ZBAR = OUT; e.UNEXT = OUT2;
      e.ldu = ld2; e.s_next = s; e.u16 = Split16{nullptr, nullptr, ld2};
      return tc::launch_gemm_tc_nt<3>(st, M, N, K, a, b, e);
    }
    case 1:
    case 2: {
      EpiDgrad e;
      e.Nprev = N; e.Npp = ldx; e.s = s; e.D1prev = X; e.ZBARprev = Y;
      e.sdfbar = kind == 2 ? v1 : nullptr; e.wsdf = kind == 2 ? v2 : nullptr; e.sdf_inv_scale = s2;
      e.z16 = none; e.store_f32 = 1;
      return tc::launch_gemm_tc_nt<3>(st, M, N, K, a, b, e);
    }
    case 3: {
      EpiChain e;
      e.Nprev = Nv; e.Npp = ldx; e.s = s; e.D1prev = X; e.QTprev = OUT; e.GE = OUT2; e.EP = ld2; e.E = N - Nv;
      e.q16 = none;
      return tc::launch_gemm_tc_nt<3>(st, M, N, K, a, b, e);
    }
    case 4: {
      EpiDgradRelu e{nullptr, xh, OUT, ldx, none};
      return tc::launch_gemm_tc_nt<3>(st, M, N, K, a, b, e);
    }
    case 5: {
      EpiGe e{OUT2, ld2, N};
      return tc::launch_gemm_tc_nt<3>(st, M, N, K, a, b, e);
    }
  }
  if (kind >= 12 && kind <= 15) {
    if (!OUT || !OUT2) return AVC_E_NULL;
    __nv_bfloat16* o16 = reinterpret_cast<__nv_bfloat16*>(OUT2);
    const Split16 split{o16, o16 + ld2, 2 * ld2};
    if (kind == 12) {
      EpiChainBwd e;
      e.N = N; e.Np = ldx; e.D1 = X; e.QT = nullptr; e.qt16 = Split16{xh, xl, ldx}; e.ZBAR = OUT; e.UNEXT = nullptr;
      e.ldu = ldx; e.s_next = s; e.u16 = split;
      return tc::launch_gemm_tc_nt<3>(st, M, N, K, a, b, e);
    }
    if (kind == 13 || kind == 14) {
      EpiDgrad e;
      e.Nprev = N; e.Npp = ldx; e.s = s; e.D1prev = X; e.ZBARprev = Y;
      e.sdfbar = kind == 14 ? v1 : nullptr; e.wsdf = kind == 14 ? v2 : nullptr; e.sdf_inv_scale = s2;
      e.z16 = split; e.store_f32 = 0;
      return tc::launch_gemm_tc_nt<3>(st, M, N, K, a, b, e);
    }
    EpiChain e;
    e.Nprev = Nv; e.Npp = ldx; e.s = s; e.D1prev = X; e.QTprev = nullptr; e.GE = OUT; e.EP = ldx; e.E = N - Nv;
    e.q16 = split;
    return tc::launch_gemm_tc_nt<3>(st, M, N, K, a, b, e);
  }
  // kinds 108..111: 8..11 with one bf16 product (the colour net at color_products = 1)
  const bool np1 = kind >= 108 && kind <= 111;
  if (np1) kind -= 100;
  if (kind < 6 || kind > 11) return AVC_E_BADCFG;
  auto launch_color = [&](const auto& e) {
    return np1 ? tc::launch_gemm_tc_nt<1>(st, M, N, K, a, b, e) : tc::launch_gemm_tc_nt<3>(st, M, N, K, a, b, e);
  };
  if (!OUT2 || (!v1 && kind != 10 && kind != 11)) return AVC_E_NULL;
  __nv_bfloat16* o16 = reinterpret_cast<__nv_bfloat16*>(OUT2);
  const Split16 split{o16, o16 + ld2, 2 * ld2};
  switch (kind) {
    case 6: {
      EpiValue<true> e{v1, Y, ldx, OUT, ldx, s, N, split};
      return tc::launch_gemm_tc_nt<3>(st, M, N, K, a, b, e);
    }
    case 7: {
      EpiBias e{v1, OUT, ldx, N, split};
      return tc::launch_gemm_tc_nt<3>(st, M, N, K, a, b, e);
    }
    case 8: {
      EpiColor0 e{v1, X, v2, ldx, OUT, ldx, split};
      return launch_color(e);
    }
    case 9: {
      EpiRelu e{v1, OUT, ldx, split};
      return launch_color(e);
    }
    case 10: {
      EpiStore e{OUT, ldx, N, split};
      return launch_color(e);
    }
    case 11: {
      EpiDgradRelu e{nullptr, xh, OUT, ldx, Split16{o16, o16 + ld2, 2 * ld2}};
      return launch_color(e);
    }
  }
  return AVC_E_BADCFG;
}

// One kernel of the NeuS path outside the GEMM tiles on caller buffers, launched by the render's own host helpers
// (argument roles in include/avc_b200.h).
int avc_neus_kernel_test(int32_t kind, const int64_t* d, const float* fs, const void* const* in, void* const* out,
                         avc_stream_t stream) {
  if (!d || !fs || !in || !out) return AVC_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  const auto F32 = [](const void* p) { return (const float*)p; };
  const auto O32 = [](void* p) { return (float*)p; };
  const auto pair = [](void* p, int ld) {      // a bf16 pair buffer [rows][2 ld]: hi in [0, ld), lo in [ld, 2 ld)
    __nv_bfloat16* h = (__nv_bfloat16*)p;
    return Split16{h, h ? h + ld : nullptr, 2 * ld};
  };
  switch (kind) {
    case 0: return ctx_init(F32(in[0]), d[0], O32(out[0]), (int)d[1], st);
    case 1:
    case 2: {
      const int S = (int)d[0], bg_kind = (int)d[2];
      const int64_t Rc = d[1];
      if (S < 1 || S > 256 || Rc < 1) return AVC_E_SIZE;
      if (bg_kind < 0 || bg_kind > 2 || (bg_kind != 0 && !in[5])) return AVC_E_BADCFG;
      CompositeArgs A;
      A.rays_d = F32(in[0]); A.z_vals = F32(in[1]); A.sdf = F32(in[2]); A.cin = F32(in[3]); A.rgb6 = F32(in[4]);
      A.background = F32(in[5]); A.bg_kind = bg_kind; A.cos_anneal = fs[0]; A.sample_dist = fs[1]; A.S = S; A.Rc = Rc;
      if (kind == 1) {
        float* ctx = O32(out[8]);
        A.ctx = ctx;
        avc_neus_outputs o;
        memset(&o, 0, sizeof(o));
        o.color_fine = O32(out[0]); o.extra_color_fine = O32(out[1]); o.s_val = O32(out[2]); o.cdf_fine = O32(out[3]);
        o.weight_sum = O32(out[4]); o.weight_max = O32(out[5]); o.weights = O32(out[6]);
        return composite_forward(A, o, O32(out[7]), ctx, st);
      }
      float* ctx = O32(out[4]);
      A.ctx = ctx;
      CompositeBwdArgs G;
      G.g_color = F32(in[6]); G.g_extra = F32(in[7]); G.g_wsum = F32(in[8]); G.g_wmax = F32(in[9]);
      G.g_w = F32(in[10]); G.g_cdf = F32(in[11]); G.g_n = F32(in[12]); G.g_gerr = F32(in[13]); G.weights = F32(in[14]);
      if (G.g_wmax && !G.weights) return AVC_E_NULL;
      G.y6bar = O32(out[0]); G.sdfbar = O32(out[1]); G.nbar = O32(out[2]); G.ray_part = O32(out[3]);
      return composite_backward(A, G, ctx, st);
    }
    case 3: {
      if (d[0] < 1 || d[1] < 1) return AVC_E_SIZE;
      return relax_count(F32(in[0]), F32(in[1]), F32(in[2]), (int)d[0], d[1], fs[0], O32(out[0]), O32(out[1]), st);
    }
    case 4: return finalize_fwd(F32(in[0]), O32(out[0]), st);
    case 5: return variance_grad(F32(in[0]), d[0], F32(in[1]), F32(in[2]), d[1], O32(out[0]), st);
    case 6: {
      const int n = (int)d[0], pitch = (int)d[1], Rc = (int)d[2];
      if (n < 1 || pitch < n || Rc < 1) return AVC_E_SIZE;
      return coarse_z(F32(in[0]), F32(in[1]), F32(in[2]), n, pitch, Rc, O32(out[0]), st);
    }
    case 7: {
      const int n = (int)d[0], pitch = (int)d[1], Rc = (int)d[2], per = (int)d[3];
      if (n < 2 || n > kPlaceMaxN || pitch < n || Rc < 1 || per < 1 || per > kPlaceMaxNew) return AVC_E_SIZE;
      return upsample(F32(in[0]), F32(in[1]), F32(in[2]), F32(in[3]), n, pitch, Rc, fs[0], per, O32(out[0]), st);
    }
    case 8: {
      const int n = (int)d[0], pitch = (int)d[1], Rc = (int)d[2], per = (int)d[3], pitch_o = (int)d[4];
      if (n < 1 || n > kPlaceMaxN || pitch < n || Rc < 1 || per < 1 || per > kPlaceMaxNew || pitch_o < n + per)
        return AVC_E_SIZE;
      if (in[3] && !out[1]) return AVC_E_NULL;
      return merge(F32(in[0]), F32(in[1]), n, pitch, F32(in[2]), F32(in[3]), per, Rc, O32(out[0]), O32(out[1]), pitch_o,
                   st);
    }
    case 18: {
      const int NI = (int)d[0], lds = (int)d[1], ldh = (int)d[2], NC = (int)d[3], si = (int)d[5], sc = (int)d[6];
      const int split = (int)d[7];
      const int64_t P = d[4];
      if (P < 1 || NC < 1 || lds < NI || ldh < NC) return AVC_E_SIZE;
      if (NI == 1) return thin_tn<1>(st, F32(in[0]), lds, fs[0], F32(in[1]), ldh, NC, P, O32(out[0]), si, sc, O32(out[1]),
                                     split, O32(out[2]), O32(out[3]));
      if (NI == 6) return thin_tn<6>(st, F32(in[0]), lds, fs[0], F32(in[1]), ldh, NC, P, O32(out[0]), si, sc, O32(out[1]),
                                     split, O32(out[2]), O32(out[3]));
      return AVC_E_BADCFG;
    }
    case 19: {
      if (d[2] < 1 || d[1] < 1 || d[0] < d[1]) return AVC_E_SIZE;
      return colsum(st, F32(in[0]), (int)d[0], (int)d[1], d[2], fs[0], O32(out[0]));
    }
    case 25: {
      if (d[0] < 1) return AVC_E_SIZE;
      return points_to_cin(F32(in[0]), d[0], O32(out[0]), st);
    }
  }
  if (kind < 9 || kind > 26) return AVC_E_BADCFG;
  if (kind >= 12 && kind <= 14) {
    // EncodeTargets: out[0] in0 or NULL, out[1..4] skip fp32 targets or NULL, out[5] the in0 pair, out[6..9] the skip
    // pairs (bf16 [P][2 ld]: hi in columns [0, ld), lo in [ld, 2 ld) of each row; NULL: none)
    const int multires = (int)d[0], E = 3 * (1 + 2 * multires), EP = (int)round_up(E, 8);
    if (multires < 0 || multires > 10 || d[1] < EP || d[2] < 0 || d[2] > 4) return AVC_E_SIZE;
    EncodeTargets t;
    memset(&t, 0, sizeof(t));
    t.in0 = O32(out[0]); t.ld0 = (int)d[1]; t.in0_16 = pair(out[5], t.ld0);
    t.n_skip = (int)d[2];
    for (int s = 0; s < t.n_skip; ++s) {
      t.skip_ptr[s] = O32(out[1 + s]); t.skip_ld[s] = (int)d[3 + s]; t.skip_col[s] = (int)d[7 + s];
      if (t.skip_col[s] < 0 || t.skip_col[s] + E > t.skip_ld[s]) return AVC_E_SIZE;
      t.skip16[s] = pair(out[6 + s], t.skip_ld[s]);
    }
    if (kind == 12) {
      if (d[11] < 1) return AVC_E_SIZE;
      return encode_points(F32(in[0]), d[11], fs[0], multires, E, EP, t, st);
    }
    if (kind == 13) {
      const int nz = (int)d[11], pitch = (int)d[12], Rc = (int)d[13];
      if (nz < 1 || pitch < nz || Rc < 1) return AVC_E_SIZE;
      return encode_samples(F32(in[0]), F32(in[1]), F32(in[2]), nz, pitch, Rc, fs[0], multires, E, EP, t, st);
    }
    const int S = (int)d[11];
    if (S < 1 || d[12] < 1 || !out[10]) return AVC_E_SIZE;
    return encode_fine(F32(in[0]), F32(in[1]), F32(in[2]), S, d[12], fs[1], fs[0], multires, E, EP, O32(out[10]),
                       O32(out[11]), O32(out[12]), t, st);
  }
  // the kinds below run on a whole configuration: in[0] is a HOST avc_neus_cfg
  NeusPlan pl;
  AVC_TRY(build_plan((const avc_neus_cfg*)in[0], &pl));
  if (kind >= 15 && d[0] < 1) return AVC_E_SIZE;      // d[0] = P
  switch (kind) {
    case 9: {
      int64_t* o = (int64_t*)out[0];
      const int64_t head[16] = {pl.L, pl.Lc, pl.E, pl.EP, pl.F, pl.Fp, pl.Hc, pl.pack_floats, pl.n_params, pl.off_var,
                                pl.pk_wsdf, pl.pk_bsdf, pl.pk_c0x, pl.pk_c0xT, pl.pk_W6, pl.pk_b6};
      for (int i = 0; i < 16; ++i) o[i] = head[i];
      int64_t* q = o + 16;
      auto put = [&](const LinDim& x) {
        const int64_t r[11] = {x.K, x.N, x.Kp, x.Np, x.skip ? 1 : 0, x.off_g, x.off_v, x.off_b, x.pk_W, x.pk_WT, x.pk_b};
        for (int i = 0; i < 11; ++i) *q++ = r[i];
      };
      for (int l = 0; l <= pl.L; ++l) put(pl.sdf[l]);
      for (int l = 0; l <= pl.Lc; ++l) put(pl.col[l]);
      put(pl.extra);
      return 0;
    }
    case 10: {
      NeusWs w;
      memset(&w, 0, sizeof(w));
      w.pack = O32(out[0]);
      if (pl.cfg.engine == 1) {
        if (!out[1]) return AVC_E_NULL;
        w.pk_hi = (__nv_bfloat16*)out[1]; w.pk_lo = w.pk_hi + pl.pack_floats;
      }
      return prepare_weights(pl, w, F32(in[1]), st);
    }
    case 11: return weight_norm_backward_all(pl, F32(in[1]), F32(in[2]), O32(out[0]), st);
    case 15: return sdf_head(pl, F32(in[1]), F32(in[2]), d[0], O32(out[0]), (int)d[1], (int)d[2], st);
    case 16: return color_heads(pl, F32(in[1]), F32(in[2]), d[0], O32(out[0]), st);
    case 17: return nbar_add_color(pl, F32(in[1]), F32(in[2]), d[0], O32(out[0]), st);
    case 20: return heads_dgrad(pl, F32(in[1]), F32(in[2]), F32(in[3]), d[0], O32(out[0]), pair(out[1], pl.Hc), st);
    case 21:
      return chain_start(pl, F32(in[1]), F32(in[2]), d[0], O32(out[0]), O32(out[1]), pair(out[2], pl.sdf[pl.L - 1].Np),
                         st);
    case 22: return normals(pl, F32(in[1]), d[0], O32(out[0]), O32(out[1]), st);
    case 23: return dge(pl, F32(in[1]), F32(in[2]), d[0], O32(out[0]), O32(out[1]), pair(out[2], pl.sdf[0].Kp), st);
    case 24: {
      const int l = (int)d[1];
      if (l < 1 || l > pl.L || !pl.sdf[l].skip) return AVC_E_BADCFG;
      return fill_gebar(pl, l, F32(in[1]), d[0], O32(out[0]), pair(out[1], pl.sdf[l].Kp), st);
    }
    case 26: return assemble_sdf_feat(pl, F32(in[1]), F32(in[2]), d[0], O32(out[0]), st);
  }
  return AVC_E_BADCFG;
}

int avc_neus_param_count(const avc_neus_cfg* cfg, int64_t* n_params) {
  if (!cfg || !n_params) return AVC_E_NULL;
  NeusPlan pl;
  AVC_TRY(build_plan(cfg, &pl));
  *n_params = pl.n_params;
  return 0;
}

int avc_neus_param_offset(const avc_neus_cfg* cfg, int net, int layer, int which, int64_t* offset, int64_t* numel) {
  if (!cfg || !offset || !numel) return AVC_E_NULL;
  NeusPlan pl;
  AVC_TRY(build_plan(cfg, &pl));
  const LinDim* d = nullptr;
  if (net == 0) { if (layer < 0 || layer > pl.L) return AVC_E_SIZE; d = &pl.sdf[layer]; }
  else if (net == 1) { if (layer < 0 || layer > pl.Lc) return AVC_E_SIZE; d = &pl.col[layer]; }
  else if (net == 2) d = &pl.extra;
  else if (net == 3) { *offset = pl.off_var; *numel = 1; return 0; }
  else return AVC_E_BADCFG;
  if (which == 0) { *offset = d->off_g; *numel = d->N; }
  else if (which == 1) { *offset = d->off_v; *numel = (int64_t)d->N * d->K; }
  else if (which == 2) { *offset = d->off_b; *numel = d->N; }
  else return AVC_E_BADCFG;
  return 0;
}

int avc_neus_workspace_bytes(const avc_neus_cfg* cfg, int64_t max_rays_per_chunk, size_t* bytes) {
  if (!cfg || !bytes) return AVC_E_NULL;
  if (max_rays_per_chunk <= 0) return AVC_E_SIZE;
  NeusPlan pl;
  AVC_TRY(build_plan(cfg, &pl));
  NeusWs w;
  carve_ws(pl, max_rays_per_chunk, nullptr, &w);
  *bytes = w.bytes;
  return 0;
}

int avc_neus_render_fwd(const avc_neus_cfg* cfg, const float* params, const float* rays_o, const float* rays_d,
                        const float* near, const float* far, const float* jitter, const float* background,
                        int bg_kind, const float* z_vals_in, float cos_anneal_ratio, int64_t R,
                        const avc_neus_outputs* out, void* workspace, size_t workspace_bytes,
                        int64_t max_rays_per_chunk, avc_stream_t stream) {
  if (!cfg || !params || !rays_o || !rays_d || !out || !workspace) return AVC_E_NULL;
  if (!z_vals_in && (!near || !far)) return AVC_E_NULL;
  if (!out->color_fine || !out->extra_color_fine || !out->s_val || !out->cdf_fine || !out->weight_sum ||
      !out->weight_max || !out->gradients || !out->weights || !out->mid_z_vals || !out->gradient_error ||
      !out->inside_sphere || !out->z_vals)
    return AVC_E_NULL;
  if (bg_kind < 0 || bg_kind > 2 || (bg_kind != 0 && !background)) return AVC_E_BADCFG;
  if (R <= 0 || max_rays_per_chunk <= 0) return AVC_E_SIZE;
  NeusPlan pl;
  AVC_TRY(build_plan(cfg, &pl));
  AVC_TRY(check_ptr16(workspace)); AVC_TRY(check_ptr16(params)); AVC_TRY(check_ptr16(out->z_vals));
  const int64_t Rc_max = R < max_rays_per_chunk ? R : max_rays_per_chunk;
  NeusWs w;
  carve_ws(pl, Rc_max, workspace, &w);
  if (w.bytes > workspace_bytes) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;

  AVC_TRY(prepare_weights(pl, w, params, st));
  AVC_TRY(ctx_init(params, pl.off_var, w.ctx, 1, st));

  for (int64_t r0 = 0; r0 < R; r0 += Rc_max) {
    const int64_t Rc = (R - r0) < Rc_max ? (R - r0) : Rc_max;
    ChunkIO io;
    io.rays_o = rays_o + r0 * 3; io.rays_d = rays_d + r0 * 3;
    io.background = (bg_kind == 2) ? background + r0 : background;
    io.bg_kind = bg_kind; io.cos_anneal = cos_anneal_ratio; io.Rc = Rc;
    io.out = offset_outputs(*out, r0, pl.S);
    if (z_vals_in && z_vals_in + r0 * pl.S == io.out.z_vals) {
      // caller passed the output buffer itself: depths already in place
    } else if (z_vals_in) {
      AVC_CUDA_TRY(cudaMemcpyAsync(io.out.z_vals, z_vals_in + r0 * pl.S, sizeof(float) * Rc * pl.S,
                                   cudaMemcpyDeviceToDevice, st));
    } else {
      AVC_TRY(place_samples(pl, w, io.rays_o, io.rays_d, near + r0, far + r0, jitter ? jitter + r0 : nullptr,
                            (int)Rc, io.out.z_vals, st));
    }
    AVC_TRY(fine_forward(pl, w, io, true, st));
  }
  return finalize_fwd(w.ctx, out->gradient_error, st);
}

int avc_neus_render_bwd(const avc_neus_cfg* cfg, const float* params, const float* rays_o, const float* rays_d,
                        const float* background, int bg_kind, float cos_anneal_ratio, int64_t R,
                        const avc_neus_outputs* fwd_out, const avc_neus_cotangents* cot, float* grad_params,
                        void* workspace, size_t workspace_bytes, int64_t max_rays_per_chunk, int32_t flags,
                        avc_stream_t stream) {
  if (!cfg || !params || !rays_o || !rays_d || !fwd_out || !cot || !grad_params || !workspace) return AVC_E_NULL;
  if (!fwd_out->z_vals || !fwd_out->weights) return AVC_E_NULL;
  if (bg_kind < 0 || bg_kind > 2 || (bg_kind != 0 && !background)) return AVC_E_BADCFG;
  if (R <= 0 || max_rays_per_chunk <= 0) return AVC_E_SIZE;
  NeusPlan pl;
  AVC_TRY(build_plan(cfg, &pl));
  AVC_TRY(check_ptr16(workspace)); AVC_TRY(check_ptr16(params)); AVC_TRY(check_ptr16(grad_params));
  const int64_t Rc_max = R < max_rays_per_chunk ? R : max_rays_per_chunk;
  NeusWs w;
  carve_ws(pl, Rc_max, workspace, &w);
  if (w.bytes > workspace_bytes) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  const bool single = (R <= Rc_max) && !(flags & AVC_BWD_RECOMPUTE);

  // The workspace still holds pack / ctx sums / (single chunk) the stash of the matching forward.
  // Multi-chunk calls rebuild the stash per chunk from the saved depths.
  AVC_CUDA_TRY(cudaMemsetAsync(w.wbar, 0, sizeof(float) * (size_t)pl.n_params, st));
  AVC_TRY(ctx_init(params, pl.off_var, w.ctx, 1, st));
  for (int64_t r0 = 0; r0 < R; r0 += Rc_max) {   // eikonal normaliser over ALL rays of the call
    const int64_t Rc = (R - r0) < Rc_max ? (R - r0) : Rc_max;
    AVC_TRY(relax_count(rays_o + r0 * 3, rays_d + r0 * 3, fwd_out->z_vals + r0 * pl.S, pl.S, Rc, 2.0f / (float)pl.n0,
                        w.ray_part, w.ctx, st));
  }
  if (!single) AVC_TRY(prepare_weights(pl, w, params, st));
  for (int64_t r0 = 0; r0 < R; r0 += Rc_max) {
    const int64_t Rc = (R - r0) < Rc_max ? (R - r0) : Rc_max;
    ChunkIO io;
    io.rays_o = rays_o + r0 * 3; io.rays_d = rays_d + r0 * 3;
    io.background = (bg_kind == 2) ? background + r0 : background;
    io.bg_kind = bg_kind; io.cos_anneal = cos_anneal_ratio; io.Rc = Rc;
    io.out = offset_outputs(*fwd_out, r0, pl.S);
    if (!single) AVC_TRY(fine_forward(pl, w, io, false, st));
    avc_neus_cotangents c = offset_cot(*cot, r0, pl.S);
    AVC_TRY(fine_backward(pl, w, io, c, st));
  }
  AVC_TRY(weight_norm_backward_all(pl, params, w.wbar, grad_params, st));
  return variance_grad(params, pl.off_var, w.ctx, cot->s_val, R, grad_params + pl.off_var, st);
}

int avc_neus_sdf_query(const avc_neus_cfg* cfg, const float* params, const float* pts, int64_t P, float* sdf_out,
                       void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!cfg || !params || !pts || !sdf_out || !workspace) return AVC_E_NULL;
  if (P <= 0) return AVC_E_SIZE;
  NeusPlan pl;
  AVC_TRY(build_plan(cfg, &pl));
  // the workspace is sized in rays; a chunk of Rc rays offers Rc * S point rows
  size_t one = 0;
  AVC_TRY(avc_neus_workspace_bytes(cfg, 1, &one));
  NeusWs w;
  int64_t Rc = 1;
  {   // largest Rc that fits (bytes grow linearly in Rc)
    NeusWs w2; carve_ws(pl, 2, nullptr, &w2);
    size_t per = w2.bytes - one;
    if (workspace_bytes < one) return AVC_E_SIZE;
    Rc = 1 + (int64_t)((workspace_bytes - one) / (per ? per : 1));
    while (Rc > 1) { carve_ws(pl, Rc, nullptr, &w); if (w.bytes <= workspace_bytes) break; --Rc; }
  }
  carve_ws(pl, Rc, workspace, &w);
  if (w.bytes > workspace_bytes) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  AVC_TRY(prepare_weights(pl, w, params, st));
  const int64_t cap = Rc * pl.S;
  EncodeTargets t = make_targets(pl, w);
  for (int64_t p0 = 0; p0 < P; p0 += cap) {
    int64_t n = (P - p0) < cap ? (P - p0) : cap;
    AVC_TRY(encode_points(pts + p0 * 3, n, pl.cfg.sdf_scale, pl.cfg.sdf_multires, pl.E, pl.EP, t, st));
    AVC_TRY(value_chain(pl, w, n, false, false, sdf_out + p0, st));
  }
  return 0;
}

// SDFNetwork.forward / .sdf_hidden_appearance / .gradient (models/fields.py:72-107) on arbitrary points: convenience
// evaluators of the boundary (not on the training path).  Always the exact-fp32 tiles (engine 0).
int avc_neus_sdf_eval(const avc_neus_cfg* cfg_in, const float* params, const float* pts, int64_t P, float* sdf_feat_out,
                      float* grad_out, void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!cfg_in || !params || !pts || !workspace) return AVC_E_NULL;
  if (!sdf_feat_out && !grad_out) return AVC_E_NULL;
  if (P <= 0) return AVC_E_SIZE;
  avc_neus_cfg cfg = *cfg_in;
  cfg.engine = 0;
  NeusPlan pl;
  AVC_TRY(build_plan(&cfg, &pl));
  size_t one = 0;
  AVC_TRY(avc_neus_workspace_bytes(&cfg, 1, &one));
  NeusWs w;
  int64_t Rc = 1;
  {
    NeusWs w2; carve_ws(pl, 2, nullptr, &w2);
    size_t per = w2.bytes - one;
    if (workspace_bytes < one) return AVC_E_SIZE;
    Rc = 1 + (int64_t)((workspace_bytes - one) / (per ? per : 1));
    while (Rc > 1) { carve_ws(pl, Rc, nullptr, &w); if (w.bytes <= workspace_bytes) break; --Rc; }
  }
  carve_ws(pl, Rc, workspace, &w);
  if (w.bytes > workspace_bytes) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  AVC_TRY(prepare_weights(pl, w, params, st));
  const int64_t cap = Rc * pl.S;
  EncodeTargets t = make_targets(pl, w);
  for (int64_t p0 = 0; p0 < P; p0 += cap) {
    int64_t n = (P - p0) < cap ? (P - p0) : cap;
    AVC_TRY(encode_points(pts + p0 * 3, n, pl.cfg.sdf_scale, pl.cfg.sdf_multires, pl.E, pl.EP, t, st));
    AVC_TRY(points_to_cin(pts + p0 * 3, n, w.cin, st));
    AVC_TRY(value_chain(pl, w, n, grad_out != nullptr, sdf_feat_out != nullptr, w.sdf, st));
    if (sdf_feat_out) AVC_TRY(assemble_sdf_feat(pl, w.sdf, w.feat, n, sdf_feat_out + p0 * (pl.F + 1), st));
    if (grad_out) AVC_TRY(gradient_chain(pl, w, n, grad_out + p0 * 3, st));
  }
  return 0;
}

// The C ABI carries betas as float; the reference's betas are the Python doubles 0.9 / 0.999.  Recover the short decimal
// the float was rounded from (6 significant digits) so that `1 - beta` and the bias corrections match torch's doubles.
static double round_beta(float b) { return (double)((long long)((double)b * 1e6 + 0.5)) / 1e6; }

int avc_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                  float beta1, float beta2, float eps, int64_t step, float grad_scale, avc_stream_t stream) {
  if (!params || !grads || !exp_avg || !exp_avg_sq) return AVC_E_NULL;
  if (n <= 0 || step < 1) return AVC_E_SIZE;
  // Python floats are doubles: torch sees beta = 0.9 / 0.999 exactly as the decimal literals, not their float roundings
  const double b1 = round_beta(beta1), b2 = round_beta(beta2);
  double bc1 = 1.0 - pow(b1, (double)step);
  double bc2 = 1.0 - pow(b2, (double)step);
  k_adam<<<blocks_for(n, 256), 256, 0, (cudaStream_t)stream>>>(params, grads, exp_avg, exp_avg_sq, n, lr, (float)b1,
                                                               (float)b2, eps, (float)bc1, (float)sqrt(bc2), grad_scale,
                                                               (float)(1.0 - b1), (float)(1.0 - b2));
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_adam_step_dev(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, float* state,
                      float beta1, float beta2, float eps, float grad_scale, avc_stream_t stream) {
  if (!params || !grads || !exp_avg || !exp_avg_sq || !state) return AVC_E_NULL;
  if (n <= 0) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  const double b1 = round_beta(beta1), b2 = round_beta(beta2);
  k_adam_state<<<1, 32, 0, st>>>(state, b1, b2);
  k_adam_dev<<<blocks_for(n, 256), 256, 0, st>>>(params, grads, exp_avg, exp_avg_sq, n, state, (float)b1, (float)b2, eps,
                                                 grad_scale, (float)(1.0 - b1), (float)(1.0 - b2));
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"
