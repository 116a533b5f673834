// avc_motion.cu -- AvatarAnimate's MotionOptimizer without its CLIP term (models/motion_generation.py:249-358): a motion
// from the motion VAE's transformer decoder, its latent optimised so that the motion passes through the candidate poses.
//
//   avc_motion_decode    MotionOptimizer.decode: decoder (4-layer post-LN nn.TransformerDecoder over the positional
//                        table, one memory token = the latent), final linear, then rotation_6d_to_matrix ->
//                        matrix_to_quaternion -> quaternion_to_axis_angle, joints 1..21
//   avc_motion_optimize  n iterations of decode, the reconstruction (and delta) loss, the backward to the latent only and
//                        avc_adam_step_dev; one iteration's launches are captured once as a CUDA graph and the graph is
//                        launched n times, so the host never waits inside the call
//
// Exact shortcuts: cross-attention attends over one memory token, so its softmax is exactly 1 and its output is
// out_proj(v_proj(latent)) on every row (Q / K get no gradient); layer 0's self-attention reads only the positional
// table, so that block (and its LayerNorm) is computed once per call.
#include <cfloat>
#include <cmath>

#include "avc_common.cuh"
#include "avc_dual.cuh"

using namespace avc;

namespace {

constexpr int kMaxT = 64;          // frames (attention rows)
constexpr int kMaxD = 512;
constexpr int kMaxHeadDim = 64;
constexpr int kMaxF = 4096;
constexpr int kMaxLayers = 16;
constexpr int kMaxCand = 16;
constexpr int kJoints = 21;        // motion[:, 3:66]: joints 1..21 of the decoder's n_out / 6
constexpr int kPose = kJoints * 3;
constexpr float kLnEps = 1e-5f;    // nn.LayerNorm default

// ---------------------------------------------------------------- parameter layout (floats)
struct Layout {
  int D, F, n_out, L;
  size_t wqkv, bqkv, wo, bo, wv, bv, wc, bc, w1, b1, w2, b2, g1, be1, g2, be2, g3, be3, stride, wf, bf, total;
};

Layout make_layout(int D, int F, int n_out, int L) {
  Layout y{};
  y.D = D; y.F = F; y.n_out = n_out; y.L = L;
  size_t o = 0;
  auto take = [&](size_t n) { size_t r = o; o += n; return r; };
  y.wqkv = take((size_t)3 * D * D); y.bqkv = take(3 * D);
  y.wo = take((size_t)D * D); y.bo = take(D);
  y.wv = take((size_t)D * D); y.bv = take(D);
  y.wc = take((size_t)D * D); y.bc = take(D);
  y.w1 = take((size_t)F * D); y.b1 = take(F);
  y.w2 = take((size_t)D * F); y.b2 = take(D);
  y.g1 = take(D); y.be1 = take(D); y.g2 = take(D); y.be2 = take(D); y.g3 = take(D); y.be3 = take(D);
  y.stride = o;
  y.wf = (size_t)L * y.stride;
  y.bf = y.wf + (size_t)n_out * D;
  y.total = y.bf + n_out;
  return y;
}

// ---------------------------------------------------------------- fp32 GEMM
// C[m][n] = epi(sum_k A[m][k] op(B)[k][n] + bias[n] + addend[m][n]); op(B)[k][n] = B[n][k] (BT: nn.Linear forward,
// B = W [N][K]) or B[k][n] (!BT: input gradient, B = W [K][N]).  EPI 0 plain; 1 GELU (aux = the pre-activation);
// 2 times GELU'(aux).  32 x 32 tiles, 256 threads, 2 x 2 outputs per thread, k in steps of 32.
constexpr int kTM = 32, kTN = 32, kTK = 32;

__device__ __forceinline__ float gelu(float x) { return 0.5f * x * (1.f + erff(x * kSqrtHalf)); }
__device__ __forceinline__ float gelu_d(float x) {
  return 0.5f * (1.f + erff(x * kSqrtHalf)) + x * expf(-0.5f * x * x) * 0.3989422804014327f;
}

template <bool BT, int EPI>
__global__ void __launch_bounds__(256)
k_gemm(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb, const float* __restrict__ bias,
       const float* __restrict__ addend, float* __restrict__ C, int ldc, float* __restrict__ aux, int M, int N, int K) {
  __shared__ float sa[kTK][kTM + 1];
  __shared__ float sb[kTK][kTN + 1];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * kTM, n0 = blockIdx.x * kTN;
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  for (int k0 = 0; k0 < K; k0 += kTK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = tid + i * 256, r = e >> 5, c = e & 31;
      const int m = m0 + r, k = k0 + c;
      sa[c][r] = (m < M && k < K) ? A[(size_t)m * lda + k] : 0.f;
      if (BT) {
        const int n = n0 + r;
        sb[c][r] = (n < N && k < K) ? B[(size_t)n * ldb + k] : 0.f;
      } else {
        const int kk = k0 + r, n = n0 + c;
        sb[r][c] = (kk < K && n < N) ? B[(size_t)kk * ldb + n] : 0.f;
      }
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < kTK; ++kk) {
      const float a0 = sa[kk][ty], a1 = sa[kk][ty + 16], b0 = sb[kk][tx], b1 = sb[kk][tx + 16];
      acc[0][0] = fmaf(a0, b0, acc[0][0]);
      acc[0][1] = fmaf(a0, b1, acc[0][1]);
      acc[1][0] = fmaf(a1, b0, acc[1][0]);
      acc[1][1] = fmaf(a1, b1, acc[1][1]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int m = m0 + ty + 16 * i, n = n0 + tx + 16 * j;
      if (m >= M || n >= N) continue;
      float v = acc[i][j];
      if (bias) v += bias[n];
      if (addend) v += addend[(size_t)m * ldc + n];
      if (EPI == 1) {
        aux[(size_t)m * ldc + n] = v;
        v = gelu(v);
      } else if (EPI == 2) {
        v *= gelu_d(aux[(size_t)m * ldc + n]);
      }
      C[(size_t)m * ldc + n] = v;
    }
}

// ---------------------------------------------------------------- attention over the T query rows, one CTA per head
// Q, K, V [T][dh] of head h are columns h dh, D + h dh, 2D + h dh of qkv [T][3D]; P [H][T][T] the softmax
__global__ void __launch_bounds__(256)
k_attn_fwd(const float* __restrict__ qkv, int T, int D, int dh, float scale, float* __restrict__ P,
           float* __restrict__ out) {
  extern __shared__ float sm[];
  const int h = blockIdx.x, ld = dh + 1, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  float *sq = sm, *sk = sq + T * ld, *sv = sk + T * ld, *sp = sv + T * ld;
  for (int i = threadIdx.x; i < T * dh; i += blockDim.x) {
    const int t = i / dh, d = i - t * dh;
    const float* row = qkv + (size_t)t * 3 * D + h * dh + d;
    sq[t * ld + d] = row[0];
    sk[t * ld + d] = row[D];
    sv[t * ld + d] = row[2 * D];
  }
  __syncthreads();
  float* p = sp + warp * kMaxT;
  for (int i = warp; i < T; i += nw) {
    float mx = -FLT_MAX;
    for (int j = lane; j < T; j += 32) {
      float s = 0.f;
      for (int d = 0; d < dh; ++d) s = fmaf(sq[i * ld + d], sk[j * ld + d], s);
      p[j] = s * scale;
      mx = fmaxf(mx, p[j]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int j = lane; j < T; j += 32) {
      p[j] = expf(p[j] - mx);
      sum += p[j];
    }
    sum = warp_sum(sum);
    for (int j = lane; j < T; j += 32) {
      p[j] /= sum;
      P[((size_t)h * T + i) * T + j] = p[j];
    }
    __syncwarp();
    for (int d = lane; d < dh; d += 32) {
      float o = 0.f;
      for (int j = 0; j < T; ++j) o = fmaf(p[j], sv[j * ld + d], o);
      out[(size_t)i * D + h * dh + d] = o;
    }
    __syncwarp();
  }
}

// input gradient of k_attn_fwd: dO [T][D] (head columns) -> dqkv [T][3D]
__global__ void __launch_bounds__(256)
k_attn_bwd(const float* __restrict__ qkv, const float* __restrict__ P, const float* __restrict__ dO, int T, int D,
           int dh, float scale, float* __restrict__ dqkv) {
  extern __shared__ float sm[];
  const int h = blockIdx.x, ld = dh + 1, lds = T + 1, warp = threadIdx.x >> 5, lane = threadIdx.x & 31,
            nw = blockDim.x >> 5;
  float *sq = sm, *sk = sq + T * ld, *sv = sk + T * ld, *sdo = sv + T * ld, *sds = sdo + T * ld, *spp = sds + T * lds;
  const float* Ph = P + (size_t)h * T * T;
  for (int i = threadIdx.x; i < T * dh; i += blockDim.x) {
    const int t = i / dh, d = i - t * dh;
    const float* row = qkv + (size_t)t * 3 * D + h * dh + d;
    sq[t * ld + d] = row[0];
    sk[t * ld + d] = row[D];
    sv[t * ld + d] = row[2 * D];
    sdo[t * ld + d] = dO[(size_t)t * D + h * dh + d];
  }
  for (int i = threadIdx.x; i < T * T; i += blockDim.x) spp[(i / T) * lds + i % T] = Ph[i];
  __syncthreads();
  // dS[i][j] = P[i][j] (dP[i][j] - sum_j' P[i][j'] dP[i][j']),  dP = dO V^T
  for (int i = warp; i < T; i += nw) {
    float rd = 0.f;
    for (int j = lane; j < T; j += 32) {
      float dp = 0.f;
      for (int d = 0; d < dh; ++d) dp = fmaf(sdo[i * ld + d], sv[j * ld + d], dp);
      sds[i * lds + j] = dp;
      rd = fmaf(spp[i * lds + j], dp, rd);
    }
    rd = warp_sum(rd);
    for (int j = lane; j < T; j += 32) sds[i * lds + j] = spp[i * lds + j] * (sds[i * lds + j] - rd);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < T * dh; e += blockDim.x) {
    const int i = e / dh, d = e - i * dh;
    float gq = 0.f, gk = 0.f, gv = 0.f;
    for (int j = 0; j < T; ++j) {
      gq = fmaf(sds[i * lds + j], sk[j * ld + d], gq);     // dQ[i] = scale sum_j dS[i][j] K[j]
      gk = fmaf(sds[j * lds + i], sq[j * ld + d], gk);     // dK[i] = scale sum_j dS[j][i] Q[j]
      gv = fmaf(spp[j * lds + i], sdo[j * ld + d], gv);    // dV[i] = sum_j P[j][i] dO[j]
    }
    float* row = dqkv + (size_t)i * 3 * D + h * dh + d;
    row[0] = gq * scale;
    row[D] = gk * scale;
    row[2 * D] = gv;
  }
}

// ---------------------------------------------------------------- LayerNorm, one warp per row
// y = LN(a + b + c) with b [T][D] or NULL and c [D] (broadcast over the rows) or NULL; xhat and rstd kept for the
// backward
__global__ void __launch_bounds__(256)
k_ln_fwd(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ c,
         const float* __restrict__ gamma, const float* __restrict__ beta, int T, int D, float* __restrict__ y,
         float* __restrict__ xhat, float* __restrict__ rstd) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= T) return;
  const size_t o = (size_t)row * D;
  float s = 0.f;
  for (int i = lane; i < D; i += 32) {
    float v = a[o + i] + (b ? b[o + i] : 0.f);
    if (c) v += c[i];
    xhat[o + i] = v;
    s += v;
  }
  const float mean = warp_sum(s) / D;
  float q = 0.f;
  for (int i = lane; i < D; i += 32) {
    const float d = xhat[o + i] - mean;
    q = fmaf(d, d, q);
  }
  const float r = rsqrtf(warp_sum(q) / D + kLnEps);
  for (int i = lane; i < D; i += 32) {
    const float xh = (xhat[o + i] - mean) * r;
    xhat[o + i] = xh;
    y[o + i] = fmaf(xh, gamma[i], beta[i]);
  }
  if (lane == 0) rstd[row] = r;
}

// dx = rstd (g - mean(g) - xhat mean(g xhat)),  g = dy gamma
__global__ void __launch_bounds__(256)
k_ln_bwd(const float* __restrict__ dy, const float* __restrict__ gamma, const float* __restrict__ xhat,
         const float* __restrict__ rstd, int T, int D, float* __restrict__ dx) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= T) return;
  const size_t o = (size_t)row * D;
  float s1 = 0.f, s2 = 0.f;
  for (int i = lane; i < D; i += 32) {
    const float g = dy[o + i] * gamma[i];
    s1 += g;
    s2 = fmaf(g, xhat[o + i], s2);
  }
  const float m1 = warp_sum(s1) / D, m2 = warp_sum(s2) / D, r = rstd[row];
  for (int i = lane; i < D; i += 32) dx[o + i] = r * (dy[o + i] * gamma[i] - m1 - xhat[o + i] * m2);
}

// ---------------------------------------------------------------- the memory token (cross-attention)
// y[l][n] = W_l[n][:] . x_l + b_l[n] for every layer l (W_l = base + l stride), one warp per output; x_l = x + l xs
__global__ void __launch_bounds__(256)
k_layer_matvec(const float* __restrict__ W, const float* __restrict__ bias, size_t stride, const float* __restrict__ x,
               int xs, int D, float* __restrict__ y) {
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), l = blockIdx.y, lane = threadIdx.x & 31;
  if (n >= D) return;
  const float* w = W + l * stride + (size_t)n * D;
  const float* xl = x + (size_t)l * xs;
  float s = 0.f;
  for (int k = lane; k < D; k += 32) s = fmaf(w[k], xl[k], s);
  s = warp_sum(s);
  if (lane == 0) y[(size_t)l * D + n] = s + bias[l * stride + n];
}

// w[k] = sum_n Wc[n][k] u[n], u[n] = sum_t dz[t][n]: the cross-attention output's gradient through out_proj
__global__ void __launch_bounds__(256)
k_cross_back(const float* __restrict__ dz, int T, int D, const float* __restrict__ Wc, float* __restrict__ w) {
  __shared__ float u[kMaxD];
  for (int n = threadIdx.x; n < D; n += blockDim.x) {
    float s = 0.f;
    for (int t = 0; t < T; ++t) s += dz[(size_t)t * D + n];
    u[n] = s;
  }
  __syncthreads();
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= D) return;
  float s = 0.f;
  for (int n = 0; n < D; ++n) s = fmaf(Wc[(size_t)n * D + k], u[n], s);
  w[k] = s;
}

// grad[k] = sum_l sum_n Wv_l[n][k] w_l[n]: the latent's gradient (it is every layer's memory token)
__global__ void k_latent_grad(const float* __restrict__ Wv, size_t stride, const float* __restrict__ w, int L, int D,
                              float* __restrict__ grad) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= D) return;
  float s = 0.f;
  for (int l = 0; l < L; ++l) {
    const float* W = Wv + l * stride;
    for (int n = 0; n < D; ++n) s = fmaf(W[(size_t)n * D + k], w[(size_t)l * D + n], s);
  }
  grad[k] = s;
}

// ---------------------------------------------------------------- rotation chain (models/utils.py), value + tangent
// S is float (values) or Dual (one forward-mode tangent, avc_dual.cuh).

// torch.norm(p=2): its gradient is 0 where the norm is 0
template <class S> __device__ __forceinline__ S norm3(S a, S b, S c) {
  const S ss = a * a + b * b + c * c;
  return val(ss) > 0.f ? dsqrt(ss) : konst<S>(0.f);
}
// x.clamp_min(eps) (F.normalize's denominator): the gradient passes where x >= eps
template <class S> __device__ __forceinline__ S clamp_min(S x, float eps) { return val(x) >= eps ? x : konst<S>(eps); }
// _sqrt_positive_part: zero subgradient at x <= 0
template <class S> __device__ __forceinline__ S sqrt_pos(S x) { return val(x) > 0.f ? dsqrt(x) : konst<S>(0.f); }
// torch.maximum(x, 0.1): the gradient goes to x above the floor, half of it at a tie
template <class S> __device__ __forceinline__ S floor01(S x);
template <> __device__ __forceinline__ float floor01<float>(float x) { return fmaxf(x, 0.1f); }
template <> __device__ __forceinline__ Dual floor01<Dual>(Dual x) {
  return x.v > 0.1f ? x : (x.v == 0.1f ? Dual{0.1f, 0.5f * x.d} : Dual{0.1f, 0.f});
}
// sin(a / 2) / a with the small-angle series below 1e-6
template <class S> __device__ __forceinline__ S sinc_half(S half, S angle) {
  return fabsf(val(angle)) < 1e-6f ? 0.5f - angle * angle / 48.f : dsin(half) / angle;
}

// d6 -> rotation_6d_to_matrix -> matrix_to_quaternion -> quaternion_to_axis_angle = aa, and aa -> axis_angle_to_matrix
// -> matrix_to_rotation_6d = g6 (the loss's view of the generated pose)
template <class S>
__device__ void rot6d_to_aa(const S* x, S* aa) {
  const S n1 = clamp_min(norm3(x[0], x[1], x[2]), 1e-12f);
  const S b1[3] = {x[0] / n1, x[1] / n1, x[2] / n1};
  const S dt = b1[0] * x[3] + b1[1] * x[4] + b1[2] * x[5];
  const S u[3] = {x[3] - dt * b1[0], x[4] - dt * b1[1], x[5] - dt * b1[2]};
  const S n2 = clamp_min(norm3(u[0], u[1], u[2]), 1e-12f);
  const S b2[3] = {u[0] / n2, u[1] / n2, u[2] / n2};
  const S b3[3] = {b1[1] * b2[2] - b1[2] * b2[1], b1[2] * b2[0] - b1[0] * b2[2], b1[0] * b2[1] - b1[1] * b2[0]};
  // rows of the matrix: b1, b2, b3
  const S m00 = b1[0], m01 = b1[1], m02 = b1[2], m10 = b2[0], m11 = b2[1], m12 = b2[2], m20 = b3[0], m21 = b3[1],
          m22 = b3[2];
  const S qa[4] = {sqrt_pos(1.f + m00 + m11 + m22), sqrt_pos(1.f + m00 - m11 - m22), sqrt_pos(1.f - m00 + m11 - m22),
                   sqrt_pos(1.f - m00 - m11 + m22)};
  int best = 0;                       // argmax: the first of equal maxima
#pragma unroll
  for (int i = 1; i < 4; ++i)
    if (val(qa[i]) > val(qa[best])) best = i;
  S q[4];
  if (best == 0) { q[0] = qa[0] * qa[0]; q[1] = m21 - m12; q[2] = m02 - m20; q[3] = m10 - m01; }
  else if (best == 1) { q[0] = m21 - m12; q[1] = qa[1] * qa[1]; q[2] = m10 + m01; q[3] = m02 + m20; }
  else if (best == 2) { q[0] = m02 - m20; q[1] = m10 + m01; q[2] = qa[2] * qa[2]; q[3] = m12 + m21; }
  else { q[0] = m10 - m01; q[1] = m20 + m02; q[2] = m21 + m12; q[3] = qa[3] * qa[3]; }
  const S den = 2.f * floor01(qa[best]);
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = q[i] / den;
  const S nv = norm3(q[1], q[2], q[3]);
  const S half = datan2(nv, q[0]);
  const S s = sinc_half(half, 2.f * half);
  aa[0] = q[1] / s; aa[1] = q[2] / s; aa[2] = q[3] / s;
}

template <class S>
__device__ void aa_to_6d(const S* aa, S* g6) {
  const S ang = norm3(aa[0], aa[1], aa[2]);
  const S half = ang * 0.5f;
  const S s = sinc_half(half, ang);
  const S r = dcos(half), i = aa[0] * s, j = aa[1] * s, k = aa[2] * s;
  const S two_s = 2.f / (r * r + i * i + j * j + k * k);
  g6[0] = 1.f - two_s * (j * j + k * k);
  g6[1] = two_s * (i * j - k * r);
  g6[2] = two_s * (i * k + j * r);
  g6[3] = two_s * (i * j + k * r);
  g6[4] = 1.f - two_s * (i * i + k * k);
  g6[5] = two_s * (j * k - i * r);
}

struct Coef {
  float c[kMaxCand];
};

// One CTA.  out [T][n_out] (the final linear) -> motion [T][63] (joints 1..21); with K candidates also the loss
// (per candidate the recon_coef-weighted min over frames of the 6D MSE; minus delta_coef times the MSE of consecutive
// frames when delta_coef > 0), written to loss_out[step] (step = the Adam counter, state[0]), and its gradient dout.
// torch.min's gradient goes to the first frame of equal minima.
__global__ void __launch_bounds__(1024)
k_motion_loss(const float* __restrict__ out, int T, int n_out, const float* __restrict__ poses, int K, Coef coef,
              float delta_coef, float* __restrict__ motion, float* __restrict__ g6buf, float* __restrict__ dout,
              float* __restrict__ loss_out, const float* __restrict__ state) {
  __shared__ float so6[kMaxCand * kJoints * 6];
  __shared__ float sl[kMaxCand * kMaxT];
  __shared__ int sarg[kMaxCand];
  __shared__ float red[32];
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int e = tid; e < T * kJoints; e += nt) {
    const int t = e / kJoints, j = e - t * kJoints;
    const float* x = out + (size_t)t * n_out + (j + 1) * 6;
    float xv[6], aa[3], g6[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) xv[i] = x[i];
    rot6d_to_aa(xv, aa);
#pragma unroll
    for (int c = 0; c < 3; ++c) motion[(size_t)t * kPose + j * 3 + c] = aa[c];
    if (K) {
      aa_to_6d(aa, g6);
#pragma unroll
      for (int c = 0; c < 6; ++c) g6buf[(size_t)e * 6 + c] = g6[c];
    }
  }
  if (!K) return;
  for (int e = tid; e < K * kJoints; e += nt) aa_to_6d(poses + (size_t)e * 3, so6 + e * 6);
  __syncthreads();
  for (int e = tid; e < K * T; e += nt) {
    const int k = e / T, t = e - k * T;
    float s = 0.f;
    for (int j = 0; j < kJoints; ++j) {
      float sj = 0.f;
      for (int c = 0; c < 6; ++c) {
        const float d = g6buf[((size_t)t * kJoints + j) * 6 + c] - so6[(k * kJoints + j) * 6 + c];
        sj = fmaf(d, d, sj);
      }
      s += sj / 6.f;
    }
    sl[e] = s / kJoints;
  }
  // delta: mean over (T - 1) x 63 of (motion[t] - motion[t + 1])^2
  float dl = 0.f;
  if (delta_coef > 0.f)
    for (int e = tid; e < (T - 1) * kPose; e += nt) {
      const float d = motion[e] - motion[e + kPose];
      dl = fmaf(d, d, dl);
    }
  dl = warp_sum(dl);
  if ((tid & 31) == 0) red[tid >> 5] = dl;
  __syncthreads();
  if (tid == 0) {
    float loss = 0.f;
    for (int k = 0; k < K; ++k) {
      int a = 0;
      for (int t = 1; t < T; ++t)
        if (sl[k * T + t] < sl[k * T + a]) a = t;
      sarg[k] = a;
      loss += sl[k * T + a] * coef.c[k];
    }
    if (delta_coef > 0.f) {
      float s = 0.f;
      for (int w = 0; w < (nt >> 5); ++w) s += red[w];
      loss -= s / ((T - 1) * kPose) * delta_coef;
    }
    if (loss_out) loss_out[(int)state[0]] = loss;
  }
  __syncthreads();
  const float gdelta = delta_coef > 0.f ? -delta_coef * 2.f / ((T - 1) * kPose) : 0.f;
  const float grecon = 2.f / (6.f * kJoints);
  for (int e = tid; e < T * kJoints; e += nt) {
    const int t = e / kJoints, j = e - t * kJoints;
    float dg[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, da[3] = {0.f, 0.f, 0.f};
    bool any = false;
    for (int k = 0; k < K; ++k)
      if (sarg[k] == t) {
        any = true;
#pragma unroll
        for (int c = 0; c < 6; ++c)
          dg[c] = fmaf(coef.c[k] * grecon, g6buf[(size_t)e * 6 + c] - so6[(k * kJoints + j) * 6 + c], dg[c]);
      }
    if (gdelta != 0.f) {
      any = true;
      const float* m = motion + (size_t)t * kPose + j * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        if (t + 1 < T) da[c] += gdelta * (m[c] - m[c + kPose]);
        if (t > 0) da[c] -= gdelta * (m[c - kPose] - m[c]);
      }
    }
    float* g = dout + (size_t)t * n_out + (j + 1) * 6;
    const float* x = out + (size_t)t * n_out + (j + 1) * 6;
#pragma unroll 1
    for (int i = 0; i < 6; ++i) {
      float r = 0.f;
      if (any) {
        Dual xd[6], aa[3], g6[6];
#pragma unroll
        for (int c = 0; c < 6; ++c) xd[c] = Dual{x[c], c == i ? 1.f : 0.f};
        rot6d_to_aa(xd, aa);
        aa_to_6d(aa, g6);
#pragma unroll
        for (int c = 0; c < 3; ++c) r = fmaf(da[c], aa[c].d, r);
#pragma unroll
        for (int c = 0; c < 6; ++c) r = fmaf(dg[c], g6[c].d, r);
      }
      g[i] = r;
    }
  }
}

// ---------------------------------------------------------------- the CLIP term (:333-343)
// Row r scores frame st + r P (P = clip_num_part, st = *st_idx) with weight clip_coef (st + r P) / T.  Rows past the
// motion get weight 0 and frame st, so that every row renders a valid pose.  One thread per (row, pose column).
__global__ void k_motion_clip_select(const float* __restrict__ motion, int T, int P, float clip_coef,
                                     const int32_t* __restrict__ st_idx, int R, float* __restrict__ pose,
                                     int32_t* __restrict__ frame, float* __restrict__ weight) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= R * kPose) return;
  const int r = e / kPose, c = e - r * kPose, st = *st_idx, t = st + r * P;
  const int f = t < T ? t : st;
  pose[e] = motion[(size_t)f * kPose + c];
  if (c == 0) {
    frame[r] = f;
    weight[r] = t < T ? clip_coef * ((float)t / (float)T) : 0.f;
  }
}

// dout[frame[r]] += J^T (weight[r] g[r]) per joint, J = d rot6d_to_aa / d (the 6D output), by the forward-mode duals
// k_motion_loss uses; loss_out[state[0]] += sum_r weight[r] loss[r].  Rows of weight 0 are skipped, and the rows of
// non-zero weight score distinct frames, so each thread owns its 6 entries of dout.
__global__ void k_motion_clip_grad(const float* __restrict__ out, int n_out, const int32_t* __restrict__ frame,
                                   const float* __restrict__ weight, int R, const float* __restrict__ g,
                                   const float* __restrict__ loss, float* __restrict__ dout,
                                   float* __restrict__ loss_out, const float* __restrict__ state) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e == 0 && loss_out) {
    float s = 0.f;
    bool any = false;
    for (int r = 0; r < R; ++r)
      if (weight[r] != 0.f) {
        any = true;
        s = fmaf(weight[r], loss[r], s);
      }
    if (any) loss_out[(int)state[0]] += s;
  }
  if (e >= R * kJoints) return;
  const int r = e / kJoints, j = e - r * kJoints;
  const float w = weight[r];
  if (w == 0.f) return;
  const size_t o = (size_t)frame[r] * n_out + (j + 1) * 6;
  const float ga[3] = {w * g[r * kPose + j * 3], w * g[r * kPose + j * 3 + 1], w * g[r * kPose + j * 3 + 2]};
#pragma unroll 1
  for (int i = 0; i < 6; ++i) {
    Dual xd[6], aa[3];
#pragma unroll
    for (int c = 0; c < 6; ++c) xd[c] = Dual{out[o + c], c == i ? 1.f : 0.f};
    rot6d_to_aa(xd, aa);
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) s = fmaf(ga[c], aa[c].d, s);
    dout[o + i] += s;
  }
}

// ---------------------------------------------------------------- host side
struct Dims {
  int D, L, H, F, T, O, dh;
};

struct Ws {
  float *lat, *m1, *m2, *grad, *state, *vc, *cvec, *wback, *out, *dout, *g6;
  float *qkv, *P, *attn, *sa, *xh1, *y1, *r1, *xh2, *y2, *r2, *u, *g, *f, *xh3, *y3, *r3;   // per layer
  float *dx, *dz3, *dg, *dh2, *dz2, *dz1, *da, *dqkv;
};

Ws carve(void* base, const Dims& d, size_t* used) {
  Carver c(base);
  Ws w{};
  const size_t TD = (size_t)d.T * d.D, TF = (size_t)d.T * d.F, L = d.L;
  w.lat = c.take<float>(d.D); w.m1 = c.take<float>(d.D); w.m2 = c.take<float>(d.D); w.grad = c.take<float>(d.D);
  w.state = c.take<float>(4);
  w.vc = c.take<float>(L * d.D); w.cvec = c.take<float>(L * d.D); w.wback = c.take<float>(L * d.D);
  w.out = c.take<float>((size_t)d.T * d.O); w.dout = c.take<float>((size_t)d.T * d.O);
  w.g6 = c.take<float>((size_t)d.T * kJoints * 6);
  w.qkv = c.take<float>(L * 3 * TD); w.P = c.take<float>(L * d.H * d.T * d.T); w.attn = c.take<float>(L * TD);
  w.sa = c.take<float>(L * TD);
  w.xh1 = c.take<float>(L * TD); w.y1 = c.take<float>(L * TD); w.r1 = c.take<float>(L * d.T);
  w.xh2 = c.take<float>(L * TD); w.y2 = c.take<float>(L * TD); w.r2 = c.take<float>(L * d.T);
  w.u = c.take<float>(L * TF); w.g = c.take<float>(L * TF); w.f = c.take<float>(L * TD);
  w.xh3 = c.take<float>(L * TD); w.y3 = c.take<float>(L * TD); w.r3 = c.take<float>(L * d.T);
  w.dx = c.take<float>(TD); w.dz3 = c.take<float>(TD); w.dg = c.take<float>(TF); w.dh2 = c.take<float>(TD);
  w.dz2 = c.take<float>(TD); w.dz1 = c.take<float>(TD); w.da = c.take<float>(TD); w.dqkv = c.take<float>(3 * TD);
  if (used) *used = c.used();
  return w;
}

size_t ws_bytes(const Dims& d) {
  size_t used = 0;
  carve(nullptr, d, &used);
  return used;
}

bool dims_ok(const Dims& d) {
  return d.D >= 32 && d.D <= kMaxD && d.H >= 1 && d.D % d.H == 0 && d.D / d.H <= kMaxHeadDim && d.L >= 1 &&
         d.L <= kMaxLayers && d.F >= 1 && d.F <= kMaxF && d.T >= 2 && d.T <= kMaxT && d.O % 6 == 0 &&
         d.O >= 6 * (kJoints + 1);
}

size_t attn_fwd_smem(const Dims& d) { return sizeof(float) * (3 * d.T * (d.dh + 1) + 8 * kMaxT); }
size_t attn_bwd_smem(const Dims& d) { return sizeof(float) * (4 * d.T * (d.dh + 1) + 2 * d.T * (d.T + 1)); }

template <bool BT, int EPI>
void gemm(cudaStream_t st, const float* A, int lda, const float* B, int ldb, const float* bias, const float* addend,
          float* C, int ldc, float* aux, int M, int N, int K) {
  dim3 grid(ceil_div(N, kTN), ceil_div(M, kTM));
  k_gemm<BT, EPI><<<grid, 256, 0, st>>>(A, lda, B, ldb, bias, addend, C, ldc, aux, M, N, K);
}

struct Net {
  Dims d;
  Layout y;
  const float* p;
  const float* pe;
  Ws w;
  float scale;
  const float* lp(int l, size_t off) const { return p + (size_t)l * y.stride + off; }
  size_t TD() const { return (size_t)d.T * d.D; }
};

void ln_fwd(cudaStream_t st, const Net& n, const float* a, const float* b, const float* c, const float* gamma,
            const float* beta, float* y, float* xh, float* r) {
  k_ln_fwd<<<ceil_div(n.d.T, 8), 256, 0, st>>>(a, b, c, gamma, beta, n.d.T, n.d.D, y, xh, r);
}

// self-attention block of layer l on x: qkv, attention, out_proj, LN1
void self_attn_fwd(cudaStream_t st, const Net& n, int l, const float* x) {
  const Dims& d = n.d;
  const size_t TD = n.TD();
  float* qkv = n.w.qkv + l * 3 * TD;
  gemm<true, 0>(st, x, d.D, n.lp(l, n.y.wqkv), d.D, n.lp(l, n.y.bqkv), nullptr, qkv, 3 * d.D, nullptr, d.T, 3 * d.D,
                d.D);
  k_attn_fwd<<<d.H, 256, attn_fwd_smem(d), st>>>(qkv, d.T, d.D, d.dh, n.scale, n.w.P + (size_t)l * d.H * d.T * d.T,
                                                  n.w.attn + l * TD);
  gemm<true, 0>(st, n.w.attn + l * TD, d.D, n.lp(l, n.y.wo), d.D, n.lp(l, n.y.bo), nullptr, n.w.sa + l * TD, d.D,
                nullptr, d.T, d.D, d.D);
  ln_fwd(st, n, x, n.w.sa + l * TD, nullptr, n.lp(l, n.y.g1), n.lp(l, n.y.be1), n.w.y1 + l * TD, n.w.xh1 + l * TD,
         n.w.r1 + (size_t)l * d.T);
}

// the decoder on the latent in n.w.lat -> n.w.out [T][O]; layer 0's self-attention block must already be in place
void forward(cudaStream_t st, const Net& n) {
  const Dims& d = n.d;
  const size_t TD = n.TD(), TF = (size_t)d.T * d.F;
  dim3 mv(ceil_div(d.D, 8), d.L);
  k_layer_matvec<<<mv, 256, 0, st>>>(n.p + n.y.wv, n.p + n.y.bv, n.y.stride, n.w.lat, 0, d.D, n.w.vc);
  k_layer_matvec<<<mv, 256, 0, st>>>(n.p + n.y.wc, n.p + n.y.bc, n.y.stride, n.w.vc, d.D, d.D, n.w.cvec);
  for (int l = 0; l < d.L; ++l) {
    if (l > 0) self_attn_fwd(st, n, l, n.w.y3 + (l - 1) * TD);
    ln_fwd(st, n, n.w.y1 + l * TD, nullptr, n.w.cvec + (size_t)l * d.D, n.lp(l, n.y.g2), n.lp(l, n.y.be2),
           n.w.y2 + l * TD, n.w.xh2 + l * TD, n.w.r2 + (size_t)l * d.T);
    gemm<true, 1>(st, n.w.y2 + l * TD, d.D, n.lp(l, n.y.w1), d.D, n.lp(l, n.y.b1), nullptr, n.w.g + l * TF, d.F,
                  n.w.u + l * TF, d.T, d.F, d.D);
    gemm<true, 0>(st, n.w.g + l * TF, d.F, n.lp(l, n.y.w2), d.F, n.lp(l, n.y.b2), nullptr, n.w.f + l * TD, d.D, nullptr,
                  d.T, d.D, d.F);
    ln_fwd(st, n, n.w.y2 + l * TD, n.w.f + l * TD, nullptr, n.lp(l, n.y.g3), n.lp(l, n.y.be3), n.w.y3 + l * TD,
           n.w.xh3 + l * TD, n.w.r3 + (size_t)l * d.T);
  }
  gemm<true, 0>(st, n.w.y3 + (d.L - 1) * TD, d.D, n.p + n.y.wf, d.D, n.p + n.y.bf, nullptr, n.w.out, d.O, nullptr, d.T,
                d.O, d.D);
}

// n.w.dout -> n.w.grad (d loss / d latent)
void backward(cudaStream_t st, const Net& n) {
  const Dims& d = n.d;
  const size_t TD = n.TD(), TF = (size_t)d.T * d.F;
  const int lnb = ceil_div(d.T, 8);
  gemm<false, 0>(st, n.w.dout, d.O, n.p + n.y.wf, d.D, nullptr, nullptr, n.w.dx, d.D, nullptr, d.T, d.D, d.O);
  for (int l = d.L - 1; l >= 0; --l) {
    k_ln_bwd<<<lnb, 256, 0, st>>>(n.w.dx, n.lp(l, n.y.g3), n.w.xh3 + l * TD, n.w.r3 + (size_t)l * d.T, d.T, d.D,
                                  n.w.dz3);
    gemm<false, 2>(st, n.w.dz3, d.D, n.lp(l, n.y.w2), d.F, nullptr, nullptr, n.w.dg, d.F, n.w.u + l * TF, d.T, d.F,
                   d.D);
    gemm<false, 0>(st, n.w.dg, d.F, n.lp(l, n.y.w1), d.D, nullptr, n.w.dz3, n.w.dh2, d.D, nullptr, d.T, d.D, d.F);
    k_ln_bwd<<<lnb, 256, 0, st>>>(n.w.dh2, n.lp(l, n.y.g2), n.w.xh2 + l * TD, n.w.r2 + (size_t)l * d.T, d.T, d.D,
                                  n.w.dz2);
    k_cross_back<<<ceil_div(d.D, 256), 256, 0, st>>>(n.w.dz2, d.T, d.D, n.lp(l, n.y.wc), n.w.wback + (size_t)l * d.D);
    if (l == 0) break;            // layer 0's self-attention block does not depend on the latent
    k_ln_bwd<<<lnb, 256, 0, st>>>(n.w.dz2, n.lp(l, n.y.g1), n.w.xh1 + l * TD, n.w.r1 + (size_t)l * d.T, d.T, d.D,
                                  n.w.dz1);
    gemm<false, 0>(st, n.w.dz1, d.D, n.lp(l, n.y.wo), d.D, nullptr, nullptr, n.w.da, d.D, nullptr, d.T, d.D, d.D);
    k_attn_bwd<<<d.H, 256, attn_bwd_smem(d), st>>>(n.w.qkv + l * 3 * TD, n.w.P + (size_t)l * d.H * d.T * d.T, n.w.da,
                                                    d.T, d.D, d.dh, n.scale, n.w.dqkv);
    gemm<false, 0>(st, n.w.dqkv, 3 * d.D, n.lp(l, n.y.wqkv), d.D, nullptr, n.w.dz1, n.w.dx, d.D, nullptr, d.T, d.D,
                   3 * d.D);
  }
  k_latent_grad<<<ceil_div(d.D, 128), 128, 0, st>>>(n.p + n.y.wv, n.y.stride, n.w.wback, d.L, d.D, n.w.grad);
}

int prepare(const avc_motion_dims* dims, const float* params, const float* pe, void* workspace, size_t workspace_bytes,
            Net* n) {
  if (!dims || !params || !pe || !workspace) return AVC_E_NULL;
  Dims d{dims->latent, dims->n_layers, dims->n_heads, dims->ff, dims->n_frames, dims->n_out, 0};
  if (!dims_ok(d)) return AVC_E_BADCFG;
  d.dh = d.D / d.H;
  if (workspace_bytes < ws_bytes(d)) return AVC_E_SIZE;
  n->d = d;
  n->y = make_layout(d.D, d.F, d.O, d.L);
  n->p = params;
  n->pe = pe;
  n->w = carve(workspace, d, nullptr);
  n->scale = 1.f / sqrtf((float)d.dh);
  AVC_CUDA_TRY(cudaFuncSetAttribute(k_attn_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_fwd_smem(d)));
  AVC_CUDA_TRY(cudaFuncSetAttribute(k_attn_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_bwd_smem(d)));
  return 0;
}

}  // namespace

extern "C" {

int avc_motion_param_count(const avc_motion_dims* dims, int64_t* count) {
  if (!dims || !count) return AVC_E_NULL;
  Dims d{dims->latent, dims->n_layers, dims->n_heads, dims->ff, dims->n_frames, dims->n_out, 0};
  if (!dims_ok(d)) return AVC_E_BADCFG;
  *count = (int64_t)make_layout(d.D, d.F, d.O, d.L).total;
  return 0;
}

int avc_motion_workspace_bytes(const avc_motion_dims* dims, size_t* bytes) {
  if (!dims || !bytes) return AVC_E_NULL;
  Dims d{dims->latent, dims->n_layers, dims->n_heads, dims->ff, dims->n_frames, dims->n_out, 0};
  if (!dims_ok(d)) return AVC_E_BADCFG;
  d.dh = d.D / d.H;
  *bytes = ws_bytes(d);
  return 0;
}

int avc_motion_decode(const avc_motion_dims* dims, const float* params, const float* pe, const float* latent,
                      float* motion_out, void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!latent || !motion_out) return AVC_E_NULL;
  Net n;
  AVC_TRY(prepare(dims, params, pe, workspace, workspace_bytes, &n));
  cudaStream_t st = (cudaStream_t)stream;
  AVC_CUDA_TRY(cudaMemcpyAsync(n.w.lat, latent, sizeof(float) * n.d.D, cudaMemcpyDeviceToDevice, st));
  self_attn_fwd(st, n, 0, pe);
  forward(st, n);
  k_motion_loss<<<1, 1024, 0, st>>>(n.w.out, n.d.T, n.d.O, nullptr, 0, Coef{}, 0.f, motion_out, nullptr, nullptr,
                                    nullptr, nullptr);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_motion_optimize(const avc_motion_dims* dims, const float* params, const float* pe, const float* poses,
                        int32_t n_poses, const float* recon_coef, float delta_coef, float lr, float beta1, float beta2,
                        float eps, int32_t n_iter, const float* latent_init, float* latent_out, float* motion_out,
                        float* loss_out, float* grad_out, void* workspace, size_t workspace_bytes,
                        avc_stream_t stream) {
  if (!poses || !recon_coef || !latent_init || !latent_out || !motion_out) return AVC_E_NULL;
  if (n_poses < 1 || n_poses > kMaxCand || n_iter < 1 || !(delta_coef >= 0.f)) return AVC_E_BADCFG;
  Net n;
  AVC_TRY(prepare(dims, params, pe, workspace, workspace_bytes, &n));
  Coef coef{};
  for (int k = 0; k < n_poses; ++k) coef.c[k] = recon_coef[k];
  const int D = n.d.D;
  // capture on a private stream (the caller's may be the legacy default stream, which cannot be captured), ordered
  // after the caller's earlier work and before its later work by events; the graph and the stream are released
  // asynchronously once the launches complete
  cudaStream_t user = (cudaStream_t)stream, st = nullptr;
  cudaEvent_t ev_in = nullptr, ev_out = nullptr;
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  int rc = 0;
  auto fail = [&](cudaError_t e) { if (!rc && e != cudaSuccess) rc = (int)e; return rc != 0; };
  if (fail(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking)) ||
      fail(cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming)) ||
      fail(cudaEventCreateWithFlags(&ev_out, cudaEventDisableTiming)) || fail(cudaEventRecord(ev_in, user)) ||
      fail(cudaStreamWaitEvent(st, ev_in, 0)))
    goto done;
  {
    const float lr_state[4] = {0.f, lr, 0.f, 0.f};
    fail(cudaMemcpyAsync(n.w.lat, latent_init, sizeof(float) * D, cudaMemcpyDeviceToDevice, st));
    fail(cudaMemsetAsync(n.w.m1, 0, sizeof(float) * D, st));
    fail(cudaMemsetAsync(n.w.m2, 0, sizeof(float) * D, st));
    fail(cudaMemsetAsync(n.w.dout, 0, sizeof(float) * n.d.T * n.d.O, st));
    fail(cudaMemcpyAsync(n.w.state, lr_state, sizeof(lr_state), cudaMemcpyHostToDevice, st));
    if (rc) goto done;
    self_attn_fwd(st, n, 0, pe);
    if (fail(cudaGetLastError())) goto done;
  }
  if (fail(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal))) goto done;
  forward(st, n);
  k_motion_loss<<<1, 1024, 0, st>>>(n.w.out, n.d.T, n.d.O, poses, n_poses, coef, delta_coef, motion_out, n.w.g6,
                                    n.w.dout, loss_out, n.w.state);
  backward(st, n);
  rc = avc_adam_step_dev(n.w.lat, n.w.grad, n.w.m1, n.w.m2, D, n.w.state, beta1, beta2, eps, 1.f, st);
  {
    const cudaError_t e = cudaStreamEndCapture(st, &graph);
    if (rc || fail(e)) goto done;
  }
  if (fail(cudaGraphInstantiate(&exec, graph, 0))) goto done;
  for (int i = 0; i < n_iter; ++i)
    if (fail(cudaGraphLaunch(exec, st))) goto done;
  if (fail(cudaMemcpyAsync(latent_out, n.w.lat, sizeof(float) * D, cudaMemcpyDeviceToDevice, st))) goto done;
  if (grad_out && fail(cudaMemcpyAsync(grad_out, n.w.grad, sizeof(float) * D, cudaMemcpyDeviceToDevice, st))) goto done;
  fail(cudaEventRecord(ev_out, st)) || fail(cudaStreamWaitEvent(user, ev_out, 0));
done:
  if (exec) cudaGraphExecDestroy(exec);
  if (graph) cudaGraphDestroy(graph);
  if (ev_in) cudaEventDestroy(ev_in);
  if (ev_out) cudaEventDestroy(ev_out);
  if (st) cudaStreamDestroy(st);
  return rc;
}

int avc_motion_clip_init(const avc_motion_dims* dims, const float* params, const float* pe, const float* latent_init,
                         float lr, void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!latent_init) return AVC_E_NULL;
  Net n;
  AVC_TRY(prepare(dims, params, pe, workspace, workspace_bytes, &n));
  cudaStream_t st = (cudaStream_t)stream;
  const float lr_state[4] = {0.f, lr, 0.f, 0.f};
  AVC_CUDA_TRY(cudaMemcpyAsync(n.w.lat, latent_init, sizeof(float) * n.d.D, cudaMemcpyDeviceToDevice, st));
  AVC_CUDA_TRY(cudaMemsetAsync(n.w.m1, 0, sizeof(float) * n.d.D, st));
  AVC_CUDA_TRY(cudaMemsetAsync(n.w.m2, 0, sizeof(float) * n.d.D, st));
  AVC_CUDA_TRY(cudaMemsetAsync(n.w.dout, 0, sizeof(float) * n.d.T * n.d.O, st));
  AVC_CUDA_TRY(cudaMemcpyAsync(n.w.state, lr_state, sizeof(lr_state), cudaMemcpyHostToDevice, st));
  self_attn_fwd(st, n, 0, pe);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_motion_clip_forward(const avc_motion_dims* dims, const float* params, const float* pe, float* motion_out,
                            void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!motion_out) return AVC_E_NULL;
  Net n;
  AVC_TRY(prepare(dims, params, pe, workspace, workspace_bytes, &n));
  cudaStream_t st = (cudaStream_t)stream;
  forward(st, n);
  k_motion_loss<<<1, 1024, 0, st>>>(n.w.out, n.d.T, n.d.O, nullptr, 0, Coef{}, 0.f, motion_out, nullptr, nullptr,
                                    nullptr, nullptr);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_motion_clip_select(const float* motion, int32_t n_frames, int32_t clip_num_part, float clip_coef,
                           const int32_t* st_idx, int32_t n_rows, float* pose_out, int32_t* frame_out,
                           float* weight_out, avc_stream_t stream) {
  if (!motion || !st_idx || !pose_out || !frame_out || !weight_out) return AVC_E_NULL;
  if (n_frames < 1 || clip_num_part < 1 || clip_num_part > n_frames || n_rows < 1 || n_rows > kMaxT ||
      !(clip_coef >= 0.f))
    return AVC_E_BADCFG;
  k_motion_clip_select<<<ceil_div(n_rows * kPose, 256), 256, 0, (cudaStream_t)stream>>>(
      motion, n_frames, clip_num_part, clip_coef, st_idx, n_rows, pose_out, frame_out, weight_out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_motion_clip_backward(const avc_motion_dims* dims, const float* params, const float* pe, const float* poses,
                             int32_t n_poses, const float* recon_coef, float delta_coef, int32_t n_rows,
                             const int32_t* frame, const float* weight, const float* pose_grad, const float* pose_loss,
                             float beta1, float beta2, float eps, float* motion_out, float* loss_out, float* grad_out,
                             void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!poses || !recon_coef || !frame || !weight || !pose_grad || !pose_loss || !motion_out) return AVC_E_NULL;
  if (n_poses < 1 || n_poses > kMaxCand || n_rows < 1 || n_rows > kMaxT || !(delta_coef >= 0.f)) return AVC_E_BADCFG;
  Net n;
  AVC_TRY(prepare(dims, params, pe, workspace, workspace_bytes, &n));
  Coef coef{};
  for (int k = 0; k < n_poses; ++k) coef.c[k] = recon_coef[k];
  cudaStream_t st = (cudaStream_t)stream;
  k_motion_loss<<<1, 1024, 0, st>>>(n.w.out, n.d.T, n.d.O, poses, n_poses, coef, delta_coef, motion_out, n.w.g6,
                                    n.w.dout, loss_out, n.w.state);
  k_motion_clip_grad<<<ceil_div(n_rows * kJoints, 128), 128, 0, st>>>(n.w.out, n.d.O, frame, weight, n_rows,
                                                                      pose_grad, pose_loss, n.w.dout, loss_out,
                                                                      n.w.state);
  backward(st, n);
  if (grad_out)
    AVC_CUDA_TRY(cudaMemcpyAsync(grad_out, n.w.grad, sizeof(float) * n.d.D, cudaMemcpyDeviceToDevice, st));
  AVC_TRY(avc_adam_step_dev(n.w.lat, n.w.grad, n.w.m1, n.w.m2, n.d.D, n.w.state, beta1, beta2, eps, 1.f, st));
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_motion_clip_latent(const avc_motion_dims* dims, const float* params, const float* pe, float* latent_out,
                           void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!latent_out) return AVC_E_NULL;
  Net n;
  AVC_TRY(prepare(dims, params, pe, workspace, workspace_bytes, &n));
  AVC_CUDA_TRY(cudaMemcpyAsync(latent_out, n.w.lat, sizeof(float) * n.d.D, cudaMemcpyDeviceToDevice,
                               (cudaStream_t)stream));
  return 0;
}

}  // extern "C"
