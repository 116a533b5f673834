// avc_pose.cu -- AvatarAnimate's pose stage (models/pose_generation.py, general.mode = pose): candidate SMPL body poses
// from a text prompt, scored by CLIP on textured renders.
//
//   avc_vposer_decode          VPoser 2.x decode: decoder_net (Linear, LeakyReLU, Linear, LeakyReLU, Linear) then the
//                              6D -> matrix (Gram-Schmidt) -> quaternion -> axis-angle tail (matrot2aa), one kernel per
//                              tile of rows
//   avc_vposer_decode_bwd      its backward, d loss / d z from d loss / d pose_body: the forward recomputed bit for bit,
//                              the matrot2aa tail's Jacobian by forward-mode duals, then the three Linear / LeakyReLU
//                              input gradients, one kernel per tile of rows
//   avc_realnvp_pack           the coupling nets' weights transposed for avc_realnvp_decode, once per checkpoint
//   avc_realnvp_decode         VPoserRealNVP.decode (:233-240): the 8 conditional coupling blocks, the text feature folded
//                              into each first linear's bias once per call, the whole chain in one kernel per tile of rows
//   avc_smpl_pose_batch        smplx SMPL with zero betas for B body poses: pose blend shapes, kinematic chain, skinning;
//                              each row is what avc_lbs_fwd computes for it (both pose through avc_smpl.cuh)
//   avc_raster_textured_batch  render.py:10-39's renders of B meshes from A eyes per group of rows, one launch per pass
//                              for the whole batch; each image is what avc_raster_textured makes of it
//   avc_cosine_topk            F.cosine_similarity of N rows against one vector + torch.topk (VPoserCodebook :322-324)
//   avc_pose_suppress          VPoserCodebook.suppress_duplicated_poses (:304-317)
//   avc_pose_score             get_pose_feature's mean over the cameras, calculate_pose_score's cosine, get_pose's
//                              per-batch argmax (:88-89, 94, 273-274)
#include <cfloat>
#include <type_traits>
#include <vector>

#include "avc_common.cuh"
#include "avc_dual.cuh"
#include "avc_raster.cuh"
#include "avc_smpl.cuh"

using namespace avc;

namespace {

constexpr float kLeaky = 0.01f;      // nn.LeakyReLU() default slope
constexpr int kVpRows = 8;           // VPoser rows per CTA
constexpr int kVpMaxH = 512;
constexpr int kVpMaxL = 64;
constexpr int kVpMaxOut = 192;       // 6 x up to 32 joints
constexpr int kNvpRows = 16;         // RealNVP rows per CTA
constexpr int kNvpMaxD = 32;
constexpr int kNvpMaxH = 256;
constexpr int kNvpMaxBlocks = 16;
constexpr int kMaxCams = 16;
constexpr int kSupMax = 64;
constexpr int kSupMaxD = 96;

// Wt[k][n] = W[n][col0 + k] for k < K  (W row-major with leading dimension ldw)
__global__ void k_transpose(const float* __restrict__ W, int N, int K, int ldw, int col0, float* __restrict__ Wt) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * K) return;
  int k = i / N, n = i - k * N;
  Wt[i] = W[(size_t)n * ldw + col0 + k];
}

// out[r][j] = act(sum_k in[r][k] Wt[k][j] + bias[j]) for ROWS rows held in shared memory; act 0 none, 1 LeakyReLU,
// 2 tanh.  Threads stride over j; each weight is read once per CTA (coalesced along j).
template <int ROWS>
__device__ __forceinline__ void dense_rows(const float* in, int ldi, int K, const float* __restrict__ Wt, int N,
                                           const float* __restrict__ bias, int act, float* out, int ldo) {
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    float acc[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) acc[r] = 0.f;
    for (int k = 0; k < K; ++k) {
      const float w = Wt[(size_t)k * N + j];
#pragma unroll
      for (int r = 0; r < ROWS; ++r) acc[r] = fmaf(in[r * ldi + k], w, acc[r]);
    }
    const float b = bias[j];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      float v = acc[r] + b;
      if (act == 1) v = v > 0.f ? v : kLeaky * v;
      else if (act == 2) v = tanhf(v);
      out[r * ldo + j] = v;
    }
  }
}

// ---------------------------------------------------------------- VPoser decode
// ContinousRotReprDecoder + matrot2aa (torchgeometry rotation_matrix_to_quaternion / quaternion_to_angle_axis) of one
// joint: x[6] read as a [3][2] matrix, columns a = (x0, x2, x4), c = (x1, x3, x5).  S = float gives the values and
// records each branch taken in br; S = Dual (avc_dual.cuh) gives one column of the Jacobian and takes the branches
// recorded in br, so the backward differentiates exactly the branches of the forward whose pose was rendered, whatever
// the duals' value arithmetic would round to.  The gradient is autograd's on the branch taken: F.normalize's clamp
// passes none where it is active, and torchgeometry's masked quaternion carries gradient only from its selected
// branch, 0.5 / sqrt(t) included.  At an exact identity rotation (s2 = 0) torch's backward is NaN (sqrt's backward at
// 0); the duals give the finite k = 2 branch's derivative there, a point no test compares.
template <class S>
__device__ __forceinline__ void rot6d_to_aa(const S* x, S* aa, float* rm, unsigned& br) {
  constexpr bool kRecord = std::is_same<S, float>::value;
  if (kRecord) br = 0u;
  auto take = [&br](unsigned bit, bool cond) {
    if (kRecord) {
      if (cond) br |= bit;
      return cond;
    }
    return (br & bit) != 0u;
  };
  S a[3] = {x[0], x[2], x[4]}, c[3] = {x[1], x[3], x[5]};
  const S la = dsqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
  const S na = take(1u, val(la) >= 1e-12f) ? la : konst<S>(1e-12f);            // F.normalize
  S b1[3] = {a[0] / na, a[1] / na, a[2] / na};
  S dot = b1[0] * c[0] + b1[1] * c[1] + b1[2] * c[2];
  S u[3] = {c[0] - dot * b1[0], c[1] - dot * b1[1], c[2] - dot * b1[2]};
  const S lu = dsqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
  const S nu = take(2u, val(lu) >= 1e-12f) ? lu : konst<S>(1e-12f);
  S b2[3] = {u[0] / nu, u[1] / nu, u[2] / nu};
  S b3[3] = {b1[1] * b2[2] - b1[2] * b2[1], b1[2] * b2[0] - b1[0] * b2[2], b1[0] * b2[1] - b1[1] * b2[0]};
  // R = stack([b1, b2, b3], -1): R[i][j] = b_j[i]
  S R[9] = {b1[0], b2[0], b3[0], b1[1], b2[1], b3[1], b1[2], b2[2], b3[2]};
  if (rm)
#pragma unroll
    for (int i = 0; i < 9; ++i) rm[i] = val(R[i]);
  // rmat_t = R^T: m(i, j) = R[j][i]
#define M(i, j) R[(j) * 3 + (i)]
  S q[4], t;
  if (take(4u, val(M(2, 2)) < 1e-6f)) {
    if (take(8u, val(M(0, 0)) > val(M(1, 1)))) {
      t = 1.f + M(0, 0) - M(1, 1) - M(2, 2);
      q[0] = M(1, 2) - M(2, 1); q[1] = t; q[2] = M(0, 1) + M(1, 0); q[3] = M(2, 0) + M(0, 2);
    } else {
      t = 1.f - M(0, 0) + M(1, 1) - M(2, 2);
      q[0] = M(2, 0) - M(0, 2); q[1] = M(0, 1) + M(1, 0); q[2] = t; q[3] = M(1, 2) + M(2, 1);
    }
  } else {
    if (take(16u, val(M(0, 0)) < -val(M(1, 1)))) {
      t = 1.f - M(0, 0) - M(1, 1) + M(2, 2);
      q[0] = M(0, 1) - M(1, 0); q[1] = M(2, 0) + M(0, 2); q[2] = M(1, 2) + M(2, 1); q[3] = t;
    } else {
      t = 1.f + M(0, 0) + M(1, 1) + M(2, 2);
      q[0] = t; q[1] = M(1, 2) - M(2, 1); q[2] = M(2, 0) - M(0, 2); q[3] = M(0, 1) - M(1, 0);
    }
  }
#undef M
  const S st = dsqrt(t);
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = (q[i] / st) * 0.5f;
  const S s2 = q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  const S s = dsqrt(s2), co = q[0];
  const S two_theta = 2.f * (take(32u, val(co) < 0.f) ? datan2(-s, -co) : datan2(s, co));
  const S k = take(64u, val(s2) > 0.f) ? two_theta / s : konst<S>(2.f);
  aa[0] = q[1] * k; aa[1] = q[2] * k; aa[2] = q[3] * k;
}

struct VpWeights {
  const float *w1t, *b1, *w2t, *b2, *w3t, *b3;   // transposed [K][N] copies in the workspace, biases as given
};

// decoder_net of the kVpRows rows from row0 (rows past B read as 0) into shared memory: sh1 / sh2 the two LeakyReLU
// outputs, so the 6 n_joints outputs.  k_vposer_decode and k_vposer_decode_bwd both run this, so the backward sees
// the forward's bits.
__device__ __forceinline__ void vposer_decoder_rows(const float* __restrict__ z, int B, int L, int H, int O,
                                                    const VpWeights& w, int row0, float* sz, float* sh1, float* sh2,
                                                    float* so) {
  for (int i = threadIdx.x; i < kVpRows * L; i += blockDim.x) {
    const int r = i / L, row = row0 + r;
    sz[i] = row < B ? z[(size_t)row * L + (i - r * L)] : 0.f;
  }
  __syncthreads();
  dense_rows<kVpRows>(sz, L, L, w.w1t, H, w.b1, 1, sh1, H);       // decoder_net.0 + LeakyReLU (Dropout: eval)
  __syncthreads();
  dense_rows<kVpRows>(sh1, H, H, w.w2t, H, w.b2, 1, sh2, H);      // decoder_net.3 + LeakyReLU
  __syncthreads();
  dense_rows<kVpRows>(sh2, H, H, w.w3t, O, w.b3, 0, so, O);       // decoder_net.5
  __syncthreads();
}

__global__ void __launch_bounds__(256)
k_vposer_decode(const float* __restrict__ z, int B, int L, int H, int NJ, VpWeights w, float* __restrict__ pose_out,
                float* __restrict__ rotmat_out) {
  __shared__ float sz[kVpRows * kVpMaxL];
  __shared__ float sh1[kVpRows * kVpMaxH];
  __shared__ float sh2[kVpRows * kVpMaxH];
  __shared__ float so[kVpRows * kVpMaxOut];
  const int row0 = blockIdx.x * kVpRows, O = NJ * 6;
  vposer_decoder_rows(z, B, L, H, O, w, row0, sz, sh1, sh2, so);
  for (int i = threadIdx.x; i < kVpRows * NJ; i += blockDim.x) {
    const int r = i / NJ, j = i - r * NJ, row = row0 + r;
    if (row >= B) continue;
    float aa[3];
    unsigned br;
    rot6d_to_aa(so + r * O + j * 6, aa, rotmat_out ? rotmat_out + ((size_t)row * NJ + j) * 9 : nullptr, br);
    float* p = pose_out + ((size_t)row * NJ + j) * 3;
    p[0] = aa[0]; p[1] = aa[1]; p[2] = aa[2];
  }
}

// out[r][k] = sum_n g[r][n] W[n][k] for ROWS rows in shared memory: the input gradient of a Linear whose weight W
// [N][K] is in nn.Linear's layout, read coalesced along k.  With leaky, out holds that Linear's LeakyReLU output on
// entry, whose sign is its input's, and the product is scaled by LeakyReLU's derivative there (1 above 0, else 0.01,
// as torch's backward takes it at 0) in place.
template <int ROWS>
__device__ __forceinline__ void dense_t_rows(const float* g, int ldg, int N, const float* __restrict__ W, int K,
                                             bool leaky, float* out, int ldo) {
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    float acc[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) acc[r] = 0.f;
    for (int n = 0; n < N; ++n) {
      const float w = W[(size_t)n * K + k];
#pragma unroll
      for (int r = 0; r < ROWS; ++r) acc[r] = fmaf(g[r * ldg + n], w, acc[r]);
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      float v = acc[r];
      if (leaky && !(out[r * ldo + k] > 0.f)) v *= kLeaky;
      out[r * ldo + k] = v;
    }
  }
}

// d loss / d z of the kVpRows rows from row0 given d loss / d pose_body g_pose [B][NJ][3]: the forward recomputed by
// vposer_decoder_rows, then per joint g6 = J^T g_aa (J [3][6] from six dual passes of rot6d_to_aa), then
// W3^T g6 . leaky'(pre2), W2^T . leaky'(pre1), W1^T, each in place over the forward's shared buffers.  pose_out, when
// given, receives the recomputed pose, bit for bit k_vposer_decode's.
__global__ void __launch_bounds__(256)
k_vposer_decode_bwd(const float* __restrict__ z, int B, int L, int H, int NJ, VpWeights w, const float* __restrict__ W1,
                    const float* __restrict__ W2, const float* __restrict__ W3, const float* __restrict__ g_pose,
                    float* __restrict__ g_z, float* __restrict__ pose_out) {
  __shared__ float sz[kVpRows * kVpMaxL];
  __shared__ float sh1[kVpRows * kVpMaxH];
  __shared__ float sh2[kVpRows * kVpMaxH];
  __shared__ float so[kVpRows * kVpMaxOut];
  const int row0 = blockIdx.x * kVpRows, O = NJ * 6;
  vposer_decoder_rows(z, B, L, H, O, w, row0, sz, sh1, sh2, so);
  for (int i = threadIdx.x; i < kVpRows * NJ; i += blockDim.x) {
    const int r = i / NJ, j = i - r * NJ, row = row0 + r;
    float* x = so + r * O + j * 6;
    float g6[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (row < B) {
      float xv[6], aa[3];
#pragma unroll
      for (int c = 0; c < 6; ++c) xv[c] = x[c];
      unsigned br;
      rot6d_to_aa(xv, aa, nullptr, br);
      const size_t o = ((size_t)row * NJ + j) * 3;
      if (pose_out) { pose_out[o] = aa[0]; pose_out[o + 1] = aa[1]; pose_out[o + 2] = aa[2]; }
      const float ga[3] = {g_pose[o], g_pose[o + 1], g_pose[o + 2]};
#pragma unroll 1
      for (int i6 = 0; i6 < 6; ++i6) {
        Dual xd[6], ad[3];
#pragma unroll
        for (int c = 0; c < 6; ++c) xd[c] = Dual{xv[c], c == i6 ? 1.f : 0.f};
        rot6d_to_aa(xd, ad, nullptr, br);
        g6[i6] = fmaf(ga[0], ad[0].d, fmaf(ga[1], ad[1].d, ga[2] * ad[2].d));
      }
    }
#pragma unroll
    for (int c = 0; c < 6; ++c) x[c] = g6[c];
  }
  __syncthreads();
  dense_t_rows<kVpRows>(so, O, O, W3, H, true, sh2, H);          // through decoder_net.5 and the LeakyReLU at 4
  __syncthreads();
  dense_t_rows<kVpRows>(sh2, H, H, W2, H, true, sh1, H);         // through decoder_net.3 and the LeakyReLU at 1
  __syncthreads();
  dense_t_rows<kVpRows>(sh1, H, H, W1, L, false, sz, L);         // through decoder_net.0
  __syncthreads();
  for (int i = threadIdx.x; i < kVpRows * L; i += blockDim.x) {
    const int r = i / L, row = row0 + r;
    if (row < B) g_z[(size_t)row * L + (i - r * L)] = sz[i];
  }
}

// ---------------------------------------------------------------- VPoser encode (.mean)
// eval-mode BatchNorm1d of ROWS rows in place: (x - running_mean) * (1 / sqrt(running_var + eps)) * weight + bias;
// bn = (weight, bias, running_mean, running_var), each [n]
__device__ __forceinline__ void batchnorm_rows(float* x, int rows, int n, const float* __restrict__ bn) {
  for (int i = threadIdx.x; i < rows * n; i += blockDim.x) {
    const int c = i % n;
    const float invstd = 1.f / sqrtf(bn[3 * n + c] + 1e-5f);
    x[i] = (x[i] - bn[2 * n + c]) * invstd * bn[c] + bn[n + c];
  }
}

struct VpEncWeights {
  const float *bn1, *w1t, *b1, *bn2, *w2t, *b2, *w3t, *b3, *wmt, *bm;
};

__global__ void __launch_bounds__(256)
k_vposer_encode(const float* __restrict__ x, int B, int NI, int H, int L, VpEncWeights w, float* __restrict__ mu_out) {
  __shared__ float sx[kVpRows * kVpMaxOut];
  __shared__ float sh1[kVpRows * kVpMaxH];
  __shared__ float sh2[kVpRows * kVpMaxH];
  const int row0 = blockIdx.x * kVpRows;
  for (int i = threadIdx.x; i < kVpRows * NI; i += blockDim.x) {
    const int r = i / NI, row = row0 + r;
    sx[i] = row < B ? x[(size_t)row * NI + (i - r * NI)] : 0.f;
  }
  __syncthreads();
  batchnorm_rows(sx, kVpRows, NI, w.bn1);                          // encoder_net.1
  __syncthreads();
  dense_rows<kVpRows>(sx, NI, NI, w.w1t, H, w.b1, 1, sh1, H);      // encoder_net.2 + LeakyReLU
  __syncthreads();
  batchnorm_rows(sh1, kVpRows, H, w.bn2);                          // encoder_net.4 (Dropout: eval)
  __syncthreads();
  dense_rows<kVpRows>(sh1, H, H, w.w2t, H, w.b2, 0, sh2, H);       // encoder_net.6
  __syncthreads();
  dense_rows<kVpRows>(sh2, H, H, w.w3t, H, w.b3, 0, sh1, H);       // encoder_net.7
  __syncthreads();
  dense_rows<kVpRows>(sh1, H, H, w.wmt, L, w.bm, 0, sh2, L);       // encoder_net.8.mu
  __syncthreads();
  for (int i = threadIdx.x; i < kVpRows * L; i += blockDim.x) {
    const int r = i / L, row = row0 + r;
    if (row < B) mu_out[(size_t)row * L + (i - r * L)] = sh2[i];
  }
}

// ---------------------------------------------------------------- RealNVP decode
// the transposed weights, packed once per checkpoint, per coupling net (block i, net n: 0 = s, 1 = t): w1t [D][H]
// (the x columns of the first linear), w2t [H][H], w3t [H][D]
struct NvpPack {
  size_t w1t, w2t, w3t, stride;
};

__host__ __device__ inline NvpPack nvp_pack(int D, int H) {
  NvpPack p;
  p.w1t = 0;
  p.w2t = p.w1t + (size_t)D * H;
  p.w3t = p.w2t + (size_t)H * H;
  p.stride = p.w3t + (size_t)H * D;
  return p;
}

// params per net: W1 [H][D+E], b1 [H], W2 [H][H], b2 [H], W3 [D][H], b3 [D]
__host__ __device__ inline size_t nvp_param_stride(int D, int E, int H) {
  return (size_t)H * (D + E) + H + (size_t)H * H + H + (size_t)D * H + D;
}

// net blockIdx.y: the three transposes into its slot of the pack
__global__ void k_realnvp_pack(const float* __restrict__ params, int D, int E, int H, float* __restrict__ pack) {
  const float* W1 = params + (size_t)blockIdx.y * nvp_param_stride(D, E, H);
  const float* W2 = W1 + (size_t)H * (D + E) + H;
  const float* W3 = W2 + (size_t)H * H + H;
  const NvpPack pk = nvp_pack(D, H);
  float* P = pack + (size_t)blockIdx.y * pk.stride;
  const int total = max(H * H, D * H);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int k = i / H, n = i - k * H;
    if (i < H * H) P[pk.w2t + i] = W2[(size_t)n * H + k];    // w2t[k][n] = W2[n][k]
    if (i < D * H) {
      P[pk.w1t + i] = W1[(size_t)n * (D + E) + k];            // w1t[k][n] = W1[n][k], k < D
      const int k3 = i / D, n3 = i - k3 * D;
      P[pk.w3t + i] = W3[(size_t)n3 * H + k3];                // w3t[k][n] = W3[n][k]
    }
  }
}

// c[net][j] = b1[j] + sum_e W1[j][D + e] f[e], one CTA per net
__global__ void k_realnvp_fold(const float* __restrict__ params, const float* __restrict__ f, int D, int E, int H,
                               float* __restrict__ fold) {
  const float* W1 = params + (size_t)blockIdx.x * nvp_param_stride(D, E, H);
  const float* b1 = W1 + (size_t)H * (D + E);
  float* c = fold + (size_t)blockIdx.x * H;
  for (int j = threadIdx.x; j < H; j += blockDim.x) {
    const float* wr = W1 + (size_t)j * (D + E) + D;
    float acc = 0.f;
    for (int e = 0; e < E; ++e) acc = fmaf(wr[e], f[e], acc);
    c[j] = acc + b1[j];
  }
}

__global__ void __launch_bounds__(256)
k_realnvp_decode(const float* __restrict__ z, int B, int D, int E, int H, int nb, const float* __restrict__ params,
                 const float* __restrict__ pack, const float* __restrict__ fold, const float* __restrict__ mask,
                 float* __restrict__ x_out) {
  __shared__ float sx[kNvpRows * kNvpMaxD], sxm[kNvpRows * kNvpMaxD];
  __shared__ float sh1[kNvpRows * kNvpMaxH], sh2[kNvpRows * kNvpMaxH];
  __shared__ float ss[kNvpRows * kNvpMaxD], st[kNvpRows * kNvpMaxD];
  const int row0 = blockIdx.x * kNvpRows;
  for (int i = threadIdx.x; i < kNvpRows * D; i += blockDim.x) {
    const int r = i / D, row = row0 + r;
    sx[i] = row < B ? z[(size_t)row * D + (i - r * D)] : 0.f;
  }
  const NvpPack pk = nvp_pack(D, H);
  const size_t ps = nvp_param_stride(D, E, H);
  for (int blk = 0; blk < nb; ++blk) {
    const float* m = mask + (size_t)blk * D;
    __syncthreads();
    for (int i = threadIdx.x; i < kNvpRows * D; i += blockDim.x) sxm[i] = sx[i] * m[i % D];   // x_ = x * mask
    for (int net = 0; net < 2; ++net) {
      const float* P = pack + (size_t)(blk * 2 + net) * pk.stride;
      const float* W = params + (size_t)(blk * 2 + net) * ps;
      const float* b2 = W + (size_t)H * (D + E) + H + (size_t)H * H;
      const float* b3 = b2 + H + (size_t)D * H;
      __syncthreads();
      dense_rows<kNvpRows>(sxm, D, D, P + pk.w1t, H, fold + (size_t)(blk * 2 + net) * H, 1, sh1, H);
      __syncthreads();
      dense_rows<kNvpRows>(sh1, H, H, P + pk.w2t, H, b2, 1, sh2, H);
      __syncthreads();
      dense_rows<kNvpRows>(sh2, H, H, P + pk.w3t, D, b3, net == 0 ? 2 : 0, net == 0 ? ss : st, D);
    }
    __syncthreads();
    // s, t = net(...) * (1 - mask);  x = x_ + (1 - mask) * (x * exp(s) + t)
    for (int i = threadIdx.x; i < kNvpRows * D; i += blockDim.x) {
      const float om = 1.f - m[i % D];
      const float s = ss[i] * om, t = st[i] * om;
      sx[i] = sxm[i] + om * (sx[i] * expf(s) + t);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kNvpRows * D; i += blockDim.x) {
    const int r = i / D, row = row0 + r;
    if (row < B) x_out[(size_t)row * D + (i - r * D)] = sx[i];
  }
}

// ---------------------------------------------------------------- SMPL for a batch of body poses
struct Orient {
  float r[3];
};

// one warp per pose row, lane j = joint j: batch_rodrigues of (global_orient, body_pose, zeros), the pose feature and
// avc_smpl.cuh's kinematic chain, written per row: A [B][NJ][12], feat [B][(NJ-1)*9]
__global__ void __launch_bounds__(128)
k_pose_chain(const float* __restrict__ body_pose, int P, int B, Orient go, const float* __restrict__ Jg,
             const int* __restrict__ parents, int NJ, float* __restrict__ A_out, float* __restrict__ feat_out) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;                        // warp-uniform
  const int j = lane;
  const bool act = j < NJ;
  float* feat = feat_out + (size_t)b * (NJ - 1) * 9;
  float R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (act) {
    float rv[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int q = (j - 1) * 3 + c;
      rv[c] = j == 0 ? go.r[c] : (q < P ? body_pose[(size_t)b * P + q] : 0.f);
    }
    rodrigues(rv[0], rv[1], rv[2], R);
    if (j >= 1)
#pragma unroll
      for (int i = 0; i < 9; ++i) feat[(j - 1) * 9 + i] = R[i] - ((i % 4 == 0) ? 1.f : 0.f);
  }
  const int par = act ? parents[j] : -1;
  const float Jx = act ? Jg[j * 3] : 0.f, Jy = act ? Jg[j * 3 + 1] : 0.f, Jz = act ? Jg[j * 3 + 2] : 0.f;
  float T[12];
  chain_world(R, j, par, act, Jx, Jy, Jz, T);
  if (act) rel_transform(T, Jx, Jy, Jz, A_out + ((size_t)b * NJ + j) * 12);
}

constexpr int kSkinRows = 8;

struct PostRot {
  float m[9];
  int on;
};

// thread per vertex, kSkinRows pose rows per CTA: the [rows][207] x [207][3V] pose blend contraction (each posedirs
// element read once for all rows, each row's terms summed in k_lbs_skin's order), then the blended transform
__global__ void __launch_bounds__(128)
k_pose_skin(const float* __restrict__ v_template, const float* __restrict__ posedirs, const float* __restrict__ feat,
            const float* __restrict__ A, const float* __restrict__ lbs_weights, int V, int NJ, int NF, int B, PostRot pr,
            float* __restrict__ verts) {
  __shared__ float sA[kSkinRows][NJ_MAX * 12];
  __shared__ float sF[kSkinRows][NJ_MAX * 9];
  const int b0 = blockIdx.y * kSkinRows;
  const int nr = min(kSkinRows, B - b0);
  stage_rows<kSkinRows>(sA, sF, A, feat, b0, nr, NJ, NF);
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  float p[kSkinRows][3];
  pose_blend_rows<kSkinRows>(p, v_template, posedirs, sF, V, NF, v);
#pragma unroll
  for (int r = 0; r < kSkinRows; ++r) {
    if (r >= nr) break;
    float T[12];
    blend_transform(lbs_weights + (size_t)v * NJ, sA[r], NJ, T);
    const float p0 = p[r][0], p1 = p[r][1], p2 = p[r][2];
    float o0 = T[0] * p0 + T[1] * p1 + T[2] * p2 + T[3];
    float o1 = T[4] * p0 + T[5] * p1 + T[6] * p2 + T[7];
    float o2 = T[8] * p0 + T[9] * p1 + T[10] * p2 + T[11];
    if (pr.on) {     // row vector times matrix: o @ m
      const float q0 = o0 * pr.m[0] + o1 * pr.m[3] + o2 * pr.m[6];
      const float q1 = o0 * pr.m[1] + o1 * pr.m[4] + o2 * pr.m[7];
      const float q2 = o0 * pr.m[2] + o1 * pr.m[5] + o2 * pr.m[8];
      o0 = q0; o1 = q1; o2 = q2;
    }
    float* out = verts + ((size_t)(b0 + r) * V + v) * 3;
    out[0] = o0; out[1] = o1; out[2] = o2;
  }
}

// ---------------------------------------------------------------- batched textured render
// images are [A][B] (angle-major); mesh b uses the cameras of its group b / G: cams[(b / G) * A + a]
__global__ void k_project_batch(const float* __restrict__ verts, int V, int B, int G, int A,
                                const LookAtCam* __restrict__ cams, float4* __restrict__ proj) {
  const int img = blockIdx.y, a = img / B, b = img - a * B;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V) return;
  const LookAtCam c = cams[(b / G) * A + a];
  project_look_at(i, verts + (size_t)b * V * 3, c, proj + (size_t)img * V);
}

__global__ void k_raster_batch(const float4* __restrict__ proj, int V, const int* __restrict__ faces, int F, int is,
                               unsigned long long* __restrict__ zbuf) {
  const int img = blockIdx.y;
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  raster_face(f, proj + (size_t)img * V, faces, is, 0.1f, 100.f, zbuf + (size_t)img * is * is);
}

__global__ void k_resolve_batch(const unsigned long long* __restrict__ zbuf, const int* __restrict__ faces,
                                const float* __restrict__ verts, const float4* __restrict__ proj,
                                const float* __restrict__ tex, int R, int V, int B, int G, int A,
                                const LookAtCam* __restrict__ cams, int n, int ss, float* __restrict__ rgb) {
  const int img = blockIdx.y, a = img / B, b = img - a * B;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n * n) return;
  const LookAtCam c = cams[(b / G) * A + a];
  resolve_textured(p, zbuf + (size_t)img * c.is * c.is, faces, verts + (size_t)b * V * 3, proj + (size_t)img * V, tex,
                   R, c, n, ss, rgb + (size_t)img * n * n * 3);
}

// ---------------------------------------------------------------- scores and selection
// one CTA per row: F.cosine_similarity(X[i], y) = sum_j (x_j / max(|x|, eps)) (y_j / max(|y|, eps)), sums in fp64
__global__ void k_rows_cos(const float* __restrict__ X, const float* __restrict__ y, int D, float eps,
                           float* __restrict__ cos_out) {
  __shared__ double red[32];
  const int i = blockIdx.x;
  double xx = 0.0, xy = 0.0, yy = 0.0;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const double a = X[(size_t)i * D + j], b = y[j];
    xx += a * a; xy += a * b; yy += b * b;
  }
  const auto add = [](double u, double v) { return u + v; };
  xx = block_reduce(xx, red, add, 0.0);
  xy = block_reduce(xy, red, add, 0.0);
  yy = block_reduce(yy, red, add, 0.0);
  if (threadIdx.x == 0) cos_out[i] = (float)(xy / (fmax(sqrt(xx), (double)eps) * fmax(sqrt(yy), (double)eps)));
}

// one CTA: k rounds, each the largest key below the previous round's (keys are distinct)
__global__ void __launch_bounds__(1024) k_topk(const float* __restrict__ v, int N, int k, int* __restrict__ idx_out) {
  __shared__ unsigned long long red[32];
  unsigned long long prev = ~0ull;
  for (int r = 0; r < k; ++r) {
    unsigned long long best = 0;
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
      const unsigned long long key = sel_key(v[i], i);
      if (key < prev && key > best) best = key;
    }
    best = block_reduce(best, red, [](unsigned long long x, unsigned long long y) { return x > y ? x : y; }, 0ull);
    if (threadIdx.x == 0) idx_out[r] = sel_index(best);
    prev = best;
  }
}

// one CTA: pairwise mean absolute differences (fp32 differences, fp64 sum, rounded to fp32 like the reference's
// tensor mean), then the greedy pass of suppress_duplicated_poses in list order
__global__ void __launch_bounds__(256)
k_pose_suppress(const float* __restrict__ poses, int P, int Dp, float threshold, int* __restrict__ keep_out,
                int* __restrict__ count_out) {
  __shared__ float sp[kSupMax * kSupMaxD];
  __shared__ float dist[kSupMax][kSupMax];
  __shared__ int kept[kSupMax];
  for (int i = threadIdx.x; i < P * Dp; i += blockDim.x) sp[i] = poses[i];
  __syncthreads();
  for (int t = threadIdx.x; t < P * P; t += blockDim.x) {
    const int i = t / P, j = t - i * P;
    if (j >= i) continue;
    double s = 0.0;
    for (int d = 0; d < Dp; ++d) s += (double)fabsf(sp[i * Dp + d] - sp[j * Dp + d]);
    dist[i][j] = (float)(s / Dp);
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  int n = 0;
  for (int i = 0; i < P; ++i) {
    float md = 10.f;
    for (int q = 0; q < n; ++q) md = fminf(dist[i][kept[q]], md);
    if (n == 0 || md > threshold) kept[n++] = i;
  }
  for (int q = 0; q < n; ++q) keep_out[q] = kept[q];
  *count_out = n;
}

// one CTA per pose b: feature = mean_a emb[a][b] (fp64 sum / A, rounded), score = cosine(feature, text) (eps 1e-8),
// then the group's first argmax through a 64-bit atomicMax
__global__ void k_pose_score(const float* __restrict__ emb, int A, int B, int Dm, const float* __restrict__ text, int G,
                             float* __restrict__ score_out, unsigned long long* __restrict__ keys) {
  __shared__ double red[32];
  const int b = blockIdx.x;
  double xx = 0.0, xy = 0.0, yy = 0.0;
  for (int j = threadIdx.x; j < Dm; j += blockDim.x) {
    double s = 0.0;
    for (int a = 0; a < A; ++a) s += emb[((size_t)a * B + b) * Dm + j];
    const double f = (float)(s / A), t = text[j];
    xx += f * f; xy += f * t; yy += t * t;
  }
  const auto add = [](double u, double v) { return u + v; };
  xx = block_reduce(xx, red, add, 0.0);
  xy = block_reduce(xy, red, add, 0.0);
  yy = block_reduce(yy, red, add, 0.0);
  if (threadIdx.x == 0) {
    const float sc = (float)(xy / (fmax(sqrt(xx), 1e-8) * fmax(sqrt(yy), 1e-8)));
    score_out[b] = sc;
    atomicMax(keys + b / G, sel_key(sc, b % G));
  }
}

__global__ void k_group_best(const unsigned long long* __restrict__ keys, int n, int* __restrict__ best) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n) best[g] = sel_index(keys[g]);
}

// ================================================================ backward of the pose optimiser's chain
// N values summed over the CTA in a fixed order: warp xor trees, then the warps in index order by thread i < N;
// the totals land in red[i * 32] (red holds N * 32 floats)
template <int N>
__device__ __forceinline__ void block_sum_n(float (&v)[N], float* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int i = 0; i < N; ++i) v[i] = warp_sum(v[i]);
  if (lane == 0)
#pragma unroll
    for (int i = 0; i < N; ++i) red[i * 32 + w] = v[i];
  __syncthreads();
  if (threadIdx.x < N) {
    float s = 0.f;
    for (int k = 0; k < nw; ++k) s += red[threadIdx.x * 32 + k];
    red[threadIdx.x * 32] = s;
  }
  __syncthreads();
}

// ---------------------------------------------------------------- SMPL posing backward
// thread per vertex, kSkinRows rows per CTA: k_pose_skin's p (pose-blended template) and blended transform T again,
// then g_o = post_rot g_v (o @ post_rot is the output), and g_p = T_3x3^T g_o
__global__ void __launch_bounds__(128)
k_pose_skin_bwd(const float* __restrict__ v_template, const float* __restrict__ posedirs, const float* __restrict__ feat,
                const float* __restrict__ A, const float* __restrict__ lbs_weights, int V, int NJ, int NF, int B,
                PostRot pr, const float* __restrict__ g_verts, float* __restrict__ p_out, float* __restrict__ go_out,
                float* __restrict__ gp_out) {
  __shared__ float sA[kSkinRows][NJ_MAX * 12];
  __shared__ float sF[kSkinRows][NJ_MAX * 9];
  const int b0 = blockIdx.y * kSkinRows;
  const int nr = min(kSkinRows, B - b0);
  stage_rows<kSkinRows>(sA, sF, A, feat, b0, nr, NJ, NF);
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  float p[kSkinRows][3];
  pose_blend_rows<kSkinRows>(p, v_template, posedirs, sF, V, NF, v);
#pragma unroll
  for (int r = 0; r < kSkinRows; ++r) {
    if (r >= nr) break;
    float T[12];
    blend_transform(lbs_weights + (size_t)v * NJ, sA[r], NJ, T);
    const size_t o = ((size_t)(b0 + r) * V + v) * 3;
    float g0 = g_verts[o], g1 = g_verts[o + 1], g2 = g_verts[o + 2];
    if (pr.on) {     // q = o @ m  ->  g_o = m g_q
      const float h0 = pr.m[0] * g0 + pr.m[1] * g1 + pr.m[2] * g2;
      const float h1 = pr.m[3] * g0 + pr.m[4] * g1 + pr.m[5] * g2;
      const float h2 = pr.m[6] * g0 + pr.m[7] * g1 + pr.m[8] * g2;
      g0 = h0; g1 = h1; g2 = h2;
    }
    p_out[o] = p[r][0]; p_out[o + 1] = p[r][1]; p_out[o + 2] = p[r][2];
    go_out[o] = g0; go_out[o + 1] = g1; go_out[o + 2] = g2;
    gp_out[o] = T[0] * g0 + T[4] * g1 + T[8] * g2;
    gp_out[o + 1] = T[1] * g0 + T[5] * g1 + T[9] * g2;
    gp_out[o + 2] = T[2] * g0 + T[6] * g1 + T[10] * g2;
  }
}

// CTA (joint j, row b): dA[b][j] = sum_v w_vj g_o(v) [p(v); 1]^T, a 3 x 4 block
__global__ void __launch_bounds__(256)
k_pose_dA(const float* __restrict__ lbs_weights, const float* __restrict__ p, const float* __restrict__ go, int V,
          int NJ, float* __restrict__ dA) {
  __shared__ float red[12 * 32];
  const int j = blockIdx.x, b = blockIdx.y;
  float acc[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) acc[i] = 0.f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    const float w = lbs_weights[(size_t)v * NJ + j];
    if (w == 0.f) continue;
    const size_t o = ((size_t)b * V + v) * 3;
    const float q[4] = {p[o], p[o + 1], p[o + 2], 1.f};
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float wg = w * go[o + r];
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[r * 4 + c] = fmaf(wg, q[c], acc[r * 4 + c]);
    }
  }
  block_sum_n<12>(acc, red);
  if (threadIdx.x < 12) dA[((size_t)b * NJ + j) * 12 + threadIdx.x] = red[threadIdx.x * 32];
}

// CTA (pose feature k, kSkinRows rows): g_feat[b][k] = posedirs[k] . g_p[b] over the 3V entries
__global__ void __launch_bounds__(256)
k_pose_gfeat(const float* __restrict__ posedirs, const float* __restrict__ gp, int V3, int NF, int B,
             float* __restrict__ gfeat) {
  __shared__ float red[kSkinRows * 32];
  const int k = blockIdx.x, b0 = blockIdx.y * kSkinRows;
  const int nr = min(kSkinRows, B - b0);
  float acc[kSkinRows];
#pragma unroll
  for (int r = 0; r < kSkinRows; ++r) acc[r] = 0.f;
  const float* pd = posedirs + (size_t)k * V3;
  for (int i = threadIdx.x; i < V3; i += blockDim.x) {
    const float d = pd[i];
#pragma unroll
    for (int r = 0; r < kSkinRows; ++r)
      if (r < nr) acc[r] = fmaf(d, gp[(size_t)(b0 + r) * V3 + i], acc[r]);
  }
  block_sum_n<kSkinRows>(acc, red);
  if (threadIdx.x < nr) gfeat[(size_t)(b0 + threadIdx.x) * NF + k] = red[threadIdx.x * 32];
}

// one warp per pose row, lane j = joint j: the kinematic chain in reverse (children before parents, each parent
// adding its children's terms in lane order), then batch_rodrigues' backward (the eps inside the norm included)
__global__ void __launch_bounds__(128)
k_pose_chain_bwd(const float* __restrict__ body_pose, int P, int B, const float* __restrict__ Jg,
                 const int* __restrict__ parents, int NJ, const float* __restrict__ A, const float* __restrict__ feat,
                 const float* __restrict__ dA, const float* __restrict__ gfeat, float* __restrict__ g_pose) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;                        // warp-uniform
  const int j = lane;
  const bool act = j < NJ;
  const int NF = (NJ - 1) * 9;
  const int par = act ? parents[j] : -1;
  const int depth = joint_depth(par);
  const int maxd = max_depth(depth);
  // forward values: R_j = feat_j + I, t_j = J_j - J_par, the parent's world rotation P3 = A[par][:, :3]
  float R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {0.f, 0.f, 0.f}, P3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  const float Jx = act ? Jg[j * 3] : 0.f, Jy = act ? Jg[j * 3 + 1] : 0.f, Jz = act ? Jg[j * 3 + 2] : 0.f;
  if (act && j >= 1) {
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = feat[(size_t)b * NF + (j - 1) * 9 + i] + ((i % 4 == 0) ? 1.f : 0.f);
    t[0] = Jx - Jg[par * 3]; t[1] = Jy - Jg[par * 3 + 1]; t[2] = Jz - Jg[par * 3 + 2];
    const float* ap = A + ((size_t)b * NJ + par) * 12;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) P3[r * 3 + c] = ap[r * 4 + c];
  }
  // A = G - [0 | G_3x3 J]:  g_G3 = dA3 - dA_t J^T, g_Gt = dA_t
  float gG[12];
  if (act) {
    const float* d = dA + ((size_t)b * NJ + j) * 12;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float dt = d[r * 4 + 3];
      gG[r * 4 + 0] = d[r * 4 + 0] - dt * Jx;
      gG[r * 4 + 1] = d[r * 4 + 1] - dt * Jy;
      gG[r * 4 + 2] = d[r * 4 + 2] - dt * Jz;
      gG[r * 4 + 3] = dt;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 12; ++i) gG[i] = 0.f;
  }
  // G_j = G_par [R_j | t_j]:  g_Gpar3 += g_G3 R^T + g_Gt t^T, g_Gpar_t += g_Gt
  for (int d = maxd; d >= 1; --d) {
    float cP[12];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
      for (int c = 0; c < 3; ++c)
        cP[r * 4 + c] = gG[r * 4] * R[c * 3] + gG[r * 4 + 1] * R[c * 3 + 1] + gG[r * 4 + 2] * R[c * 3 + 2] +
                        gG[r * 4 + 3] * t[c];
      cP[r * 4 + 3] = gG[r * 4 + 3];
    }
    const bool send = act && depth == d;
    for (int src = 0; src < 32; ++src) {
      const int ps = __shfl_sync(0xffffffffu, send ? par : -1, src);
      float add[12];
#pragma unroll
      for (int i = 0; i < 12; ++i) add[i] = __shfl_sync(0xffffffffu, cP[i], src);
      if (ps == j)
#pragma unroll
        for (int i = 0; i < 12; ++i) gG[i] += add[i];
    }
  }
  if (!act || j == 0) return;
  // G3 = P3 R:  g_R = P3^T g_G3, plus the pose feature's (feat = R - I)
  float gR[9];
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int c = 0; c < 3; ++c)
      gR[k * 3 + c] = P3[k] * gG[c] + P3[3 + k] * gG[4 + c] + P3[6 + k] * gG[8 + c] +
                      gfeat[(size_t)b * NF + (j - 1) * 9 + k * 3 + c];
  float rv[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int q = (j - 1) * 3 + c;
    rv[c] = q < P ? body_pose[(size_t)b * P + q] : 0.f;
  }
  const Rodrigues rq = rodrigues_terms(rv[0], rv[1], rv[2]);
  const float ang = rq.ang, s = rq.s, c = rq.c;
  const float* K = rq.K;
  const float* KK = rq.KK;
  // R = I + s K + (1 - c) K K
  float gs = 0.f, gc = 0.f;
#pragma unroll
  for (int i = 0; i < 9; ++i) { gs += gR[i] * K[i]; gc -= gR[i] * KK[i]; }
  const float omc = 1.f - c;
  float gK[9];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int bb = 0; bb < 3; ++bb) {
      // d(KK) -> g_K += g_KK K^T + K^T g_KK with g_KK = (1 - c) g_R
      float m = 0.f;
#pragma unroll
      for (int k = 0; k < 3; ++k) m += gR[a * 3 + k] * K[bb * 3 + k] + K[k * 3 + a] * gR[k * 3 + bb];
      gK[a * 3 + bb] = s * gR[a * 3 + bb] + omc * m;
    }
  const float gx = gK[7] - gK[5], gy = gK[2] - gK[6], gz = gK[3] - gK[1];
  const float gang = gs * c - gc * s - (gx * rv[0] + gy * rv[1] + gz * rv[2]) / (ang * ang);
  const float ga[3] = {gx, gy, gz};
#pragma unroll
  for (int cc = 0; cc < 3; ++cc) {
    const int q = (j - 1) * 3 + cc;
    if (q < P) g_pose[(size_t)b * P + q] = ga[cc] / ang + gang * (rv[cc] + kRodriguesEps) / ang;
  }
}

// ---------------------------------------------------------------- textured render backward
// per supersample of image img: the lit colour the forward averaged (ss_rgb) and dl = g_ss . unlit sample, this
// supersample's share of the gradient of its face's light (g_ss = g_pixel / ss^2, avg-pool's backward); background 0
__global__ void k_rb_samples(const unsigned long long* __restrict__ zbuf, const int* __restrict__ faces,
                             const float* __restrict__ verts, const float4* __restrict__ proj,
                             const float* __restrict__ tex, int R, int V, int B, int G, int A,
                             const LookAtCam* __restrict__ cams, int n, int ss, const float* __restrict__ g_rgb,
                             float* __restrict__ ss_rgb, float* __restrict__ dl) {
  const int img = blockIdx.y, a = img / B, b = img - a * B;
  const LookAtCam c = cams[(b / G) * A + a];
  const int is = c.is;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= is * is) return;
  const int row = q / is, xi = q - row * is;
  const size_t o = (size_t)img * is * is + q;
  const unsigned long long zb = zbuf[o];
  float* out = ss_rgb + o * 3;
  if (zb == ~0ull) {
    out[0] = 0.f; out[1] = 0.f; out[2] = 0.f;
    dl[o] = 0.f;
    return;
  }
  const int f = (int)(zb & 0xffffffffu);
  const float zp = __uint_as_float((unsigned)(zb >> 32));
  float col[3], light;
  textured_sample(row, xi, f, zp, faces, verts + (size_t)b * V * 3, proj + (size_t)img * V, tex, R, c, col, &light);
  out[0] = col[0] * light; out[1] = col[1] * light; out[2] = col[2] * light;
  const float* g = g_rgb + ((size_t)img * n * n + (size_t)(row / ss) * n + xi / ss) * 3;
  const float inv = 1.f / (float)(ss * ss);
  dl[o] = (g[0] * inv) * col[0] + (g[1] * inv) * col[1] + (g[2] * inv) * col[2];
}

__device__ __forceinline__ int face_at(const unsigned long long* zbuf, size_t i) {
  return (int)(unsigned)(zbuf[i] & 0xffffffffu);      // background ~0 -> -1
}

// neural_renderer's backward_pixel_map of face f in one image (rgb only, fp32), its corners in the winding of the
// drawn copy: pxy [3][2] their NDC x, y; adds d loss / d (x, y) of each corner to gxy.  Pixel coordinates and the
// crossings are rounded op by op (no contraction), so an fp32 restatement makes the same pixel choices.
__device__ __forceinline__ void edge_sweep(const float (&pxy)[3][2], int f, const unsigned long long* __restrict__ zbuf,
                           const float* __restrict__ rgb, const float* __restrict__ g_rgb, int is, int n, int ss,
                           float (&gxy)[3][2]) {
  const float eps = 1e-4f;                   // neural_renderer's DEFAULT_EPS
  const float inv = 1.f / (float)(ss * ss);
  const float fis = (float)is;
  float pp[3][2];
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int d = 0; d < 2; ++d) pp[k][d] = __fmul_rn(0.5f, __fadd_rn(__fadd_rn(__fmul_rn(pxy[k][d], fis), fis), -1.f));
  auto gpix = [&](size_t i) {                // g at supersample i = (row, col)
    const int row = (int)(i / is), col = (int)(i - (size_t)row * is);
    return g_rgb + ((size_t)(row / ss) * n + col / ss) * 3;
  };
  // unrolled, so that every index into pp and gxy is a constant (no local memory)
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    const int pi[3] = {e, (e + 1) % 3, (e + 2) % 3};
#pragma unroll
    for (int axis = 0; axis < 2; ++axis) {
      float p[3][2];
#pragma unroll
      for (int k = 0; k < 3; ++k) { p[k][0] = pp[pi[k]][axis]; p[k][1] = pp[pi[k]][1 - axis]; }
      if (p[0][0] == p[1][0]) continue;      // neural_renderer divides 0 by 0 here
      int direction = p[0][0] < p[1][0] ? -1 : 1;
      if (axis == 1) direction = -direction;
      const float span = __fadd_rn(p[1][0], -p[0][0]);
      const float slope = __fdiv_rn(__fadd_rn(p[1][1], -p[0][1]), span);
      const int d0_from = max((int)ceilf(fminf(p[0][0], p[1][0])), 0);
      const int d0_to = min((int)floorf(fmaxf(p[0][0], p[1][0])), is - 1);
      for (int d0 = d0_from; d0 <= d0_to; ++d0) {
        const float fd0 = (float)d0;
        const float d1_cross = __fadd_rn(__fmul_rn(slope, __fadd_rn(fd0, -p[0][0])), p[0][1]);
        const int d1_in = direction > 0 ? (int)floorf(d1_cross) : (int)ceilf(d1_cross);
        const int d1_out = d1_in + direction;
        if (d1_in < 0 || d1_in >= is || d1_out < 0 || d1_out >= is) continue;
        auto pix = [&](int d1) {
          return axis == 0 ? (size_t)(is - 1 - d1) * is + d0 : (size_t)(is - 1 - d0) * is + d1;
        };
        const float* rin = rgb + pix(d1_in) * 3;
        const float* rout = rgb + pix(d1_out) * 3;
        // the two distance factors of the edge's end points
        const bool use0 = p[1][0] != fd0, use1 = p[0][0] != fd0;
        const float f0 = use0 ? span / (p[1][0] - fd0) : 0.f;
        const float f1 = use1 ? span / (fd0 - p[0][0]) : 0.f;
        auto add = [&](int d1, float diff) {
          const float base = (d1 - d1_cross) * 2.f / fis;
          if (use0) {
            float dist = f0 * base;
            dist = dist > 0.f ? dist + eps : dist - eps;
            gxy[pi[0]][1 - axis] -= diff / dist;
          }
          if (use1) {
            float dist = f1 * base;
            dist = dist > 0.f ? dist + eps : dist - eps;
            gxy[pi[1]][1 - axis] -= diff / dist;
          }
        };
        // out: the in-pixel is f's, sweep the pixels beyond the edge up to the border
        if (face_at(zbuf, pix(d1_in)) == f) {
          const int lim = direction > 0 ? is - 1 : 0;
          const int lo = min(d1_out, lim), hi = max(d1_out, lim);
          for (int d1 = lo; d1 <= hi; ++d1) {
            const size_t i = pix(d1);
            const float* r = rgb + i * 3;
            const float* g = gpix(i);
            const float diff = (r[0] - rin[0]) * (g[0] * inv) + (r[1] - rin[1]) * (g[1] * inv) +
                               (r[2] - rin[2]) * (g[2] * inv);
            if (diff > 0.f) add(d1, diff);
          }
        }
        // in: f's pixels from the edge to the face's opposite edge
        {
          float cross2;
          if ((fd0 - p[0][0]) * (fd0 - p[2][0]) < 0.f)
            cross2 = __fadd_rn(__fmul_rn(__fdiv_rn(__fadd_rn(p[2][1], -p[0][1]), __fadd_rn(p[2][0], -p[0][0])),
                                         __fadd_rn(fd0, -p[0][0])), p[0][1]);
          else
            cross2 = __fadd_rn(__fmul_rn(__fdiv_rn(__fadd_rn(p[1][1], -p[2][1]), __fadd_rn(p[1][0], -p[2][0])),
                                         __fadd_rn(fd0, -p[2][0])), p[2][1]);
          int lim = d1_in;                   // a vertical opposite edge through the column: only d1_in
          if (isfinite(cross2)) {
            const float l = direction > 0 ? ceilf(cross2) : floorf(cross2);
            lim = (int)fminf(fmaxf(l, -1.f), (float)is);
          }
          const int lo = max(min(d1_in, lim), 0), hi = min(max(d1_in, lim), is - 1);
          for (int d1 = lo; d1 <= hi; ++d1) {
            const size_t i = pix(d1);
            if (face_at(zbuf, i) != f) continue;
            const float* r = rgb + i * 3;
            const float* g = gpix(i);
            const float diff = (r[0] - rout[0]) * (g[0] * inv) + (r[1] - rout[1]) * (g[1] * inv) +
                               (r[2] - rout[2]) * (g[2] * inv);
            if (diff > 0.f) add(d1, diff);
          }
        }
      }
    }
  }
}

// thread per (image, face): the edge sweep of the drawn copy, the projection's backward, and the light's backward,
// written per corner: gface [A B][F][3][3] (world frame of the vertices as given to the forward)
// (128, 4): with one block per SM as the target ptxas held the kernel to 96 registers and spilled 12 bytes
__global__ void __launch_bounds__(128, 4)
k_rb_faces(const unsigned long long* __restrict__ zbuf, const int* __restrict__ faces, int F,
           const float* __restrict__ verts, const float4* __restrict__ proj, int V, int B, int G, int A,
           const LookAtCam* __restrict__ cams, int n, int ss, const float* __restrict__ ss_rgb,
           const float* __restrict__ dl, const float* __restrict__ g_rgb, float* __restrict__ gface) {
  const int img = blockIdx.y, a = img / B, b = img - a * B;
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const LookAtCam c = cams[(b / G) * A + a];
  const int is = c.is;
  const size_t npix = (size_t)is * is;
  const unsigned long long* zb = zbuf + (size_t)img * npix;
  const float4* pj = proj + (size_t)img * V;
  const float* vb = verts + (size_t)b * V * 3;
  const int idx[3] = {faces[f * 3], faces[f * 3 + 1], faces[f * 3 + 2]};
  const float4 q[3] = {pj[idx[0]], pj[idx[1]], pj[idx[2]]};
  float g[3][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
  float* out = gface + ((size_t)img * F + f) * 9;
  if (q[0].z <= 0.f || q[1].z <= 0.f || q[2].z <= 0.f) {       // never drawn
#pragma unroll
    for (int i = 0; i < 9; ++i) out[i] = 0.f;
    return;
  }
  // (b) the edge sweep of the drawn copy: the face as given when it faces the camera (neural_renderer's backside
  // test), else fill_back's reversed copy (v2, v1, v0)
  const bool front = (q[2].y - q[0].y) * (q[1].x - q[0].x) >= (q[1].y - q[0].y) * (q[2].x - q[0].x);
  const float4 o[3] = {front ? q[0] : q[2], q[1], front ? q[2] : q[0]};     // corners in the drawn winding
  float pxy[3][2], gxy[3][2];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    pxy[k][0] = o[k].x; pxy[k][1] = o[k].y;
    gxy[k][0] = 0.f; gxy[k][1] = 0.f;
  }
  edge_sweep(pxy, f, zb, ss_rgb + (size_t)img * npix * 3, g_rgb + (size_t)img * n * n * 3, is, n, ss, gxy);
  // (a) light: the sum of dl over f's supersamples, in raster_face's bounding box, row-major
  float dlight = 0.f;
  {
    const float xmin = fminf(q[0].x, fminf(q[1].x, q[2].x)), xmax = fmaxf(q[0].x, fmaxf(q[1].x, q[2].x));
    const float ymin = fminf(q[0].y, fminf(q[1].y, q[2].y)), ymax = fmaxf(q[0].y, fmaxf(q[1].y, q[2].y));
    // one pixel wider than raster_face's box: f's supersamples lie inside however the bounds round
    const int xi0 = max(0, (int)ceilf((xmin * is + is - 1.f) * 0.5f) - 1);
    const int xi1 = min(is - 1, (int)floorf((xmax * is + is - 1.f) * 0.5f) + 1);
    const int yi0 = max(0, (int)ceilf((ymin * is + is - 1.f) * 0.5f) - 1);
    const int yi1 = min(is - 1, (int)floorf((ymax * is + is - 1.f) * 0.5f) + 1);
    const float* d = dl + (size_t)img * npix;
    for (int yi = yi1; yi >= yi0; --yi)
      for (int xi = xi0; xi <= xi1; ++xi) {
        const size_t i = (size_t)(is - 1 - yi) * is + xi;
        if (face_at(zb, i) == f) dlight += d[i];
      }
  }
  if (dlight != 0.f) {
    const float* v0 = vb + 3 * idx[0];
    const float* v1 = vb + 3 * idx[1];
    const float* v2 = vb + 3 * idx[2];
    const float ea[3] = {v0[0] - v1[0], v0[1] - v1[1], v0[2] - v1[2]};
    const float eb[3] = {v2[0] - v1[0], v2[1] - v1[1], v2[2] - v1[2]};
    const float nx = ea[1] * eb[2] - ea[2] * eb[1], ny = ea[2] * eb[0] - ea[0] * eb[2], nz = ea[0] * eb[1] - ea[1] * eb[0];
    const float len = sqrtf(nx * nx + ny * ny + nz * nz);
    const float nl = fmaxf(len, 1e-5f);
    const float s = (nx * (c.eye[0] - v1[0]) + ny * (c.eye[1] - v1[1]) + nz * (c.eye[2] - v1[2])) >= 0.f ? 1.f : -1.f;
    if (s * ny / nl > 0.f) {                 // relu's gradient is 0 at <= 0
      // light = 0.5 + 0.5 s n_y / max(|n|, 1e-5)
      const float k = 0.5f * s * dlight;
      float gn[3] = {0.f, k / nl, 0.f};
      if (len > 1e-5f) {
        const float m = k * ny / (len * len * len);
        gn[0] -= m * nx; gn[1] -= m * ny; gn[2] -= m * nz;
      }
      // n = ea x eb:  g_ea = eb x g_n, g_eb = g_n x ea
      const float ga[3] = {eb[1] * gn[2] - eb[2] * gn[1], eb[2] * gn[0] - eb[0] * gn[2], eb[0] * gn[1] - eb[1] * gn[0]};
      const float gb[3] = {gn[1] * ea[2] - gn[2] * ea[1], gn[2] * ea[0] - gn[0] * ea[2], gn[0] * ea[1] - gn[1] * ea[0]};
#pragma unroll
      for (int k3 = 0; k3 < 3; ++k3) {
        g[0][k3] += ga[k3];
        g[2][k3] += gb[k3];
        g[1][k3] -= ga[k3] + gb[k3];
      }
    }
  }
  // (c) projection: x' = x_c / z_c / tan 30, y' likewise; c = R (v - eye)
  float gw[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float gx = gxy[k][0], gy = gxy[k][1];
    const float iz = 1.f / o[k].z;
    const float gcx = gx * c.inv_width * iz, gcy = gy * c.inv_width * iz, gcz = -(gx * o[k].x + gy * o[k].y) * iz;
#pragma unroll
    for (int d = 0; d < 3; ++d) gw[k][d] = c.rx[d] * gcx + c.ry[d] * gcy + c.rz[d] * gcz;
  }
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    g[0][d] += front ? gw[0][d] : gw[2][d];
    g[1][d] += gw[1][d];
    g[2][d] += front ? gw[2][d] : gw[0][d];
  }
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int d = 0; d < 3; ++d) out[k * 3 + d] = g[k][d];
}

// thread per (row b, vertex v): g_verts[b][v] = sum over the angles, then over v's faces in ascending order, of the
// corners of those faces that are v
__global__ void k_rb_gather(const float* __restrict__ gface, const int* __restrict__ faces, int F,
                            const int* __restrict__ offsets, const int* __restrict__ vf, int V, int B, int A,
                            float* __restrict__ g_verts) {
  const int b = blockIdx.y;
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  const int e0 = offsets[v], e1 = offsets[v + 1];
  for (int a = 0; a < A; ++a) {
    const float* gf = gface + (size_t)(a * B + b) * F * 9;
    int prev = -1;
    for (int e = e0; e < e1; ++e) {
      const int f = vf[e];
      if (f == prev) continue;               // a face naming v twice is listed twice
      prev = f;
#pragma unroll
      for (int k = 0; k < 3; ++k)
        if (faces[f * 3 + k] == v) {
          const float* x = gf + (size_t)f * 9 + k * 3;
          s0 += x[0]; s1 += x[1]; s2 += x[2];
        }
    }
  }
  float* o = g_verts + ((size_t)b * V + v) * 3;
  o[0] = s0; o[1] = s1; o[2] = s2;
}

// ---------------------------------------------------------------- CLIP prep and loss
// thread per (row b, source pixel): avc_clip_prep_nearest's backward, the output pixels that read it summed in
// row-major order, each divided by its channel's std
__global__ void k_clip_prep_nearest_bwd(const float* __restrict__ g_out, int B, int n, int S, float* __restrict__ g_img) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * n * n) return;
  const int sx = (int)(i % n), sy = (int)((i / n) % n), b = (int)(i / ((long long)n * n));
  const float scale = (float)n / (float)S;
  const int y0 = max(0, (int)((float)sy / scale) - 2), y1 = min(S - 1, (int)((float)(sy + 1) / scale) + 2);
  const int x0 = max(0, (int)((float)sx / scale) - 2), x1 = min(S - 1, (int)((float)(sx + 1) / scale) + 2);
  float acc[3] = {0.f, 0.f, 0.f};
  for (int y = y0; y <= y1; ++y) {
    if (min((int)floorf(y * scale), n - 1) != sy) continue;
    for (int x = x0; x <= x1; ++x) {
      if (min((int)floorf(x * scale), n - 1) != sx) continue;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const double stdv = ch == 0 ? 0.26862954 : (ch == 1 ? 0.26130258 : 0.27577711);
        acc[ch] += (float)((double)g_out[(((size_t)b * 3 + ch) * S + y) * S + x] / stdv);
      }
    }
  }
  float* o = g_img + (size_t)i * 3;
  o[0] = acc[0]; o[1] = acc[1]; o[2] = acc[2];
}

// one CTA per pose b: loss[b] = 1 - cos(mean_a emb[a][b], text) as k_pose_score computes the cosine, and
// g_emb[a][b] = d loss[b] / d emb[a][b]
__global__ void k_pose_clip_loss(const float* __restrict__ emb, int A, int B, int Dm, const float* __restrict__ text,
                                 float* __restrict__ loss, float* __restrict__ g_emb) {
  __shared__ double red[32];
  const int b = blockIdx.x;
  double xx = 0.0, xy = 0.0, yy = 0.0;
  for (int j = threadIdx.x; j < Dm; j += blockDim.x) {
    double s = 0.0;
    for (int a = 0; a < A; ++a) s += emb[((size_t)a * B + b) * Dm + j];
    const double f = (float)(s / A), t = text[j];
    xx += f * f; xy += f * t; yy += t * t;
  }
  const auto add = [](double u, double v) { return u + v; };
  xx = block_reduce(xx, red, add, 0.0);
  xy = block_reduce(xy, red, add, 0.0);
  yy = block_reduce(yy, red, add, 0.0);
  const double lf = sqrt(xx), nf = fmax(lf, 1e-8), nt = fmax(sqrt(yy), 1e-8);
  const double cs = xy / (nf * nt);
  if (threadIdx.x == 0 && loss) loss[b] = (float)(1.0 - (double)(float)cs);
  for (int j = threadIdx.x; j < Dm; j += blockDim.x) {
    double s = 0.0;
    for (int a = 0; a < A; ++a) s += emb[((size_t)a * B + b) * Dm + j];
    const double f = (float)(s / A);
    double dc = text[j] / (nf * nt);
    if (lf > 1e-8) dc -= cs * f / (nf * lf);
    const float gv = (float)(-dc / A);
    for (int a = 0; a < A; ++a) g_emb[((size_t)a * B + b) * Dm + j] = gv;
  }
}

}  // namespace

// the batched render's passes with its cameras copied (kind: from host or device memory) into the workspace
static int raster_batch_run(const float* verts, int B, int group, const int* faces, const float* textures, int V,
                            int F, int R, const void* cams_src, cudaMemcpyKind kind, int A, int image_size,
                            int supersample, float* rgb_out, void* workspace, avc_stream_t stream) {
  const int ngroups = (B + group - 1) / group;
  const int is = image_size * supersample;
  cudaStream_t st = (cudaStream_t)stream;
  Carver c(workspace);
  LookAtCam* cams = c.take<LookAtCam>((size_t)ngroups * A);
  float4* proj = c.take<float4>((size_t)A * B * V);
  unsigned long long* zbuf = c.take<unsigned long long>((size_t)A * B * is * is);
  AVC_CUDA_TRY(cudaMemcpyAsync(cams, cams_src, sizeof(LookAtCam) * (size_t)ngroups * A, kind, st));
  AVC_CUDA_TRY(cudaMemsetAsync(zbuf, 0xff, sizeof(unsigned long long) * (size_t)A * B * is * is, st));
  const unsigned nimg = (unsigned)(A * B);
  k_project_batch<<<dim3((V + 255) / 256, nimg), 256, 0, st>>>(verts, V, B, group, A, cams, proj);
  k_raster_batch<<<dim3((F + 127) / 128, nimg), 128, 0, st>>>(proj, V, faces, F, is, zbuf);
  k_resolve_batch<<<dim3((image_size * image_size + 255) / 256, nimg), 256, 0, st>>>(
      zbuf, faces, verts, proj, textures, R, V, B, group, A, cams, image_size, supersample, rgb_out);
  AVC_LAUNCH_TRY();
  return 0;
}

// decoder_net's weights transposed to [K][N] into the workspace (avc_vposer_decode_workspace_bytes), as
// k_vposer_decode and k_vposer_decode_bwd read them
static VpWeights vposer_weights(int L, int H, int n_joints, const float* W1, const float* b1, const float* W2,
                                const float* b2, const float* W3, const float* b3, void* workspace, cudaStream_t st) {
  const int O = n_joints * 6;
  Carver c(workspace);
  float* w1t = c.take<float>((size_t)L * H);
  float* w2t = c.take<float>((size_t)H * H);
  float* w3t = c.take<float>((size_t)H * O);
  k_transpose<<<(H * L + 255) / 256, 256, 0, st>>>(W1, H, L, L, 0, w1t);
  k_transpose<<<(H * H + 255) / 256, 256, 0, st>>>(W2, H, H, H, 0, w2t);
  k_transpose<<<(O * H + 255) / 256, 256, 0, st>>>(W3, O, H, H, 0, w3t);
  return VpWeights{w1t, b1, w2t, b2, w3t, b3};
}

extern "C" {

int avc_vposer_decode_workspace_bytes(int32_t latent, int32_t hidden, int32_t n_joints, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (latent < 1 || latent > kVpMaxL || hidden < 1 || hidden > kVpMaxH || n_joints < 1 || n_joints * 6 > kVpMaxOut)
    return AVC_E_SIZE;
  Carver c(nullptr);
  c.take<float>((size_t)latent * hidden);
  c.take<float>((size_t)hidden * hidden);
  c.take<float>((size_t)hidden * n_joints * 6);
  *bytes = c.used();
  return 0;
}

int avc_vposer_decode(const float* z, int32_t B, int32_t latent, const float* W1, const float* b1, int32_t hidden,
                      const float* W2, const float* b2, const float* W3, const float* b3, int32_t n_joints,
                      float* pose_out, float* rotmat_out, void* workspace, size_t workspace_bytes,
                      avc_stream_t stream) {
  if (!z || !W1 || !b1 || !W2 || !b2 || !W3 || !b3 || !pose_out || !workspace) return AVC_E_NULL;
  size_t need = 0;
  AVC_TRY(avc_vposer_decode_workspace_bytes(latent, hidden, n_joints, &need));
  if (B < 1 || workspace_bytes < need) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  const VpWeights w = vposer_weights(latent, hidden, n_joints, W1, b1, W2, b2, W3, b3, workspace, st);
  k_vposer_decode<<<(B + kVpRows - 1) / kVpRows, 256, 0, st>>>(z, B, latent, hidden, n_joints, w, pose_out,
                                                               rotmat_out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_vposer_decode_bwd_workspace_bytes(int32_t latent, int32_t hidden, int32_t n_joints, size_t* bytes) {
  return avc_vposer_decode_workspace_bytes(latent, hidden, n_joints, bytes);
}

int avc_vposer_decode_bwd(const float* z, int32_t B, int32_t latent, const float* W1, const float* b1, int32_t hidden,
                          const float* W2, const float* b2, const float* W3, const float* b3, int32_t n_joints,
                          const float* g_pose, float* g_z, float* pose_out, void* workspace, size_t workspace_bytes,
                          avc_stream_t stream) {
  if (!z || !W1 || !b1 || !W2 || !b2 || !W3 || !b3 || !g_pose || !g_z || !workspace) return AVC_E_NULL;
  size_t need = 0;
  AVC_TRY(avc_vposer_decode_bwd_workspace_bytes(latent, hidden, n_joints, &need));
  if (B < 1 || workspace_bytes < need) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  const VpWeights w = vposer_weights(latent, hidden, n_joints, W1, b1, W2, b2, W3, b3, workspace, st);
  k_vposer_decode_bwd<<<(B + kVpRows - 1) / kVpRows, 256, 0, st>>>(z, B, latent, hidden, n_joints, w, W1, W2, W3,
                                                                   g_pose, g_z, pose_out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_vposer_encode_workspace_bytes(int32_t n_in, int32_t hidden, int32_t latent, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (n_in < 1 || n_in > kVpMaxOut || hidden < 1 || hidden > kVpMaxH || latent < 1 || latent > kVpMaxL)
    return AVC_E_SIZE;
  Carver c(nullptr);
  c.take<float>((size_t)n_in * hidden);
  c.take<float>((size_t)hidden * hidden);
  c.take<float>((size_t)hidden * hidden);
  c.take<float>((size_t)hidden * latent);
  *bytes = c.used();
  return 0;
}

int avc_vposer_encode(const float* x, int32_t B, int32_t n_in, const float* bn1, const float* W1, const float* b1,
                      int32_t hidden, const float* bn2, const float* W2, const float* b2, const float* W3,
                      const float* b3, const float* Wmu, const float* bmu, int32_t latent, float* mu_out,
                      void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!x || !bn1 || !W1 || !b1 || !bn2 || !W2 || !b2 || !W3 || !b3 || !Wmu || !bmu || !mu_out || !workspace)
    return AVC_E_NULL;
  size_t need = 0;
  AVC_TRY(avc_vposer_encode_workspace_bytes(n_in, hidden, latent, &need));
  if (B < 1 || workspace_bytes < need) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  const int NI = n_in, H = hidden, L = latent;
  Carver c(workspace);
  float* w1t = c.take<float>((size_t)NI * H);
  float* w2t = c.take<float>((size_t)H * H);
  float* w3t = c.take<float>((size_t)H * H);
  float* wmt = c.take<float>((size_t)H * L);
  k_transpose<<<(H * NI + 255) / 256, 256, 0, st>>>(W1, H, NI, NI, 0, w1t);
  k_transpose<<<(H * H + 255) / 256, 256, 0, st>>>(W2, H, H, H, 0, w2t);
  k_transpose<<<(H * H + 255) / 256, 256, 0, st>>>(W3, H, H, H, 0, w3t);
  k_transpose<<<(L * H + 255) / 256, 256, 0, st>>>(Wmu, L, H, H, 0, wmt);
  VpEncWeights w{bn1, w1t, b1, bn2, w2t, b2, w3t, b3, wmt, bmu};
  k_vposer_encode<<<(B + kVpRows - 1) / kVpRows, 256, 0, st>>>(x, B, NI, H, L, w, mu_out);
  AVC_LAUNCH_TRY();
  return 0;
}

static bool nvp_sizes_ok(int dim, int hidden, int n_blocks) {
  return dim >= 1 && dim <= kNvpMaxD && hidden >= 1 && hidden <= kNvpMaxH && n_blocks >= 1 && n_blocks <= kNvpMaxBlocks;
}

int avc_realnvp_pack_floats(int32_t dim, int32_t hidden, int32_t n_blocks, size_t* floats) {
  if (!floats) return AVC_E_NULL;
  if (!nvp_sizes_ok(dim, hidden, n_blocks)) return AVC_E_SIZE;
  *floats = nvp_pack(dim, hidden).stride * 2 * n_blocks;
  return 0;
}

int avc_realnvp_pack(const float* params, int32_t dim, int32_t feat_dim, int32_t hidden, int32_t n_blocks, float* pack,
                     avc_stream_t stream) {
  if (!params || !pack) return AVC_E_NULL;
  if (!nvp_sizes_ok(dim, hidden, n_blocks) || feat_dim < 0) return AVC_E_SIZE;
  const int H = hidden;
  const dim3 grid((max(H, dim) * H + 255) / 256, 2 * n_blocks);
  k_realnvp_pack<<<grid, 256, 0, (cudaStream_t)stream>>>(params, dim, feat_dim, H, pack);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_realnvp_decode_workspace_bytes(int32_t dim, int32_t hidden, int32_t n_blocks, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (!nvp_sizes_ok(dim, hidden, n_blocks)) return AVC_E_SIZE;
  Carver c(nullptr);
  c.take<float>((size_t)hidden * 2 * n_blocks);
  *bytes = c.used();
  return 0;
}

int avc_realnvp_decode(const float* z, int32_t B, int32_t dim, const float* feature, int32_t feat_dim,
                       const float* params, const float* pack, const float* mask, int32_t n_blocks, int32_t hidden,
                       float* x_out, void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!z || !feature || !params || !pack || !mask || !x_out || !workspace) return AVC_E_NULL;
  size_t need = 0;
  AVC_TRY(avc_realnvp_decode_workspace_bytes(dim, hidden, n_blocks, &need));
  if (B < 1 || feat_dim < 0 || workspace_bytes < need) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  const int D = dim, E = feat_dim, H = hidden;
  float* fold = static_cast<float*>(workspace);
  k_realnvp_fold<<<2 * n_blocks, 256, 0, st>>>(params, feature, D, E, H, fold);
  k_realnvp_decode<<<(B + kNvpRows - 1) / kNvpRows, 256, 0, st>>>(z, B, D, E, H, n_blocks, params, pack, fold, mask,
                                                                  x_out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_smpl_pose_batch_workspace_bytes(int32_t B, int32_t n_joints, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (B < 1 || n_joints < 2 || n_joints > NJ_MAX) return AVC_E_SIZE;
  Carver c(nullptr);
  c.take<float>((size_t)n_joints * 3);
  c.take<float>((size_t)B * n_joints * 12);
  c.take<float>((size_t)B * (n_joints - 1) * 9);
  *bytes = c.used();
  return 0;
}

int avc_smpl_pose_batch(const float* v_template, const float* J_regressor, const int32_t* parents,
                        const float* posedirs, const float* lbs_weights, int32_t V, int32_t n_joints,
                        const float* body_pose, int32_t pose_dim, int32_t B, const float* global_orient,
                        const float* post_rot, float* verts_out, void* workspace, size_t workspace_bytes,
                        avc_stream_t stream) {
  if (!v_template || !J_regressor || !parents || !posedirs || !lbs_weights || !body_pose || !global_orient ||
      !verts_out || !workspace)
    return AVC_E_NULL;
  size_t need = 0;
  AVC_TRY(avc_smpl_pose_batch_workspace_bytes(B, n_joints, &need));
  if (V < 1 || pose_dim < 0 || pose_dim > (n_joints - 1) * 3 || workspace_bytes < need) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  Carver c(workspace);
  float* J = c.take<float>((size_t)n_joints * 3);
  float* A = c.take<float>((size_t)B * n_joints * 12);
  float* feat = c.take<float>((size_t)B * (n_joints - 1) * 9);
  Orient go{{global_orient[0], global_orient[1], global_orient[2]}};
  PostRot pr{};
  pr.on = post_rot != nullptr;
  if (post_rot)
    for (int i = 0; i < 9; ++i) pr.m[i] = post_rot[i];
  k_smpl_joints<<<1, 256, 0, st>>>(v_template, J_regressor, V, n_joints, J);
  k_pose_chain<<<(B + 3) / 4, 128, 0, st>>>(body_pose, pose_dim, B, go, J, parents, n_joints, A, feat);
  dim3 grid((V + 127) / 128, (B + kSkinRows - 1) / kSkinRows);
  k_pose_skin<<<grid, 128, 0, st>>>(v_template, posedirs, feat, A, lbs_weights, V, n_joints, (n_joints - 1) * 9, B, pr,
                                    verts_out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_raster_textured_batch_workspace_bytes(int32_t V, int32_t n_images, int32_t n_cams, int32_t image_size,
                                              int32_t supersample, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (V < 1 || n_images < 1 || n_images > 65535 || n_cams < 1 || image_size < 1 || image_size > 4096 ||
      supersample < 1 || supersample > 4)
    return AVC_E_SIZE;
  const size_t is = (size_t)image_size * supersample;
  Carver c(nullptr);
  c.take<LookAtCam>(n_cams);
  c.take<float4>((size_t)n_images * V);
  c.take<unsigned long long>((size_t)n_images * is * is);
  *bytes = c.used();
  return 0;
}

int avc_raster_textured_batch(const float* verts, int32_t B, int32_t group, const int32_t* faces,
                              const float* textures, int32_t V, int32_t F, int32_t R, const float* eyes, int32_t A,
                              const float* at, const float* up, int32_t image_size, int32_t supersample,
                              float* rgb_out, void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!verts || !faces || !textures || !eyes || !at || !up || !rgb_out || !workspace) return AVC_E_NULL;
  if (B < 1 || group < 1 || A < 1 || A > kMaxCams || F < 1 || R < 2 || R > 64) return AVC_E_SIZE;
  const int ngroups = (B + group - 1) / group;
  size_t need = 0;
  AVC_TRY(avc_raster_textured_batch_workspace_bytes(V, A * B, ngroups * A, image_size, supersample, &need));
  if (workspace_bytes < need) return AVC_E_SIZE;
  const int is = image_size * supersample;
  std::vector<LookAtCam> hc((size_t)ngroups * A);
  for (int i = 0; i < ngroups * A; ++i)
    if (!make_look_at_cam(eyes + 3 * i, at, up, is, &hc[i])) return AVC_E_BADCFG;
  // from pageable memory: the call returns once hc is staged, so it may be freed on return
  return raster_batch_run(verts, B, group, faces, textures, V, F, R, hc.data(), cudaMemcpyHostToDevice, A, image_size,
                          supersample, rgb_out, workspace, stream);
}

int avc_look_at_cam_bytes(size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  *bytes = sizeof(LookAtCam);
  return 0;
}

int avc_look_at_cams(const float* eyes, int32_t n, const float* at, const float* up, int32_t image_size,
                     int32_t supersample, void* cams_out, avc_stream_t stream) {
  if (!eyes || !at || !up || !cams_out) return AVC_E_NULL;
  if (n < 1 || image_size < 1 || image_size > 4096 || supersample < 1 || supersample > 4) return AVC_E_SIZE;
  std::vector<LookAtCam> hc((size_t)n);
  for (int i = 0; i < n; ++i)
    if (!make_look_at_cam(eyes + 3 * i, at, up, image_size * supersample, &hc[i])) return AVC_E_BADCFG;
  AVC_CUDA_TRY(cudaMemcpyAsync(cams_out, hc.data(), sizeof(LookAtCam) * hc.size(), cudaMemcpyHostToDevice,
                               (cudaStream_t)stream));
  return 0;
}

int avc_raster_textured_batch_dev(const float* verts, int32_t B, int32_t group, const int32_t* faces,
                                  const float* textures, int32_t V, int32_t F, int32_t R, const void* cams, int32_t A,
                                  int32_t image_size, int32_t supersample, float* rgb_out, void* workspace,
                                  size_t workspace_bytes, avc_stream_t stream) {
  if (!verts || !faces || !textures || !cams || !rgb_out || !workspace) return AVC_E_NULL;
  if (B < 1 || group < 1 || A < 1 || A > kMaxCams || F < 1 || R < 2 || R > 64) return AVC_E_SIZE;
  const int ngroups = (B + group - 1) / group;
  size_t need = 0;
  AVC_TRY(avc_raster_textured_batch_workspace_bytes(V, A * B, ngroups * A, image_size, supersample, &need));
  if (workspace_bytes < need) return AVC_E_SIZE;
  return raster_batch_run(verts, B, group, faces, textures, V, F, R, cams, cudaMemcpyDeviceToDevice, A, image_size,
                          supersample, rgb_out, workspace, stream);
}

int avc_raster_textured_batch_bwd_workspace_bytes(int32_t F, int32_t n_images, int32_t image_size,
                                                  int32_t supersample, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (F < 1 || n_images < 1 || n_images > 65535 || image_size < 1 || image_size > 4096 || supersample < 1 ||
      supersample > 4)
    return AVC_E_SIZE;
  const size_t npix = (size_t)image_size * supersample * image_size * supersample;
  Carver c(nullptr);
  c.take<float>((size_t)n_images * npix * 3);
  c.take<float>((size_t)n_images * npix);
  c.take<float>((size_t)n_images * F * 9);
  *bytes = c.used();
  return 0;
}

int avc_raster_textured_batch_bwd(const float* verts, int32_t B, int32_t group, const int32_t* faces,
                                  const float* textures, int32_t V, int32_t F, int32_t R, int32_t A,
                                  int32_t image_size, int32_t supersample, const int32_t* offsets, const int32_t* vf,
                                  const float* g_rgb, float* g_verts, const void* fwd_workspace,
                                  size_t fwd_workspace_bytes, void* workspace, size_t workspace_bytes,
                                  avc_stream_t stream) {
  if (!verts || !faces || !textures || !offsets || !vf || !g_rgb || !g_verts || !fwd_workspace || !workspace)
    return AVC_E_NULL;
  if (B < 1 || group < 1 || A < 1 || A > kMaxCams || F < 1 || R < 2 || R > 64) return AVC_E_SIZE;
  const int ngroups = (B + group - 1) / group;
  size_t need_f = 0, need = 0;
  AVC_TRY(avc_raster_textured_batch_workspace_bytes(V, A * B, ngroups * A, image_size, supersample, &need_f));
  AVC_TRY(avc_raster_textured_batch_bwd_workspace_bytes(F, A * B, image_size, supersample, &need));
  if (fwd_workspace_bytes < need_f || workspace_bytes < need) return AVC_E_SIZE;
  const int is = image_size * supersample;
  const size_t npix = (size_t)is * is;
  Carver cf(const_cast<void*>(fwd_workspace));
  const LookAtCam* cams = cf.take<LookAtCam>((size_t)ngroups * A);
  const float4* proj = cf.take<float4>((size_t)A * B * V);
  const unsigned long long* zbuf = cf.take<unsigned long long>((size_t)A * B * npix);
  Carver c(workspace);
  float* ss_rgb = c.take<float>((size_t)A * B * npix * 3);
  float* dl = c.take<float>((size_t)A * B * npix);
  float* gface = c.take<float>((size_t)A * B * F * 9);
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned nimg = (unsigned)(A * B);
  k_rb_samples<<<dim3((unsigned)((npix + 255) / 256), nimg), 256, 0, st>>>(
      zbuf, faces, verts, proj, textures, R, V, B, group, A, cams, image_size, supersample, g_rgb, ss_rgb, dl);
  k_rb_faces<<<dim3((F + 127) / 128, nimg), 128, 0, st>>>(zbuf, faces, F, verts, proj, V, B, group, A, cams,
                                                          image_size, supersample, ss_rgb, dl, g_rgb, gface);
  k_rb_gather<<<dim3((V + 127) / 128, B), 128, 0, st>>>(gface, faces, F, offsets, vf, V, B, A, g_verts);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_smpl_pose_batch_bwd_workspace_bytes(int32_t B, int32_t V, int32_t n_joints, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (B < 1 || V < 1 || n_joints < 2 || n_joints > NJ_MAX) return AVC_E_SIZE;
  Carver c(nullptr);
  c.take<float>((size_t)n_joints * 3);
  c.take<float>((size_t)B * n_joints * 12);
  c.take<float>((size_t)B * (n_joints - 1) * 9);
  for (int i = 0; i < 3; ++i) c.take<float>((size_t)B * V * 3);
  c.take<float>((size_t)B * n_joints * 12);
  c.take<float>((size_t)B * (n_joints - 1) * 9);
  *bytes = c.used();
  return 0;
}

int avc_smpl_pose_batch_bwd(const float* v_template, const float* J_regressor, const int32_t* parents,
                            const float* posedirs, const float* lbs_weights, int32_t V, int32_t n_joints,
                            const float* body_pose, int32_t pose_dim, int32_t B, const float* global_orient,
                            const float* post_rot, const float* g_verts, float* g_body_pose, void* workspace,
                            size_t workspace_bytes, avc_stream_t stream) {
  if (!v_template || !J_regressor || !parents || !posedirs || !lbs_weights || !body_pose || !global_orient ||
      !g_verts || !g_body_pose || !workspace)
    return AVC_E_NULL;
  size_t need = 0;
  AVC_TRY(avc_smpl_pose_batch_bwd_workspace_bytes(B, V, n_joints, &need));
  if (pose_dim < 1 || pose_dim > (n_joints - 1) * 3 || workspace_bytes < need) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  const int NF = (n_joints - 1) * 9;
  Carver c(workspace);
  float* J = c.take<float>((size_t)n_joints * 3);
  float* A = c.take<float>((size_t)B * n_joints * 12);
  float* feat = c.take<float>((size_t)B * NF);
  float* p = c.take<float>((size_t)B * V * 3);
  float* go = c.take<float>((size_t)B * V * 3);
  float* gp = c.take<float>((size_t)B * V * 3);
  float* dA = c.take<float>((size_t)B * n_joints * 12);
  float* gfeat = c.take<float>((size_t)B * NF);
  Orient o{{global_orient[0], global_orient[1], global_orient[2]}};
  PostRot pr{};
  pr.on = post_rot != nullptr;
  if (post_rot)
    for (int i = 0; i < 9; ++i) pr.m[i] = post_rot[i];
  k_smpl_joints<<<1, 256, 0, st>>>(v_template, J_regressor, V, n_joints, J);
  k_pose_chain<<<(B + 3) / 4, 128, 0, st>>>(body_pose, pose_dim, B, o, J, parents, n_joints, A, feat);
  const unsigned rows = (unsigned)((B + kSkinRows - 1) / kSkinRows);
  k_pose_skin_bwd<<<dim3((V + 127) / 128, rows), 128, 0, st>>>(v_template, posedirs, feat, A, lbs_weights, V, n_joints,
                                                               NF, B, pr, g_verts, p, go, gp);
  k_pose_dA<<<dim3(n_joints, B), 256, 0, st>>>(lbs_weights, p, go, V, n_joints, dA);
  k_pose_gfeat<<<dim3(NF, rows), 256, 0, st>>>(posedirs, gp, V * 3, NF, B, gfeat);
  k_pose_chain_bwd<<<(B + 3) / 4, 128, 0, st>>>(body_pose, pose_dim, B, J, parents, n_joints, A, feat, dA, gfeat,
                                                g_body_pose);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_clip_prep_nearest_bwd(const float* g_out, int32_t B, int32_t n, int32_t out_size, float* g_images,
                              avc_stream_t stream) {
  if (!g_out || !g_images) return AVC_E_NULL;
  if (B < 1 || n < 1 || out_size < 1) return AVC_E_SIZE;
  const long long total = (long long)B * n * n;
  k_clip_prep_nearest_bwd<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(g_out, B, n, out_size,
                                                                                              g_images);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_pose_clip_loss(const float* emb, int32_t A, int32_t B, int32_t dim, const float* text, float* loss_out,
                       float* g_emb, avc_stream_t stream) {
  if (!emb || !text || !g_emb) return AVC_E_NULL;
  if (A < 1 || B < 1 || dim < 1) return AVC_E_SIZE;
  k_pose_clip_loss<<<B, 128, 0, (cudaStream_t)stream>>>(emb, A, B, dim, text, loss_out, g_emb);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_cosine_topk(const float* rows, int32_t N, int32_t D, const float* vec, float eps, int32_t k, float* cos_out,
                    int32_t* idx_out, avc_stream_t stream) {
  if (!rows || !vec || !cos_out || !idx_out) return AVC_E_NULL;
  if (N < 1 || D < 1 || k < 1 || k > N) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  k_rows_cos<<<N, 128, 0, st>>>(rows, vec, D, eps, cos_out);
  k_topk<<<1, 1024, 0, st>>>(cos_out, N, k, idx_out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_pose_suppress(const float* poses, int32_t P, int32_t dim, float threshold, int32_t* keep_out,
                      int32_t* count_out, avc_stream_t stream) {
  if (!poses || !keep_out || !count_out) return AVC_E_NULL;
  if (P < 1 || P > kSupMax || dim < 1 || dim > kSupMaxD) return AVC_E_SIZE;
  k_pose_suppress<<<1, 256, 0, (cudaStream_t)stream>>>(poses, P, dim, threshold, keep_out, count_out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_pose_score(const float* emb, int32_t A, int32_t B, int32_t dim, const float* text, int32_t group,
                   float* score_out, int32_t* best_out, void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!emb || !text || !score_out || !best_out || !workspace) return AVC_E_NULL;
  if (A < 1 || B < 1 || dim < 1 || group < 1) return AVC_E_SIZE;
  const int ng = (B + group - 1) / group;
  if (workspace_bytes < sizeof(unsigned long long) * ng) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* keys = static_cast<unsigned long long*>(workspace);
  AVC_CUDA_TRY(cudaMemsetAsync(keys, 0, sizeof(unsigned long long) * ng, st));
  k_pose_score<<<B, 128, 0, st>>>(emb, A, B, dim, text, group, score_out, keys);
  k_group_best<<<(ng + 255) / 256, 256, 0, st>>>(keys, ng, best_out);
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"
