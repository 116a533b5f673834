// avc_smpl.cuh -- SMPL forward kinematics, shared by avc_lbs_fwd (avc_lbs.cu), avc_lbs_rel_transforms (avc_drive.cu)
// and avc_smpl_pose_batch with its backward (avc_pose.cu), so that every path poses a joint with the same arithmetic in
// the same order.  It restates smplx's vertices2joints / batch_rigid_transform (in-tree copies: drive.py:51-160) and
// AvatarCLIP's batch_rodrigues (models/utils.py:72-106).  A kinematic chain is walked by one warp, lane j owning joint j;
// the callers differ only in how they read a joint's local rotation.
#pragma once

#include "avc_common.cuh"

namespace avc {

constexpr int NJ_MAX = 32;   // joints of a skeleton: one warp lane each

// J[j] = J_regressor[j] . v for every joint, one warp per joint at a time (vertices2joints, drive.py:51-70).  J is
// [NJ][3], in shared or global memory.
__device__ __forceinline__ void regress_joints(const float* __restrict__ v, const float* __restrict__ J_regressor, int V,
                                               int NJ, float* J) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int j = warp; j < NJ; j += nw) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    const float* jr = J_regressor + (size_t)j * V;
    for (int i = lane; i < V; i += 32) {
      const float w = jr[i];
      a0 = fmaf(w, v[i * 3 + 0], a0); a1 = fmaf(w, v[i * 3 + 1], a1); a2 = fmaf(w, v[i * 3 + 2], a2);
    }
    a0 = warp_sum(a0); a1 = warp_sum(a1); a2 = warp_sum(a2);
    if (lane == 0) { J[j * 3] = a0; J[j * 3 + 1] = a1; J[j * 3 + 2] = a2; }
  }
}

// regress_joints into global memory, for the launches that pose many rows from one J (defined in avc_lbs.cu)
__global__ void k_smpl_joints(const float* __restrict__ v_template, const float* __restrict__ J_regressor, int V, int NJ,
                              float* __restrict__ J);

// batch_rodrigues of one axis-angle r: angle |r + eps| (the eps inside the norm), unit axis r / angle with its
// cross-product matrix K, and R = I + s K + (1 - c) K K.  The pieces are what the backward differentiates.
constexpr float kRodriguesEps = 1e-8f;

struct Rodrigues {
  float ang, s, c;
  float K[9], KK[9];
};

__device__ __forceinline__ Rodrigues rodrigues_terms(float rx, float ry, float rz) {
  Rodrigues q;
  const float eps = kRodriguesEps;
  q.ang = sqrtf((rx + eps) * (rx + eps) + (ry + eps) * (ry + eps) + (rz + eps) * (rz + eps));
  const float x = rx / q.ang, y = ry / q.ang, z = rz / q.ang;
  sincosf(q.ang, &q.s, &q.c);   // its Payne-Hanek path for |ang| > 105615 is the callers' 32-byte stack frame
  const float K[9] = {0, -z, y, z, 0, -x, -y, x, 0};
#pragma unroll
  for (int i = 0; i < 9; ++i) q.K[i] = K[i];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) q.KK[a * 3 + b] = K[a * 3] * K[b] + K[a * 3 + 1] * K[3 + b] + K[a * 3 + 2] * K[6 + b];
  return q;
}

__device__ __forceinline__ void rodrigues(float rx, float ry, float rz, float R[9]) {
  const Rodrigues q = rodrigues_terms(rx, ry, rz);
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = ((i % 4 == 0) ? 1.f : 0.f) + q.s * q.K[i] + (1.f - q.c) * q.KK[i];
}

// depth of the lane's joint in the tree (root 0) by pointer chasing through shuffles; par is -1 at the root and on
// lanes past the last joint
__device__ __forceinline__ int joint_depth(int par) {
  int depth = 0, p = par;
  for (int it = 0; it < NJ_MAX; ++it) {
    const int pp = __shfl_sync(0xffffffffu, par, p < 0 ? 0 : p);
    if (p >= 0) { ++depth; p = pp; }
  }
  return depth;
}

// the deepest level of the warp's tree.  Every lane ends with the same value, lanes past the last joint included, so
// the level loops that follow stay warp-uniform and each of their full-warp shuffles is reached by all 32 lanes.
__device__ __forceinline__ int max_depth(int depth) {
  int maxd = depth;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) maxd = max(maxd, __shfl_xor_sync(0xffffffffu, maxd, o));
  return maxd;
}

// Lane j = joint j with local rotation R, parent par and rest joint (Jx, Jy, Jz); act is j < NJ.  The world transform
// T = T_parent [R | J - J_parent], filled level by level (batch_rigid_transform, drive.py:122-136).
__device__ __forceinline__ void chain_world(const float R[9], int j, int par, bool act, float Jx, float Jy, float Jz,
                                            float T[12]) {
  float tx = Jx, ty = Jy, tz = Jz;
  {
    const int p = par < 0 ? 0 : par;
    const float px = __shfl_sync(0xffffffffu, Jx, p), py = __shfl_sync(0xffffffffu, Jy, p),
                pz = __shfl_sync(0xffffffffu, Jz, p);
    if (act && j >= 1) { tx -= px; ty -= py; tz -= pz; }
  }
  T[0] = R[0]; T[1] = R[1]; T[2] = R[2]; T[3] = tx;
  T[4] = R[3]; T[5] = R[4]; T[6] = R[5]; T[7] = ty;
  T[8] = R[6]; T[9] = R[7]; T[10] = R[8]; T[11] = tz;
  const int depth = joint_depth(par);
  const int maxd = max_depth(depth);
  for (int d = 1; d <= maxd; ++d) {
    float P[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) P[i] = __shfl_sync(0xffffffffu, T[i], par < 0 ? 0 : par);
    if (act && depth == d) {
      float Nw[12];
#pragma unroll
      for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) Nw[r * 4 + c] = P[r * 4] * T[c] + P[r * 4 + 1] * T[4 + c] + P[r * 4 + 2] * T[8 + c];
        Nw[r * 4 + 3] = P[r * 4] * T[3] + P[r * 4 + 1] * T[7] + P[r * 4 + 2] * T[11] + P[r * 4 + 3];
      }
#pragma unroll
      for (int i = 0; i < 12; ++i) T[i] = Nw[i];
    }
  }
}

// rel_transforms: A = T - [0 | T_rot J]  (drive.py:143-146)
__device__ __forceinline__ void rel_transform(const float T[12], float Jx, float Jy, float Jz, float* a) {
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    a[r * 4 + 0] = T[r * 4]; a[r * 4 + 1] = T[r * 4 + 1]; a[r * 4 + 2] = T[r * 4 + 2];
    a[r * 4 + 3] = T[r * 4 + 3] - (T[r * 4] * Jx + T[r * 4 + 1] * Jy + T[r * 4 + 2] * Jz);
  }
}

// ---------------------------------------------------------------- skinning of ROWS pose rows per CTA
// the transforms A [B][NJ][12] and pose features [B][NF] of rows b0 .. b0 + ROWS - 1 into shared memory, zeros for the
// rows past B (nr rows are live)
template <int ROWS>
__device__ __forceinline__ void stage_rows(float (*sA)[NJ_MAX * 12], float (*sF)[NJ_MAX * 9], const float* __restrict__ A,
                                           const float* __restrict__ feat, int b0, int nr, int NJ, int NF) {
  for (int i = threadIdx.x; i < ROWS * NJ * 12; i += blockDim.x) {
    const int r = i / (NJ * 12), k = i - r * NJ * 12;
    sA[r][k] = r < nr ? A[(size_t)(b0 + r) * NJ * 12 + k] : 0.f;
  }
  for (int i = threadIdx.x; i < ROWS * NF; i += blockDim.x) {
    const int r = i / NF, k = i - r * NF;
    sF[r][k] = r < nr ? feat[(size_t)(b0 + r) * NF + k] : 0.f;
  }
  __syncthreads();
}

// the pose-blended template of every row at vertex v: p[r] = v_template[v] + sum_k feat[r][k] posedirs[k][v], the
// terms in k_lbs_skin's order, each posedirs element read once for all rows  (models/utils.py:195-205)
template <int ROWS>
__device__ __forceinline__ void pose_blend_rows(float p[ROWS][3], const float* __restrict__ v_template,
                                                const float* __restrict__ posedirs, const float (*sF)[NJ_MAX * 9], int V,
                                                int NF, int v) {
  const float t0 = v_template[v * 3], t1 = v_template[v * 3 + 1], t2 = v_template[v * 3 + 2];
#pragma unroll
  for (int r = 0; r < ROWS; ++r) { p[r][0] = t0; p[r][1] = t1; p[r][2] = t2; }
  const size_t ld = (size_t)V * 3;
  for (int k = 0; k < NF; ++k) {
    const float* pd = posedirs + (size_t)k * ld + (size_t)v * 3;
    const float d0 = pd[0], d1 = pd[1], d2 = pd[2];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const float f = sF[r][k];
      p[r][0] = fmaf(f, d0, p[r][0]); p[r][1] = fmaf(f, d1, p[r][1]); p[r][2] = fmaf(f, d2, p[r][2]);
    }
  }
}

// the blended transform T = sum_j W[v,j] A_j of one row, w = lbs_weights + v * NJ  (models/utils.py:213-218)
__device__ __forceinline__ void blend_transform(const float* __restrict__ w, const float* a, int NJ, float T[12]) {
#pragma unroll
  for (int i = 0; i < 12; ++i) T[i] = 0.f;
  for (int j = 0; j < NJ; ++j) {
    const float wj = w[j];
#pragma unroll
    for (int i = 0; i < 12; ++i) T[i] = fmaf(wj, a[j * 12 + i], T[i]);
  }
}

}  // namespace avc
