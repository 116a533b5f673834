// avc_lbs.cu -- SMPL linear-blend skinning as AvatarCLIP uses it: my_lbs / batch_rodrigues
// (AvatarGen/AppearanceGen/models/utils.py:72-106,176-224) with smplx's vertices2joints / batch_rigid_transform
// (in-tree copies: drive.py:51-160).  Two launches:
//   k_lbs_joints_chain  one CTA: joint regression by warp-shuffle reductions (one warp per joint at a time), then
//                       warp 0 walks the kinematic tree (both from avc_smpl.cuh)
//   k_lbs_skin          one thread per vertex: pose blend shapes (207-term dot against coalesced posedirs columns),
//                       blended 3x4 transform from the 24 joint transforms held in shared memory, skinned vertex
// Also defines k_smpl_joints (declared in avc_smpl.cuh), the joint regression that avc_lbs_rel_transforms and
// avc_smpl_pose_batch launch.
#include "avc_smpl.cuh"

using namespace avc;

__global__ void __launch_bounds__(256)
avc::k_smpl_joints(const float* __restrict__ v_template, const float* __restrict__ J_regressor, int V, int NJ,
                   float* __restrict__ J) {
  regress_joints(v_template, J_regressor, V, NJ, J);
}

namespace {

__global__ void __launch_bounds__(256)
k_lbs_joints_chain(const float* __restrict__ v_shaped, const float* __restrict__ pose, int pose2rot,
                   const float* __restrict__ J_regressor, const int* __restrict__ parents, int V, int NJ,
                   float* __restrict__ A_out /*[NJ][12]*/, float* __restrict__ joints_out /*[NJ][3]*/,
                   float* __restrict__ feat_out /*[(NJ-1)*9]*/) {
  __shared__ float sJ[NJ_MAX][3];
  regress_joints(v_shaped, J_regressor, V, NJ, &sJ[0][0]);
  __syncthreads();
  if ((threadIdx.x >> 5) != 0) return;
  // ---- lane j <-> joint j
  const int j = threadIdx.x & 31;
  const bool act = j < NJ;
  float R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (act) {
    if (pose2rot) {
      rodrigues(pose[j * 3], pose[j * 3 + 1], pose[j * 3 + 2], R);
    } else {
      for (int i = 0; i < 9; ++i) R[i] = pose[j * 9 + i];
    }
    if (j >= 1)
      for (int i = 0; i < 9; ++i) feat_out[(j - 1) * 9 + i] = R[i] - ((i % 4 == 0) ? 1.f : 0.f);   // pose_feature (:193)
  }
  const int par = act ? parents[j] : -1;
  const float Jx = act ? sJ[j][0] : 0.f, Jy = act ? sJ[j][1] : 0.f, Jz = act ? sJ[j][2] : 0.f;
  float T[12];
  chain_world(R, j, par, act, Jx, Jy, Jz, T);
  if (act) {
    joints_out[j * 3 + 0] = T[3]; joints_out[j * 3 + 1] = T[7]; joints_out[j * 3 + 2] = T[11];   // posed joints (:140)
    rel_transform(T, Jx, Jy, Jz, A_out + j * 12);
  }
}

__global__ void __launch_bounds__(256)
k_lbs_skin(const float* __restrict__ v_shaped, const float* __restrict__ posedirs, const float* __restrict__ feat,
           const float* __restrict__ A, const float* __restrict__ lbs_weights, int V, int NJ, int NF,
           float* __restrict__ verts) {
  __shared__ float sA[NJ_MAX * 12];
  __shared__ float sF[NJ_MAX * 9];
  for (int i = threadIdx.x; i < NJ * 12; i += blockDim.x) sA[i] = A[i];
  for (int i = threadIdx.x; i < NF; i += blockDim.x) sF[i] = feat[i];
  __syncthreads();
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  // pose blend shapes: v_posed = v_shaped + pose_feature @ posedirs   (models/utils.py:195-205)
  float p0 = v_shaped[v * 3], p1 = v_shaped[v * 3 + 1], p2 = v_shaped[v * 3 + 2];
  const size_t ld = (size_t)V * 3;
  for (int k = 0; k < NF; ++k) {
    const float f = sF[k];
    const float* pd = posedirs + (size_t)k * ld + (size_t)v * 3;
    p0 = fmaf(f, pd[0], p0); p1 = fmaf(f, pd[1], p1); p2 = fmaf(f, pd[2], p2);
  }
  // T = sum_j W[v,j] A_j ; verts = T [v_posed; 1]   (:213-222)
  float T[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) T[i] = 0.f;
  for (int j = 0; j < NJ; ++j) {
    const float w = lbs_weights[(size_t)v * NJ + j];
#pragma unroll
    for (int i = 0; i < 12; ++i) T[i] = fmaf(w, sA[j * 12 + i], T[i]);
  }
  verts[v * 3 + 0] = T[0] * p0 + T[1] * p1 + T[2] * p2 + T[3];
  verts[v * 3 + 1] = T[4] * p0 + T[5] * p1 + T[6] * p2 + T[7];
  verts[v * 3 + 2] = T[8] * p0 + T[9] * p1 + T[10] * p2 + T[11];
}

}  // namespace

extern "C" {

int avc_lbs_workspace_bytes(int32_t n_joints, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (n_joints < 1 || n_joints > NJ_MAX) return AVC_E_BADCFG;
  *bytes = sizeof(float) * (size_t)(n_joints * 12 + n_joints * 9 + 64);
  return 0;
}

int avc_lbs_fwd(const float* v_shaped, const float* pose, int32_t pose2rot, const float* J_regressor,
                const int32_t* parents, const float* posedirs, const float* lbs_weights, int32_t V, int32_t n_joints,
                float* verts_out, float* joints_out, void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!v_shaped || !pose || !J_regressor || !parents || !posedirs || !lbs_weights || !verts_out || !joints_out || !workspace)
    return AVC_E_NULL;
  if (V < 1) return AVC_E_SIZE;
  size_t need = 0;
  AVC_TRY(avc_lbs_workspace_bytes(n_joints, &need));
  if (workspace_bytes < need) return AVC_E_SIZE;
  float* A = (float*)workspace;
  float* feat = A + n_joints * 12;
  cudaStream_t st = (cudaStream_t)stream;
  k_lbs_joints_chain<<<1, 256, 0, st>>>(v_shaped, pose, pose2rot, J_regressor, parents, V, n_joints, A, joints_out, feat);
  k_lbs_skin<<<(V + 255) / 256, 256, 0, st>>>(v_shaped, posedirs, feat, A, lbs_weights, V, n_joints, (n_joints - 1) * 9,
                                              verts_out);
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"
