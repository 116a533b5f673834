// avc_drive.cu -- the animation step after the exported mesh: AvatarGen/AppearanceGen/drive.py's cleanup_mesh (:172-210),
// find_nearest_ind (:235-240), inv_lbs (:242-253) and lbs (:255-265) over a motion sequence.
//   k_nearest_vertex    exact argmin of the squared distance to a reference point set, in fp64 (drive.py) or fp32
//                       (Avatar2FBX's find_nearest_ind); reference points staged through shared memory in tiles,
//                       NN_QPT query points per thread held in registers
//   k_cc_*              connected components of the triangle-edge graph: lock-free union-find (hook the larger root
//                       under the smaller by CAS, path halving), flatten + atomicAdd sizes, one 64-bit atomicMax picks
//                       the largest component (ties: smallest minimum vertex index, the reference's discovery order)
//   k_smpl_joints       J = J_regressor . v_template (avc_smpl.cuh)
//   k_drive_chain       one warp per frame: rotations (or batch_rodrigues of axis-angle), then avc_smpl.cuh's kinematic
//                       chain, A[f][j][3x4]
//   k_inv_lbs           T = sum_j w_j A_j (fp64), p_T = M^-1 (p - t / s) in fp64 (torch.inverse(T) . [p; 1], rows 0-2)
//   k_skin_frames       out[f][v] = (sum_j w_j A[f]_j) . [p_T; 1] for a range of frames, in the PC2 payload layout
#include "avc_smpl.cuh"

using namespace avc;

namespace {

// ---------------------------------------------------------------- nearest vertex (drive.py:235-240)
constexpr int NN_THREADS = 128, NN_QPT = 4, NN_TILE = 256;

// The distance arithmetic of numpy's ((tv - v) ** 2).sum(-1) in the precision T of its operands: every op rounded on
// its own (no contraction into FMAs).  double: drive.py (float32 template minus float64 points); float: Avatar2FBX's
// ply_utils.py:84-89 (both operands float32).
template <typename T> struct NnOps;
template <> struct NnOps<double> {
  static __device__ __forceinline__ double inf() { return __longlong_as_double(0x7ff0000000000000ll); }
  static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
};
template <> struct NnOps<float> {
  static __device__ __forceinline__ float inf() { return __int_as_float(0x7f800000); }
  static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
};

template <typename T>
__global__ void __launch_bounds__(NN_THREADS)
k_nearest_vertex(const float* __restrict__ query, int N, const float* __restrict__ ref, int M,
                 int32_t* __restrict__ nearest) {
  using O = NnOps<T>;
  __shared__ T sR[NN_TILE * 3];
  T qx[NN_QPT], qy[NN_QPT], qz[NN_QPT], best[NN_QPT];
  int bi[NN_QPT];
  const int base = blockIdx.x * (NN_THREADS * NN_QPT) + threadIdx.x;
#pragma unroll
  for (int k = 0; k < NN_QPT; ++k) {
    const int i = base + k * NN_THREADS;
    const bool ok = i < N;
    qx[k] = ok ? (T)query[(size_t)i * 3 + 0] : (T)0;
    qy[k] = ok ? (T)query[(size_t)i * 3 + 1] : (T)0;
    qz[k] = ok ? (T)query[(size_t)i * 3 + 2] : (T)0;
    best[k] = O::inf();
    bi[k] = 0;
  }
  for (int t0 = 0; t0 < M; t0 += NN_TILE) {
    const int n = min(NN_TILE, M - t0);
    __syncthreads();
    for (int i = threadIdx.x; i < n * 3; i += NN_THREADS) sR[i] = (T)ref[(size_t)t0 * 3 + i];
    __syncthreads();
#pragma unroll 2
    for (int j = 0; j < n; ++j) {
      const T rx = sR[j * 3], ry = sR[j * 3 + 1], rz = sR[j * 3 + 2];
#pragma unroll
      for (int k = 0; k < NN_QPT; ++k) {
        // numpy: ((tv - v) ** 2).sum(-1) = (dx*dx + dy*dy) + dz*dz, each op rounded (no FMA)
        const T dx = O::sub(rx, qx[k]), dy = O::sub(ry, qy[k]), dz = O::sub(rz, qz[k]);
        const T d = O::add(O::add(O::mul(dx, dx), O::mul(dy, dy)), O::mul(dz, dz));
        if (d < best[k]) { best[k] = d; bi[k] = t0 + j; }      // strict <, increasing index: ties keep the first
      }
    }
  }
#pragma unroll
  for (int k = 0; k < NN_QPT; ++k) {
    const int i = base + k * NN_THREADS;
    if (i < N) nearest[i] = bi[k];
  }
}

// ---------------------------------------------------------------- connected components (drive.py:172-210)
// Invariant: parent[v] <= v, and parent[v] == v exactly at roots, so a root is the smallest index of its tree.
__device__ __forceinline__ int cc_root(volatile int* parent, int v) {
  int cur = parent[v];
  if (cur != v) {
    int prev = v, next;
    while (cur > (next = parent[cur])) {
      parent[prev] = next;        // path halving: only ever points a non-root further up its own tree
      prev = cur;
      cur = next;
    }
  }
  return cur;
}

__device__ __forceinline__ void cc_union(int* parent, int a, int b) {
  int ra = cc_root(parent, a), rb = cc_root(parent, b);
  while (ra != rb) {
    if (ra < rb) { int t = ra; ra = rb; rb = t; }
    const int old = atomicCAS(parent + ra, ra, rb);   // hook the larger root under the smaller one
    if (old == ra) break;
    ra = cc_root(parent, old);                        // ra stopped being a root meanwhile: climb and retry
    rb = cc_root(parent, rb);
  }
}

__global__ void k_cc_init(int V, int* __restrict__ labels, int* __restrict__ sizes, unsigned long long* __restrict__ key) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) { labels[v] = v; sizes[v] = 0; }
  if (v == 0) *key = 0ull;
}

__global__ void k_cc_hook(const int32_t* __restrict__ faces, int F, int V, int* labels) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= F) return;
  const int a = faces[(size_t)t * 3], b = faces[(size_t)t * 3 + 1], c = faces[(size_t)t * 3 + 2];
  if ((unsigned)a >= (unsigned)V || (unsigned)b >= (unsigned)V || (unsigned)c >= (unsigned)V) return;
  cc_union(labels, a, b);     // edge (c, a) joins nothing that (a, b) and (b, c) have not joined
  cc_union(labels, b, c);
}

// No path halving here: a halving write parent[prev] = next could land after prev's own thread stored its root, leaving
// prev labelled with an inner node of its tree.  Every write of this pass stores a root, so the walk always ends there.
__device__ __forceinline__ int cc_find(const volatile int* parent, int v) {
  int cur = v, next;
  while ((next = parent[cur]) != cur) cur = next;
  return cur;
}

__global__ void k_cc_flatten(int V, int* labels, int* __restrict__ sizes) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int r = cc_find(labels, v);
  labels[v] = r;
  atomicAdd(sizes + r, 1);
}

__global__ void k_cc_best(int V, const int* __restrict__ labels, const int* __restrict__ sizes,
                          unsigned long long* __restrict__ key) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V || labels[v] != v) return;
  // larger size wins; equal sizes: the smaller label (= smallest vertex index, the island the reference found first)
  atomicMax(key, ((unsigned long long)sizes[v] << 32) | (unsigned long long)(unsigned)(INT32_MAX - v));
}

__global__ void k_cc_kept(const unsigned long long* __restrict__ key, int32_t* __restrict__ kept) {
  const unsigned long long k = *key;
  kept[0] = INT32_MAX - (int)(unsigned)(k & 0xffffffffull);
  kept[1] = (int)(k >> 32);
}

// ---------------------------------------------------------------- rigid transforms (drive.py:93-148, batched)
constexpr int CHAIN_WARPS = 4;

__global__ void __launch_bounds__(CHAIN_WARPS * 32)
k_drive_chain(const float* __restrict__ joints, const float* __restrict__ pose, int pose2rot,
              const int32_t* __restrict__ parents, int NJ, int F, float* __restrict__ A_out /*[F][NJ][12]*/) {
  const int f = blockIdx.x * CHAIN_WARPS + (threadIdx.x >> 5);
  if (f >= F) return;                 // whole warps leave together
  const int j = threadIdx.x & 31;
  const bool act = j < NJ;
  float R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (act) {
    if (pose2rot) {
      const float* r = pose + ((size_t)f * NJ + j) * 3;
      rodrigues(r[0], r[1], r[2], R);
    } else {
      const float* r = pose + ((size_t)f * NJ + j) * 9;
#pragma unroll
      for (int i = 0; i < 9; ++i) R[i] = r[i];
    }
  }
  const int par = act ? parents[j] : -1;
  const float Jx = act ? joints[j * 3] : 0.f, Jy = act ? joints[j * 3 + 1] : 0.f, Jz = act ? joints[j * 3 + 2] : 0.f;
  float T[12];
  chain_world(R, j, par, act, Jx, Jy, Jz, T);
  if (act) rel_transform(T, Jx, Jy, Jz, A_out + ((size_t)f * NJ + j) * 12);
}

// ---------------------------------------------------------------- inverse LBS (drive.py:242-253)
__global__ void __launch_bounds__(256)
k_inv_lbs(const float* __restrict__ verts, const int32_t* __restrict__ nearest, int N,
          const float* __restrict__ weights, int NJ, const float* __restrict__ A, float* __restrict__ out) {
  __shared__ float sA[NJ_MAX * 12];
  for (int i = threadIdx.x; i < NJ * 12; i += blockDim.x) sA[i] = A[i];
  __syncthreads();
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N) return;
  const float* w = weights + (size_t)(nearest ? nearest[v] : v) * NJ;
  double T[12], s = 0.0;
#pragma unroll
  for (int i = 0; i < 12; ++i) T[i] = 0.0;
  for (int j = 0; j < NJ; ++j) {
    const double wj = (double)w[j];
    s += wj;                          // T's bottom row is [0, 0, 0, s]
#pragma unroll
    for (int i = 0; i < 12; ++i) T[i] = fma(wj, (double)sA[j * 12 + i], T[i]);
  }
  // torch.inverse(T) . [p; 1], rows 0-2, for T = [[M, t], [0, s]]:  M^-1 (p - t / s)
  const double qx = (double)verts[(size_t)v * 3 + 0] - T[3] / s;
  const double qy = (double)verts[(size_t)v * 3 + 1] - T[7] / s;
  const double qz = (double)verts[(size_t)v * 3 + 2] - T[11] / s;
  const double a = T[0], b = T[1], c = T[2], d = T[4], e = T[5], f = T[6], g = T[8], h = T[9], k = T[10];
  const double c00 = e * k - f * h, c01 = c * h - b * k, c02 = b * f - c * e;
  const double c10 = f * g - d * k, c11 = a * k - c * g, c12 = c * d - a * f;
  const double c20 = d * h - e * g, c21 = b * g - a * h, c22 = a * e - b * d;
  const double inv = 1.0 / (a * c00 + b * c10 + c * c20);
  out[(size_t)v * 3 + 0] = (float)((c00 * qx + c01 * qy + c02 * qz) * inv);
  out[(size_t)v * 3 + 1] = (float)((c10 * qx + c11 * qy + c12 * qz) * inv);
  out[(size_t)v * 3 + 2] = (float)((c20 * qx + c21 * qy + c22 * qz) * inv);
}

// ---------------------------------------------------------------- per-frame skinning (drive.py:255-265)
constexpr int SKIN_FRAMES = 16;   // frames per CTA, their transforms staged in shared memory

__global__ void __launch_bounds__(256)
k_skin_frames(const float* __restrict__ tpose, const int32_t* __restrict__ nearest, int N,
              const float* __restrict__ weights, int NJ, const float* __restrict__ A, int f_begin, int f_count,
              float* __restrict__ out) {
  __shared__ float sA[SKIN_FRAMES * NJ_MAX * 12];
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = v < N;
  float w[NJ_MAX];
  float px = 0.f, py = 0.f, pz = 0.f;
  {
    const float* wr = weights + (size_t)(live ? (nearest ? nearest[v] : v) : 0) * NJ;
#pragma unroll
    for (int j = 0; j < NJ_MAX; ++j) w[j] = (live && j < NJ) ? wr[j] : 0.f;
    if (live) { px = tpose[(size_t)v * 3]; py = tpose[(size_t)v * 3 + 1]; pz = tpose[(size_t)v * 3 + 2]; }
  }
  const int ngroups = (f_count + SKIN_FRAMES - 1) / SKIN_FRAMES;
  for (int gi = blockIdx.y; gi < ngroups; gi += gridDim.y) {
    const int g0 = gi * SKIN_FRAMES, nf = min(SKIN_FRAMES, f_count - g0);
    __syncthreads();
    for (int i = threadIdx.x; i < nf * NJ * 12; i += blockDim.x) sA[i] = A[((size_t)(f_begin + g0) * NJ) * 12 + i];
    __syncthreads();
    if (!live) continue;
    for (int fl = 0; fl < nf; ++fl) {
      const float* a = sA + fl * NJ * 12;
      float T[12];
#pragma unroll
      for (int i = 0; i < 12; ++i) T[i] = 0.f;
#pragma unroll
      for (int j = 0; j < NJ_MAX; ++j) {
        if (j < NJ) {
#pragma unroll
          for (int i = 0; i < 12; ++i) T[i] = fmaf(w[j], a[j * 12 + i], T[i]);
        }
      }
      float* o = out + ((size_t)(g0 + fl) * N + v) * 3;
      o[0] = T[0] * px + T[1] * py + T[2] * pz + T[3];
      o[1] = T[4] * px + T[5] * py + T[6] * pz + T[7];
      o[2] = T[8] * px + T[9] * py + T[10] * pz + T[11];
    }
  }
}

}  // namespace

extern "C" {

int avc_nearest_vertex(const float* query, int32_t N, const float* ref, int32_t M, int32_t* nearest, avc_stream_t stream) {
  if (!query || !ref || !nearest) return AVC_E_NULL;
  if (N < 1 || M < 1) return AVC_E_SIZE;
  k_nearest_vertex<double><<<ceil_div(N, NN_THREADS * NN_QPT), NN_THREADS, 0, (cudaStream_t)stream>>>(query, N, ref, M,
                                                                                                       nearest);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_nearest_vertex_f32(const float* query, int32_t N, const float* ref, int32_t M, int32_t* nearest,
                           avc_stream_t stream) {
  if (!query || !ref || !nearest) return AVC_E_NULL;
  if (N < 1 || M < 1) return AVC_E_SIZE;
  k_nearest_vertex<float><<<ceil_div(N, NN_THREADS * NN_QPT), NN_THREADS, 0, (cudaStream_t)stream>>>(query, N, ref, M,
                                                                                                      nearest);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_mesh_components_workspace_bytes(int32_t V, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (V < 1) return AVC_E_SIZE;
  *bytes = (((size_t)V * sizeof(int32_t) + 15) & ~(size_t)15) + 16;
  return 0;
}

int avc_mesh_components(const int32_t* faces, int32_t F, int32_t V, int32_t* labels, int32_t* kept, void* workspace,
                        size_t workspace_bytes, avc_stream_t stream) {
  if ((!faces && F > 0) || !labels || !kept || !workspace) return AVC_E_NULL;
  if (F < 0) return AVC_E_SIZE;
  size_t need = 0;
  AVC_TRY(avc_mesh_components_workspace_bytes(V, &need));
  if (workspace_bytes < need) return AVC_E_SIZE;
  int* sizes = (int*)workspace;
  unsigned long long* key = (unsigned long long*)((char*)workspace + need - 16);
  cudaStream_t st = (cudaStream_t)stream;
  k_cc_init<<<ceil_div(V, 256), 256, 0, st>>>(V, labels, sizes, key);
  if (F > 0) k_cc_hook<<<ceil_div(F, 256), 256, 0, st>>>(faces, F, V, labels);
  k_cc_flatten<<<ceil_div(V, 256), 256, 0, st>>>(V, labels, sizes);
  k_cc_best<<<ceil_div(V, 256), 256, 0, st>>>(V, labels, sizes, key);
  k_cc_kept<<<1, 1, 0, st>>>(key, kept);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_lbs_rel_transforms(const float* v_template, const float* J_regressor, const int32_t* parents, int32_t V,
                           int32_t n_joints, const float* pose, int32_t pose2rot, int32_t n_frames, float* joints_out,
                           float* A_out, avc_stream_t stream) {
  if (!v_template || !J_regressor || !parents || !pose || !joints_out || !A_out) return AVC_E_NULL;
  if (n_joints < 1 || n_joints > NJ_MAX) return AVC_E_BADCFG;
  if (V < 1 || n_frames < 1) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  k_smpl_joints<<<1, 256, 0, st>>>(v_template, J_regressor, V, n_joints, joints_out);
  k_drive_chain<<<ceil_div(n_frames, CHAIN_WARPS), CHAIN_WARPS * 32, 0, st>>>(joints_out, pose, pose2rot, parents,
                                                                              n_joints, n_frames, A_out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_inv_lbs(const float* verts, const int32_t* nearest, int32_t N, const float* lbs_weights, int32_t M,
                int32_t n_joints, const float* A, float* tpose_out, avc_stream_t stream) {
  if (!verts || !lbs_weights || !A || !tpose_out) return AVC_E_NULL;
  if (n_joints < 1 || n_joints > NJ_MAX) return AVC_E_BADCFG;
  if (N < 1 || M < 1 || (!nearest && M < N)) return AVC_E_SIZE;
  k_inv_lbs<<<ceil_div(N, 256), 256, 0, (cudaStream_t)stream>>>(verts, nearest, N, lbs_weights, n_joints, A, tpose_out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_lbs_frames(const float* tpose, const int32_t* nearest, int32_t N, const float* lbs_weights, int32_t M,
                   int32_t n_joints, const float* A, int32_t n_frames, int32_t frame_begin, int32_t frame_count,
                   float* out, avc_stream_t stream) {
  if (!tpose || !lbs_weights || !A || !out) return AVC_E_NULL;
  if (n_joints < 1 || n_joints > NJ_MAX) return AVC_E_BADCFG;
  if (N < 1 || M < 1 || (!nearest && M < N)) return AVC_E_SIZE;
  if (frame_begin < 0 || frame_count < 1 || frame_begin > n_frames - frame_count) return AVC_E_SIZE;
  const int groups = (frame_count + SKIN_FRAMES - 1) / SKIN_FRAMES;
  dim3 grid(ceil_div(N, 256), groups < 65535 ? groups : 65535);
  k_skin_frames<<<grid, 256, 0, (cudaStream_t)stream>>>(tpose, nearest, N, lbs_weights, n_joints, A, frame_begin,
                                                        frame_count, out);
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"
