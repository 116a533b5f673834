// avc_bake.cu -- the texture atlas of a baked avatar (avatarclip_b200/bake.py): a closed-form per-face UV layout, the
// surface point behind every texel, and the smooth vertex normals the textured glTF carries.
//   k_bake_texel     per texel: owning face (or unused), clamped barycentrics at the texel centre, the surface point
//   k_bake_uv        per face: the UV of its three corners
//   k_bake_normals   per vertex: sum of the un-normalised face cross products in CSR order (no float atomics), normalised
// Semantics in include/avc_b200.h.
#include <math.h>

#include "avc_common.cuh"

using namespace avc;

namespace {

constexpr int kThreads = 256;
constexpr int kMinCell = 8;          // texels per cell side: the two inset triangles need legs of at least 4 texels
constexpr int kMaxTexture = 16384;   // T * T texel indices fit int32

inline unsigned blocks(long long n, int t) { return (unsigned)((n + t - 1) / t); }

// m = ceil(sqrt(ceil(F / 2))) in integers
int grid_side(int32_t F) {
  const long long n = ((long long)F + 1) / 2;
  long long m = (long long)sqrt((double)n);
  while (m * m < n) ++m;
  while (m > 1 && (m - 1) * (m - 1) >= n) --m;
  return (int)m;
}

struct Atlas {
  int F, V, T, m, c;
};

// Cell-local layout (x right, y down, in texels; texel (i, j) covers [i, i + 1) x [j, j + 1)).  Face 2k owns the texels
// with i >= j and maps its corners to (3, 1), (c - 1, 1), (c - 1, c - 3); face 2k + 1 owns i < j and is the mirror image
// across the diagonal.  In the owner's (mirrored) frame p = P0 + a (P1 - P0) + b (P2 - P0) with P1 - P0 = (L, 0) and
// P2 - P0 = (L, L), L = c - 4.
__global__ void __launch_bounds__(kThreads)
k_bake_texel(const float* __restrict__ verts, const int* __restrict__ faces, Atlas a, int* __restrict__ owner,
             float* __restrict__ points) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)a.T * a.T) return;
  const int y = (int)(t / a.T), x = (int)(t - (long long)y * a.T);
  const int q = x / a.c, r = y / a.c;
  int f = -1;
  float px = 0.f, py = 0.f;
  if (q < a.m && r < a.m) {
    const int i = x - q * a.c, j = y - r * a.c;
    const int side = i >= j ? 0 : 1;
    const long long ff = 2LL * ((long long)r * a.m + q) + side;
    if (ff < a.F) {
      f = (int)ff;
      px = (side ? j : i) + 0.5f;
      py = (side ? i : j) + 0.5f;
    }
  }
  int i0 = 0, i1 = 0, i2 = 0;
  if (f >= 0) {
    i0 = faces[(size_t)f * 3], i1 = faces[(size_t)f * 3 + 1], i2 = faces[(size_t)f * 3 + 2];
    if ((unsigned)i0 >= (unsigned)a.V || (unsigned)i1 >= (unsigned)a.V || (unsigned)i2 >= (unsigned)a.V) f = -1;
  }
  owner[t] = f;
  float* o = points + t * 3;
  if (f < 0) {
    o[0] = o[1] = o[2] = 0.f;
    return;
  }
  const float inv_l = 1.f / (float)(a.c - 4);
  const float be = (py - 1.f) * inv_l;
  const float al = (px - py - 2.f) * inv_l;
  float b0 = fmaxf(1.f - al - be, 0.f), b1 = fmaxf(al, 0.f), b2 = fmaxf(be, 0.f);
  const float s = 1.f / (b0 + b1 + b2);        // > 0: the unclamped weights sum to 1
  b0 *= s; b1 *= s; b2 *= s;
  const float* A = verts + (size_t)i0 * 3;
  const float* B = verts + (size_t)i1 * 3;
  const float* C = verts + (size_t)i2 * 3;
#pragma unroll
  for (int d = 0; d < 3; ++d) o[d] = b0 * A[d] + b1 * B[d] + b2 * C[d];
}

__global__ void __launch_bounds__(kThreads) k_bake_uv(Atlas a, float* __restrict__ uv) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= a.F) return;
  const int k = f >> 1, side = f & 1;
  const int r = k / a.m, q = k - r * a.m;
  const float c = (float)a.c, inv_t = 1.f / (float)a.T;
  const float ox = (float)(q * a.c), oy = (float)(r * a.c);
  const float P[3][2] = {{3.f, 1.f}, {c - 1.f, 1.f}, {c - 1.f, c - 3.f}};
  float* o = uv + (size_t)f * 6;
#pragma unroll
  for (int v = 0; v < 3; ++v) {
    const float lx = side ? P[v][1] : P[v][0], ly = side ? P[v][0] : P[v][1];
    o[2 * v] = (ox + lx) * inv_t;
    o[2 * v + 1] = (oy + ly) * inv_t;
  }
}

__global__ void __launch_bounds__(kThreads)
k_bake_normals(const float* __restrict__ verts, const int* __restrict__ faces, const int* __restrict__ offsets,
               const int* __restrict__ vf, int V, float* __restrict__ normals) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  float nx = 0.f, ny = 0.f, nz = 0.f;
  for (int j = offsets[v], e = offsets[v + 1]; j < e; ++j) {
    const int f = vf[j];
    const float* a = verts + (size_t)faces[(size_t)f * 3] * 3;
    const float* b = verts + (size_t)faces[(size_t)f * 3 + 1] * 3;
    const float* d = verts + (size_t)faces[(size_t)f * 3 + 2] * 3;
    const float ux = b[0] - a[0], uy = b[1] - a[1], uz = b[2] - a[2];
    const float wx = d[0] - a[0], wy = d[1] - a[1], wz = d[2] - a[2];
    nx += uy * wz - uz * wy;
    ny += uz * wx - ux * wz;
    nz += ux * wy - uy * wx;
  }
  const float len = sqrtf(nx * nx + ny * ny + nz * nz);
  float* o = normals + (size_t)v * 3;
  if (len > 0.f) {
    o[0] = nx / len; o[1] = ny / len; o[2] = nz / len;
  } else {
    o[0] = 0.f; o[1] = 1.f; o[2] = 0.f;
  }
}

}  // namespace

extern "C" {

int avc_bake_atlas_grid(int32_t F, int32_t T, int32_t* m, int32_t* c) {
  if (!m || !c) return AVC_E_NULL;
  if (F < 1 || F > (1 << 30) || T < 1 || T > kMaxTexture) return AVC_E_SIZE;
  *m = grid_side(F);
  *c = T / *m;
  return *c < kMinCell ? AVC_E_BADCFG : 0;
}

int avc_bake_texel_points(const float* verts, const int32_t* faces, int32_t V, int32_t F, int32_t T, int32_t* owner,
                          float* points, float* uv, avc_stream_t stream) {
  if (!verts || !faces || !owner || !points) return AVC_E_NULL;
  if (V < 1) return AVC_E_SIZE;
  int32_t m = 0, c = 0;
  AVC_TRY(avc_bake_atlas_grid(F, T, &m, &c));
  cudaStream_t st = (cudaStream_t)stream;
  const Atlas a{F, V, T, m, c};
  k_bake_texel<<<blocks((long long)T * T, kThreads), kThreads, 0, st>>>(verts, faces, a, owner, points);
  if (uv) k_bake_uv<<<blocks(F, kThreads), kThreads, 0, st>>>(a, uv);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_bake_vertex_normals(const float* verts, const int32_t* faces, const int32_t* offsets, const int32_t* vf,
                            int32_t V, int32_t F, float* normals, avc_stream_t stream) {
  if (!verts || !faces || !offsets || !vf || !normals) return AVC_E_NULL;
  if (V < 1 || F < 1 || F > (1 << 29)) return AVC_E_SIZE;
  k_bake_normals<<<blocks(V, kThreads), kThreads, 0, (cudaStream_t)stream>>>(verts, faces, offsets, vf, V, normals);
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"
