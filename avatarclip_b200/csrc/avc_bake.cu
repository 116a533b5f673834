// avc_bake.cu -- the texture atlas of a baked avatar (avatarclip_b200/bake.py): a closed-form per-face UV layout, the
// surface point behind every texel, the smooth vertex normals the textured glTF carries, and its tangent-space normal
// map.
//   k_bake_texel     per texel: owning face (or unused), clamped barycentrics at the texel centre, the surface point
//   k_bake_uv        per face: the UV of its three corners
//   k_bake_normals   per vertex: sum of the un-normalised face cross products in CSR order (no float atomics), normalised
//   k_bake_tangents  per face: dP/du Gram-Schmidt'd against each corner's normal, and the handedness w
//   k_bake_frames    per used texel: the interpolated (T, B, N) frame at the texel centre
//   k_snap_*         per used texel: the search samples along N, the sign-change bracket nearest t = 0, bisection
//   k_normal_encode  per used texel: the SDF gradient in the texel's frame, as RGB bytes
// Semantics in include/avc_b200.h.
#include <math.h>

#include "avc_common.cuh"

using namespace avc;

namespace {

constexpr int kThreads = 256;
constexpr int kMinCell = 8;          // texels per cell side: the two inset triangles need legs of at least 4 texels
constexpr int kMaxTexture = 16384;   // T * T texel indices fit int32

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
// The owner of texel t (x = t mod T, y = t / T), or -1 for an unused texel, with its corners vi and its centre (px, py)
// in the owner's (mirrored) cell frame.  k_bake_texel and k_bake_frames share it and texel_bary, so a texel's frame is
// taken at exactly the point avc_bake_texel_points writes.
__device__ __forceinline__ int texel_owner(const int* __restrict__ faces, const Atlas& a, long long t, int (&vi)[3],
                                           float& px, float& py) {
  const int y = (int)(t / a.T), x = (int)(t - (long long)y * a.T);
  const int q = x / a.c, r = y / a.c;
  int f = -1;
  px = 0.f, py = 0.f;
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
  vi[0] = vi[1] = vi[2] = 0;
  if (f >= 0) {
    vi[0] = faces[(size_t)f * 3], vi[1] = faces[(size_t)f * 3 + 1], vi[2] = faces[(size_t)f * 3 + 2];
    if ((unsigned)vi[0] >= (unsigned)a.V || (unsigned)vi[1] >= (unsigned)a.V || (unsigned)vi[2] >= (unsigned)a.V)
      f = -1;
  }
  return f;
}

// The clamped barycentrics of the cell-frame point (px, py) in the owner's UV triangle.
__device__ __forceinline__ void texel_bary(const Atlas& a, float px, float py, float (&b)[3]) {
  const float inv_l = 1.f / (float)(a.c - 4);
  const float be = (py - 1.f) * inv_l;
  const float al = (px - py - 2.f) * inv_l;
  float b0 = fmaxf(1.f - al - be, 0.f), b1 = fmaxf(al, 0.f), b2 = fmaxf(be, 0.f);
  const float s = 1.f / (b0 + b1 + b2);        // > 0: the unclamped weights sum to 1
  b[0] = b0 * s; b[1] = b1 * s; b[2] = b2 * s;
}

__global__ void __launch_bounds__(kThreads)
k_bake_texel(const float* __restrict__ verts, const int* __restrict__ faces, Atlas a, int* __restrict__ owner,
             float* __restrict__ points) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)a.T * a.T) return;
  int vi[3];
  float px, py;
  const int f = texel_owner(faces, a, t, vi, px, py);
  owner[t] = f;
  float* o = points + t * 3;
  if (f < 0) {
    o[0] = o[1] = o[2] = 0.f;
    return;
  }
  float b[3];
  texel_bary(a, px, py, b);
  const float* A = verts + (size_t)vi[0] * 3;
  const float* B = verts + (size_t)vi[1] * 3;
  const float* C = verts + (size_t)vi[2] * 3;
#pragma unroll
  for (int d = 0; d < 3; ++d) o[d] = b[0] * A[d] + b[1] * B[d] + b[2] * C[d];
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

// ---------------------------------------------------------------- normal map
constexpr int kSnapSamples = 16;     // K: samples of the search segment [-D, D]
constexpr float kMinGrad = 1e-6f;    // |grad sdf| below this bakes the flat normal

struct V3 {
  float x, y, z;
};
__device__ __forceinline__ V3 ld3(const float* p) { return {p[0], p[1], p[2]}; }
__device__ __forceinline__ V3 sub(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ V3 scl(V3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
__device__ __forceinline__ float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ V3 cross(V3 a, V3 b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}

// t Gram-Schmidt'd against the unit n and normalised; when that leaves |o| <= 1e-6 |t| (t = 0 or along n), the unit
// axis e of n's smallest |component| (the first of equals) Gram-Schmidt'd instead.
__device__ __forceinline__ V3 tangent_against(V3 t, V3 n) {
  V3 o = sub(t, scl(n, dot(t, n)));
  float len = sqrtf(dot(o, o));
  if (!(len > 1e-6f * sqrtf(dot(t, t)))) {
    const float ax = fabsf(n.x), ay = fabsf(n.y), az = fabsf(n.z);
    const V3 e = (ax <= ay && ax <= az) ? V3{1.f, 0.f, 0.f} : (ay <= az ? V3{0.f, 1.f, 0.f} : V3{0.f, 0.f, 1.f});
    o = sub(e, scl(n, dot(e, n)));
    len = sqrtf(dot(o, o));
  }
  return scl(o, 1.f / len);
}

__global__ void __launch_bounds__(kThreads)
k_bake_tangents(const float* __restrict__ verts, const int* __restrict__ faces, const float* __restrict__ normals,
                const float* __restrict__ uv, int F, float* __restrict__ tangents) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int vi[3] = {faces[(size_t)f * 3], faces[(size_t)f * 3 + 1], faces[(size_t)f * 3 + 2]};
  const V3 p0 = ld3(verts + (size_t)vi[0] * 3);
  const V3 e1 = sub(ld3(verts + (size_t)vi[1] * 3), p0), e2 = sub(ld3(verts + (size_t)vi[2] * 3), p0);
  const float* w = uv + (size_t)f * 6;
  const float du1 = w[2] - w[0], dv1 = w[3] - w[1], du2 = w[4] - w[0], dv2 = w[5] - w[1];
  const float det = du1 * dv2 - du2 * dv1;
  const float sg = det < 0.f ? -1.f : 1.f;
  const V3 tf = scl(sub(scl(e1, dv2), scl(e2, dv1)), sg);     // dP/du times |det|
  const V3 bv = scl(sub(scl(e2, du1), scl(e1, du2)), sg);     // dP/dv times |det|
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const V3 n = ld3(normals + (size_t)vi[k] * 3);
    const V3 t = tangent_against(tf, n);
    float* o = tangents + ((size_t)f * 3 + k) * 4;
    o[0] = t.x; o[1] = t.y; o[2] = t.z;
    o[3] = (det != 0.f && dot(cross(n, t), bv) > 0.f) ? -1.f : 1.f;
  }
}

// frames [n][3][3]: rows T, B, N of texel texels[i]; all 0 for an unused texel
__global__ void __launch_bounds__(kThreads)
k_bake_frames(const int* __restrict__ faces, const float* __restrict__ normals, const float* __restrict__ tangents,
              Atlas a, const int* __restrict__ texels, int n, float* __restrict__ frames) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float* o = frames + (size_t)i * 9;
  const int t = texels[i];
  int vi[3];
  float px, py, b[3];
  const int f = (unsigned)t < (unsigned)a.T * (unsigned)a.T ? texel_owner(faces, a, t, vi, px, py) : -1;
  if (f < 0) {
#pragma unroll
    for (int d = 0; d < 9; ++d) o[d] = 0.f;
    return;
  }
  texel_bary(a, px, py, b);
  V3 N{0.f, 0.f, 0.f}, Ti{0.f, 0.f, 0.f};
  float w = 0.f;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const V3 nk = ld3(normals + (size_t)vi[k] * 3);
    const float* tk = tangents + ((size_t)f * 3 + k) * 4;
    N = {N.x + b[k] * nk.x, N.y + b[k] * nk.y, N.z + b[k] * nk.z};
    Ti = {Ti.x + b[k] * tk[0], Ti.y + b[k] * tk[1], Ti.z + b[k] * tk[2]};
    w += b[k] * tk[3];
  }
  const float len = sqrtf(dot(N, N));
  N = len > 0.f ? scl(N, 1.f / len) : V3{0.f, 1.f, 0.f};
  const V3 T = tangent_against(Ti, N);
  const V3 B = scl(cross(N, T), w >= 0.f ? 1.f : -1.f);
  o[0] = T.x; o[1] = T.y; o[2] = T.z;
  o[3] = B.x; o[4] = B.y; o[5] = B.z;
  o[6] = N.x; o[7] = N.y; o[8] = N.z;
}

// t_k = (2k - 15) D / 15, the k-th of the K equally spaced search offsets
__device__ __forceinline__ float snap_t(int k, float D) {
  return (float)(2 * k - (kSnapSamples - 1)) * D / (float)(kSnapSamples - 1);
}

__device__ __forceinline__ void along(const float* __restrict__ p, const float* __restrict__ frame, float t,
                                      float* __restrict__ o) {
  o[0] = p[0] + t * frame[6];
  o[1] = p[1] + t * frame[7];
  o[2] = p[2] + t * frame[8];
}

__global__ void __launch_bounds__(kThreads)
k_snap_samples(const float* __restrict__ points, const float* __restrict__ frames, int n, float D,
               float* __restrict__ samples) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= (long long)n * kSnapSamples) return;
  const int i = (int)(j / kSnapSamples), k = (int)(j - (long long)i * kSnapSamples);
  along(points + (size_t)i * 3, frames + (size_t)i * 9, snap_t(k, D), samples + j * 3);
}

// Candidates on the position scale p = 0 .. 2K - 2: sample k (p = 2k) when its sdf is exactly 0, the interval
// [t_k, t_k+1] (p = 2k + 1) when its ends have strictly opposite signs.  The winner has the least |p - (K - 1)| (the
// distance from t = 0), the larger p on a tie.
__global__ void __launch_bounds__(kThreads)
k_snap_bracket(const float* __restrict__ sdf, int n, float D, float2* __restrict__ bracket, int* __restrict__ state) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* s = sdf + (size_t)i * kSnapSamples;
  int best = -1, best_key = 1 << 30;
  float prev = s[0];
  if (prev == 0.f) best = 0, best_key = kSnapSamples - 1;
#pragma unroll
  for (int k = 1; k < kSnapSamples; ++k) {
    const float cur = s[k];
    const int pi = 2 * k - 1, pk = 2 * k;
    if (((prev < 0.f && cur > 0.f) || (prev > 0.f && cur < 0.f)) && abs(pi - (kSnapSamples - 1)) <= best_key)
      best = pi, best_key = abs(pi - (kSnapSamples - 1));
    if (cur == 0.f && abs(pk - (kSnapSamples - 1)) <= best_key) best = pk, best_key = abs(pk - (kSnapSamples - 1));
    prev = cur;
  }
  if (best < 0) {
    bracket[i] = make_float2(0.f, 0.f);
    state[i] = 0;
  } else if (best & 1) {
    const int k = best >> 1;
    bracket[i] = make_float2(snap_t(k, D), snap_t(k + 1, D));
    state[i] = s[k] < 0.f ? 1 : 2;
  } else {
    const float t = snap_t(best >> 1, D);
    bracket[i] = make_float2(t, t);
    state[i] = 1;
  }
}

__device__ __forceinline__ float mid(float2 b) { return (b.x + b.y) * 0.5f; }

__global__ void __launch_bounds__(kThreads)
k_snap_midpoints(const float* __restrict__ points, const float* __restrict__ frames,
                 const float2* __restrict__ bracket, int n, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  along(points + (size_t)i * 3, frames + (size_t)i * 9, mid(bracket[i]), out + (size_t)i * 3);
}

__global__ void __launch_bounds__(kThreads)
k_snap_bisect(const float* __restrict__ sdf_mid, int n, float2* __restrict__ bracket, const int* __restrict__ state) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int st = state[i];
  if (st == 0) return;
  float2 b = bracket[i];
  const float m = mid(b), s = sdf_mid[i];
  if (s == 0.f) b = make_float2(m, m);
  else if ((s < 0.f) == (st == 1)) b.x = m;
  else b.y = m;
  bracket[i] = b;
}

__global__ void __launch_bounds__(kThreads)
k_normal_encode(const float* __restrict__ frames, const float* __restrict__ grad, const int* __restrict__ state,
                const int* __restrict__ texels, int n, unsigned TT, unsigned char* __restrict__ image,
                int* __restrict__ counts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned t = (unsigned)texels[i];
  if (t >= TT) return;
  const V3 g = ld3(grad + (size_t)i * 3);
  const float len = sqrtf(dot(g, g));
  unsigned char* o = image + (size_t)t * 3;
  if (state[i] == 0 || !(len >= kMinGrad)) {
    o[0] = 128; o[1] = 128; o[2] = 255;
    atomicAdd(counts, 1);
    return;
  }
  const V3 nn = scl(g, 1.f / len);
  const float* fr = frames + (size_t)i * 9;
  const float c[3] = {dot(ld3(fr), nn), dot(ld3(fr + 3), nn), dot(ld3(fr + 6), nn)};
#pragma unroll
  for (int d = 0; d < 3; ++d) o[d] = (unsigned char)fminf(fmaxf(rintf(127.5f * c[d] + 127.5f), 0.f), 255.f);
  if (c[2] <= 0.f) atomicAdd(counts + 1, 1);
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
  k_bake_texel<<<ceil_div((long long)T * T, kThreads), kThreads, 0, st>>>(verts, faces, a, owner, points);
  if (uv) k_bake_uv<<<ceil_div(F, kThreads), kThreads, 0, st>>>(a, uv);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_bake_vertex_normals(const float* verts, const int32_t* faces, const int32_t* offsets, const int32_t* vf,
                            int32_t V, int32_t F, float* normals, avc_stream_t stream) {
  if (!verts || !faces || !offsets || !vf || !normals) return AVC_E_NULL;
  if (V < 1 || F < 1 || F > (1 << 29)) return AVC_E_SIZE;
  k_bake_normals<<<ceil_div(V, kThreads), kThreads, 0, (cudaStream_t)stream>>>(verts, faces, offsets, vf, V, normals);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_bake_corner_tangents(const float* verts, const int32_t* faces, const float* normals, const float* uv,
                             int32_t V, int32_t F, float* tangents, avc_stream_t stream) {
  if (!verts || !faces || !normals || !uv || !tangents) return AVC_E_NULL;
  if (V < 1 || F < 1 || F > (1 << 29)) return AVC_E_SIZE;
  k_bake_tangents<<<ceil_div(F, kThreads), kThreads, 0, (cudaStream_t)stream>>>(verts, faces, normals, uv, F, tangents);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_bake_texel_frames(const int32_t* faces, const float* normals, const float* tangents, int32_t V, int32_t F,
                          int32_t T, const int32_t* texels, int32_t n, float* frames, avc_stream_t stream) {
  if (!faces || !normals || !tangents || !texels || !frames) return AVC_E_NULL;
  if (V < 1 || n < 1) return AVC_E_SIZE;
  int32_t m = 0, c = 0;
  AVC_TRY(avc_bake_atlas_grid(F, T, &m, &c));
  const Atlas a{F, V, T, m, c};
  k_bake_frames<<<ceil_div(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(faces, normals, tangents, a, texels, n,
                                                                               frames);
  AVC_LAUNCH_TRY();
  return 0;
}

static bool snap_d_ok(float D) { return D > 0.f && D <= 3.0e38f; }

int avc_bake_snap_samples(const float* points, const float* frames, int32_t n, float D, float* samples,
                          avc_stream_t stream) {
  if (!points || !frames || !samples) return AVC_E_NULL;
  if (n < 1) return AVC_E_SIZE;
  if (!snap_d_ok(D)) return AVC_E_BADCFG;
  k_snap_samples<<<ceil_div((long long)n * kSnapSamples, kThreads), kThreads, 0, (cudaStream_t)stream>>>(points, frames,
                                                                                                      n, D, samples);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_bake_snap_bracket(const float* sdf, int32_t n, float D, float* bracket, int32_t* state, avc_stream_t stream) {
  if (!sdf || !bracket || !state) return AVC_E_NULL;
  if (n < 1) return AVC_E_SIZE;
  if (!snap_d_ok(D)) return AVC_E_BADCFG;
  k_snap_bracket<<<ceil_div(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(sdf, n, D, (float2*)bracket, state);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_bake_snap_midpoints(const float* points, const float* frames, const float* bracket, int32_t n, float* out,
                            avc_stream_t stream) {
  if (!points || !frames || !bracket || !out) return AVC_E_NULL;
  if (n < 1) return AVC_E_SIZE;
  k_snap_midpoints<<<ceil_div(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(points, frames, (const float2*)bracket,
                                                                                  n, out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_bake_snap_bisect(const float* sdf_mid, int32_t n, float* bracket, const int32_t* state, avc_stream_t stream) {
  if (!sdf_mid || !bracket || !state) return AVC_E_NULL;
  if (n < 1) return AVC_E_SIZE;
  k_snap_bisect<<<ceil_div(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(sdf_mid, n, (float2*)bracket, state);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_bake_normal_encode(const float* frames, const float* grad, const int32_t* state, const int32_t* texels,
                           int32_t n, int32_t T, uint8_t* image, int32_t* counts, avc_stream_t stream) {
  if (!frames || !grad || !state || !texels || !image || !counts) return AVC_E_NULL;
  if (n < 1 || T < 1 || T > kMaxTexture) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  AVC_CUDA_TRY(cudaMemsetAsync(counts, 0, 2 * sizeof(int32_t), st));
  k_normal_encode<<<ceil_div(n, kThreads), kThreads, 0, st>>>(frames, grad, state, texels, n, (unsigned)T * (unsigned)T,
                                                              image, counts);
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"
