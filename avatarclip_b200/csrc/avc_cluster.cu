// avc_cluster.cu -- Avatar2FBX's mesh simplification (utils/ply_utils.py:16-19): open3d's
// TriangleMesh::simplify_vertex_clustering(voxel_size = max(max_bound - min_bound) / 256, contraction = Average), on the
// device, in the order open3d produces (semantics in include/avc_b200.h).
//   k_cl_bounds        per-axis min / max of the positions (order-preserving int encoding, atomicMin / atomicMax)
//   k_cl_vkey          voxel of every vertex in fp64 (the bounds and voxel size recomputed per thread from the six
//                      reduced values, no host round trip), packed 21 bits per axis into a 64-bit key
//   k_cl_vinsert       open-addressing table of vertex ids keyed by voxel: CAS an empty slot, or atomicMin the id into
//                      the slot of the same voxel, so each slot ends holding the first vertex of its voxel
//   k_cl_flag          flags the first vertex of each voxel; exclusive_scan (avc_scan.cu, in index order) of the flags
//                      numbers the output vertices
//   k_cl_vaccum/final  fp64 position sums (exact for float32 inputs at mesh scale, so order-independent) and integer
//                      colour sums by atomics, then the means
//   k_cl_tremap        triangles to output vertices; two corners in one voxel -> dropped
//   k_cl_tinsert       the same table scheme keyed by the rotation that puts the smallest index first: each slot ends
//                      holding the first triangle of its rotation class (a reversed triangle is another class)
//   k_cl_flag/temit    kept triangles compacted in input order by exclusive_scan, each in the rotation it first
//                      appeared in
// Every stage is linear in V + F: no per-vertex or per-voxel loops over neighbours, so a fan of many triangles around one
// vertex or many vertices in one voxel costs no more than spread-out ones.
#include "avc_common.cuh"

using namespace avc;

namespace {

constexpr int CL_THREADS = 256;
constexpr int KEY_BITS = 21;                                  // per axis; the largest voxel index is resolution + 1
constexpr int KEY_MAX = (1 << KEY_BITS) - 1;
constexpr int MAX_RESOLUTION = KEY_MAX - 1;
constexpr int MAX_ELEMS = 1 << 30;                             // tables of 2^31 slots still index with int

__device__ __forceinline__ int f2o(float f) {                  // float order == int order
  const int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float o2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {   // splitmix64's finaliser
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27; x *= 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

// Insert `id` into the open-addressing table `tab` (-1 = empty, load <= 1/2).  A slot only ever goes from empty to an id
// and then down to smaller ids of the same key, so eq(prev) never sees a slot change its key.  Returns the slot.
template <class Eq>
__device__ __forceinline__ int table_insert(int* tab, unsigned mask, unsigned long long h, int id, Eq eq) {
  unsigned s = (unsigned)h & mask;
  while (true) {
    const int prev = atomicCAS(tab + s, -1, id);
    if (prev == -1) return (int)s;
    if (eq(prev)) { atomicMin(tab + s, id); return (int)s; }
    s = (s + 1) & mask;
  }
}

// ---------------------------------------------------------------- bounds and voxel keys
__global__ void k_cl_init(int* bounds, int32_t* counts) {
  if (threadIdx.x < 3) { bounds[threadIdx.x] = INT32_MAX; bounds[3 + threadIdx.x] = INT32_MIN; }
  if (threadIdx.x < 2) counts[threadIdx.x] = 0;
}

__global__ void __launch_bounds__(CL_THREADS) k_cl_bounds(const float* __restrict__ v, int V, int* bounds) {
  int mn[3] = {INT32_MAX, INT32_MAX, INT32_MAX}, mx[3] = {INT32_MIN, INT32_MIN, INT32_MIN};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < V; i += gridDim.x * blockDim.x) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const int o = f2o(v[(size_t)i * 3 + a]);
      mn[a] = min(mn[a], o);
      mx[a] = max(mx[a], o);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn[a] = min(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      mx[a] = max(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
    }
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) { atomicMin(bounds + a, mn[a]); atomicMax(bounds + 3 + a, mx[a]); }
  }
}

// open3d: voxel_min_bound = min_bound - voxel / 2; idx = floor((v - voxel_min_bound) / voxel), all fp64, no contraction.
// voxel = max over axes of (max - min) / resolution, as the reference computes it with numpy.
__global__ void __launch_bounds__(CL_THREADS)
k_cl_vkey(const float* __restrict__ v, int V, const int* __restrict__ bounds, int resolution,
          unsigned long long* __restrict__ vkey) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V) return;
  double mn[3], ext = 0.0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    mn[a] = (double)o2f(bounds[a]);
    ext = fmax(ext, __dsub_rn((double)o2f(bounds[3 + a]), mn[a]));
  }
  const double vox = __ddiv_rn(ext, (double)resolution);
  unsigned long long key = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    int idx = 0;
    if (vox > 0.0) {     // vox == 0: every vertex is the same point, one voxel
      const double lo = __dsub_rn(mn[a], __dmul_rn(vox, 0.5));
      const double r = floor(__ddiv_rn(__dsub_rn((double)v[(size_t)i * 3 + a], lo), vox));
      idx = r > 0.0 ? (int)fmin(r, (double)KEY_MAX) : 0;   // only non-finite inputs leave [0, resolution + 1]
    }
    key = (key << KEY_BITS) | (unsigned long long)idx;
  }
  vkey[i] = key;
}

__global__ void __launch_bounds__(CL_THREADS)
k_cl_vinsert(const unsigned long long* __restrict__ vkey, int V, int* tab, unsigned mask, int* __restrict__ vslot) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V) return;
  const unsigned long long k = vkey[i];
  vslot[i] = table_insert(tab, mask, mix64(k), i, [&](int p) { return vkey[p] == k; });
}

// flag[i] = 1 where i is the entry its slot ended with (the first vertex of its voxel / triangle of its class)
__global__ void __launch_bounds__(CL_THREADS)
k_cl_flag(const int* __restrict__ slot, const int* __restrict__ tab, int n, int* __restrict__ flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = slot[i];
  flag[i] = (s >= 0 && tab[s] == i) ? 1 : 0;
}

// ---------------------------------------------------------------- vertex means
__global__ void __launch_bounds__(CL_THREADS)
k_cl_vaccum(const float* __restrict__ v, const uint8_t* __restrict__ col, int V, const int* __restrict__ vslot,
            const int* __restrict__ tab, const int* __restrict__ vscan, int* __restrict__ vcl, double* sums,
            int* cnt, unsigned* csum) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V) return;
  const int c = vscan[tab[vslot[i]]];   // the output index is the scan value of the voxel's first vertex
  vcl[i] = c;
#pragma unroll
  for (int a = 0; a < 3; ++a) atomicAdd(sums + (size_t)c * 3 + a, (double)v[(size_t)i * 3 + a]);
  atomicAdd(cnt + c, 1);
  if (col) {
#pragma unroll
    for (int a = 0; a < 3; ++a) atomicAdd(csum + (size_t)c * 3 + a, (unsigned)col[(size_t)i * 3 + a]);
  }
}

__global__ void __launch_bounds__(CL_THREADS)
k_cl_vfinal(const double* __restrict__ sums, const int* __restrict__ cnt, const unsigned* __restrict__ csum,
            const int32_t* __restrict__ counts, float* __restrict__ vout, float* __restrict__ cout) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= counts[0]) return;
  const double n = (double)cnt[c];
#pragma unroll
  for (int a = 0; a < 3; ++a) vout[(size_t)c * 3 + a] = (float)__ddiv_rn(sums[(size_t)c * 3 + a], n);
  if (cout) {      // open3d reads a uchar colour as c / 255 and averages those; the integer sum is exact
#pragma unroll
    for (int a = 0; a < 3; ++a)
      cout[(size_t)c * 3 + a] = (float)__ddiv_rn(__ddiv_rn((double)csum[(size_t)c * 3 + a], 255.0), n);
  }
}

// ---------------------------------------------------------------- triangles
__global__ void __launch_bounds__(CL_THREADS)
k_cl_tremap(const int32_t* __restrict__ tris, int F, int V, const int* __restrict__ vcl, int* __restrict__ rtri) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= F) return;
  const int a = tris[(size_t)t * 3], b = tris[(size_t)t * 3 + 1], c = tris[(size_t)t * 3 + 2];
  int A = -1, B = -1, C = -1;
  if ((unsigned)a < (unsigned)V && (unsigned)b < (unsigned)V && (unsigned)c < (unsigned)V) {
    A = vcl[a]; B = vcl[b]; C = vcl[c];
    if (A == B || A == C || B == C) A = -1;                 // two corners in one voxel: dropped
  }
  rtri[(size_t)t * 3] = A; rtri[(size_t)t * 3 + 1] = B; rtri[(size_t)t * 3 + 2] = C;
}

__device__ __forceinline__ void canon(const int* r, int& m, int& x, int& y) {   // the rotation with the smallest first
  const int a = r[0], b = r[1], c = r[2];
  if (a < b && a < c) { m = a; x = b; y = c; }
  else if (b < c) { m = b; x = c; y = a; }
  else { m = c; x = a; y = b; }
}

__global__ void __launch_bounds__(CL_THREADS)
k_cl_tinsert(const int* __restrict__ rtri, int F, int* tab, unsigned mask, int* __restrict__ tslot) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= F) return;
  if (rtri[(size_t)t * 3] < 0) { tslot[t] = -1; return; }
  int m, x, y;
  canon(rtri + (size_t)t * 3, m, x, y);
  const unsigned long long h = mix64(mix64(((unsigned long long)(unsigned)m << 32) | (unsigned)x) ^ (unsigned)y);
  tslot[t] = table_insert(tab, mask, h, t, [&](int p) {
    int pm, px, py;
    canon(rtri + (size_t)p * 3, pm, px, py);
    return pm == m && px == x && py == y;
  });
}

__global__ void __launch_bounds__(CL_THREADS)
k_cl_temit(const int* __restrict__ rtri, const int* __restrict__ tslot, const int* __restrict__ tab,
           const int* __restrict__ tscan, int F, int32_t* __restrict__ tout) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= F) return;
  const int s = tslot[t];
  if (s < 0 || tab[s] != t) return;
  const int o = tscan[t];
#pragma unroll
  for (int k = 0; k < 3; ++k) tout[(size_t)o * 3 + k] = rtri[(size_t)t * 3 + k];
}

// ---------------------------------------------------------------- workspace layout
size_t pow2_at_least(size_t n) {
  size_t p = 64;
  while (p < n) p <<= 1;
  return p;
}

struct Layout {
  size_t bounds, vtab, vkey, vslot, vscan, vcl, sums, cnt, csum, rtri, ttab, tslot, tscan, scan_sums, total;
  unsigned vmask, tmask;
};

Layout layout(int V, int F) {
  Layout L{};
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  const size_t hv = pow2_at_least((size_t)V * 2), ht = pow2_at_least((size_t)F * 2);
  L.vmask = (unsigned)(hv - 1);
  L.tmask = (unsigned)(ht - 1);
  L.bounds = take(6 * sizeof(int));
  L.vtab = take(hv * sizeof(int));
  L.vkey = take((size_t)V * sizeof(unsigned long long));
  L.vslot = take((size_t)V * sizeof(int));
  L.vscan = take((size_t)V * sizeof(int));
  L.vcl = take((size_t)V * sizeof(int));
  L.sums = take((size_t)V * 3 * sizeof(double));
  L.cnt = take((size_t)V * sizeof(int));
  L.csum = take((size_t)V * 3 * sizeof(unsigned));
  L.rtri = take((size_t)F * 3 * sizeof(int));
  L.ttab = take(ht * sizeof(int));
  L.tslot = take((size_t)F * sizeof(int));
  L.tscan = take((size_t)F * sizeof(int));
  L.scan_sums = take(exclusive_scan_sums(V > F ? V : F) * sizeof(int));
  L.total = off;
  return L;
}

}  // namespace

extern "C" {

int avc_mesh_cluster_workspace_bytes(int32_t V, int32_t F, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (V < 1 || V > MAX_ELEMS || F < 0 || F > MAX_ELEMS) return AVC_E_SIZE;
  *bytes = layout(V, F).total;
  return 0;
}

int avc_mesh_cluster(const float* verts, const uint8_t* colors, int32_t V, const int32_t* tris, int32_t F,
                     int32_t resolution, float* verts_out, float* colors_out, int32_t* tris_out, int32_t* counts,
                     void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!verts || !verts_out || !counts || !workspace || (F > 0 && (!tris || !tris_out)) ||
      (colors && !colors_out))
    return AVC_E_NULL;
  if (resolution < 1 || resolution > MAX_RESOLUTION) return AVC_E_BADCFG;
  size_t need = 0;
  AVC_TRY(avc_mesh_cluster_workspace_bytes(V, F, &need));
  if (workspace_bytes < need) return AVC_E_SIZE;
  const Layout L = layout(V, F);
  char* ws = (char*)workspace;
  int* bounds = (int*)(ws + L.bounds);
  int* vtab = (int*)(ws + L.vtab);
  unsigned long long* vkey = (unsigned long long*)(ws + L.vkey);
  int *vslot = (int*)(ws + L.vslot), *vscan = (int*)(ws + L.vscan), *vcl = (int*)(ws + L.vcl);
  double* sums = (double*)(ws + L.sums);
  int* cnt = (int*)(ws + L.cnt);
  unsigned* csum = (unsigned*)(ws + L.csum);
  int *rtri = (int*)(ws + L.rtri), *ttab = (int*)(ws + L.ttab), *tslot = (int*)(ws + L.tslot);
  int *tscan = (int*)(ws + L.tscan), *scan_sums = (int*)(ws + L.scan_sums);
  cudaStream_t st = (cudaStream_t)stream;

  AVC_CUDA_TRY(cudaMemsetAsync(vtab, 0xff, (size_t)(L.vmask + 1) * sizeof(int), st));
  AVC_CUDA_TRY(cudaMemsetAsync(sums, 0, L.csum + (size_t)V * 3 * sizeof(unsigned) - L.sums, st));  // sums, cnt, csum
  k_cl_init<<<1, 32, 0, st>>>(bounds, counts);
  k_cl_bounds<<<min(ceil_div(V, CL_THREADS), 264), CL_THREADS, 0, st>>>(verts, V, bounds);
  k_cl_vkey<<<ceil_div(V, CL_THREADS), CL_THREADS, 0, st>>>(verts, V, bounds, resolution, vkey);
  k_cl_vinsert<<<ceil_div(V, CL_THREADS), CL_THREADS, 0, st>>>(vkey, V, vtab, L.vmask, vslot);
  k_cl_flag<<<ceil_div(V, CL_THREADS), CL_THREADS, 0, st>>>(vslot, vtab, V, vscan);
  exclusive_scan(vscan, V, scan_sums, counts, st);
  k_cl_vaccum<<<ceil_div(V, CL_THREADS), CL_THREADS, 0, st>>>(verts, colors, V, vslot, vtab, vscan, vcl, sums, cnt,
                                                              csum);
  k_cl_vfinal<<<ceil_div(V, CL_THREADS), CL_THREADS, 0, st>>>(sums, cnt, csum, counts, verts_out,
                                                              colors ? colors_out : nullptr);
  if (F > 0) {
    AVC_CUDA_TRY(cudaMemsetAsync(ttab, 0xff, (size_t)(L.tmask + 1) * sizeof(int), st));
    k_cl_tremap<<<ceil_div(F, CL_THREADS), CL_THREADS, 0, st>>>(tris, F, V, vcl, rtri);
    k_cl_tinsert<<<ceil_div(F, CL_THREADS), CL_THREADS, 0, st>>>(rtri, F, ttab, L.tmask, tslot);
    k_cl_flag<<<ceil_div(F, CL_THREADS), CL_THREADS, 0, st>>>(tslot, ttab, F, tscan);
    exclusive_scan(tscan, F, scan_sums, counts + 1, st);
    k_cl_temit<<<ceil_div(F, CL_THREADS), CL_THREADS, 0, st>>>(rtri, tslot, ttab, tscan, F, tris_out);
  }
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"
