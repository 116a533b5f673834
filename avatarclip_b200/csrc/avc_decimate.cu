// avc_decimate.cu -- quadric-error edge collapse (Garland & Heckbert 1997) of a triangle mesh to a target face count,
// in rounds of independent collapses (semantics in include/avc_b200.h, avc_mesh_decimate).
//   k_dc_init        positions / colours to the workspace, faces to the working copy, validity, the survivor map
//   k_dc_quadric     per vertex the fp64 sum, in ascending face order (avc_video_adjacency's CSR), of its faces' area-
//                    weighted plane quadrics and its boundary edges' penalty quadrics
//   per round, over the live faces only (avc_video_adjacency on the gathered live faces gives the vertex -> face lists):
//   k_dc_classify    per half-edge: the faces on its edge, and whether it is the edge's smallest 3 face + corner;
//                    non-manifold edges lock their endpoints, boundary edges mark theirs
//   k_dc_keys        per edge: checks, the optimal point, the key (float32 cost bits, edge id), and the per-vertex
//                    minimum key (64-bit atomicMin: the minimum does not depend on the order)
//   k_dc_select      an edge whose key is the minimum over every vertex of the faces around its endpoints
//   k_dc_cap         one block: the longest prefix of the selection in key order that removes no more faces than allowed
//   k_dc_apply       the collapses (their neighbourhoods are disjoint, so no two touch the same vertex or face)
//   k_dc_filter      the live faces that remain, and the next round's gathered faces
//   k_dc_flag_v + exclusive_scan + k_dc_emit_*   surviving vertices and faces compacted in input order by the
//                    device-wide scan of avc_scan.cu
// The lists built by atomics each round (live faces, CSR entries, the selection) come out in an order that depends on
// scheduling; nothing computed from them does: counts, minima and the collapses of disjoint neighbourhoods.
#include "avc_common.cuh"

using namespace avc;

namespace {

constexpr int kThreads = 256;
constexpr int kCapThreads = 1024;
constexpr int kMaxDeg = 32;   // an edge with an endpoint in more live faces is not a candidate this round: the link and
                              // flip tests loop O(deg^2) per edge, and a fan of thousands would stall its warp
constexpr double kBoundaryWeight = 10.0;    // boundary penalty weight per squared edge length
constexpr double kDetEps = 1e-9;            // det(A) > kDetEps tr(A)^3: the 3x3 system is solved
constexpr double kFlipCos = 0.25;           // a moved face keeps n_new . n_old > kFlipCos |n_new| |n_old|
constexpr unsigned long long kNoKey = ~0ull;
constexpr int kMaxElems = 1 << 29;          // avc_video_adjacency's face limit; 3 F edge ids fit in an int

enum { C_LIVE = 0, C_NEXT, C_SEL, C_REM, C_NV, C_NF, C_WORDS = 8 };

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }

struct D3 { double x, y, z; };

__device__ __forceinline__ D3 ld3(const float* p, int v) {
  return {(double)p[(size_t)v * 3], (double)p[(size_t)v * 3 + 1], (double)p[(size_t)v * 3 + 2]};
}
__device__ __forceinline__ D3 sub3(D3 a, D3 b) { return {dsub(a.x, b.x), dsub(a.y, b.y), dsub(a.z, b.z)}; }
__device__ __forceinline__ D3 cross3(D3 a, D3 b) {
  return {dsub(dmul(a.y, b.z), dmul(a.z, b.y)), dsub(dmul(a.z, b.x), dmul(a.x, b.z)),
          dsub(dmul(a.x, b.y), dmul(a.y, b.x))};
}
__device__ __forceinline__ double dot3(D3 a, D3 b) { return dadd(dadd(dmul(a.x, b.x), dmul(a.y, b.y)), dmul(a.z, b.z)); }

// q[10] += w p p^T for the plane p = (n / |n|, -(n / |n|) . o); nothing (an exact +0) when |n| = 0
__device__ __forceinline__ void add_plane(double* q, D3 n, D3 o, double w_per_len, bool w_is_len) {
  const double len = __dsqrt_rn(dot3(n, n));
  double p[4] = {0.0, 0.0, 0.0, 0.0}, w = 0.0;
  if (len != 0.0) {
    const D3 u{__ddiv_rn(n.x, len), __ddiv_rn(n.y, len), __ddiv_rn(n.z, len)};
    p[0] = u.x; p[1] = u.y; p[2] = u.z; p[3] = -dot3(u, o);
    w = w_is_len ? dmul(0.5, len) : w_per_len;
  }
  int k = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = i; j < 4; ++j, ++k) q[k] = dadd(q[k], dmul(w, dmul(p[i], p[j])));
}

__device__ __forceinline__ void ldq(const double* Q, int v, double* q) {
#pragma unroll
  for (int k = 0; k < 10; ++k) q[k] = Q[(size_t)v * 10 + k];
}

// v^T Q v with v = (x, y, z, 1), in the order of the header
__device__ __forceinline__ double qcost(const double* q, D3 v) {
  const double s0 = dadd(dadd(dadd(dmul(q[0], v.x), dmul(q[1], v.y)), dmul(q[2], v.z)), q[3]);
  const double s1 = dadd(dadd(dadd(dmul(q[1], v.x), dmul(q[4], v.y)), dmul(q[5], v.z)), q[6]);
  const double s2 = dadd(dadd(dadd(dmul(q[2], v.x), dmul(q[5], v.y)), dmul(q[7], v.z)), q[8]);
  const double s3 = dadd(dadd(dadd(dmul(q[3], v.x), dmul(q[6], v.y)), dmul(q[8], v.z)), q[9]);
  return dadd(dadd(dadd(dmul(v.x, s0), dmul(v.y, s1)), dmul(v.z, s2)), s3);
}

// the collapse point of edge (a, b) under q = Q_a + Q_b, and its cost clamped at 0
__device__ __forceinline__ D3 optimal_point(const double* q, D3 pa, D3 pb, double* cost) {
  const double c00 = dsub(dmul(q[4], q[7]), dmul(q[5], q[5]));
  const double c01 = dsub(dmul(q[5], q[2]), dmul(q[1], q[7]));
  const double c02 = dsub(dmul(q[1], q[5]), dmul(q[4], q[2]));
  const double c11 = dsub(dmul(q[0], q[7]), dmul(q[2], q[2]));
  const double c12 = dsub(dmul(q[1], q[2]), dmul(q[0], q[5]));
  const double c22 = dsub(dmul(q[0], q[4]), dmul(q[1], q[1]));
  const double det = dadd(dadd(dmul(q[0], c00), dmul(q[1], c01)), dmul(q[2], c02));
  const double tr = dadd(dadd(q[0], q[4]), q[7]);
  const D3 m{dmul(dadd(pa.x, pb.x), 0.5), dmul(dadd(pa.y, pb.y), 0.5), dmul(dadd(pa.z, pb.z), 0.5)};
  const D3 e = sub3(pb, pa);
  if (det > dmul(kDetEps, dmul(dmul(tr, tr), tr))) {
    const double r0 = -q[3], r1 = -q[6], r2 = -q[8];
    const D3 v{__ddiv_rn(dadd(dadd(dmul(r0, c00), dmul(r1, c01)), dmul(r2, c02)), det),
               __ddiv_rn(dadd(dadd(dmul(r0, c01), dmul(r1, c11)), dmul(r2, c12)), det),
               __ddiv_rn(dadd(dadd(dmul(r0, c02), dmul(r1, c12)), dmul(r2, c22)), det)};
    const D3 dv = sub3(v, m);
    if (dot3(dv, dv) <= dot3(e, e)) {
      *cost = fmax(qcost(q, v), 0.0);
      return v;
    }
  }
  const double ca = qcost(q, pa), cb = qcost(q, pb), cm = qcost(q, m);
  D3 v = m;
  double c = cm;
  if (ca <= cb && ca <= cm) { v = pa; c = ca; }
  else if (cb <= cm) { v = pb; c = cb; }
  *cost = fmax(c, 0.0);
  return v;
}

__device__ __forceinline__ bool has(const int* t, int v) { return t[0] == v || t[1] == v || t[2] == v; }

// ---------------------------------------------------------------- set-up
__global__ void __launch_bounds__(kThreads)
k_dc_init_v(const float* __restrict__ verts, const float* __restrict__ colors, int V, float* __restrict__ pos,
            float* __restrict__ col, int* __restrict__ remap, int* __restrict__ lock) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    pos[(size_t)v * 3 + a] = verts[(size_t)v * 3 + a];
    if (colors) col[(size_t)v * 3 + a] = colors[(size_t)v * 3 + a];
  }
  remap[v] = v;
  lock[v] = 0;
}

__global__ void __launch_bounds__(kThreads)
k_dc_init_f(const int32_t* __restrict__ tris, int F, int V, int* __restrict__ tri, int* __restrict__ alive,
            int* __restrict__ live, int* ctr) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int a = tris[(size_t)f * 3], b = tris[(size_t)f * 3 + 1], c = tris[(size_t)f * 3 + 2];
  tri[(size_t)f * 3] = a; tri[(size_t)f * 3 + 1] = b; tri[(size_t)f * 3 + 2] = c;
  const bool ok = (unsigned)a < (unsigned)V && (unsigned)b < (unsigned)V && (unsigned)c < (unsigned)V && a != b &&
                  b != c && a != c;
  alive[f] = ok;
  if (ok) live[atomicAdd(ctr + C_LIVE, 1)] = f;
}

// faces of the CSR list of v (live indices) that hold both v and w
__device__ __forceinline__ int faces_on_edge(const int* __restrict__ off, const int* __restrict__ vf,
                                             const int* __restrict__ lf, int v, int w) {
  int n = 0;
  for (int j = off[v]; j < off[v + 1]; ++j) n += has(lf + (size_t)vf[j] * 3, w);
  return n;
}

// per vertex: the sum in ascending face order of each valid face's quadric, then its boundary edges' (corner order)
__global__ void __launch_bounds__(kThreads)
k_dc_quadric(const float* __restrict__ pos, const int* __restrict__ tri, const int* __restrict__ alive, int V,
             const int* __restrict__ off, const int* __restrict__ vf, double* __restrict__ Q) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  double q[10];
#pragma unroll
  for (int k = 0; k < 10; ++k) q[k] = 0.0;
  for (int j = off[v]; j < off[v + 1]; ++j) {
    const int f = vf[j];
    if (!alive[f]) continue;                       // a valid face names v once
    const int* t = tri + (size_t)f * 3;
    const D3 p0 = ld3(pos, t[0]), p1 = ld3(pos, t[1]), p2 = ld3(pos, t[2]);
    const D3 n = cross3(sub3(p1, p0), sub3(p2, p0));
    add_plane(q, n, p0, 0.0, true);
    for (int k = 0; k < 3; ++k) {
      const int a = t[k], b = t[k == 2 ? 0 : k + 1];
      if (a != v && b != v) continue;
      int nf = 0;                                  // valid faces on edge (a, b), from v's list
      for (int i = off[v]; i < off[v + 1]; ++i) {
        const int g = vf[i];
        if (alive[g]) nf += has(tri + (size_t)g * 3, a == v ? b : a);
      }
      if (nf != 1) continue;
      const D3 pa = ld3(pos, a), e = sub3(ld3(pos, b), pa);
      add_plane(q, cross3(e, n), pa, dmul(kBoundaryWeight, dot3(e, e)), false);
    }
  }
#pragma unroll
  for (int k = 0; k < 10; ++k) Q[(size_t)v * 10 + k] = q[k];
}

// ---------------------------------------------------------------- rounds
__global__ void __launch_bounds__(kThreads)
k_dc_gather(const int* __restrict__ live, const int* __restrict__ ctr, const int* __restrict__ tri,
            int* __restrict__ lf) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ctr[C_LIVE]) return;
  const int g = live[i];
#pragma unroll
  for (int k = 0; k < 3; ++k) lf[(size_t)i * 3 + k] = tri[(size_t)g * 3 + k];
}

// hnf[3 i + c] = the number of live faces on the edge of corner c of live face i when that corner is the edge's
// smallest 3 face + corner, else 0
__global__ void __launch_bounds__(kThreads)
k_dc_classify(const int* __restrict__ lf, const int* __restrict__ live, const int* __restrict__ ctr,
              const int* __restrict__ off, const int* __restrict__ vf, int* __restrict__ hnf, int* lock, int* bnd) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= 3 * ctr[C_LIVE]) return;
  const int i = h / 3, c = h - 3 * i;
  const int a = lf[h], b = lf[3 * i + (c == 2 ? 0 : c + 1)];
  const int x = (off[b + 1] - off[b] < off[a + 1] - off[a]) ? b : a;
  const int own = 3 * live[i] + c;
  int nf = 0, mn = own;
  for (int j = off[x]; j < off[x + 1]; ++j) {
    const int* t = lf + (size_t)vf[j] * 3;
    if (!has(t, a) || !has(t, b)) continue;
    ++nf;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int u = t[k], w = t[k == 2 ? 0 : k + 1];
      if ((u == a && w == b) || (u == b && w == a)) mn = min(mn, 3 * live[vf[j]] + k);
    }
  }
  hnf[h] = mn == own ? nf : 0;
  if (mn != own) return;
  if (nf > 2) { lock[a] = 1; lock[b] = 1; }
  if (nf == 1) { bnd[a] = 1; bnd[b] = 1; }
}

// does some face in v's list hold the vertex set {v, c, d}?
__device__ __forceinline__ bool has_face(const int* __restrict__ off, const int* __restrict__ vf,
                                         const int* __restrict__ lf, int v, int c, int d) {
  for (int j = off[v]; j < off[v + 1]; ++j) {
    const int* t = lf + (size_t)vf[j] * 3;
    if (has(t, c) && has(t, d)) return true;
  }
  return false;
}

// every face in v's list that does not hold `other`, with v moved to p, keeps its orientation and a non-zero area
__device__ __forceinline__ bool no_flip(const float* __restrict__ pos, const int* __restrict__ off,
                                        const int* __restrict__ vf, const int* __restrict__ lf, int v, int other,
                                        D3 p) {
  for (int j = off[v]; j < off[v + 1]; ++j) {
    const int* t = lf + (size_t)vf[j] * 3;
    if (has(t, other)) continue;
    const D3 p0 = ld3(pos, t[0]), p1 = ld3(pos, t[1]), p2 = ld3(pos, t[2]);
    const D3 n = cross3(sub3(p1, p0), sub3(p2, p0));
    const D3 q0 = t[0] == v ? p : p0, q1 = t[1] == v ? p : p1, q2 = t[2] == v ? p : p2;
    const D3 m = cross3(sub3(q1, q0), sub3(q2, q0));
    if (!(dot3(n, m) > dmul(kFlipCos, dmul(__dsqrt_rn(dot3(n, n)), __dsqrt_rn(dot3(m, m)))))) return false;
  }
  return true;
}

__device__ __forceinline__ void edge_ends(const int* lf, int h, int& a, int& b) {
  const int i = h / 3, c = h - 3 * i;
  const int u = lf[h], w = lf[3 * i + (c == 2 ? 0 : c + 1)];
  a = min(u, w);
  b = max(u, w);
}

// min blocks 1: without it ptxas holds the kernel to 64 registers and spills the summed quadric
__global__ void __launch_bounds__(kThreads, 1)
k_dc_keys(const float* __restrict__ pos, const double* __restrict__ Q, const int* __restrict__ lf,
          const int* __restrict__ live, const int* __restrict__ ctr, const int* __restrict__ off,
          const int* __restrict__ vf, const int* __restrict__ hnf, const int* __restrict__ lock,
          const int* __restrict__ bnd, unsigned long long* __restrict__ key, unsigned long long* vmin) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= 3 * ctr[C_LIVE]) return;
  key[h] = kNoKey;
  const int nf = hnf[h];
  if (nf < 1 || nf > 2) return;
  int a, b;
  edge_ends(lf, h, a, b);
  if (lock[a] || lock[b] || off[a + 1] - off[a] > kMaxDeg || off[b + 1] - off[b] > kMaxDeg) return;
  if (nf == 2 && bnd[a] && bnd[b]) return;
  // link condition: the common neighbours of a and b are exactly the opposite vertices of the faces on ab
  int o0 = -1, o1 = -1, common = 0;
  for (int j = off[a]; j < off[a + 1]; ++j) {
    const int* t = lf + (size_t)vf[j] * 3;
    const bool on_ab = has(t, b);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int w = t[k];
      if (w == a || w == b) continue;
      if (on_ab) { if (o0 < 0) o0 = w; else o1 = w; }
      bool seen = false;
      for (int i = off[a]; i < j && !seen; ++i) seen = has(lf + (size_t)vf[i] * 3, w);
      if (!seen && faces_on_edge(off, vf, lf, b, w) > 0) ++common;
    }
  }
  if (common != nf) return;
  if (nf == 2 && (o0 == o1 || (has_face(off, vf, lf, a, o0, o1) && has_face(off, vf, lf, b, o0, o1))))
    return;
  double q[10], qb[10], cost;
  ldq(Q, a, q);
  ldq(Q, b, qb);
#pragma unroll
  for (int k = 0; k < 10; ++k) q[k] = dadd(q[k], qb[k]);
  const D3 v = optimal_point(q, ld3(pos, a), ld3(pos, b), &cost);
  const D3 vr{(double)(float)v.x, (double)(float)v.y, (double)(float)v.z};
  if (!no_flip(pos, off, vf, lf, a, b, vr) || !no_flip(pos, off, vf, lf, b, a, vr)) return;
  const int id = 3 * live[h / 3] + (h - 3 * (h / 3));
  const unsigned long long k = depth_key(__double2float_rn(cost), id);
  key[h] = k;
  atomicMin(vmin + a, k);
  atomicMin(vmin + b, k);
}

__device__ __forceinline__ bool ring_min(const int* __restrict__ off, const int* __restrict__ vf,
                                         const int* __restrict__ lf, const unsigned long long* __restrict__ vmin,
                                         int v, unsigned long long k) {
  for (int j = off[v]; j < off[v + 1]; ++j) {
    const int* t = lf + (size_t)vf[j] * 3;
    if (vmin[t[0]] < k || vmin[t[1]] < k || vmin[t[2]] < k) return false;
  }
  return true;
}

__global__ void __launch_bounds__(kThreads)
k_dc_select(const int* __restrict__ lf, int* ctr, const int* __restrict__ off, const int* __restrict__ vf,
            const int* __restrict__ hnf, const unsigned long long* __restrict__ key,
            const unsigned long long* __restrict__ vmin, int* __restrict__ sel) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= 3 * ctr[C_LIVE]) return;
  const unsigned long long k = key[h];
  if (k == kNoKey) return;
  int a, b;
  edge_ends(lf, h, a, b);
  if (!ring_min(off, vf, lf, vmin, a, k) || !ring_min(off, vf, lf, vmin, b, k)) return;
  sel[atomicAdd(ctr + C_SEL, 1)] = h;
  atomicAdd(ctr + C_REM, hnf[h]);
}

// thr[0]: the collapses applied are the selected keys < thr[0]: the longest prefix in key order that removes at most
// live - target faces, and at least the smallest
__global__ void __launch_bounds__(kCapThreads)
k_dc_cap(const int* __restrict__ ctr, const int* __restrict__ sel, const unsigned long long* __restrict__ key,
         const int* __restrict__ hnf, int target, unsigned long long* thr) {
  __shared__ unsigned long long shk[kCapThreads / 32];
  __shared__ int shi[kCapThreads / 32];
  const int n = ctr[C_SEL];
  const long long budget = (long long)ctr[C_LIVE] - target;
  auto sum = [](int x, int y) { return x + y; };
  if ((long long)ctr[C_REM] <= budget) {
    if (threadIdx.x == 0) *thr = kNoKey;
    return;
  }
  unsigned long long mn = kNoKey;
  for (int i = threadIdx.x; i < n; i += kCapThreads) mn = min(mn, key[sel[i]]);
  mn = block_reduce(mn, shk, [](unsigned long long x, unsigned long long y) { return x < y ? x : y; }, kNoKey);
  unsigned long long ans = 0;
  for (int bit = 63; bit >= 0; --bit) {
    const unsigned long long cand = ans | (1ull << bit);
    int s = 0;
    for (int i = threadIdx.x; i < n; i += kCapThreads) s += key[sel[i]] < cand ? hnf[sel[i]] : 0;
    s = block_reduce(s, shi, sum, 0);
    if (s <= budget) ans = cand;
  }
  if (threadIdx.x == 0) *thr = ans > mn ? ans : mn + 1;
}

__global__ void __launch_bounds__(kThreads)
k_dc_apply(const int* __restrict__ ctr, const int* __restrict__ sel, const unsigned long long* __restrict__ key,
           const unsigned long long* __restrict__ thr, const int* __restrict__ lf, const int* __restrict__ live,
           const int* __restrict__ off, const int* __restrict__ vf, float* pos, float* col, double* Q, int* remap,
           int* tri, int* alive) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= ctr[C_SEL]) return;
  const int h = sel[s];
  if (!(key[h] < *thr)) return;
  int a, b;
  edge_ends(lf, h, a, b);
  double q[10], qb[10], cost;
  ldq(Q, a, q);
  ldq(Q, b, qb);
#pragma unroll
  for (int k = 0; k < 10; ++k) q[k] = dadd(q[k], qb[k]);
  const D3 pa = ld3(pos, a), pb = ld3(pos, b);
  const D3 v = optimal_point(q, pa, pb, &cost);
  if (col) {
    const D3 e = sub3(pb, pa);
    const double ee = dot3(e, e);
    double t = ee > 0.0 ? __ddiv_rn(dot3(sub3(v, pa), e), ee) : 0.0;
    t = fmin(fmax(t, 0.0), 1.0);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double ca = col[(size_t)a * 3 + c], cb = col[(size_t)b * 3 + c];
      col[(size_t)a * 3 + c] = __double2float_rn(dadd(ca, dmul(t, dsub(cb, ca))));
    }
  }
  pos[(size_t)a * 3] = __double2float_rn(v.x);
  pos[(size_t)a * 3 + 1] = __double2float_rn(v.y);
  pos[(size_t)a * 3 + 2] = __double2float_rn(v.z);
#pragma unroll
  for (int k = 0; k < 10; ++k) Q[(size_t)a * 10 + k] = q[k];
  remap[b] = a;
  for (int j = off[b]; j < off[b + 1]; ++j) {
    const int g = live[vf[j]];
    int* t = tri + (size_t)g * 3;
    if (has(t, a)) { alive[g] = 0; continue; }
#pragma unroll
    for (int k = 0; k < 3; ++k) if (t[k] == b) t[k] = a;
  }
}

__global__ void __launch_bounds__(kThreads)
k_dc_filter(const int* __restrict__ live, int* ctr, const int* __restrict__ alive, int* __restrict__ next) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ctr[C_LIVE]) return;
  const int g = live[i];
  if (alive[g]) next[atomicAdd(ctr + C_NEXT, 1)] = g;
}

// ---------------------------------------------------------------- output in input order
__global__ void __launch_bounds__(kThreads)
k_dc_flag_v(const int* __restrict__ remap, int V, int* __restrict__ vscan) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) vscan[v] = remap[v] == v;
}

__global__ void __launch_bounds__(kThreads)
k_dc_emit_v(const int* __restrict__ remap, const int* __restrict__ vscan, const float* __restrict__ pos,
            const float* __restrict__ col, int V, float* __restrict__ vout, float* __restrict__ cout) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V || remap[v] != v) return;
  const int o = vscan[v];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    vout[(size_t)o * 3 + a] = pos[(size_t)v * 3 + a];
    if (cout) cout[(size_t)o * 3 + a] = col[(size_t)v * 3 + a];
  }
}

__global__ void __launch_bounds__(kThreads)
k_dc_emit_f(const int* __restrict__ alive, const int* __restrict__ fscan, const int* __restrict__ tri,
            const int* __restrict__ vscan, int F, int32_t* __restrict__ tout) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F || !alive[f]) return;
  const int o = fscan[f];
#pragma unroll
  for (int k = 0; k < 3; ++k) tout[(size_t)o * 3 + k] = vscan[tri[(size_t)f * 3 + k]];
}

__global__ void k_dc_passthrough_counts(int V, int F, int rounds, int32_t* counts) {
  counts[0] = V; counts[1] = F; counts[2] = rounds;
}

__global__ void k_dc_counts(const int* __restrict__ ctr, int rounds, int32_t* counts) {
  counts[0] = ctr[C_NV]; counts[1] = ctr[C_NF]; counts[2] = rounds;
}

// ---------------------------------------------------------------- workspace
struct Ws {
  float *pos, *col;
  double* Q;
  int *remap, *lock, *bnd, *tri, *alive, *live, *next, *lf, *off, *vf, *hnf, *sel, *vscan, *fscan, *sums, *ctr;
  unsigned long long *key, *vmin, *thr;
  void* adj;
  size_t adj_bytes, total;
};

Ws carve(void* base, int V, int F) {
  Carver c(base);
  Ws w{};
  w.pos = c.take<float>((size_t)V * 3);
  w.col = c.take<float>((size_t)V * 3);
  w.Q = c.take<double>((size_t)V * 10);
  w.vmin = c.take<unsigned long long>(V);
  w.key = c.take<unsigned long long>((size_t)F * 3);
  w.thr = c.take<unsigned long long>(1);
  w.remap = c.take<int>(V);
  w.lock = c.take<int>(V);
  w.bnd = c.take<int>(V);
  w.vscan = c.take<int>(V);
  w.off = c.take<int>((size_t)V + 1);
  w.tri = c.take<int>((size_t)F * 3);
  w.lf = c.take<int>((size_t)F * 3);
  w.vf = c.take<int>((size_t)F * 3);
  w.hnf = c.take<int>((size_t)F * 3);
  w.alive = c.take<int>(F);
  w.live = c.take<int>(F);
  w.next = c.take<int>(F);
  w.sel = c.take<int>(F);
  w.fscan = c.take<int>(F);
  w.sums = c.take<int>(exclusive_scan_sums(V > F ? V : F));
  w.ctr = c.take<int>(C_WORDS);
  size_t adj = 0;
  avc_video_adjacency_workspace_bytes(V, &adj);
  w.adj_bytes = adj;
  w.adj = c.take<char>(adj);
  w.total = c.used();
  return w;
}

}  // namespace

extern "C" {

int avc_mesh_decimate_workspace_bytes(int32_t V, int32_t F, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (V < 1 || V > kMaxElems || F < 1 || F > kMaxElems) return AVC_E_SIZE;
  *bytes = carve(nullptr, V, F).total;
  return 0;
}

int avc_mesh_decimate(const float* verts, const float* colors, int32_t V, const int32_t* tris, int32_t F,
                      int32_t target_faces, float* verts_out, float* colors_out, int32_t* tris_out, int32_t* counts,
                      void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!verts || !tris || !verts_out || !tris_out || !counts || !workspace || (colors && !colors_out))
    return AVC_E_NULL;
  size_t need = 0;
  AVC_TRY(avc_mesh_decimate_workspace_bytes(V, F, &need));
  if (target_faces < 1) return AVC_E_BADCFG;
  if (workspace_bytes < need) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  if (F <= target_faces) {
    AVC_CUDA_TRY(cudaMemcpyAsync(verts_out, verts, sizeof(float) * 3 * (size_t)V, cudaMemcpyDeviceToDevice, st));
    if (colors)
      AVC_CUDA_TRY(cudaMemcpyAsync(colors_out, colors, sizeof(float) * 3 * (size_t)V, cudaMemcpyDeviceToDevice, st));
    AVC_CUDA_TRY(cudaMemcpyAsync(tris_out, tris, sizeof(int32_t) * 3 * (size_t)F, cudaMemcpyDeviceToDevice, st));
    k_dc_passthrough_counts<<<1, 1, 0, st>>>(V, F, 0, counts);
    AVC_LAUNCH_TRY();
    return 0;
  }
  const Ws w = carve(workspace, V, F);
  float* col = colors ? w.col : nullptr;
  AVC_CUDA_TRY(cudaMemsetAsync(w.ctr, 0, sizeof(int) * C_WORDS, st));
  k_dc_init_v<<<ceil_div(V, kThreads), kThreads, 0, st>>>(verts, colors, V, w.pos, col, w.remap, w.lock);
  k_dc_init_f<<<ceil_div(F, kThreads), kThreads, 0, st>>>(tris, F, V, w.tri, w.alive, w.live, w.ctr);
  AVC_TRY(avc_video_adjacency(w.tri, V, F, w.off, w.vf, w.adj, w.adj_bytes, stream));
  k_dc_quadric<<<ceil_div(V, kThreads), kThreads, 0, st>>>(w.pos, w.tri, w.alive, V, w.off, w.vf, w.Q);
  AVC_LAUNCH_TRY();

  int host[C_WORDS];
  AVC_CUDA_TRY(cudaMemcpyAsync(host, w.ctr, sizeof(host), cudaMemcpyDeviceToHost, st));
  AVC_CUDA_TRY(cudaStreamSynchronize(st));
  int live_n = host[C_LIVE], rounds = 0;
  int *live = w.live, *next = w.next;
  while (live_n > target_faces) {
    const int nb = ceil_div(live_n, kThreads), nh = ceil_div(3LL * live_n, kThreads);
    k_dc_gather<<<nb, kThreads, 0, st>>>(live, w.ctr, w.tri, w.lf);
    AVC_TRY(avc_video_adjacency(w.lf, V, live_n, w.off, w.vf, w.adj, w.adj_bytes, stream));
    AVC_CUDA_TRY(cudaMemsetAsync(w.bnd, 0, sizeof(int) * (size_t)V, st));
    AVC_CUDA_TRY(cudaMemsetAsync(w.vmin, 0xff, sizeof(unsigned long long) * (size_t)V, st));
    AVC_CUDA_TRY(cudaMemsetAsync(w.ctr + C_NEXT, 0, sizeof(int) * 3, st));     // next, selected, removed
    k_dc_classify<<<nh, kThreads, 0, st>>>(w.lf, live, w.ctr, w.off, w.vf, w.hnf, w.lock, w.bnd);
    k_dc_keys<<<nh, kThreads, 0, st>>>(w.pos, w.Q, w.lf, live, w.ctr, w.off, w.vf, w.hnf, w.lock, w.bnd, w.key,
                                       w.vmin);
    k_dc_select<<<nh, kThreads, 0, st>>>(w.lf, w.ctr, w.off, w.vf, w.hnf, w.key, w.vmin, w.sel);
    k_dc_cap<<<1, kCapThreads, 0, st>>>(w.ctr, w.sel, w.key, w.hnf, target_faces, w.thr);
    k_dc_apply<<<nb, kThreads, 0, st>>>(w.ctr, w.sel, w.key, w.thr, w.lf, live, w.off, w.vf, w.pos, col, w.Q,
                                        w.remap, w.tri, w.alive);
    k_dc_filter<<<nb, kThreads, 0, st>>>(live, w.ctr, w.alive, next);
    AVC_CUDA_TRY(cudaMemcpyAsync(w.ctr + C_LIVE, w.ctr + C_NEXT, sizeof(int), cudaMemcpyDeviceToDevice, st));
    AVC_LAUNCH_TRY();
    AVC_CUDA_TRY(cudaMemcpyAsync(host, w.ctr, sizeof(host), cudaMemcpyDeviceToHost, st));   // the round's counts
    AVC_CUDA_TRY(cudaStreamSynchronize(st));
    if (host[C_SEL] == 0) break;
    ++rounds;
    live_n = host[C_LIVE];
    int* t = live; live = next; next = t;
  }

  k_dc_flag_v<<<ceil_div(V, kThreads), kThreads, 0, st>>>(w.remap, V, w.vscan);
  exclusive_scan(w.vscan, V, w.sums, w.ctr + C_NV, st);
  AVC_CUDA_TRY(cudaMemcpyAsync(w.fscan, w.alive, sizeof(int) * (size_t)F, cudaMemcpyDeviceToDevice, st));
  exclusive_scan(w.fscan, F, w.sums, w.ctr + C_NF, st);
  k_dc_emit_v<<<ceil_div(V, kThreads), kThreads, 0, st>>>(w.remap, w.vscan, w.pos, col, V, verts_out,
                                                          colors ? colors_out : nullptr);
  k_dc_emit_f<<<ceil_div(F, kThreads), kThreads, 0, st>>>(w.alive, w.fscan, w.tri, w.vscan, F, tris_out);
  k_dc_counts<<<1, 1, 0, st>>>(w.ctr, rounds, counts);
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"
