// avc_mesh.cu -- iso-surface extraction for NeuSRenderer.extract_geometry (AvatarGen/AppearanceGen/models/renderer.py:
// 27-36,399-404) on the device.
//
// The reference hands the [N][N][N] field u = -sdf to PyMCubes (`mcubes.marching_cubes(u, threshold)`, a third-party
// native CPU extension that is neither vendored nor installable here) and rescales the index-space vertices to the
// bounding box.  This file extracts the same iso-surface {u = threshold} with MARCHING TETRAHEDRA: every grid cube is cut
// into the six tetrahedra around its main diagonal (corner 0 -> corner 7; face diagonals agree between neighbouring
// cubes, so the mesh is watertight), each tetrahedron contributes 0, 1 or 2 triangles with vertices linearly
// interpolated along its edges, oriented so that normals point towards decreasing u (out of the body).  The surface is
// the same to O(h^2); the triangulation is not PyMCubes' (documented in DESIGN.md; PARITY UNPINNED: mcubes is absent).
//
//   pass 1 (emit = false): triangles per cube -> counts[cube]
//   host: exclusive scan of counts (torch.cumsum: plumbing)
//   pass 2 (emit = true):  vertices [3 T][3] in index coordinates + a 64-bit key of the grid edge each vertex lies on
//                          (min point index * 8 + edge direction code 1..7) for welding (torch.unique on the keys); a
//                          crossing whose outside corner equals iso is that grid point and takes the point's key
//                          (point index * 8 + code 0), so the caller welds it once and drops the triangles it collapses
#include "avc_common.cuh"

using namespace avc;

namespace {

__constant__ int kTet[6][4] = {{0, 1, 3, 7}, {0, 1, 5, 7}, {0, 2, 3, 7}, {0, 2, 6, 7}, {0, 4, 5, 7}, {0, 4, 6, 7}};

struct Grid {
  int nx, ny, nz;
  float iso;
};

__device__ __forceinline__ int3 corner(int c) { return make_int3(c & 1, (c >> 1) & 1, (c >> 2) & 1); }

template <bool EMIT>
__global__ void k_march_tets(const float* __restrict__ u, Grid g, int* __restrict__ counts,
                             const int* __restrict__ offsets, float* __restrict__ verts,
                             long long* __restrict__ keys) {
  const long long ncubes = (long long)(g.nx - 1) * (g.ny - 1) * (g.nz - 1);
  long long cid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (cid >= ncubes) return;
  const int cz = (int)(cid % (g.nz - 1));
  const int cy = (int)((cid / (g.nz - 1)) % (g.ny - 1));
  const int cx = (int)(cid / ((long long)(g.nz - 1) * (g.ny - 1)));
  float val[8];
  bool any_in = false, any_out = false;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    int3 o = corner(c);
    val[c] = u[((size_t)(cx + o.x) * g.ny + (cy + o.y)) * g.nz + (cz + o.z)];
    if (val[c] > g.iso) any_in = true; else any_out = true;
  }
  if (!(any_in && any_out)) {
    if (!EMIT) counts[cid] = 0;
    return;
  }
  int ntri = 0;
  int out = EMIT ? offsets[cid] : 0;
  for (int t = 0; t < 6; ++t) {
    int in_idx[4], out_idx[4], ni = 0, no = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      int c = kTet[t][k];
      if (val[c] > g.iso) in_idx[ni++] = c; else out_idx[no++] = c;
    }
    if (ni == 0 || ni == 4) continue;
    const int nt = (ni == 2) ? 2 : 1;
    if (!EMIT) { ntri += nt; continue; }
    // crossing points: every (inside, outside) pair of the tetrahedron is a cut edge
    float P[4][3];
    long long K[4];
    int M[4][3];                                          // twice the cut edge's midpoint, cube-local
    int np = 0;
    int cin[3] = {0, 0, 0}, cout[3] = {0, 0, 0};
    for (int a = 0; a < ni; ++a) { int3 o = corner(in_idx[a]); cin[0] += o.x; cin[1] += o.y; cin[2] += o.z; }
    for (int b = 0; b < no; ++b) { int3 o = corner(out_idx[b]); cout[0] += o.x; cout[1] += o.y; cout[2] += o.z; }
    for (int a = 0; a < ni; ++a)
      for (int b = 0; b < no; ++b) {
        int ci = in_idx[a], co = out_idx[b];
        int3 pi = corner(ci), po = corner(co);
        float tt = (g.iso - val[ci]) / (val[co] - val[ci]);
        P[np][0] = cx + pi.x + tt * (po.x - pi.x);
        P[np][1] = cy + pi.y + tt * (po.y - pi.y);
        P[np][2] = cz + pi.z + tt * (po.z - pi.z);
        M[np][0] = pi.x + po.x; M[np][1] = pi.y + po.y; M[np][2] = pi.z + po.z;
        // key: the grid edge {p, q}: lower point's linear index and the direction code (bits of |q - p|); an outside
        // corner equal to iso puts the crossing on that grid point (tt == 1), keyed by the point itself with code 0
        // so that every edge ending there welds to one vertex
        const bool on_point = val[co] == g.iso;
        int lo = on_point ? co : min(ci, co), hi = on_point ? co : max(ci, co);   // lo is componentwise <= hi
        int3 pl = corner(lo);
        long long base = ((long long)(cx + pl.x) * g.ny + (cy + pl.y)) * g.nz + (cz + pl.z);
        K[np] = base * 8 + (hi - lo);
        ++np;
      }
    // ni == 1 or 3: np == 3 (one triangle); ni == 2: np == 4, ordered (a0b0, a0b1, a1b0, a1b1) -> quad a0b0,a0b1,a1b1,a1b0
    int tri[2][3] = {{0, 1, 2}, {0, 0, 0}};
    if (ni == 2) { tri[0][0] = 0; tri[0][1] = 1; tri[0][2] = 3; tri[1][0] = 0; tri[1][1] = 3; tri[1][2] = 2; }
    // orientation: the normal must leave the body, i.e. n . (inside centroid - outside centroid) < 0.  The triangle's
    // plane separates the inside corners from the outside ones for every crossing strictly inside its edge, so the sign
    // is the same for all of them: it is taken exactly, in integers, with the crossings at the edge midpoints (ni * no
    // times the centroid difference), rather than from the fp32 positions, whose sign is arbitrary on triangles that
    // fp32 index coordinates (2^-15 apart at 512) make degenerate
    const int dir[3] = {no * cin[0] - ni * cout[0], no * cin[1] - ni * cout[1], no * cin[2] - ni * cout[2]};
    for (int q = 0; q < nt; ++q) {
      int i0 = tri[q][0], i1 = tri[q][1], i2 = tri[q][2];
      int e1[3] = {M[i1][0] - M[i0][0], M[i1][1] - M[i0][1], M[i1][2] - M[i0][2]};
      int e2[3] = {M[i2][0] - M[i0][0], M[i2][1] - M[i0][1], M[i2][2] - M[i0][2]};
      int n[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
      if (n[0] * dir[0] + n[1] * dir[1] + n[2] * dir[2] > 0) { int s = i1; i1 = i2; i2 = s; }
      int idx[3] = {i0, i1, i2};
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        size_t w = (size_t)(out + ntri) * 3 + k;
        verts[w * 3] = P[idx[k]][0]; verts[w * 3 + 1] = P[idx[k]][1]; verts[w * 3 + 2] = P[idx[k]][2];
        keys[w] = K[idx[k]];
      }
      ++ntri;
    }
  }
  if (!EMIT) counts[cid] = ntri;
}

}  // namespace

extern "C" {

int avc_march_count(const float* field, int32_t nx, int32_t ny, int32_t nz, float iso, int32_t* counts,
                    avc_stream_t stream) {
  if (!field || !counts) return AVC_E_NULL;
  if (nx < 2 || ny < 2 || nz < 2) return AVC_E_SIZE;
  Grid g{nx, ny, nz, iso};
  long long n = (long long)(nx - 1) * (ny - 1) * (nz - 1);
  k_march_tets<false><<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(field, g, counts, nullptr, nullptr,
                                                                                      nullptr);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_march_emit(const float* field, int32_t nx, int32_t ny, int32_t nz, float iso, const int32_t* offsets,
                   float* verts, int64_t* keys, avc_stream_t stream) {
  if (!field || !offsets || !verts || !keys) return AVC_E_NULL;
  if (nx < 2 || ny < 2 || nz < 2) return AVC_E_SIZE;
  Grid g{nx, ny, nz, iso};
  long long n = (long long)(nx - 1) * (ny - 1) * (nz - 1);
  k_march_tets<true><<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(field, g, nullptr, offsets, verts,
                                                                                     (long long*)keys);
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"
