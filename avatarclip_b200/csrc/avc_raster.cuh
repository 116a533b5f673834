// avc_raster.cuh -- the z-buffer pass shared by the white-textured template rasteriser (avc_view.cu) and the textured
// look_at rasteriser (avc_shape.cu).  Both restate neural_renderer's rasterisation: per supersample the nearest
// face by barycentric 1/z interpolation, near / far clipping, image row 0 at the top.
#pragma once

namespace {

__device__ __forceinline__ unsigned long long pack_depth(float z, int face) {
  return ((unsigned long long)__float_as_uint(z) << 32) | (unsigned int)face;   // z > 0: uint order == float order
}

// one thread per face: walk the bounding box, z-test with a 64-bit atomicMin (depth bits, face index).  Both windings
// are drawn (fill_back=True doubles every face with reversed winding and the rasteriser culls back faces: exactly one
// copy of each triangle survives), the lighting normal is the one facing the camera.
__global__ void k_raster_faces(const float4* __restrict__ proj, const int* __restrict__ faces, int F, int is,
                               float near, float far, unsigned long long* __restrict__ zbuf) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  float4 a = proj[faces[f * 3]], b = proj[faces[f * 3 + 1]], c = proj[faces[f * 3 + 2]];
  if (a.z <= 0.f || b.z <= 0.f || c.z <= 0.f) return;           // behind the camera: not clipped by the reference either
  float xmin = fminf(a.x, fminf(b.x, c.x)), xmax = fmaxf(a.x, fmaxf(b.x, c.x));
  float ymin = fminf(a.y, fminf(b.y, c.y)), ymax = fmaxf(a.y, fmaxf(b.y, c.y));
  // pixel centre xi <-> x_ndc = (2 xi + 1 - is) / is
  int xi0 = max(0, (int)ceilf((xmin * is + is - 1.f) * 0.5f)), xi1 = min(is - 1, (int)floorf((xmax * is + is - 1.f) * 0.5f));
  int yi0 = max(0, (int)ceilf((ymin * is + is - 1.f) * 0.5f)), yi1 = min(is - 1, (int)floorf((ymax * is + is - 1.f) * 0.5f));
  if (xi0 > xi1 || yi0 > yi1) return;
  float det = (b.y - c.y) * (a.x - c.x) + (c.x - b.x) * (a.y - c.y);
  if (fabsf(det) < 1e-20f) return;
  float inv_det = 1.f / det;
  for (int yi = yi0; yi <= yi1; ++yi) {
    float yp = (2.f * yi + 1.f - is) / is;
    for (int xi = xi0; xi <= xi1; ++xi) {
      float xp = (2.f * xi + 1.f - is) / is;
      float w0 = ((b.y - c.y) * (xp - c.x) + (c.x - b.x) * (yp - c.y)) * inv_det;
      float w1 = ((c.y - a.y) * (xp - c.x) + (a.x - c.x) * (yp - c.y)) * inv_det;
      float w2 = 1.f - w0 - w1;
      if (w0 < 0.f || w1 < 0.f || w2 < 0.f) continue;
      float zp = 1.f / (w0 / a.z + w1 / b.z + w2 / c.z);
      if (zp <= near || zp >= far) continue;
      // image row 0 is the top: row = is - 1 - yi
      atomicMin(&zbuf[(size_t)(is - 1 - yi) * is + xi], pack_depth(zp, f));
    }
  }
}

}  // namespace
