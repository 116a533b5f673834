// avc_raster.cuh -- the passes shared by the white-textured template rasteriser (avc_view.cu), the textured look_at
// rasteriser (avc_shape.cu) and its batched form (avc_pose.cu).  All restate neural_renderer's rasterisation: per
// supersample the nearest face by barycentric 1/z interpolation, near / far clipping, image row 0 at the top.
// The per-element bodies are device functions so that the single-image kernels and the batched ones (one image per
// blockIdx.y) run the same arithmetic.
#pragma once

namespace {

// one face: walk the bounding box, z-test with a 64-bit atomicMin (depth bits, face index).  Both windings are drawn
// (fill_back=True doubles every face with reversed winding and the rasteriser culls back faces: exactly one copy of
// each triangle survives), the lighting normal is the one facing the camera.
__device__ __forceinline__ void raster_face(int f, const float4* __restrict__ proj, const int* __restrict__ faces,
                                            int is, float near, float far, unsigned long long* __restrict__ zbuf) {
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
      atomicMin(&zbuf[(size_t)(is - 1 - yi) * is + xi], avc::depth_key(zp, f));
    }
  }
}

// one thread per face
__global__ void k_raster_faces(const float4* __restrict__ proj, const int* __restrict__ faces, int F, int is,
                               float near, float far, unsigned long long* __restrict__ zbuf) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  raster_face(f, proj, faces, is, near, far, zbuf);
}

// ---------------------------------------------------------------- textured look_at camera
struct LookAtCam {
  float eye[3];
  float rx[3], ry[3], rz[3];   // rows of look_at()'s rotation
  float inv_width;             // 1 / tan(viewing_angle = 30 deg)
  int is;                      // supersampled image size
};

// look_at() + perspective() of vertex i, the vertices as given: x_ndc, y_ndc, z_cam
__device__ __forceinline__ void project_look_at(int i, const float* __restrict__ v, const LookAtCam& c,
                                                float4* __restrict__ proj) {
  float dx = v[i * 3] - c.eye[0], dy = v[i * 3 + 1] - c.eye[1], dz = v[i * 3 + 2] - c.eye[2];
  float cx = c.rx[0] * dx + c.rx[1] * dy + c.rx[2] * dz;
  float cy = c.ry[0] * dx + c.ry[1] * dy + c.ry[2] * dz;
  float cz = c.rz[0] * dx + c.rz[1] * dy + c.rz[2] * dz;
  proj[i] = make_float4(cx / cz * c.inv_width, cy / cz * c.inv_width, cz, 0.f);
}

__global__ void k_project_look_at(const float* __restrict__ v, int V, LookAtCam c, float4* __restrict__ proj) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V) return;
  project_look_at(i, v, c, proj);
}

// the supersample (row, xi) won by face f at depth zp: the unlit trilinear sample col of f's R^3 cube at the
// perspective-corrected barycentrics, and f's light
__device__ __forceinline__ void textured_sample(int row, int xi, int f, float zp, const int* __restrict__ faces,
                                                const float* __restrict__ verts, const float4* __restrict__ proj,
                                                const float* __restrict__ tex, int R, const LookAtCam& c, float* col,
                                                float* light_out) {
  const int is = c.is;
  const int i0 = faces[f * 3], i1 = faces[f * 3 + 1], i2 = faces[f * 3 + 2];
  // lighting in the world frame: n = normalize((v0 - v1) x (v2 - v1)), the copy facing the eye is the one drawn
  const float* v0 = verts + 3 * i0;
  const float* v1 = verts + 3 * i1;
  const float* v2 = verts + 3 * i2;
  float a[3] = {v0[0] - v1[0], v0[1] - v1[1], v0[2] - v1[2]}, b[3] = {v2[0] - v1[0], v2[1] - v1[1], v2[2] - v1[2]};
  float nx = a[1] * b[2] - a[2] * b[1], ny = a[2] * b[0] - a[0] * b[2], nz = a[0] * b[1] - a[1] * b[0];
  float nl = fmaxf(sqrtf(nx * nx + ny * ny + nz * nz), 1e-5f);
  float s = (nx * (c.eye[0] - v1[0]) + ny * (c.eye[1] - v1[1]) + nz * (c.eye[2] - v1[2])) >= 0.f ? 1.f : -1.f;
  const float light = 0.5f + 0.5f * fmaxf(s * ny / nl, 0.f);
  // screen barycentrics at the supersample centre, then w_k (R - 1) z_pixel / z_k
  const float4 pa = proj[i0], pb = proj[i1], pc = proj[i2];
  const int yi = is - 1 - row;
  const float xp = (2.f * xi + 1.f - is) / is, yp = (2.f * yi + 1.f - is) / is;
  const float det = (pb.y - pc.y) * (pa.x - pc.x) + (pc.x - pb.x) * (pa.y - pc.y);
  const float w0 = ((pb.y - pc.y) * (xp - pc.x) + (pc.x - pb.x) * (yp - pc.y)) / det;
  const float w1 = ((pc.y - pa.y) * (xp - pc.x) + (pa.x - pc.x) * (yp - pc.y)) / det;
  const float w2 = 1.f - w0 - w1;
  const float wz[3] = {w0 * zp / pa.z, w1 * zp / pb.z, w2 * zp / pc.z};
  float ti[3];
  int tb[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    ti[k] = fminf(fmaxf(wz[k] * (R - 1), 0.f), (float)(R - 1) - 1e-5f);
    tb[k] = (int)ti[k];
    ti[k] -= (float)tb[k];
  }
  const float* cube = tex + (size_t)f * R * R * R * 3;
  col[0] = 0.f; col[1] = 0.f; col[2] = 0.f;
#pragma unroll
  for (int corner = 0; corner < 8; ++corner) {
    float w = 1.f;
    int idx = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int hi = (corner >> k) & 1;
      w *= hi ? ti[k] : 1.f - ti[k];
      idx = idx * R + min(tb[k] + hi, R - 1);
    }
    col[0] += w * cube[idx * 3];
    col[1] += w * cube[idx * 3 + 1];
    col[2] += w * cube[idx * 3 + 2];
  }
  *light_out = light;
}

// resolve pixel p: per supersample the winning face's colour -- trilinear sample of its R^3 cube at the perspective-
// corrected barycentrics, times the face's light -- then the ss x ss average.  No flip (neural_renderer's image).
__device__ __forceinline__ void resolve_textured(int p, const unsigned long long* __restrict__ zbuf,
                                                 const int* __restrict__ faces, const float* __restrict__ verts,
                                                 const float4* __restrict__ proj, const float* __restrict__ tex, int R,
                                                 const LookAtCam& c, int n, int ss, float* __restrict__ rgb) {
  int y = p / n, x = p - y * n;
  const int is = c.is;
  float acc[3] = {0.f, 0.f, 0.f};
  for (int sy = 0; sy < ss; ++sy)
    for (int sx = 0; sx < ss; ++sx) {
      const int row = y * ss + sy, xi = x * ss + sx;
      unsigned long long zb = zbuf[(size_t)row * is + xi];
      if (zb == ~0ull) continue;
      const int f = (int)(zb & 0xffffffffu);
      const float zp = __uint_as_float((unsigned)(zb >> 32));
      float col[3], light;
      textured_sample(row, xi, f, zp, faces, verts, proj, tex, R, c, col, &light);
      acc[0] += col[0] * light;
      acc[1] += col[1] * light;
      acc[2] += col[2] * light;
    }
  const float inv = 1.f / (float)(ss * ss);
  float* o = rgb + (size_t)p * 3;
  o[0] = acc[0] * inv; o[1] = acc[1] * inv; o[2] = acc[2] * inv;
}

__global__ void k_resolve_textured(const unsigned long long* __restrict__ zbuf, const int* __restrict__ faces,
                                   const float* __restrict__ verts, const float4* __restrict__ proj,
                                   const float* __restrict__ tex, int R, LookAtCam c, int n, int ss,
                                   float* __restrict__ rgb) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n * n) return;
  resolve_textured(p, zbuf, faces, verts, proj, tex, R, c, n, ss, rgb);
}

// look_at(): z = normalize(at - eye), x = normalize(cross(up, z)), y = normalize(cross(z, x)); false when eye == at or
// up is parallel to the viewing direction
inline bool make_look_at_cam(const float* eye, const float* at, const float* up, int is, LookAtCam* cam) {
  auto cross3 = [](const float* a, const float* b, float* o) {
    o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
  };
  auto normalize3 = [](float* a) {
    float n = sqrtf(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
    if (!(n > 0.f)) return false;
    a[0] /= n; a[1] /= n; a[2] /= n;
    return true;
  };
  for (int i = 0; i < 3; ++i) { cam->eye[i] = eye[i]; cam->rz[i] = at[i] - eye[i]; }
  if (!normalize3(cam->rz)) return false;
  cross3(up, cam->rz, cam->rx);
  if (!normalize3(cam->rx)) return false;
  cross3(cam->rz, cam->rx, cam->ry);
  normalize3(cam->ry);
  cam->inv_width = 1.0f / tanf(30.0f * 3.14159265358979323846f / 180.0f);
  cam->is = is;
  return true;
}

}  // namespace
