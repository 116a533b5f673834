// avc_video.cu -- video frames of one large vertex-coloured mesh over many frames (avatarclip_b200/video.py): the
// vertex -> incident-face lists once per mesh, then per chunk of frames one launch of each stage over every frame.
//   k_vid_count / exclusive_scan / k_vid_fill / k_vid_sort   CSR adjacency: count, the device-wide exclusive scan of
//                     avc_scan.cu, fill, then each vertex's list sorted by face id (independent of scheduling)
//   k_vid_project     per (frame, vertex): world -> camera [R | t] -> supersampled pixel coordinates and depth
//   k_vid_normals     per (frame, vertex): sum of the un-normalised face cross products in CSR order (no float atomics)
//   k_vid_raster      per (frame, face): z-buffer by a 64-bit atomicMin of (depth bits | face id)
//   k_vid_resolve     per (frame, pixel): perspective-correct colour and normal of each sample's face, headlight
//                     shading, background, the supersample mean rounded to uint8
// Semantics in include/avc_b200.h.
#include "avc_common.cuh"

using namespace avc;

namespace {

constexpr int kThreads = 256;
constexpr float kNear = 1e-2f;
constexpr float kAmbient = 0.25f, kDiffuse = 0.75f;
constexpr float kGrey = 200.f;
constexpr int kMaxFrames = 65535;     // grid.y

// ---------------------------------------------------------------- adjacency
__global__ void k_vid_count(const int* __restrict__ faces, int F, int V, int* __restrict__ counts) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3LL * F) return;
  const int v = faces[i];
  if (v >= 0 && v < V) atomicAdd(counts + v, 1);
}

__global__ void k_vid_fill(const int* __restrict__ faces, int F, int V, int* __restrict__ cursor, int* __restrict__ vf) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3LL * F) return;
  const int v = faces[i];
  if (v >= 0 && v < V) vf[atomicAdd(cursor + v, 1)] = (int)(i / 3);
}

// insertion sort of each vertex's list: a vertex has a handful of faces in a surface mesh
__global__ void k_vid_sort(const int* __restrict__ offsets, int V, int* __restrict__ vf) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int b = offsets[v], e = offsets[v + 1];
  for (int i = b + 1; i < e; ++i) {
    const int x = vf[i];
    int j = i - 1;
    while (j >= b && vf[j] > x) { vf[j + 1] = vf[j]; --j; }
    vf[j + 1] = x;
  }
}

// ---------------------------------------------------------------- render
struct VidCfg {
  int V, F, n, ss, is;
  long long stride;       // floats between frames of verts (0: one vertex set for every frame)
};

// cams [frame][13] = R (row-major 3x3) | t, focal (output pixels); proj = (u, v, z, 0): u, v in supersampled pixels
// (pixel xi covers [xi, xi + 1)), z the camera depth
__global__ void __launch_bounds__(kThreads)
k_vid_project(const float* __restrict__ verts, const float* __restrict__ cams, VidCfg c, float4* __restrict__ proj) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= c.V) return;
  const int fr = blockIdx.y;
  const float* p = verts + fr * c.stride + (size_t)v * 3;
  const float* k = cams + fr * 13;
  const float x = p[0], y = p[1], z = p[2];
  const float X = k[0] * x + k[1] * y + k[2] * z + k[3];
  const float Y = k[4] * x + k[5] * y + k[6] * z + k[7];
  const float Z = k[8] * x + k[9] * y + k[10] * z + k[11];
  const float fs = k[12] * c.ss, h = 0.5f * c.is;
  proj[(size_t)fr * c.V + v] = make_float4(fs * X / Z + h, fs * Y / Z + h, Z, 0.f);
}

__global__ void __launch_bounds__(kThreads)
k_vid_normals(const float* __restrict__ verts, const int* __restrict__ faces, const int* __restrict__ offsets,
              const int* __restrict__ vf, VidCfg c, float4* __restrict__ nrm) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= c.V) return;
  const int fr = blockIdx.y;
  const float* P = verts + fr * c.stride;
  float nx = 0.f, ny = 0.f, nz = 0.f;
  for (int j = offsets[v], e = offsets[v + 1]; j < e; ++j) {
    const int f = vf[j];
    const float* a = P + (size_t)faces[f * 3] * 3;
    const float* b = P + (size_t)faces[f * 3 + 1] * 3;
    const float* d = P + (size_t)faces[f * 3 + 2] * 3;
    const float ux = b[0] - a[0], uy = b[1] - a[1], uz = b[2] - a[2];
    const float wx = d[0] - a[0], wy = d[1] - a[1], wz = d[2] - a[2];
    nx += uy * wz - uz * wy;
    ny += uz * wx - ux * wz;
    nz += ux * wy - uy * wx;
  }
  nrm[(size_t)fr * c.V + v] = make_float4(nx, ny, nz, 0.f);
}

// one thread per (frame, face): walk the pixel-centre bounding box, both windings
__global__ void __launch_bounds__(kThreads)
k_vid_raster(const float4* __restrict__ proj, const int* __restrict__ faces, VidCfg c,
             unsigned long long* __restrict__ zbuf) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= c.F) return;
  const int fr = blockIdx.y;
  const int i0 = faces[f * 3], i1 = faces[f * 3 + 1], i2 = faces[f * 3 + 2];
  if ((unsigned)i0 >= (unsigned)c.V || (unsigned)i1 >= (unsigned)c.V || (unsigned)i2 >= (unsigned)c.V) return;
  const float4* P = proj + (size_t)fr * c.V;
  const float4 a = P[i0], b = P[i1], d = P[i2];
  if (!(a.z > kNear && b.z > kNear && d.z > kNear)) return;
  const float xmin = fminf(a.x, fminf(b.x, d.x)), xmax = fmaxf(a.x, fmaxf(b.x, d.x));
  const float ymin = fminf(a.y, fminf(b.y, d.y)), ymax = fmaxf(a.y, fmaxf(b.y, d.y));
  // pixel centre xi + 0.5; clamp in float first so a far-off vertex cannot overflow the int conversion
  const float lim = (float)c.is;
  const int x0 = (int)ceilf(fmaxf(xmin - 0.5f, 0.f)), x1 = (int)floorf(fminf(xmax - 0.5f, lim - 1.f));
  const int y0 = (int)ceilf(fmaxf(ymin - 0.5f, 0.f)), y1 = (int)floorf(fminf(ymax - 0.5f, lim - 1.f));
  if (x0 > x1 || y0 > y1) return;
  const float det = (b.y - d.y) * (a.x - d.x) + (d.x - b.x) * (a.y - d.y);
  if (!(fabsf(det) > 0.f)) return;
  const float inv_det = 1.f / det;
  unsigned long long* Z = zbuf + (size_t)fr * c.is * c.is;
  for (int yi = y0; yi <= y1; ++yi) {
    const float yp = yi + 0.5f;
    for (int xi = x0; xi <= x1; ++xi) {
      const float xp = xi + 0.5f;
      const float w0 = ((b.y - d.y) * (xp - d.x) + (d.x - b.x) * (yp - d.y)) * inv_det;
      const float w1 = ((d.y - a.y) * (xp - d.x) + (a.x - d.x) * (yp - d.y)) * inv_det;
      const float w2 = 1.f - w0 - w1;
      if (w0 < 0.f || w1 < 0.f || w2 < 0.f) continue;
      const float zp = 1.f / (w0 / a.z + w1 / b.z + w2 / d.z);
      atomicMin(Z + (size_t)yi * c.is + xi, depth_key(zp, f));
    }
  }
}

__global__ void __launch_bounds__(kThreads)
k_vid_resolve(const unsigned long long* __restrict__ zbuf, const float4* __restrict__ proj,
              const float4* __restrict__ nrm, const int* __restrict__ faces, const uint8_t* __restrict__ colors,
              const float* __restrict__ cams, VidCfg c, uchar3 bg, uint8_t* __restrict__ rgb,
              int* __restrict__ face_out) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= c.n * c.n) return;
  const int fr = blockIdx.y;
  const int y = p / c.n, x = p - y * c.n;
  const float4* P = proj + (size_t)fr * c.V;
  const float4* N = nrm + (size_t)fr * c.V;
  const unsigned long long* Z = zbuf + (size_t)fr * c.is * c.is;
  const float r20 = cams[fr * 13 + 8], r21 = cams[fr * 13 + 9], r22 = cams[fr * 13 + 10];   // camera z axis
  float acc[3] = {0.f, 0.f, 0.f};
  for (int sy = 0; sy < c.ss; ++sy)
    for (int sx = 0; sx < c.ss; ++sx) {
      const int yi = y * c.ss + sy, xi = x * c.ss + sx;
      const unsigned long long zb = Z[(size_t)yi * c.is + xi];
      if (face_out) face_out[((size_t)fr * c.is + yi) * c.is + xi] = zb == ~0ull ? -1 : (int)(zb & 0xffffffffu);
      if (zb == ~0ull) {
        acc[0] += bg.x; acc[1] += bg.y; acc[2] += bg.z;
        continue;
      }
      const int f = (int)(zb & 0xffffffffu);
      const float zp = __uint_as_float((unsigned)(zb >> 32));
      const int i0 = faces[f * 3], i1 = faces[f * 3 + 1], i2 = faces[f * 3 + 2];
      const float4 a = P[i0], b = P[i1], d = P[i2];
      const float xp = xi + 0.5f, yp = yi + 0.5f;
      const float det = (b.y - d.y) * (a.x - d.x) + (d.x - b.x) * (a.y - d.y);
      const float w0 = ((b.y - d.y) * (xp - d.x) + (d.x - b.x) * (yp - d.y)) / det;
      const float w1 = ((d.y - a.y) * (xp - d.x) + (a.x - d.x) * (yp - d.y)) / det;
      const float w2 = 1.f - w0 - w1;
      const float b0 = w0 * zp / a.z, b1 = w1 * zp / b.z, b2 = w2 * zp / d.z;   // perspective-correct
      float col[3];
      if (colors) {
#pragma unroll
        for (int ch = 0; ch < 3; ++ch)
          col[ch] = b0 * colors[(size_t)i0 * 3 + ch] + b1 * colors[(size_t)i1 * 3 + ch] + b2 * colors[(size_t)i2 * 3 + ch];
      } else {
        col[0] = col[1] = col[2] = kGrey;
      }
      const float4 na = N[i0], nb = N[i1], nd = N[i2];
      const float nx = b0 * na.x + b1 * nb.x + b2 * nd.x;
      const float ny = b0 * na.y + b1 * nb.y + b2 * nd.y;
      const float nz = b0 * na.z + b1 * nb.z + b2 * nd.z;
      const float len = sqrtf(nx * nx + ny * ny + nz * nz);
      // v = -(camera z axis): n . v flipped to face the camera is |n . z_cam| / |n|
      const float ndotv = len > 0.f ? fabsf(r20 * nx + r21 * ny + r22 * nz) / len : 0.f;
      const float shade = kAmbient + kDiffuse * fminf(ndotv, 1.f);
      acc[0] += col[0] * shade; acc[1] += col[1] * shade; acc[2] += col[2] * shade;
    }
  const float inv = 1.f / (float)(c.ss * c.ss);
  uint8_t* o = rgb + (((size_t)fr * c.n + y) * c.n + x) * 3;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) o[ch] = (uint8_t)min(max(__float2int_rn(acc[ch] * inv), 0), 255);
}

bool video_dims_ok(int32_t V, int32_t F, int32_t n_frames, int32_t image_size, int32_t supersample) {
  return V >= 1 && F >= 1 && F <= (1 << 29) && n_frames >= 1 && n_frames <= kMaxFrames && image_size >= 1 &&
         image_size <= 4096 && supersample >= 1 && supersample <= 4;
}

}  // namespace

extern "C" {

int avc_video_adjacency_workspace_bytes(int32_t V, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (V < 1) return AVC_E_SIZE;
  Carver c(nullptr);
  c.take<int>(V);
  c.take<int>(exclusive_scan_sums(V));
  *bytes = c.used();
  return 0;
}

int avc_video_adjacency(const int32_t* faces, int32_t V, int32_t F, int32_t* offsets, int32_t* vf, void* workspace,
                        size_t workspace_bytes, avc_stream_t stream) {
  if (!faces || !offsets || !vf || !workspace) return AVC_E_NULL;
  size_t need = 0;
  AVC_TRY(avc_video_adjacency_workspace_bytes(V, &need));
  if (F < 1 || F > (1 << 29) || workspace_bytes < need) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  Carver c(workspace);
  int* cursor = c.take<int>(V);
  int* sums = c.take<int>(exclusive_scan_sums(V));
  AVC_CUDA_TRY(cudaMemsetAsync(offsets, 0, sizeof(int) * ((size_t)V + 1), st));
  k_vid_count<<<ceil_div(3LL * F, kThreads), kThreads, 0, st>>>(faces, F, V, offsets);
  exclusive_scan(offsets, V, sums, offsets + V, st);
  AVC_CUDA_TRY(cudaMemcpyAsync(cursor, offsets, sizeof(int) * (size_t)V, cudaMemcpyDeviceToDevice, st));
  k_vid_fill<<<ceil_div(3LL * F, kThreads), kThreads, 0, st>>>(faces, F, V, cursor, vf);
  k_vid_sort<<<ceil_div(V, kThreads), kThreads, 0, st>>>(offsets, V, vf);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_video_render_workspace_bytes(int32_t V, int32_t F, int32_t n_frames, int32_t image_size, int32_t supersample,
                                     size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (!video_dims_ok(V, F, n_frames, image_size, supersample)) return AVC_E_BADCFG;
  const size_t is = (size_t)image_size * supersample;
  Carver c(nullptr);
  c.take<float>((size_t)n_frames * 13);
  c.take<float4>((size_t)n_frames * V);
  c.take<float4>((size_t)n_frames * V);
  c.take<unsigned long long>((size_t)n_frames * is * is);
  *bytes = c.used();
  return 0;
}

int avc_video_render(const float* verts, int64_t frame_stride, const int32_t* faces, const int32_t* offsets,
                     const int32_t* vf, const uint8_t* colors, int32_t V, int32_t F, const float* cameras,
                     int32_t n_frames, int32_t image_size, int32_t supersample, const uint8_t* background,
                     uint8_t* rgb_out, int32_t* face_out, void* workspace, size_t workspace_bytes,
                     avc_stream_t stream) {
  if (!verts || !faces || !offsets || !vf || !cameras || !background || !rgb_out || !workspace) return AVC_E_NULL;
  size_t need = 0;
  AVC_TRY(avc_video_render_workspace_bytes(V, F, n_frames, image_size, supersample, &need));
  if (frame_stride < 0) return AVC_E_BADCFG;
  if (workspace_bytes < need) return AVC_E_SIZE;
  for (int i = 0; i < n_frames; ++i)
    if (!(cameras[(size_t)i * 13 + 12] > 0.f)) return AVC_E_BADCFG;
  cudaStream_t st = (cudaStream_t)stream;
  const int is = image_size * supersample;
  Carver c(workspace);
  float* cams = c.take<float>((size_t)n_frames * 13);
  float4* proj = c.take<float4>((size_t)n_frames * V);
  float4* nrm = c.take<float4>((size_t)n_frames * V);
  unsigned long long* zbuf = c.take<unsigned long long>((size_t)n_frames * is * is);
  AVC_CUDA_TRY(cudaMemcpyAsync(cams, cameras, sizeof(float) * 13 * (size_t)n_frames, cudaMemcpyHostToDevice, st));
  AVC_CUDA_TRY(cudaMemsetAsync(zbuf, 0xff, sizeof(unsigned long long) * (size_t)n_frames * is * is, st));
  const VidCfg cfg{V, F, image_size, supersample, is, (long long)frame_stride};
  const uchar3 bg = make_uchar3(background[0], background[1], background[2]);
  k_vid_project<<<dim3(ceil_div(V, kThreads), n_frames), kThreads, 0, st>>>(verts, cams, cfg, proj);
  k_vid_normals<<<dim3(ceil_div(V, kThreads), n_frames), kThreads, 0, st>>>(verts, faces, offsets, vf, cfg, nrm);
  k_vid_raster<<<dim3(ceil_div(F, kThreads), n_frames), kThreads, 0, st>>>(proj, faces, cfg, zbuf);
  k_vid_resolve<<<dim3(ceil_div((long long)image_size * image_size, kThreads), n_frames), kThreads, 0, st>>>(
        zbuf, proj, nrm, faces, colors, cams, cfg, bg, rgb_out, face_out);
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"
