// avc_view.cu -- per-step view preparation of Runner.train_clip on the device (SURVEY.md 8f rank 1):
//
//   avc_raster_template   render_one_batch (models/utils.py:108-125): neural_renderer `Renderer(camera_mode='look')`
//                         of the white-textured SMPL template -> 256 x 256 RGB (+ silhouette rgb != 0)
//   avc_dilate_count      10 x binary_dilation with the full 3 x 3 structure + pixel count (dataset.py:255-257)
//   avc_mask_compact      nearest resize of the dilated mask to the canvas + row-major list of the True pixels
//                         (dataset.py:269-273: rays_v[resized_dilated_mask > 0])
//   avc_view_targets      nearest resize of the template render to the canvas and the loss mask (main.py:377-380,407-410)
//   avc_background_field  background modes 1 / 2 of main.py:392-402 (clamped Gaussian field; blurred chessboard)
//   avc_uniform_fill      counter-based uniform draws (the per-ray jitter of renderer.py:317-319)
//
// neural_renderer is a third-party CUDA extension that is neither vendored by the reference nor installable here; the
// rasteriser restates its published algorithm (daniilidis-group/neural_renderer, the PyTorch port the reference's
// requirements name): vertices -> look() -> perspective(30 deg) -> per-pixel nearest front-facing face by barycentric
// 1/z interpolation at 2x supersampling, flat ambient 0.5 + directional 0.5 lighting along +y of the rasteriser's
// frame, white texture, black background, 2 x 2 average pooling.  PARITY UNPINNED (oracle/raster.py says the same).
#include <cfloat>

#include "avc_common.cuh"

using namespace avc;

namespace {

struct RasterCam {
  float eye[3];
  float rx[3], ry[3], rz[3];   // rows of look()'s rotation: camera x, y, z (z = viewing direction)
  float inv_width;              // 1 / tan(viewing_angle = 30 deg)
  int is;                       // supersampled image size
};

// vertices: SMPL frame -> rasteriser frame (utils.py:115-119: v @ [[1,0,0],[0,0,-1],[0,1,0]] = (x, z, -y)), then
// look() + perspective().  out: [V][4] = x_ndc, y_ndc, z_cam, unused;  rot: [V][3] the rotated vertex (for lighting)
__global__ void k_raster_project(const float* __restrict__ v, int V, RasterCam c, float4* __restrict__ proj,
                                 float* __restrict__ rot) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V) return;
  float x = v[i * 3], y = v[i * 3 + 2], z = -v[i * 3 + 1];
  rot[i * 3] = x; rot[i * 3 + 1] = y; rot[i * 3 + 2] = z;
  float dx = x - c.eye[0], dy = y - c.eye[1], dz = z - c.eye[2];
  float cx = c.rx[0] * dx + c.rx[1] * dy + c.rx[2] * dz;
  float cy = c.ry[0] * dx + c.ry[1] * dy + c.ry[2] * dz;
  float cz = c.rz[0] * dx + c.rz[1] * dy + c.rz[2] * dz;
  proj[i] = make_float4(cx / cz * c.inv_width, cy / cz * c.inv_width, cz, 0.f);
}

}  // namespace

#include "avc_raster.cuh"      // k_raster_faces (the z-buffer pass)

namespace {

// resolve: intensity of the winning face per supersample, ss x ss average, horizontal flip (utils.py:124), silhouette
__global__ void k_raster_resolve(const unsigned long long* __restrict__ zbuf, const int* __restrict__ faces,
                                 const float* __restrict__ rot, RasterCam c, int n, int ss, float* __restrict__ rgb,
                                 uint8_t* __restrict__ mask) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n * n) return;
  int y = p / n, x = p - y * n;
  float acc = 0.f;
  for (int sy = 0; sy < ss; ++sy)
    for (int sx = 0; sx < ss; ++sx) {
      unsigned long long z = zbuf[(size_t)(y * ss + sy) * c.is + (x * ss + sx)];
      if (z == ~0ull) continue;
      int f = (int)(z & 0xffffffffu);
      const float* a = rot + 3 * faces[f * 3];
      const float* b = rot + 3 * faces[f * 3 + 1];
      const float* d = rot + 3 * faces[f * 3 + 2];
      float e1[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, e2[3] = {d[0] - a[0], d[1] - a[1], d[2] - a[2]};
      float nx = e1[1] * e2[2] - e1[2] * e2[1], ny = e1[2] * e2[0] - e1[0] * e2[2], nz = e1[0] * e2[1] - e1[1] * e2[0];
      float nl = sqrtf(nx * nx + ny * ny + nz * nz) + 1e-20f;
      // orient towards the camera
      float vx = c.eye[0] - a[0], vy = c.eye[1] - a[1], vz = c.eye[2] - a[2];
      float s = (nx * vx + ny * vy + nz * vz) >= 0.f ? 1.f : -1.f;
      float cosl = fmaxf(s * ny / nl, 0.f);                  // light direction (0, 1, 0)
      acc += 0.5f + 0.5f * cosl;                            // ambient 0.5 + directional 0.5, white texture
    }
  float val = acc / (float)(ss * ss);
  int xo = n - 1 - x;                                       // images[:, ::-1]
  float* o = rgb + ((size_t)y * n + xo) * 3;
  o[0] = o[1] = o[2] = val;
  mask[(size_t)y * n + xo] = val != 0.f ? 1 : 0;
}

// 10 dilations with the 3 x 3 full structure == one (2 it + 1)^2 box maximum; zero outside the image
__global__ void k_dilate_count(const uint8_t* __restrict__ m, int n, int it, uint8_t* __restrict__ out,
                               int* __restrict__ count) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  int v = 0;
  if (p < n * n) {
    int y = p / n, x = p - y * n;
    for (int dy = -it; dy <= it && !v; ++dy) {
      int yy = y + dy;
      if (yy < 0 || yy >= n) continue;
      for (int dx = -it; dx <= it; ++dx) {
        int xx = x + dx;
        if (xx >= 0 && xx < n && m[yy * n + xx]) { v = 1; break; }
      }
    }
    out[p] = (uint8_t)v;
  }
  unsigned b = __ballot_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(count, __popc(b));
}

// nearest resize (F.interpolate default: src = floor(dst * n / W)) + ordered compaction, ONE block of 1024 threads
__global__ void __launch_bounds__(1024, 1)
k_mask_compact(const uint8_t* __restrict__ dil, int n, int W, int cap, uint8_t* __restrict__ in_mask,
               int* __restrict__ pix, int* __restrict__ count) {
  __shared__ int warp_tot[33];
  const int total = W * W;
  const int per = (total + 1023) / 1024;
  const int t = threadIdx.x;
  const float scale = (float)n / (float)W;
  int begin = t * per, end = min(total, begin + per);
  int mine = 0;
  for (int p = begin; p < end; ++p) {
    int y = p / W, x = p - y * W;
    int sy = min((int)floorf(y * scale), n - 1), sx = min((int)floorf(x * scale), n - 1);
    int v = dil[sy * n + sx] ? 1 : 0;
    in_mask[p] = (uint8_t)v;
    mine += v;
  }
  int kept;
  int off = block_exclusive_scan<1024>(mine, warp_tot, kept);
  for (int p = begin; p < end; ++p)
    if (in_mask[p]) {
      if (off < cap) pix[off] = p;
      ++off;
    }
  if (t == 0) *count = kept;
}

__global__ void k_view_targets(const float* __restrict__ rgb, int n, int W, int threshold_mask,
                               float* __restrict__ true_rgb, float* __restrict__ mask) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= W * W) return;
  int y = p / W, x = p - y * W;
  const float scale = (float)n / (float)W;
  int sy = min((int)floorf(y * scale), n - 1), sx = min((int)floorf(x * scale), n - 1);
  const float* s = rgb + ((size_t)sy * n + sx) * 3;
  true_rgb[p * 3] = s[0]; true_rgb[p * 3 + 1] = s[1]; true_rgb[p * 3 + 2] = s[2];
  // main.py:378-380: mask[true_rgb != 0] = 1; mask = mask[..., :1]; :407-410: (mask > .5) or all ones when mask_weight == 0
  mask[p] = threshold_mask ? (s[0] != 0.f ? 1.f : 0.f) : 1.f;
}

// ---- counter-based generator: one 64-bit hash per (seed, index) -> two uniforms in (0, 1]
__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ void uniforms(unsigned seed, unsigned idx, float& u0, float& u1) {
  unsigned long long h = mix64(((unsigned long long)seed << 32) | idx);
  u0 = ((float)(unsigned)(h >> 40) + 0.5f) * (1.0f / 16777216.0f);
  u1 = ((float)(unsigned)((h >> 8) & 0xffffffu) + 0.5f) * (1.0f / 16777216.0f);
}

__global__ void k_uniform_fill(unsigned seed, int n, float lo, float hi, float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float u0, u1;
  uniforms(seed, (unsigned)i, u0, u1);
  out[i] = lo + (hi - lo) * (u0 - 0.5f / 16777216.0f);      // [lo, hi)
}

// main.py:393-395: clamp(N(0.5, 0.2), 0, 1) per pixel (Box-Muller on the counter-based uniforms)
__global__ void k_bg_gauss(unsigned seed, int n, float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float u0, u1;
  uniforms(seed ^ 0x5bd1e995u, (unsigned)i, u0, u1);
  float g = sqrtf(-2.f * logf(u0)) * cospif(2.f * u1);
  out[i] = fminf(fmaxf(0.5f + 0.2f * g, 0.f), 1.f);
}

// main.py:396-402: 0.2 / 0.8 chessboard with squares of `len` pixels, GaussianBlur(kernel (5, 9), sigma) -- torchvision:
// kernel_size = (kx, ky) = (5, 9) i.e. 5 taps along x (width), 9 along y (height), reflect padding, same sigma on both axes.
// chess_board[white_i, white_j] with meshgrid 'xy': value at [row = i, col = j] where (i // len + j // len) even.
__device__ __forceinline__ float chess_at(int y, int x, int len) { return (((y / len) + (x / len)) & 1) ? 0.2f : 0.8f; }
__device__ __forceinline__ int reflect(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }
__global__ void k_bg_chess(int H, int W, int len, float sigma, float* __restrict__ out) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= H * W) return;
  int y = p / W, x = p - y * W;
  float kx[5], ky[9], sx = 0.f, sy = 0.f;
#pragma unroll
  for (int i = 0; i < 5; ++i) { float t = (float)(i - 2) / sigma; kx[i] = expf(-0.5f * t * t); sx += kx[i]; }
#pragma unroll
  for (int i = 0; i < 9; ++i) { float t = (float)(i - 4) / sigma; ky[i] = expf(-0.5f * t * t); sy += ky[i]; }
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < 9; ++j) {
    int yy = reflect(y + j - 4, H);
    float row = 0.f;
#pragma unroll
    for (int i = 0; i < 5; ++i) row += kx[i] * chess_at(yy, reflect(x + i - 2, W), len);
    acc += ky[j] * row;
  }
  out[p] = acc / (sx * sy);
}

__global__ void k_gather_f32(const float* __restrict__ src, const int* __restrict__ idx, int n, float* __restrict__ dst) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[idx[i]];
}

inline void cross3(const float* a, const float* b, float* o) {
  o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
inline void normalize3(float* a) {
  float n = sqrtf(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
  if (n > 0.f) { a[0] /= n; a[1] /= n; a[2] /= n; }
}

}  // namespace

extern "C" {

int avc_raster_workspace_bytes(int32_t V, int32_t image_size, int32_t supersample, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (V < 1 || image_size < 1 || supersample < 1 || supersample > 4) return AVC_E_SIZE;
  Carver c(nullptr);
  c.take<float4>(V);
  c.take<float>((size_t)V * 3);
  c.take<unsigned long long>((size_t)image_size * supersample * image_size * supersample);
  *bytes = c.used();
  return 0;
}

int avc_raster_template(const float* verts, const int32_t* faces, int32_t V, int32_t F, const float* eye,
                        const float* at, int32_t image_size, int32_t supersample, float* rgb_out, uint8_t* mask_out,
                        void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!verts || !faces || !eye || !at || !rgb_out || !mask_out || !workspace) return AVC_E_NULL;
  size_t need = 0;
  AVC_TRY(avc_raster_workspace_bytes(V, image_size, supersample, &need));
  if (workspace_bytes < need || F < 1) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  Carver c(workspace);
  float4* proj = c.take<float4>(V);
  float* rot = c.take<float>((size_t)V * 3);
  const int is = image_size * supersample;
  unsigned long long* zbuf = c.take<unsigned long long>((size_t)is * is);
  RasterCam cam;
  // utils.py:120-122: renderer.eye = eye; camera_direction = normalize(at - eye); look(): z = direction,
  // x = normalize(cross(up = +y, z)), y = normalize(cross(z, x))
  float up[3] = {0.f, 1.f, 0.f};
  for (int i = 0; i < 3; ++i) { cam.eye[i] = eye[i]; cam.rz[i] = at[i] - eye[i]; }
  normalize3(cam.rz);
  cross3(up, cam.rz, cam.rx); normalize3(cam.rx);
  cross3(cam.rz, cam.rx, cam.ry); normalize3(cam.ry);
  cam.inv_width = 1.0f / tanf(30.0f * 3.14159265358979323846f / 180.0f);
  cam.is = is;
  AVC_CUDA_TRY(cudaMemsetAsync(zbuf, 0xff, sizeof(unsigned long long) * (size_t)is * is, st));
  k_raster_project<<<(V + 255) / 256, 256, 0, st>>>(verts, V, cam, proj, rot);
  k_raster_faces<<<(F + 127) / 128, 128, 0, st>>>(proj, faces, F, is, 0.1f, 100.f, zbuf);
  k_raster_resolve<<<(image_size * image_size + 255) / 256, 256, 0, st>>>(zbuf, faces, rot, cam, image_size, supersample,
                                                                            rgb_out, mask_out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_dilate_count(const uint8_t* mask, int32_t n, int32_t iterations, uint8_t* dilated, int32_t* count_out,
                     avc_stream_t stream) {
  if (!mask || !dilated || !count_out) return AVC_E_NULL;
  if (n < 1 || iterations < 0 || iterations > 64) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  AVC_CUDA_TRY(cudaMemsetAsync(count_out, 0, sizeof(int32_t), st));
  k_dilate_count<<<(n * n + 255) / 256, 256, 0, st>>>(mask, n, iterations, dilated, count_out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_mask_compact(const uint8_t* dilated, int32_t n, int32_t W, int32_t cap, uint8_t* in_mask, int32_t* pix,
                     int32_t* count_out, avc_stream_t stream) {
  if (!dilated || !in_mask || !pix || !count_out) return AVC_E_NULL;
  if (n < 1 || W < 1 || W > 1024 || cap < 1) return AVC_E_SIZE;
  k_mask_compact<<<1, 1024, 0, (cudaStream_t)stream>>>(dilated, n, W, cap, in_mask, pix, count_out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_view_targets(const float* rgb, int32_t n, int32_t W, int32_t threshold_mask, float* true_rgb, float* mask,
                     avc_stream_t stream) {
  if (!rgb || !true_rgb || !mask) return AVC_E_NULL;
  if (n < 1 || W < 1) return AVC_E_SIZE;
  k_view_targets<<<(W * W + 255) / 256, 256, 0, (cudaStream_t)stream>>>(rgb, n, W, threshold_mask, true_rgb, mask);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_background_field(int32_t kind, int32_t H, int32_t W, uint32_t seed, int32_t chess_len, float sigma,
                         float* canvas_bg, const int32_t* pix, int32_t R, float* ray_bg, avc_stream_t stream) {
  if (!canvas_bg) return AVC_E_NULL;
  if (H < 1 || W < 1 || (kind != 1 && kind != 2)) return AVC_E_BADCFG;
  if (kind == 2 && (chess_len < 1 || !(sigma > 0.f))) return AVC_E_BADCFG;
  cudaStream_t st = (cudaStream_t)stream;
  const int n = H * W;
  if (kind == 1) k_bg_gauss<<<(n + 255) / 256, 256, 0, st>>>(seed, n, canvas_bg);
  else k_bg_chess<<<(n + 255) / 256, 256, 0, st>>>(H, W, chess_len, sigma, canvas_bg);
  if (pix && ray_bg && R > 0)      // main.py:412-413: background_rgb.reshape(H, W, 1)[dilated_mask]
    k_gather_f32<<<(R + 255) / 256, 256, 0, st>>>(canvas_bg, pix, R, ray_bg);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_uniform_fill(uint32_t seed, int32_t n, float lo, float hi, float* out, avc_stream_t stream) {
  if (!out) return AVC_E_NULL;
  if (n < 1) return AVC_E_SIZE;
  k_uniform_fill<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(seed, n, lo, hi, out);
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"
