// avc_shape.cu -- ShapeGen's coarse body shape from a text prompt (AvatarGen/ShapeGen/main.py:93-123, utils.py:9-35):
//
//   avc_vae_decode         LinearVAE.decode (main.py:67-68): out[b] = W2 . (W1 . z[b] + b1) + b2 + v_template, B <= 8
//   avc_load_textures      neural_renderer's load_textures (nr.load_obj(..., load_texture=True, texture_size=8),
//                          utils.py:7): per-face R x R x R colour cubes bilinearly sampled from the UV image
//   avc_raster_textured    render_one_batch (utils.py:9-32): neural_renderer Renderer(camera_mode='look_at') of the
//                          textured mesh from one eye, ambient 0.5 + directional 0.5 along +y, 2 x 2 average pool
//   avc_clip_prep_nearest  F.interpolate(images, size=224) (nearest) + the CLIP Normalize (main.py:101-103)
//   avc_codebook_argmax    cos = F.normalize(C - e) . F.normalize(delta) and its first argmax (main.py:106-108)
//
// neural_renderer is neither vendored by the reference nor installable here: the texture loading and the textured
// rasteriser restate its published algorithm, as avc_view.cu does for the white template.  PARITY UNPINNED (oracle/
// shapegen.py says the same).
#include <cfloat>

#include "avc_common.cuh"
#include "avc_raster.cuh"

using namespace avc;

namespace {

// ---------------------------------------------------------------- LinearVAE.decode
constexpr int kDecMaxB = 8;
constexpr int kDecWarps = 8;           // 256 threads
constexpr int kDecRows = 4;            // W2 rows per warp
constexpr int kDecKT = 1024;           // hidden units staged in shared memory per tile

// h[b][j] = W1[j] . z[b] + b1[j]  (dec1, fp32 like nn.Linear)
__global__ void k_vae_hidden(const float* __restrict__ z, const float* __restrict__ W1, const float* __restrict__ b1,
                             int B, int L, int H, float* __restrict__ h) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * H) return;
  int b = i / H, j = i - b * H;
  float acc = 0.f;
  for (int k = 0; k < L; ++k) acc = fmaf(W1[(size_t)j * L + k], z[b * L + k], acc);
  h[i] = acc + b1[j];
}

// out[b][r] = (W2[r] . h[b] + b2[r]) + vt[r].  A pure stream of W2: each row is read once (evict-first float4 loads)
// for all B latents; the hidden vectors are staged tile by tile in shared memory.  A warp owns kDecRows rows.
template <int NB>
__global__ void __launch_bounds__(kDecWarps * 32)
k_vae_out(const float* __restrict__ h, const float* __restrict__ W2, const float* __restrict__ b2,
          const float* __restrict__ vt, int D, int H, float* __restrict__ out) {
  __shared__ __align__(16) float sh[NB * kDecKT];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int row0 = (blockIdx.x * kDecWarps + warp) * kDecRows;
  float acc[kDecRows][NB];
#pragma unroll
  for (int r = 0; r < kDecRows; ++r)
#pragma unroll
    for (int b = 0; b < NB; ++b) acc[r][b] = 0.f;
  const float4* wrow[kDecRows];
#pragma unroll
  for (int r = 0; r < kDecRows; ++r) wrow[r] = reinterpret_cast<const float4*>(W2 + (size_t)min(row0 + r, D - 1) * H);
  for (int k0 = 0; k0 < H; k0 += kDecKT) {
    const int kt = min(kDecKT, H - k0);
    __syncthreads();
    for (int i = threadIdx.x; i < NB * (kt >> 2); i += blockDim.x) {
      int b = i / (kt >> 2), q = i - b * (kt >> 2);
      reinterpret_cast<float4*>(sh + b * kDecKT)[q] = reinterpret_cast<const float4*>(h + (size_t)b * H + k0)[q];
    }
    __syncthreads();
#pragma unroll 2
    for (int q = lane; q < (kt >> 2); q += 32) {
      float4 w[kDecRows];
#pragma unroll
      for (int r = 0; r < kDecRows; ++r) w[r] = __ldcs(wrow[r] + (k0 >> 2) + q);
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        float4 x = reinterpret_cast<const float4*>(sh + b * kDecKT)[q];
#pragma unroll
        for (int r = 0; r < kDecRows; ++r)
          acc[r][b] = fmaf(w[r].x, x.x, fmaf(w[r].y, x.y, fmaf(w[r].z, x.z, fmaf(w[r].w, x.w, acc[r][b]))));
      }
    }
  }
#pragma unroll
  for (int r = 0; r < kDecRows; ++r)
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      float v = acc[r][b];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      acc[r][b] = v;
    }
  if (lane < kDecRows * NB) {       // lane (r, b) stores one output
    const int r = lane / NB, b = lane - r * NB, row = row0 + r;
    float v = 0.f;
#pragma unroll
    for (int rr = 0; rr < kDecRows; ++rr)
#pragma unroll
      for (int bb = 0; bb < NB; ++bb)
        if (rr == r && bb == b) v = acc[rr][bb];
    if (row < D) out[(size_t)b * D + row] = (v + b2[row]) + vt[row];
  }
}

template <int NB>
void launch_vae_out(const float* h, const float* W2, const float* b2, const float* vt, int D, int H, float* out,
                    cudaStream_t st) {
  const int rows_per_block = kDecWarps * kDecRows;
  k_vae_out<NB><<<(D + rows_per_block - 1) / rows_per_block, kDecWarps * 32, 0, st>>>(h, W2, b2, vt, D, H, out);
}

// ---------------------------------------------------------------- load_textures
// One thread per texel of the [F][R][R][R] cubes of the faces with is_update != 0.  Texel (i, j, k) holds the colour
// at the barycentric point (i, j, k) / (i + j + k) of the face's UV triangle ((0, 0, 0) samples the first corner);
// UVs wrap into [0, 1) (REPEAT); the image is flipped vertically (row 0 of `image` is the top of the picture, v = 0
// its bottom) and sampled bilinearly with the +1 neighbours clamped to the last row / column.
__global__ void k_load_textures(const float* __restrict__ image, int IH, int IW, const float* __restrict__ uv,
                                const int* __restrict__ is_update, int F, int R, float* __restrict__ tex) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long R3 = (long long)R * R * R;
  if (t >= (long long)F * R3) return;
  const int f = (int)(t / R3);
  if (!is_update[f]) return;
  const int c = (int)(t - (long long)f * R3);
  // positions in fp64: an fp32 uv * (size - 1) is off by ~size * 6e-8 pixels, visible against a sharp texture
  double d0 = (c / (R * R)) / (R - 1.0), d1 = ((c / R) % R) / (R - 1.0), d2 = (c % R) / (R - 1.0);
  const double s = d0 + d1 + d2;
  if (s > 0.0) { d0 /= s; d1 /= s; d2 /= s; }
  double u[3], v[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    double a = uv[(size_t)f * 6 + 2 * k], b = uv[(size_t)f * 6 + 2 * k + 1];
    u[k] = a - floor(a);
    v[k] = b - floor(b);
  }
  const double px = (u[0] * d0 + u[1] * d1 + u[2] * d2) * (IW - 1);
  const double py = (v[0] * d0 + v[1] * d1 + v[2] * d2) * (IH - 1);
  const int x0 = (int)px, y0 = (int)py;
  const int x1 = min(x0 + 1, IW - 1), y1 = min(y0 + 1, IH - 1);
  const double wx1 = px - x0, wx0 = 1.0 - wx1, wy1 = py - y0, wy0 = 1.0 - wy1;
  // flipped row y of the image = stored row IH - 1 - y
  const float* r0 = image + (size_t)(IH - 1 - y0) * IW * 3;
  const float* r1 = image + (size_t)(IH - 1 - y1) * IW * 3;
  float* o = tex + (size_t)t * 3;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch)
    o[ch] = (float)(r0[x0 * 3 + ch] * (wx0 * wy0) + r1[x0 * 3 + ch] * (wx0 * wy1) + r0[x1 * 3 + ch] * (wx1 * wy0) +
                    r1[x1 * 3 + ch] * (wx1 * wy1));
}

// ---------------------------------------------------------------- CLIP preprocessing
// images [B][n][n][3] -> out [B][3][S][S]: nearest (src = floor(dst * n / S)), then (x - mean) / std, each step in
// double rounded to float like the reference's in-place ops on a float32 tensor with float64 operands.
__global__ void k_clip_prep_nearest(const float* __restrict__ img, int B, int n, int S, float* __restrict__ out) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * 3 * S * S) return;
  const int x = (int)(i % S), y = (int)((i / S) % S), ch = (int)((i / ((long long)S * S)) % 3);
  const int b = (int)(i / (3LL * S * S));
  const double mean = ch == 0 ? 0.48145466 : (ch == 1 ? 0.4578275 : 0.40821073);
  const double stdv = ch == 0 ? 0.26862954 : (ch == 1 ? 0.26130258 : 0.27577711);
  const float scale = (float)n / (float)S;
  const int sy = min((int)floorf(y * scale), n - 1), sx = min((int)floorf(x * scale), n - 1);
  float v = img[(((size_t)b * n + sy) * n + sx) * 3 + ch];
  v = (float)((double)v - mean);
  out[i] = (float)((double)v / stdv);
}

// ---------------------------------------------------------------- codebook search
// one block per codebook row: cos[i] = sum_j (C[i][j] - e[j]) / max(|C[i] - e|, 1e-12) * d[j] / max(|d|, 1e-12);
// sums in fp64.  key = (ordered cos bits, ~index): the 64-bit atomicMax keeps the largest cos, on ties the smallest i.
__global__ void k_codebook_cos(const float* __restrict__ C, const float* __restrict__ e, const float* __restrict__ d,
                               int N, int D, float* __restrict__ cos_out, unsigned long long* __restrict__ key) {
  const int i = blockIdx.x;
  __shared__ double red[32];
  double cc = 0.0, cd = 0.0, dd = 0.0;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const double a = (double)(C[(size_t)i * D + j] - e[j]), g = (double)d[j];
    cc += a * a; cd += a * g; dd += g * g;
  }
  const auto add = [](double u, double v) { return u + v; };
  cc = block_reduce(cc, red, add, 0.0);
  cd = block_reduce(cd, red, add, 0.0);
  dd = block_reduce(dd, red, add, 0.0);
  if (threadIdx.x == 0) {
    const float c = (float)(cd / (fmax(sqrt(cc), 1e-12) * fmax(sqrt(dd), 1e-12)));
    cos_out[i] = c;
    atomicMax(key, sel_key(c, i));
  }
}

__global__ void k_codebook_best(const unsigned long long* __restrict__ key, int* __restrict__ best) {
  *best = sel_index(*key);
}

}  // namespace

extern "C" {

int avc_vae_decode_workspace_bytes(int32_t B, int32_t hidden, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (B < 1 || B > kDecMaxB || hidden < 4 || hidden % 4) return AVC_E_SIZE;
  Carver c(nullptr);
  c.take<float>((size_t)B * hidden);
  *bytes = c.used();
  return 0;
}

int avc_vae_decode(const float* z, int32_t B, int32_t latent, const float* W1, const float* b1, int32_t hidden,
                   const float* W2, const float* b2, const float* v_template, int32_t out_dim, float* out,
                   void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!z || !W1 || !b1 || !W2 || !b2 || !v_template || !out || !workspace) return AVC_E_NULL;
  size_t need = 0;
  AVC_TRY(avc_vae_decode_workspace_bytes(B, hidden, &need));
  if (latent < 1 || out_dim < 1 || workspace_bytes < need) return AVC_E_SIZE;
  if (reinterpret_cast<uintptr_t>(W2) % 16) return AVC_E_ALIGN;
  cudaStream_t st = (cudaStream_t)stream;
  Carver c(workspace);
  float* h = c.take<float>((size_t)B * hidden);
  k_vae_hidden<<<(B * hidden + 255) / 256, 256, 0, st>>>(z, W1, b1, B, latent, hidden, h);
  switch (B) {
    case 1: launch_vae_out<1>(h, W2, b2, v_template, out_dim, hidden, out, st); break;
    case 2: launch_vae_out<2>(h, W2, b2, v_template, out_dim, hidden, out, st); break;
    case 3: launch_vae_out<3>(h, W2, b2, v_template, out_dim, hidden, out, st); break;
    case 4: launch_vae_out<4>(h, W2, b2, v_template, out_dim, hidden, out, st); break;
    case 5: launch_vae_out<5>(h, W2, b2, v_template, out_dim, hidden, out, st); break;
    case 6: launch_vae_out<6>(h, W2, b2, v_template, out_dim, hidden, out, st); break;
    case 7: launch_vae_out<7>(h, W2, b2, v_template, out_dim, hidden, out, st); break;
    default: launch_vae_out<8>(h, W2, b2, v_template, out_dim, hidden, out, st); break;
  }
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_load_textures(const float* image, int32_t height, int32_t width, const float* face_uv,
                      const int32_t* is_update, int32_t F, int32_t R, float* textures, avc_stream_t stream) {
  if (!image || !face_uv || !is_update || !textures) return AVC_E_NULL;
  if (height < 1 || width < 1 || F < 1 || R < 2 || R > 64) return AVC_E_SIZE;
  const long long n = (long long)F * R * R * R;
  k_load_textures<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(image, height, width, face_uv,
                                                                                   is_update, F, R, textures);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_raster_textured_workspace_bytes(int32_t V, int32_t image_size, int32_t supersample, size_t* bytes) {
  if (!bytes) return AVC_E_NULL;
  if (V < 1 || image_size < 1 || image_size > 4096 || supersample < 1 || supersample > 4) return AVC_E_SIZE;
  Carver c(nullptr);
  c.take<float4>(V);
  c.take<unsigned long long>((size_t)image_size * supersample * image_size * supersample);
  *bytes = c.used();
  return 0;
}

int avc_raster_textured(const float* verts, const int32_t* faces, const float* textures, int32_t V, int32_t F,
                        int32_t R, const float* eye, const float* at, const float* up, int32_t image_size,
                        int32_t supersample, float* rgb_out, void* workspace, size_t workspace_bytes,
                        avc_stream_t stream) {
  if (!verts || !faces || !textures || !eye || !at || !up || !rgb_out || !workspace) return AVC_E_NULL;
  size_t need = 0;
  AVC_TRY(avc_raster_textured_workspace_bytes(V, image_size, supersample, &need));
  if (workspace_bytes < need || F < 1 || R < 2 || R > 64) return AVC_E_SIZE;
  const int is = image_size * supersample;
  LookAtCam cam;
  if (!make_look_at_cam(eye, at, up, is, &cam)) return AVC_E_BADCFG;
  cudaStream_t st = (cudaStream_t)stream;
  Carver c(workspace);
  float4* proj = c.take<float4>(V);
  unsigned long long* zbuf = c.take<unsigned long long>((size_t)is * is);
  AVC_CUDA_TRY(cudaMemsetAsync(zbuf, 0xff, sizeof(unsigned long long) * (size_t)is * is, st));
  k_project_look_at<<<(V + 255) / 256, 256, 0, st>>>(verts, V, cam, proj);
  k_raster_faces<<<(F + 127) / 128, 128, 0, st>>>(proj, faces, F, is, 0.1f, 100.f, zbuf);
  k_resolve_textured<<<(image_size * image_size + 255) / 256, 256, 0, st>>>(zbuf, faces, verts, proj, textures, R, cam,
                                                                            image_size, supersample, rgb_out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_clip_prep_nearest(const float* images, int32_t B, int32_t n, int32_t out_size, float* out,
                          avc_stream_t stream) {
  if (!images || !out) return AVC_E_NULL;
  if (B < 1 || n < 1 || out_size < 1) return AVC_E_SIZE;
  const long long total = (long long)B * 3 * out_size * out_size;
  k_clip_prep_nearest<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(images, B, n, out_size, out);
  AVC_LAUNCH_TRY();
  return 0;
}

int avc_codebook_argmax(const float* codebook, const float* image_emb, const float* delta, int32_t N, int32_t D,
                        float* cos_out, int32_t* best_out, void* workspace, size_t workspace_bytes,
                        avc_stream_t stream) {
  if (!codebook || !image_emb || !delta || !cos_out || !best_out || !workspace) return AVC_E_NULL;
  if (N < 1 || D < 1 || workspace_bytes < sizeof(unsigned long long)) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* key = static_cast<unsigned long long*>(workspace);
  AVC_CUDA_TRY(cudaMemsetAsync(key, 0, sizeof(unsigned long long), st));
  k_codebook_cos<<<N, 128, 0, st>>>(codebook, image_emb, delta, N, D, cos_out, key);
  k_codebook_best<<<1, 1, 0, st>>>(key, best_out);
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"
