// avc_neus_kernels.cuh -- device code of the NeuS path other than the GEMM tiles: weight packing,
// hierarchical sample placement, positional encoding, the thin (<= 8 wide) contractions, the
// per-ray compositing forward / backward and the epilogue functors plugged into the GEMM tiles.
//
// Reference citations are relative to AvatarGen/AppearanceGen of hongfz16/AvatarCLIP.
#pragma once
#include <cuda_bf16.h>

#include "avc_common.cuh"

namespace avc {

// Optional second copy of an activation as a two-term bf16 split (hi + lo), the operand format of the
// tcgen05 engine (avc_gemm_tc.cuh).  hi == nullptr: fp32 engine, nothing is written.
struct Split16 {
  __nv_bfloat16* hi; __nv_bfloat16* lo; int ld;
};
__device__ __forceinline__ void split16_put(const Split16& s, size_t row, int col, float v) {
  if (!s.hi) return;
  __nv_bfloat16 h = __float2bfloat16_rn(v);
  s.hi[row * s.ld + col] = h;
  s.lo[row * s.ld + col] = __float2bfloat16_rn(v - __bfloat162float(h));
}
// value of the two-term split at 4 consecutive columns: hi + lo (what the tcgen05 GEMMs see of this operand)
__device__ __forceinline__ void split16_get4(uint2 hi, uint2 lo, float v[4]) {
  v[0] = __uint_as_float(hi.x << 16) + __uint_as_float(lo.x << 16);
  v[1] = __uint_as_float(hi.x & 0xffff0000u) + __uint_as_float(lo.x & 0xffff0000u);
  v[2] = __uint_as_float(hi.y << 16) + __uint_as_float(lo.y << 16);
  v[3] = __uint_as_float(hi.y & 0xffff0000u) + __uint_as_float(lo.y & 0xffff0000u);
}
__device__ __forceinline__ float split16_get(const Split16& s, size_t row, int col) {
  return __bfloat162float(s.hi[row * s.ld + col]) + __bfloat162float(s.lo[row * s.ld + col]);
}
__device__ __forceinline__ void split16_put4(const Split16& s, size_t row, int col, const float v[4]) {
  if (!s.hi) return;
  const uint32_t h01 = bf16x2_bits(v[0], v[1]), h23 = bf16x2_bits(v[2], v[3]);
  const float r0 = v[0] - __uint_as_float(h01 << 16), r1 = v[1] - __uint_as_float(h01 & 0xffff0000u);
  const float r2 = v[2] - __uint_as_float(h23 << 16), r3 = v[3] - __uint_as_float(h23 & 0xffff0000u);
  *reinterpret_cast<uint2*>(s.hi + row * s.ld + col) = make_uint2(h01, h23);
  *reinterpret_cast<uint2*>(s.lo + row * s.ld + col) = make_uint2(bf16x2_bits(r0, r1), bf16x2_bits(r2, r3));
}

// SFU (ex2/lg2.approx based) softplus for the tcgen05 engine's epilogues, which are instruction-issue bound:
// |error| <~ 1e-8 absolute on softplus (value / 100), ~2 ulp on softplus'.  The fp32 engine keeps libm accuracy.
__device__ __forceinline__ float softplus100_fast(float z) {
  float bz = z * kBeta;
  return bz > kThresh ? z : __logf(1.0f + __expf(bz)) * (1.0f / kBeta);
}
// softplus' with SFU exp/div
__device__ __forceinline__ float softplus100_d1_fast(float z) {
  float bz = z * kBeta;
  float e = __expf(bz);
  return bz > kThresh ? 1.0f : __fdividef(e, e + 1.0f);
}
// =============================================================================================
// Weight packing: W = g * v / ||v||_row  (torch.nn.utils.weight_norm, models/fields.py:65-66,142-143)
// One block per output row.  Destinations: up to two column segments, each written row-major
// (W, leading dim ldw) and transposed (WT, leading dim ldwt); rows < row_shift of segment 0 go to
// `row0` instead (the sdf row of the last SDF linear).
// =============================================================================================
struct PackJob {
  const float* v; const float* g; const float* b;
  int N, K;
  int c0[2], c1[2];          // source column ranges of the two segments (c1 <= c0 => unused)
  float* W[2]; int ldw[2];   // W[s][(n - row_shift) * ldw + (c - c0)]
  float* WT[2]; int ldwt[2]; // WT[s][(c - c0) * ldwt + (n - row_shift)]
  int row_shift;             // 0, or 1 for the last SDF linear
  float* row0; float* row0_b;  // destination of row 0 when row_shift == 1
  float* bias; int bias_shift; // bias[n - bias_shift] for n >= bias_shift
  int dst_row_off;           // added to (n - row_shift): packs lin{Lc} and extra_lin into W6
};

// All linears of a call are packed by ONE launch: blockIdx.y selects the job, blockIdx.x the output row.
constexpr int kMaxJobs = 36;
struct PackJobs { int n; PackJob j[kMaxJobs]; };

__global__ void __launch_bounds__(128) k_pack_linear(const __grid_constant__ PackJobs jobs) {
  const PackJob& j = jobs.j[blockIdx.y];
  const int n = blockIdx.x;
  if (n >= j.N) return;
  const float* vr = j.v + (size_t)n * j.K;
  float ss = 0.f;
  for (int k = threadIdx.x; k < j.K; k += blockDim.x) ss += vr[k] * vr[k];
  __shared__ float red[4];
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = red[0] + red[1] + red[2] + red[3];
  const float sc = j.g[n] / sqrtf(tot);
  if (n < j.row_shift) {
    for (int k = threadIdx.x; k < j.K; k += blockDim.x) j.row0[k] = sc * vr[k];
    if (threadIdx.x == 0 && j.row0_b) j.row0_b[0] = j.b[n];
    return;
  }
  const int dn = n - j.row_shift + j.dst_row_off;
  for (int s = 0; s < 2; ++s) {
    if (j.c1[s] <= j.c0[s]) continue;
    for (int k = j.c0[s] + threadIdx.x; k < j.c1[s]; k += blockDim.x) {
      float w = sc * vr[k];
      if (j.W[s]) j.W[s][(size_t)dn * j.ldw[s] + (k - j.c0[s])] = w;
      if (j.WT[s]) j.WT[s][(size_t)(k - j.c0[s]) * j.ldwt[s] + dn] = w;
    }
  }
  if (threadIdx.x == 0 && j.bias && n >= j.bias_shift) j.bias[n - j.bias_shift + j.dst_row_off] = j.b[n];
}

// Weight-norm backward: Wbar (dense, in the v slot of `wbar`) -> gbar, vbar; bias grads copied.
//   gbar = sum_k Wbar * vhat ; vbar = g/||v|| (Wbar - gbar vhat)        (vhat = v/||v||)
struct WnJob { const float* v; const float* g; const float* Wbar; const float* bbar; int N, K; float* gg; float* gv; float* gb; };
struct WnJobs { int n; WnJob j[kMaxJobs]; };

__global__ void __launch_bounds__(128)
k_wn_backward(const __grid_constant__ WnJobs jobs) {
  const WnJob& J = jobs.j[blockIdx.y];
  const float* __restrict__ v = J.v; const float* __restrict__ g = J.g; const float* __restrict__ Wbar = J.Wbar;
  const float* __restrict__ bbar = J.bbar;
  const int N = J.N, K = J.K;
  float* __restrict__ gg = J.gg; float* __restrict__ gv = J.gv; float* __restrict__ gb = J.gb;
  const int n = blockIdx.x;
  if (n >= N) return;
  const float* vr = v + (size_t)n * K;
  const float* wr = Wbar + (size_t)n * K;
  float ss = 0.f, dot = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) { ss += vr[k] * vr[k]; dot += wr[k] * vr[k]; }
  __shared__ float r1[4], r2[4];
  ss = warp_sum(ss); dot = warp_sum(dot);
  if ((threadIdx.x & 31) == 0) { r1[threadIdx.x >> 5] = ss; r2[threadIdx.x >> 5] = dot; }
  __syncthreads();
  ss = r1[0] + r1[1] + r1[2] + r1[3];
  dot = r2[0] + r2[1] + r2[2] + r2[3];
  const float nv = sqrtf(ss);
  const float gbar = dot / nv;
  const float gn = g[n] / nv;
  for (int k = threadIdx.x; k < K; k += blockDim.x) gv[(size_t)n * K + k] = gn * (wr[k] - gbar * vr[k] / nv);
  if (threadIdx.x == 0) { gg[n] = gbar; gb[n] = bbar[n]; }
}

// =============================================================================================
// Positional encoding (models/embedder.py:11-36): e = [y, sin(2^k y), cos(2^k y)]_{k<L}, y = scale*x.
// =============================================================================================
struct EncodeTargets {
  float* in0; int ld0;              // in[0]: [P][EP]  <- e (padding columns zeroed)
  int n_skip;                       // skip layers: in[l][:, K-E .. K) <- e / sqrt(2)
  float* skip_ptr[4]; int skip_ld[4]; int skip_col[4];
  Split16 in0_16; Split16 skip16[4];   // tcgen05 engine copies (hi == nullptr: unused)
};

// One point is encoded by 8 cooperating lanes (group g = lane & 7): g = 0 writes the identity columns and the zero
// padding, g = 1.. write one frequency each (sin xyz, cos xyz; frequencies beyond 7 wrap around), so that the 8 lanes
// of a point cover its whole 160-byte row with adjacent pieces (coalesced) instead of one thread writing 40 floats.
__device__ __forceinline__ void encode_group(float x0, float x1, float x2, float scale, int multires, int E, int EP,
                                             int64_t p, int g, const EncodeTargets& t) {
  const float y[3] = {x0 * scale, x1 * scale, x2 * scale};
  // fp32 destinations may be NULL: the tcgen05 engine reads the encoding only through the bf16 pairs (except the fp32
  // input of the thin sdf head when the LAST linear takes the skip concat)
  float* r0 = t.in0 ? t.in0 + (size_t)p * t.ld0 : nullptr;
  auto put = [&](int c, float v) {
    if (r0) r0[c] = v;
    split16_put(t.in0_16, (size_t)p, c, v);
    for (int s = 0; s < t.n_skip; ++s) {
      if (t.skip_ptr[s]) t.skip_ptr[s][(size_t)p * t.skip_ld[s] + t.skip_col[s] + c] = v * kSqrtHalf;
      split16_put(t.skip16[s], (size_t)p, t.skip_col[s] + c, v * kSqrtHalf);
    }
  };
  if (g == 0) {
    put(0, y[0]); put(1, y[1]); put(2, y[2]);
    for (int c = E; c < EP; ++c) { if (r0) r0[c] = 0.f; split16_put(t.in0_16, (size_t)p, c, 0.f); }
  }
  for (int k = g - 1; k >= 0 && k < multires; k += 7) {
    const float f = (float)(1 << k);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float sn, cs;
      sincosf(y[c] * f, &sn, &cs);
      put(3 + 6 * k + c, sn);
      put(6 + 6 * k + c, cs);
    }
  }
}

// Sampling passes: points p = r * nz + j taken from z[r][j] (row pitch `pitch`).
__global__ void k_encode_samples(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                 const float* __restrict__ z, int nz, int pitch, int Rc, float scale, int multires, int E,
                                 int EP, EncodeTargets t) {
  int64_t id = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t p = id >> 3;
  if (p >= (int64_t)nz * Rc) return;
  int r = (int)(p / nz);
  float zz = z[(size_t)r * pitch + (p - (int64_t)r * nz)];
  // renderer.py:337 / :182: pts = rays_o + rays_d * z  (separately rounded mul and add, as torch does)
  float x0 = __fadd_rn(rays_o[r * 3 + 0], __fmul_rn(rays_d[r * 3 + 0], zz));
  float x1 = __fadd_rn(rays_o[r * 3 + 1], __fmul_rn(rays_d[r * 3 + 1], zz));
  float x2 = __fadd_rn(rays_o[r * 3 + 2], __fmul_rn(rays_d[r * 3 + 2], zz));
  encode_group(x0, x1, x2, scale, multires, E, EP, p, (int)(id & 7), t);
}

// Arbitrary query points [P][3] (SDFNetwork.sdf for extract_fields).
__global__ void k_encode_points(const float* __restrict__ pts, int64_t P, float scale, int multires, int E, int EP,
                                EncodeTargets t) {
  int64_t id = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t p = id >> 3;
  if (p >= P) return;
  encode_group(pts[p * 3 + 0], pts[p * 3 + 1], pts[p * 3 + 2], scale, multires, E, EP, p, (int)(id & 7), t);
}

// Fine pass (render_core, renderer.py:208-219): ray-major p = r * S + j.  Section midpoints, dists,
// mid_z / inside_sphere outputs, cin[p] = (x, 0,0,0, 0,0), encoding.
__global__ void k_encode_fine(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                              const float* __restrict__ z_vals, int S, int64_t Rc, float sample_dist,
                              float scale, int multires, int E, int EP, float* __restrict__ cin,
                              float* __restrict__ mid_z_out, float* __restrict__ inside_out, EncodeTargets t) {
  int64_t id = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t p = id >> 3;
  if (p >= Rc * S) return;
  const int g = (int)(id & 7);
  int64_t r = p / S;
  int j = (int)(p - r * S);
  float z0 = z_vals[p];
  float dist = (j + 1 < S) ? __fsub_rn(z_vals[p + 1], z0) : sample_dist;
  float mid = __fadd_rn(z0, __fmul_rn(dist, 0.5f));
  float x0 = __fadd_rn(rays_o[r * 3 + 0], __fmul_rn(rays_d[r * 3 + 0], mid));
  float x1 = __fadd_rn(rays_o[r * 3 + 1], __fmul_rn(rays_d[r * 3 + 1], mid));
  float x2 = __fadd_rn(rays_o[r * 3 + 2], __fmul_rn(rays_d[r * 3 + 2], mid));
  if (g == 7) {       // the lane without a frequency of its own (multires <= 6) writes the per-point extras
    float4* c = reinterpret_cast<float4*>(cin + (size_t)p * 8);
    c[0] = make_float4(x0, x1, x2, 0.f);
    c[1] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (mid_z_out) mid_z_out[p] = mid;
    if (inside_out) {
      float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x0, x0), __fmul_rn(x1, x1)), __fmul_rn(x2, x2)));
      inside_out[p] = nrm < 1.0f ? 1.f : 0.f;
    }
  }
  encode_group(x0, x1, x2, scale, multires, E, EP, p, g, t);
}

// =============================================================================================
// Hierarchical sample placement (renderer.py:302-352, 133-193, 39-69).  One thread per ray; every
// per-ray array lives in sample-major global buffers [j][r] so that a warp's accesses coalesce.
// Discontinuous decisions (bin search, radius < 1) use separately rounded mul/add like torch eager.
// =============================================================================================
__device__ __forceinline__ float torch_linspace(float start, float end, int n, int j) {
  // at::linspace's CUDA kernel (float): step = (end-start)/(n-1); first half start + step*j, second half
  // end - step*(n-1-j), each contracted into one FMA as torch's build compiles it
  if (n == 1) return start;
  float step = (end - start) / (float)(n - 1);
  return (j < n / 2) ? __fmaf_rn(step, (float)j, start) : __fmaf_rn(-step, (float)(n - 1 - j), end);
}

// Placement buffers are RAY-MAJOR [ray][pitch]; one warp per ray.
__global__ void k_coarse_z(const float* __restrict__ near, const float* __restrict__ far,
                           const float* __restrict__ jitter, int n, int pitch, int Rc, float* __restrict__ z) {
  int64_t id = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (int64_t)Rc * n) return;
  int r = (int)(id / n), j = (int)(id % n);
  float nr = near[r], fr = far[r];
  float span = __fsub_rn(fr, nr);
  float zz = __fadd_rn(nr, __fmul_rn(span, torch_linspace(0.f, 1.f, n, j)));   // renderer.py:305-306
  // renderer.py:319; torch divides a CUDA tensor by a scalar as a product with the scalar's fp32 reciprocal
  if (jitter) zz = __fadd_rn(zz, __fmul_rn(__fmul_rn(jitter[r], 2.0f), __frcp_rn((float)n)));
  z[(size_t)r * pitch + j] = zz;
}

__device__ __forceinline__ float ray_radius(const float* o, const float* d, float z) {
  float x0 = __fadd_rn(o[0], __fmul_rn(d[0], z));
  float x1 = __fadd_rn(o[1], __fmul_rn(d[1], z));
  float x2 = __fadd_rn(o[2], __fmul_rn(d[2], z));
  return sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x0, x0), __fmul_rn(x1, x1)), __fmul_rn(x2, x2)));
}

__device__ __forceinline__ float warp_excl_prod_f(float v, float* total) {
  const int lane = threadIdx.x & 31;
  float inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc *= t;
  }
  *total = __shfl_sync(0xffffffffu, inc, 31);
  float ex = __shfl_up_sync(0xffffffffu, inc, 1);
  return lane == 0 ? 1.f : ex;
}

constexpr int kPlaceMaxN = 256;     // samples per ray handled by the placement kernels
constexpr int kPlaceMaxNew = 64;    // new samples per round

// up_sample (renderer.py:133-177) + sample_pdf(det=True) (:39-69).  n = current samples per ray.
// One warp per ray: section terms in blocks of 32 (neighbour values by shuffle), transmittance by a prefix-product
// scan, cdf by a prefix-sum scan into shared memory, one inverse-CDF lookup (binary search) per new sample.
__global__ void __launch_bounds__(256)
k_upsample(const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ z,
           const float* __restrict__ sdf, int n, int pitch, int Rc, float inv_s, int per, float* __restrict__ newz) {
  __shared__ float s_z[8][kPlaceMaxN];
  __shared__ float s_cdf[8][kPlaceMaxN];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + wib;
  if (r >= Rc) return;
  float* sz = s_z[wib];
  float* scdf = s_cdf[wib];
  const float o[3] = {rays_o[r * 3], rays_o[r * 3 + 1], rays_o[r * 3 + 2]};
  const float d[3] = {rays_d[r * 3], rays_d[r * 3 + 1], rays_d[r * 3 + 2]};
  const float* zr = z + (size_t)r * pitch;
  const float* sr = sdf + (size_t)r * pitch;
  const int nsec = n - 1;
  const int nb = (nsec + 31) >> 5;
  float wreg[kPlaceMaxN / 32];
  float carry_cos = 0.f, carry_T = 1.f, wsum = 0.f;
  for (int j = lane; j < n; j += 32) sz[j] = zr[j];
#pragma unroll
  for (int b = 0; b < kPlaceMaxN / 32; ++b) {
    wreg[b] = 0.f;
    if (b >= nb) continue;
    const int j = b * 32 + lane;
    const bool ok = j < nsec;
    float z0 = 0.f, z1 = 0.f, s0 = 0.f, s1 = 0.f;
    if (ok) { z0 = zr[j]; z1 = zr[j + 1]; s0 = sr[j]; s1 = sr[j + 1]; }
    const float dist = __fsub_rn(z1, z0);
    float cosv = ok ? __fdiv_rn(__fsub_rn(s1, s0), __fadd_rn(dist, 1e-5f)) : 0.f;
    float prev = __shfl_up_sync(0xffffffffu, cosv, 1);
    if (lane == 0) prev = carry_cos;                              // prev_cos of the first section is 0 (:162)
    carry_cos = __shfl_sync(0xffffffffu, cosv, 31);
    float alpha = 0.f;
    if (ok) {
      float inside = (ray_radius(o, d, z0) < 1.0f || ray_radius(o, d, z1) < 1.0f) ? 1.f : 0.f;
      float cm = fminf(fmaxf(fminf(prev, cosv), -1e3f), 0.0f) * inside;
      float mid_sdf = __fmul_rn(__fadd_rn(s0, s1), 0.5f);
      float half = __fmul_rn(__fmul_rn(cm, dist), 0.5f);
      float pc = sigmoidf_acc(__fmul_rn(__fsub_rn(mid_sdf, half), inv_s));
      float nc = sigmoidf_acc(__fmul_rn(__fadd_rn(mid_sdf, half), inv_s));
      alpha = __fdiv_rn(__fadd_rn(__fsub_rn(pc, nc), 1e-5f), __fadd_rn(pc, 1e-5f));
    }
    float total;
    float T = carry_T * warp_excl_prod_f(ok ? __fadd_rn(__fsub_rn(1.0f, alpha), 1e-7f) : 1.f, &total);
    carry_T *= total;
    float w = ok ? __fadd_rn(__fmul_rn(alpha, T), 1e-5f) : 0.f;    // weights + 1e-5 (renderer.py:41)
    wreg[b] = w;
    wsum += w;
  }
  wsum = warp_sum(wsum);
  // cdf[0] = 0, cdf[j+1] = cdf[j] + w_j / sum
  float carry = 0.f;
  if (lane == 0) scdf[0] = 0.f;
#pragma unroll
  for (int b = 0; b < kPlaceMaxN / 32; ++b) {
    if (b >= nb) continue;
    const int j = b * 32 + lane;
    float inc = __fdiv_rn(wreg[b], wsum);
#pragma unroll
    for (int of = 1; of < 32; of <<= 1) {
      float t = __shfl_up_sync(0xffffffffu, inc, of);
      if (lane >= of) inc += t;
    }
    if (j < nsec) scdf[j + 1] = carry + inc;
    carry += __shfl_sync(0xffffffffu, inc, 31);
  }
  __syncwarp();
  const float ustart = 0.5f / (float)per, uend = 1.0f - 0.5f / (float)per;
  for (int t = lane; t < per; t += 32) {
    const float u = torch_linspace(ustart, uend, per, t);
    int lo = 0, hi = n;                       // searchsorted(right=True): number of cdf entries <= u
    while (lo < hi) { int mid = (lo + hi) >> 1; if (scdf[mid] <= u) lo = mid + 1; else hi = mid; }
    const int below = max(lo - 1, 0), above = min(lo, n - 1);
    const float cb = scdf[below], ca = scdf[above], zb = sz[below], za = sz[above];
    float denom = __fsub_rn(ca, cb);
    if (denom < 1e-5f) denom = 1.0f;
    const float tt = __fdiv_rn(__fsub_rn(u, cb), denom);
    newz[(size_t)r * per + t] = __fadd_rn(zb, __fmul_rn(tt, __fsub_rn(za, zb)));
  }
}

// cat_z_vals (renderer.py:179-193): merge two ascending lists (old entries first on ties) by rank computation:
// rank(old i) = i + #{new < z_i}, rank(new t) = t + #{old <= newz_t}.  One warp per ray.
__global__ void __launch_bounds__(256)
k_merge(const float* __restrict__ z, const float* __restrict__ sdf, int n, int pitch, const float* __restrict__ newz,
        const float* __restrict__ news, int per, int Rc, float* __restrict__ zo, float* __restrict__ so, int pitch_o) {
  __shared__ float s_z[8][kPlaceMaxN];
  __shared__ float s_n[8][kPlaceMaxNew];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + wib;
  if (r >= Rc) return;
  float* sz = s_z[wib];
  float* sn = s_n[wib];
  for (int j = lane; j < n; j += 32) sz[j] = z[(size_t)r * pitch + j];
  for (int t = lane; t < per; t += 32) sn[t] = newz[(size_t)r * per + t];
  __syncwarp();
  for (int i = lane; i < n; i += 32) {
    const float v = sz[i];
    int lo = 0, hi = per;                    // # new strictly less than v
    while (lo < hi) { int mid = (lo + hi) >> 1; if (sn[mid] < v) lo = mid + 1; else hi = mid; }
    zo[(size_t)r * pitch_o + i + lo] = v;
    if (news) so[(size_t)r * pitch_o + i + lo] = sdf[(size_t)r * pitch + i];
  }
  for (int t = lane; t < per; t += 32) {
    const float v = sn[t];
    int lo = 0, hi = n;                      // # old less than or equal to v
    while (lo < hi) { int mid = (lo + hi) >> 1; if (sz[mid] <= v) lo = mid + 1; else hi = mid; }
    zo[(size_t)r * pitch_o + t + lo] = v;
    if (news) so[(size_t)r * pitch_o + t + lo] = news[(size_t)r * per + t];
  }
}

// =============================================================================================
// Thin contractions (<= 8 outputs): one warp per row, lanes stride the reduction with float4 loads.
//   v[i] = sum_k A[p,k] * W[i*ldw + k]  (+ b[i]);  Out functor consumes the NI values.
// =============================================================================================
// A warp takes kThinPPW consecutive rows: their loads are issued together (the pass is DRAM-latency bound: one row per
// warp left 1 KB in flight per warp) and every W chunk is read once for the four rows.  Per row the arithmetic and its
// order are those of the one-row form (lane-strided partial sums, then the xor butterfly).
constexpr int kThinPPW = 4;
template <int NI, typename Out>
__global__ void __launch_bounds__(256)
k_thin_nt(const float* __restrict__ A, int lda, int K, const float* __restrict__ W, int ldw,
          const float* __restrict__ b, int64_t P, Out out) {
  const int64_t p0 = ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * kThinPPW;
  if (p0 >= P) return;
  const int lane = threadIdx.x & 31;
  float acc[kThinPPW][NI];
#pragma unroll
  for (int j = 0; j < kThinPPW; ++j)
#pragma unroll
    for (int i = 0; i < NI; ++i) acc[j][i] = 0.f;
  for (int k = lane * 4; k < K; k += 128) {
    float4 a[kThinPPW];
#pragma unroll
    for (int j = 0; j < kThinPPW; ++j)       // rows past P re-read row p0 (valid memory); their result is dropped
      a[j] = *reinterpret_cast<const float4*>(A + (size_t)(p0 + j < P ? p0 + j : p0) * lda + k);
#pragma unroll
    for (int i = 0; i < NI; ++i) {
      const float4 w = *reinterpret_cast<const float4*>(W + (size_t)i * ldw + k);
#pragma unroll
      for (int j = 0; j < kThinPPW; ++j)
        acc[j][i] = fmaf(a[j].x, w.x, fmaf(a[j].y, w.y, fmaf(a[j].z, w.z, fmaf(a[j].w, w.w, acc[j][i]))));
    }
  }
#pragma unroll
  for (int j = 0; j < kThinPPW; ++j)
#pragma unroll
    for (int i = 0; i < NI; ++i) acc[j][i] = warp_sum(acc[j][i]) + (b ? b[i] : 0.f);
#pragma unroll
  for (int j = 0; j < kThinPPW; ++j)
    if (lane == j && p0 + j < P) out(p0 + j, acc[j]);
}

struct OutSdf {     // sdf = z_L[0] / scale   (models/fields.py:88); point p = r * nz + j is stored at [r][j] (row pitch)
  float* sdf; float inv_scale; int nz; int pitch;
  __device__ void operator()(int64_t p, const float* v) const {
    int64_t o = nz > 0 ? (p / nz) * pitch + (p % nz) : p;
    sdf[o] = v[0] * inv_scale;
  }
};
struct OutHeads {   // sigmoid of both colour heads (models/fields.py:180-184) -> rgb6[p][8]
  float* rgb6;
  __device__ void operator()(int64_t p, const float* v) const {
    float4 a = make_float4(sigmoidf_acc(v[0]), sigmoidf_acc(v[1]), sigmoidf_acc(v[2]), sigmoidf_acc(v[3]));
    float4 b = make_float4(sigmoidf_acc(v[4]), sigmoidf_acc(v[5]), 0.f, 0.f);
    reinterpret_cast<float4*>(rgb6 + (size_t)p * 8)[0] = a;
    reinterpret_cast<float4*>(rgb6 + (size_t)p * 8)[1] = b;
  }
};
struct OutNbarAdd { // nbar[p][0..2] += d loss / d normal coming through colour lin0 (columns 3..5)
  float* nbar;
  __device__ void operator()(int64_t p, const float* v) const {
    nbar[(size_t)p * 4 + 0] += v[3]; nbar[(size_t)p * 4 + 1] += v[4]; nbar[(size_t)p * 4 + 2] += v[5];
  }
};

// (A variant with 16-byte loads, four row lanes per block meeting in shared memory and 64-row blocks was measured:
// 45 us per launch against 27 us for this one -- twice the atomics and three resident blocks per SM; not kept.)
// out[i*si + c*sc] += sum_p S[p*lds + i] * Hm[p*ldh + c]   (i < NI, c < NC);  optional s_scale on S;
// optional bout[i] += sum_p S[p,i].  Rows i >= split go to (out2, bout2) with index i - split (two linears that share
// the activation Hm, e.g. the two colour heads, in one pass over it).  Blocks split the rows; threads own columns.
template <int NI>
__global__ void __launch_bounds__(256)
k_thin_tn(const float* __restrict__ S, int lds, float s_scale, const float* __restrict__ Hm, int ldh, int NC,
          int64_t P, int rows_per_block, float* __restrict__ out, int si, int sc, float* __restrict__ bout,
          int split, float* __restrict__ out2, float* __restrict__ bout2) {
  __shared__ float sS[64][NI];
  const int64_t p0 = (int64_t)blockIdx.x * rows_per_block;
  const int64_t p1 = min(P, p0 + (int64_t)rows_per_block);
  float bacc = 0.f;
  for (int cb = 0; cb < NC; cb += blockDim.x) {
    const int c = cb + threadIdx.x;
    float acc[NI];
#pragma unroll
    for (int i = 0; i < NI; ++i) acc[i] = 0.f;
    for (int64_t pb = p0; pb < p1; pb += 64) {
      int nr = (int)min((int64_t)64, p1 - pb);
      __syncthreads();
      for (int t = threadIdx.x; t < nr * NI; t += blockDim.x) {
        int rr = t / NI, ii = t % NI;
        sS[rr][ii] = S[(size_t)(pb + rr) * lds + ii] * s_scale;
      }
      __syncthreads();
      if (c < NC) {
        const float* hp = Hm + (size_t)pb * ldh + c;
        int rr = 0;
        for (; rr + 8 <= nr; rr += 8) {          // 8 independent loads in flight per thread
          float h[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) h[u] = hp[(size_t)(rr + u) * ldh];
#pragma unroll
          for (int u = 0; u < 8; ++u)
#pragma unroll
            for (int i = 0; i < NI; ++i) acc[i] = fmaf(sS[rr + u][i], h[u], acc[i]);
        }
        for (; rr < nr; ++rr) {
          float h = hp[(size_t)rr * ldh];
#pragma unroll
          for (int i = 0; i < NI; ++i) acc[i] = fmaf(sS[rr][i], h, acc[i]);
        }
      }
      if ((bout || bout2) && cb == 0 && threadIdx.x < NI)
        for (int rr = 0; rr < nr; ++rr) bacc += sS[rr][threadIdx.x];
    }
    if (c < NC) {
#pragma unroll
      for (int i = 0; i < NI; ++i) {
        float* o = (i < split) ? out + (size_t)i * si : out2 + (size_t)(i - split) * si;
        atomicAdd(o + (size_t)c * sc, acc[i]);
      }
    }
  }
  if (threadIdx.x < NI) {
    const int i = threadIdx.x;
    if (i < split) { if (bout) atomicAdd(bout + i, bacc); }
    else if (bout2) atomicAdd(bout2 + (i - split), bacc);
  }
}

// out[c] += scale * sum_p X[p*ld + c], c < NC
__global__ void __launch_bounds__(256)
k_colsum(const float* __restrict__ X, int ld, int NC, int64_t P, int rows_per_block, float scale,
         float* __restrict__ out) {
  const int64_t p0 = (int64_t)blockIdx.x * rows_per_block;
  const int64_t p1 = min(P, p0 + (int64_t)rows_per_block);
  for (int c = threadIdx.x; c < NC; c += blockDim.x) {
    float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};      // eight loads in flight per thread: the pass streams X once
    int64_t p = p0;
    for (; p + 7 < p1; p += 8) {
      float x[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) x[u] = X[(size_t)(p + u) * ld + c];
#pragma unroll
      for (int u = 0; u < 8; ++u) a[u] += x[u];
    }
    for (; p < p1; ++p) a[0] += X[(size_t)p * ld + c];
    atomicAdd(out + c, (((a[0] + a[1]) + (a[2] + a[3])) + ((a[4] + a[5]) + (a[6] + a[7]))) * scale);
  }
}

// =============================================================================================
// Gradient chain helpers (SDFNetwork.gradient, models/fields.py:96-107, as a reverse sweep).
// =============================================================================================
// u_L = row 0 of W_L (constant):  qt[L-1] = softplus'(z[L-1]) * ua_L ; ge initialised.  `zprev` is the stash of
// softplus'(z[L-1]) the value pass left (EpiValue::D1).
__global__ void k_chain_start(const float* __restrict__ wsdf, int KL, int skipL, int E, int EP,
                              const float* __restrict__ zprev, int Nprev, int Npp, int64_t P,
                              float* __restrict__ qt, float* __restrict__ ge, Split16 qt16) {
  // 4 consecutive columns per thread (Npp % 4 == 0)
  int64_t i4 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  int64_t tot = P * (int64_t)Npp;
  if (i4 < tot) {
    int64_t p = i4 / Npp;
    int c = (int)(i4 - p * Npp);
    const float4 z = *reinterpret_cast<const float4*>(zprev + i4);
    const float zz[4] = {z.x, z.y, z.z, z.w};
    float v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
      v[i] = (c + i < Nprev) ? zz[i] * wsdf[c + i] * (skipL ? kSqrtHalf : 1.f) : 0.f;
    if (qt) *reinterpret_cast<float4*>(qt + i4) = make_float4(v[0], v[1], v[2], v[3]);
    split16_put4(qt16, (size_t)p, c, v);
  }
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P * (int64_t)EP) {
    int64_t p = i / EP;
    int e = (int)(i - p * EP);
    ge[i] = (skipL && e < E) ? wsdf[KL - E + e] * kSqrtHalf : 0.f;
  }
}

// n = D(y)^T ge  (grad_x sdf); writes cin[p][3..5] and the `gradients` output.
__global__ void k_normal(const float* __restrict__ ge, int EP, int multires, float scale, int64_t P,
                         float* __restrict__ cin, float* __restrict__ grad_out) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const float* g = ge + (size_t)p * EP;
  float* c = cin + (size_t)p * 8;
  float n[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    float y = c[a] * scale;
    float acc = g[a];
    float f = 1.f;
    for (int k = 0; k < multires; ++k) {
      float sn, cs;
      sincosf(y * f, &sn, &cs);
      acc += f * (cs * g[3 + 6 * k + a] - sn * g[6 + 6 * k + a]);
      f *= 2.f;
    }
    n[a] = acc;
  }
  c[3] = n[0]; c[4] = n[1]; c[5] = n[2];
  if (grad_out) { grad_out[p * 3 + 0] = n[0]; grad_out[p * 3 + 1] = n[1]; grad_out[p * 3 + 2] = n[2]; }
}

// gebar = D(y) nbar -> ubar0[p][ldu] (padding zeroed; the fp32 copy may be NULL) and gebar[p][EP].  8 lanes per
// point as in encode_group: lane 0 writes the identity columns and the padding, lanes 1..7 one frequency each
// (6 adjacent columns), so the lanes of a point cover its row with adjacent pieces.
__global__ void k_dge(const float* __restrict__ cin, const float* __restrict__ nbar, int EP, int E, int multires,
                      float scale, int64_t P, float* __restrict__ ubar0, int ldu, float* __restrict__ gebar,
                      Split16 u16) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t p = t >> 3;
  const int gl = (int)(t & 7);
  if (p >= P) return;
  const float* c = cin + (size_t)p * 8;
  const float nb[3] = {nbar[p * 4 + 0], nbar[p * 4 + 1], nbar[p * 4 + 2]};
  float* u = ubar0 ? ubar0 + (size_t)p * ldu : nullptr;
  float* g = gebar + (size_t)p * EP;
  auto put = [&](int col, float v) { if (u) u[col] = v; g[col] = v; split16_put(u16, (size_t)p, col, v); };
  if (gl == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) put(a, nb[a]);
    for (int col = E; col < EP; ++col) put(col, 0.f);
    for (int col = EP; col < ldu; ++col) { if (u) u[col] = 0.f; split16_put(u16, (size_t)p, col, 0.f); }
    return;
  }
  for (int k = gl - 1; k < multires; k += 7) {
    const float f = ldexpf(1.f, k);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      float sn, cs;
      sincosf(c[a] * scale * f, &sn, &cs);
      put(3 + 6 * k + a, f * cs * nb[a]);
      put(6 + 6 * k + a, -f * sn * nb[a]);
    }
  }
}

// ubar[p][col0 + e] = gebar[p][e] / sqrt(2)   (the encoding half of a skip layer's input adjoint)
__global__ void k_fill_gebar(const float* __restrict__ gebar, int EP, int E, int64_t P, float* __restrict__ ubar,
                             int ldu, int col0, Split16 u16) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P * (int64_t)E) return;
  int64_t p = i / E;
  int e = (int)(i - p * E);
  float v = gebar[(size_t)p * EP + e] * kSqrtHalf;
  ubar[(size_t)p * ldu + col0 + e] = v;
  split16_put(u16, (size_t)p, col0 + e, v);
}

// cbar[p][c] = (sum_i y6bar[p][i] * W6[i][c]) * [h[p][c] > 0]   (heads dgrad + ReLU mask)
__global__ void k_heads_dgrad(const float* __restrict__ y6bar, const float* __restrict__ W6, int Hc,
                              const float* __restrict__ h, int64_t P, float* __restrict__ cbar, Split16 c16) {
  // 4 consecutive columns per thread (Hc % 4 == 0): float4 loads / stores
  int64_t i4 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i4 >= P * (int64_t)Hc) return;
  int64_t p = i4 / Hc;
  int c = (int)(i4 - p * Hc);
  const float4 y0 = *reinterpret_cast<const float4*>(y6bar + (size_t)p * 8);
  const float4 y1 = *reinterpret_cast<const float4*>(y6bar + (size_t)p * 8 + 4);
  const float y[6] = {y0.x, y0.y, y0.z, y0.w, y1.x, y1.y};
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const float4 w = *reinterpret_cast<const float4*>(W6 + (size_t)k * Hc + c);
    acc[0] = fmaf(y[k], w.x, acc[0]); acc[1] = fmaf(y[k], w.y, acc[1]);
    acc[2] = fmaf(y[k], w.z, acc[2]); acc[3] = fmaf(y[k], w.w, acc[3]);
  }
  const float4 hv = *reinterpret_cast<const float4*>(h + i4);
  float v[4] = {hv.x > 0.f ? acc[0] : 0.f, hv.y > 0.f ? acc[1] : 0.f, hv.z > 0.f ? acc[2] : 0.f, hv.w > 0.f ? acc[3] : 0.f};
  if (cbar) *reinterpret_cast<float4*>(cbar + i4) = make_float4(v[0], v[1], v[2], v[3]);
  split16_put4(c16, (size_t)p, c, v);
}

// =============================================================================================
// GEMM epilogue functors.  (row, col..col+3, acc) with col % 4 == 0; N = valid output width.
//
// Every functor splits its work in two so that the wgmma epilogue can issue the global loads that do NOT depend on the
// accumulator ahead of the arithmetic, the first ones while the MMAs still run (the epilogue is bound by bytes in flight,
// not by issue slots):
//     Aux  prefetch(row, col)                      the stashed activations / biases this output group needs
//     void operator()(row, col, acc, aux)          the arithmetic and the stores
// operator()(row, col, acc) is the two back to back (what the fp32 FFMA engine calls).
// =============================================================================================
#define AVC_EPI_UNPACK float v[4] = {a.x, a.y, a.z, a.w}
#define AVC_EPI_DIRECT \
  __device__ __forceinline__ void operator()(int row, int col, float4 a) const { (*this)(row, col, a, prefetch(row, col)); }

// Ring-stored outputs (avc_gemm_tc.cuh) of the functors that write an fp32 copy and its split in whole 4-column groups
// (every group with col < n): output 0 the fp32 copy, outputs 1 / 2 the hi / lo halves, extent n rounded up to 4.
inline tc::OutOp epi_group_out(int i, float* out, int ldo, const Split16& s, int n) {
  const int cols = (n + 3) & ~3;
  return i == 0 ? tc::OutOp{out, ldo, cols} : tc::OutOp{i == 1 ? s.hi : s.lo, s.ld, cols};
}

// start of the last whole 4-column group below n, or `col` when that is smaller: an always-valid prefetch address
__device__ __forceinline__ int clamp_group(int col, int n) { return max(0, min(col, (n - 4) & ~3)); }

__device__ __forceinline__ float4 load4_guarded(const float* p, int col, int N) {
  float4 r;
  r.x = col < N ? p[col] : 0.f; r.y = col + 1 < N ? p[col + 1] : 0.f;
  r.z = col + 2 < N ? p[col + 2] : 0.f; r.w = col + 3 < N ? p[col + 3] : 0.f;
  return r;
}

// value chain: z = acc + b ; OUT[row][col] = softplus(z) * oscale (col < N) ; D1[row][col] = softplus'(z) (padding
// zero): the stash every later pass needs -- the gradient chain, the second-order sweep and the value backward only
// ever use softplus' (softplus'' = beta * sp' * (1 - sp')), so the pre-activation itself is not kept.
template <bool FAST>
struct EpiValue {
  static constexpr int kProbeId = 1;      // slot of the optional NT stall probe (avc_gemm_tc.cuh)
  const float* bias; float* D1; int ldz; float* OUT; int ldo; float oscale; int N; Split16 o16;
  struct Aux { float4 b; };
  __device__ __forceinline__ Aux prefetch(int, int col) const { return {load4_guarded(bias, col, N)}; }
  __device__ __forceinline__ void vals(int col, float4 a, const Aux& x, float hh[4], float dd[4]) const {
    AVC_EPI_UNPACK;
    const float bb[4] = {x.b.x, x.b.y, x.b.z, x.b.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      softplus100_both<FAST>(v[i] + bb[i], &hh[i], &dd[i]);
      hh[i] *= oscale;
      if (col + i >= N) { hh[i] = 0.f; dd[i] = 0.f; }
    }
  }
  // the NT tiles ring-store D1 (the whole padded width: its padding is zero), OUT and its split (columns < N: the rest
  // of a skip layer's input row is the encoding, written by k_encode_fine)
  using Out = tc::Outs<4, 4, 2, 2>;
  tc::OutOp out_op(int i, int) const {
    return i == 0 ? tc::OutOp{D1, ldz, ldz} : i == 1 ? tc::OutOp{OUT, ldo, N}
                                                     : tc::OutOp{i == 2 ? o16.hi : o16.lo, o16.ld, N};
  }
  template <typename S>
  __device__ __forceinline__ void ring(int, int col, float4 a, const Aux& x, const S& s) const {
    float dd[4], hh[4];
    vals(col, a, x, hh, dd);
    s.f32(0, dd); s.f32(1, hh); s.split(2, hh);
  }
  __device__ __forceinline__ void operator()(int row, int col, float4 a, const Aux& x) const {
    float dd[4], hh[4];
    vals(col, a, x, hh, dd);
    if (D1) *reinterpret_cast<float4*>(D1 + (size_t)row * ldz + col) = make_float4(dd[0], dd[1], dd[2], dd[3]);
    if (col + 3 < N) {
      if (OUT) *reinterpret_cast<float4*>(OUT + (size_t)row * ldo + col) = make_float4(hh[0], hh[1], hh[2], hh[3]);
      split16_put4(o16, (size_t)row, col, hh);
    } else {
      for (int i = 0; i < 4 && col + i < N; ++i) {
        if (OUT) OUT[(size_t)row * ldo + col + i] = hh[i];
        split16_put(o16, (size_t)row, col + i, hh[i]);
      }
    }
  }
  AVC_EPI_DIRECT
};

// out = acc + b (feature rows of the last SDF linear)
struct EpiBias {
  static constexpr int kProbeId = 9;      // slot of the optional NT stall probe (avc_gemm_tc.cuh)
  const float* bias; float* OUT; int ldo; int N; Split16 o16;
  struct Aux { float4 b; };
  __device__ __forceinline__ Aux prefetch(int, int col) const { return {load4_guarded(bias, col, N)}; }
  __device__ __forceinline__ void vals(int col, float4 a, const Aux& x, float v[4]) const {
    const float aa[4] = {a.x, a.y, a.z, a.w}, bb[4] = {x.b.x, x.b.y, x.b.z, x.b.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = (col + i < N) ? aa[i] + bb[i] : 0.f;
  }
  using Out = tc::Outs<4, 2, 2>;
  tc::OutOp out_op(int i, int n) const { return epi_group_out(i, OUT, ldo, o16, n); }
  template <typename S>
  __device__ __forceinline__ void ring(int, int col, float4 a, const Aux& x, const S& s) const {
    float v[4];
    vals(col, a, x, v);
    s.f32(0, v); s.split(1, v);
  }
  __device__ __forceinline__ void operator()(int row, int col, float4 a, const Aux& x) const {
    float v[4];
    vals(col, a, x, v);
    if (OUT) *reinterpret_cast<float4*>(OUT + (size_t)row * ldo + col) = make_float4(v[0], v[1], v[2], v[3]);
    split16_put4(o16, (size_t)row, col, v);
  }
  AVC_EPI_DIRECT
};

// gradient chain, layer l >= 1: u = acc (width K_l).  Columns < Nprev: ua = u * s, qt_prev = sp'(z_prev) * ua;
// columns >= Nprev (only when l is a skip layer): ge[col - Nprev] += u / sqrt(2).  Padding of qt_prev zeroed.
// D1prev = the softplus' stash of layer l-1.  QTprev (fp32 copy) may be NULL: the tcgen05 engine keeps only the split.
struct EpiChain {
  static constexpr int kProbeId = 2;      // slot of the optional NT stall probe (avc_gemm_tc.cuh)
  int Nprev, Npp; float s; const float* D1prev; float* QTprev; float* GE; int EP; int E; Split16 q16;
  struct Aux { float4 d; };
  __device__ __forceinline__ Aux prefetch(int row, int col) const {
    const int c = clamp_group(col, Npp);      // always a valid address; the value is only used where col + i < Nprev
    return {*reinterpret_cast<const float4*>(D1prev + (size_t)row * Npp + c)};
  }
  using Stage = tc::Staged<4>;                // the NT tiles stage D1prev in shared memory
  tc::StageOp stage_op(int) const { return {D1prev, Npp, Npp}; }
  static __device__ __forceinline__ Aux from_stage(const uint4 (&r)[1]) {
    return {make_float4(__uint_as_float(r[0].x), __uint_as_float(r[0].y), __uint_as_float(r[0].z), __uint_as_float(r[0].w))};
  }
  // qt_prev of the 4 columns (0 at columns >= Nprev); the ge accumulations of the columns >= Nprev are issued here
  __device__ __forceinline__ void vals(int row, int col, float4 a, const Aux& x, float q[4]) const {
    AVC_EPI_UNPACK;
    const float dd[4] = {x.d.x, x.d.y, x.d.z, x.d.w};      // D1prev[row][col + i] where col + i < Nprev <= Npp
    if (col + 3 < Nprev) {        // fast path: whole group inside the hidden part
#pragma unroll
      for (int i = 0; i < 4; ++i) q[i] = dd[i] * v[i] * s;
      return;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = col + i;
      q[i] = c < Nprev ? dd[i] * v[i] * s : 0.f;
      const int e = c - Nprev;
      // exclusive element: a fire-and-forget RED instead of a dependent load + store (written as red.global: with
      // atomicAdd the ring-storing NT tiles at BN = 128 spill about 300 bytes)
      if (c >= Nprev && e < E)
        asm volatile("red.global.add.f32 [%0], %1;" ::"l"(GE + (size_t)row * EP + e), "f"(v[i] * kSqrtHalf) : "memory");
    }
  }
  // The NT tiles ring-store qt_prev or its split (not both: the outputs are written over the staged sp' stash, whose
  // 16 x 32 fp32 box of a warp holds the fp32 copy or the hi and lo boxes) over the padded width Npp, whose padding gets
  // zeros.  The ge accumulations stay red.global from ring().
  using Out = tc::Outs<4, 2, 2>;
  tc::OutOp out_op(int i, int) const {
    return i == 0 ? tc::OutOp{QTprev, Npp, Npp} : tc::OutOp{i == 1 ? q16.hi : q16.lo, q16.ld, Npp};
  }
  __host__ __device__ static constexpr tc::Over over(int i) { return i == 0 ? tc::Over{0, 0, 1} : tc::Over{0, i - 1, 1}; }
  template <typename S>
  __device__ __forceinline__ void ring(int row, int col, float4 a, const Aux& x, const S& sk) const {
    float q[4];
    vals(row, col, a, x, q);
    sk.f32(0, q); sk.split(1, q);
  }
  __device__ __forceinline__ void operator()(int row, int col, float4 a, const Aux& x) const {
    float q[4];
    vals(row, col, a, x, q);
    if (col + 3 < Nprev) {
      if (QTprev) *reinterpret_cast<float4*>(QTprev + (size_t)row * Npp + col) = make_float4(q[0], q[1], q[2], q[3]);
      split16_put4(q16, (size_t)row, col, q);
      return;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = col + i;
      if (c < Npp) {
        if (QTprev) QTprev[(size_t)row * Npp + c] = q[i];
        split16_put(q16, (size_t)row, c, q[i]);
      }
    }
  }
  AVC_EPI_DIRECT
};

// gradient chain, layer 0: ge += acc  (width E)
struct EpiGe {
  static constexpr int kProbeId = 10;      // slot of the optional NT stall probe (avc_gemm_tc.cuh)
  float* GE; int EP; int E;
  struct Aux { float4 g; };
  __device__ __forceinline__ Aux prefetch(int row, int col) const {     // EP % 4 == 0: the padding is addressable
    return {*reinterpret_cast<const float4*>(GE + (size_t)row * EP + clamp_group(col, EP))};
  }
  __device__ __forceinline__ void operator()(int row, int col, float4 a, const Aux& x) const {
    AVC_EPI_UNPACK;
    const float gg[4] = {x.g.x, x.g.y, x.g.z, x.g.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (col + i < E) GE[(size_t)row * EP + col + i] = gg[i] + v[i];
  }
  // The NT tiles ring-store ge over its padded width EP: a padding column gets ge + acc = ge back (acc is 0 at columns
  // >= E = N, whose B rows TMA reads as zeros), so only the columns < E change, as on the register path.
  using Out = tc::Outs<4>;
  tc::OutOp out_op(int, int) const { return {GE, EP, EP}; }
  template <typename S>
  __device__ __forceinline__ void ring(int, int, float4 a, const Aux& x, const S& s) const {
    const float v[4] = {x.g.x + a.x, x.g.y + a.y, x.g.z + a.z, x.g.w + a.w};
    s.f32(0, v);
  }
  AVC_EPI_DIRECT
};

// colour lin0: z = acc + b + cin6 . Wx[col] ; out = relu(z)        (models/fields.py:162-171)
// WxT = the 6 point / normal columns of W0, transposed: [6][ldt] (one float4 per input for 4 output columns)
struct EpiColor0 {
  static constexpr int kProbeId = 7;      // slot of the optional NT stall probe (avc_gemm_tc.cuh)
  const float* bias; const float* cin; const float* WxT; int ldt; float* OUT; int ldo; Split16 o16;
  struct Aux { float4 c0, c1; };
  __device__ __forceinline__ Aux prefetch(int row, int) const {
    return {*reinterpret_cast<const float4*>(cin + (size_t)row * 8), *reinterpret_cast<const float4*>(cin + (size_t)row * 8 + 4)};
  }
  __device__ __forceinline__ void vals(int col, float4 a, const Aux& x, float v[4]) const {
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    const float cj[6] = {x.c0.x, x.c0.y, x.c0.z, x.c0.w, x.c1.x, x.c1.y};
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] += bias[col + i];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const float4 w = *reinterpret_cast<const float4*>(WxT + (size_t)j * ldt + col);
      v[0] = fmaf(cj[j], w.x, v[0]); v[1] = fmaf(cj[j], w.y, v[1]);
      v[2] = fmaf(cj[j], w.z, v[2]); v[3] = fmaf(cj[j], w.w, v[3]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = fmaxf(v[i], 0.f);
  }
  // (not ring-stored: with the ring path the NT tiles spill a few registers at BN = 128)
  __device__ __forceinline__ void operator()(int row, int col, float4 a, const Aux& x) const {
    float v[4];
    vals(col, a, x, v);
    if (OUT) *reinterpret_cast<float4*>(OUT + (size_t)row * ldo + col) = make_float4(v[0], v[1], v[2], v[3]);
    split16_put4(o16, (size_t)row, col, v);
  }
  AVC_EPI_DIRECT
};

struct EpiRelu {
  static constexpr int kProbeId = 5;      // slot of the optional NT stall probe (avc_gemm_tc.cuh)
  const float* bias; float* OUT; int ldo; Split16 o16;
  struct Aux { float4 b; };
  __device__ __forceinline__ Aux prefetch(int, int col) const {
    return {make_float4(bias[col], bias[col + 1], bias[col + 2], bias[col + 3])};
  }
  __device__ __forceinline__ static void vals(float4 a, const Aux& x, float v[4]) {
    v[0] = fmaxf(a.x + x.b.x, 0.f); v[1] = fmaxf(a.y + x.b.y, 0.f);
    v[2] = fmaxf(a.z + x.b.z, 0.f); v[3] = fmaxf(a.w + x.b.w, 0.f);
  }
  using Out = tc::Outs<4, 2, 2>;
  tc::OutOp out_op(int i, int n) const { return epi_group_out(i, OUT, ldo, o16, n); }
  template <typename S>
  __device__ __forceinline__ void ring(int, int, float4 a, const Aux& x, const S& s) const {
    float v[4];
    vals(a, x, v);
    s.f32(0, v); s.split(1, v);
  }
  __device__ __forceinline__ void operator()(int row, int col, float4 a, const Aux& x) const {
    float v[4];
    vals(a, x, v);
    if (OUT) *reinterpret_cast<float4*>(OUT + (size_t)row * ldo + col) = make_float4(v[0], v[1], v[2], v[3]);
    split16_put4(o16, (size_t)row, col, v);
  }
  AVC_EPI_DIRECT
};

// colour dgrad: out = acc * [h > 0].  The mask comes from the fp32 activation Hm or, when Hm is NULL, from the hi
// half of its split (h >= 0 after the ReLU, so h > 0 <=> the bf16 is not +-0).  OUT (fp32 copy) may be NULL.
struct EpiDgradRelu {
  static constexpr int kProbeId = 6;      // slot of the optional NT stall probe (avc_gemm_tc.cuh)
  const float* Hm; const __nv_bfloat16* Hhi; float* OUT; int ld; Split16 o16;
  struct Aux { uint4 raw; };
  __device__ __forceinline__ Aux prefetch(int row, int col) const {
    if (Hm) return {*reinterpret_cast<const uint4*>(Hm + (size_t)row * ld + col)};
    const uint2 h = *reinterpret_cast<const uint2*>(Hhi + (size_t)row * o16.ld + col);
    return {make_uint4(h.x, h.y, 0u, 0u)};
  }
  using Out = tc::Outs<4, 2, 2>;
  tc::OutOp out_op(int i, int n) const { return epi_group_out(i, OUT, ld, o16, n); }
  template <typename S>
  __device__ __forceinline__ void ring(int, int, float4 a, const Aux& x, const S& s) const {
    float v[4];
    vals(a, x, v);
    s.f32(0, v); s.split(1, v);
  }
  __device__ __forceinline__ void operator()(int row, int col, float4 a, const Aux& x) const {
    float v[4];
    vals(a, x, v);
    if (OUT) *reinterpret_cast<float4*>(OUT + (size_t)row * ld + col) = make_float4(v[0], v[1], v[2], v[3]);
    split16_put4(o16, (size_t)row, col, v);
  }
  __device__ __forceinline__ void vals(float4 a, const Aux& x, float v[4]) const {
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    bool on[4];
    if (Hm) {
      on[0] = __uint_as_float(x.raw.x) > 0.f; on[1] = __uint_as_float(x.raw.y) > 0.f;
      on[2] = __uint_as_float(x.raw.z) > 0.f; on[3] = __uint_as_float(x.raw.w) > 0.f;
    } else {
      on[0] = (x.raw.x & 0x00007fffu) != 0u; on[1] = (x.raw.x & 0x7fff0000u) != 0u;
      on[2] = (x.raw.y & 0x00007fffu) != 0u; on[3] = (x.raw.y & 0x7fff0000u) != 0u;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = on[i] ? v[i] : 0.f;
  }
  AVC_EPI_DIRECT
};

struct EpiStore {
  static constexpr int kProbeId = 8;      // slot of the optional NT stall probe (avc_gemm_tc.cuh)
  float* OUT; int ldo; int N; Split16 o16;
  __device__ __forceinline__ void vals(int col, float4 a, float v[4]) const {
    const float aa[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = (col + i < N) ? aa[i] : 0.f;
  }
  using Out = tc::Outs<4, 2, 2>;
  tc::OutOp out_op(int i, int n) const { return epi_group_out(i, OUT, ldo, o16, n); }
  template <typename S>
  __device__ __forceinline__ void ring(int, int col, float4 a, const S& s) const {
    float v[4];
    vals(col, a, v);
    s.f32(0, v); s.split(1, v);
  }
  __device__ __forceinline__ void operator()(int row, int col, float4 a) const {
    float v[4];
    vals(col, a, v);
    if (OUT) *reinterpret_cast<float4*>(OUT + (size_t)row * ldo + col) = make_float4(v[0], v[1], v[2], v[3]);
    split16_put4(o16, (size_t)row, col, v);
  }
};

// second-order sweep, layer l < L: qbar = acc (width N_l).  D1 = softplus'(z_l) stash.
//   ubar_next[row][col] = sp'(z_l) * qbar * s_next            (col < N_l)
//   zbar_l[row][col]    = beta (1 - sp'(z_l)) * qt_l * qbar    (= softplus'' * ua_{l+1} * qbar), padding zeroed
struct EpiChainBwd {
  static constexpr int kProbeId = 3;      // slot of the optional NT stall probe (avc_gemm_tc.cuh)
  int N, Np; const float* D1; const float* QT; Split16 qt16; float* ZBAR; float* UNEXT; int ldu; float s_next; Split16 u16;
  // qt_l comes from its fp32 copy QT or, when QT is NULL (tcgen05 engine), from the split hi + lo
  struct Aux { float4 d; uint4 q; };
  __device__ __forceinline__ Aux prefetch(int row, int col) const {
    const size_t o = (size_t)row * Np + clamp_group(col, Np);
    Aux x;
    x.d = *reinterpret_cast<const float4*>(D1 + o);
    if (QT) {
      x.q = *reinterpret_cast<const uint4*>(QT + o);
    } else {
      const size_t o16 = (size_t)row * qt16.ld + clamp_group(col, Np);
      const uint2 h = *reinterpret_cast<const uint2*>(qt16.hi + o16), l = *reinterpret_cast<const uint2*>(qt16.lo + o16);
      x.q = make_uint4(h.x, h.y, l.x, l.y);
    }
    return x;
  }
  // the NT tiles stage D1 and the split of qt in shared memory (they never get the fp32 copy QT)
  using Stage = tc::Staged<4, 2, 2>;
  tc::StageOp stage_op(int i) const {
    if (QT || Np % 4 || N > Np) return {nullptr, 0, 0};
    return i == 0 ? tc::StageOp{D1, Np, Np} : tc::StageOp{i == 1 ? qt16.hi : qt16.lo, qt16.ld, Np};
  }
  static __device__ __forceinline__ Aux from_stage(const uint4 (&r)[3]) {
    return {make_float4(__uint_as_float(r[0].x), __uint_as_float(r[0].y), __uint_as_float(r[0].z), __uint_as_float(r[0].w)),
            make_uint4(r[1].x, r[1].y, r[2].x, r[2].y)};
  }
  // Both engines call with col < N and col % 4 == 0, and Np (a multiple of 8) >= N: every group lies inside the PADDED
  // width.  The padding of the sp' stash and of qt is zero (EpiValue / EpiChain), so the padding columns of a group get
  // the zeros the padding of ubar / zbar must hold.
  __device__ __forceinline__ void vals(float4 a, const Aux& x, float u[4], float zb[4]) const {
    AVC_EPI_UNPACK;
    const float dd[4] = {x.d.x, x.d.y, x.d.z, x.d.w};
    float qq[4];
    if (QT) { qq[0] = __uint_as_float(x.q.x); qq[1] = __uint_as_float(x.q.y); qq[2] = __uint_as_float(x.q.z); qq[3] = __uint_as_float(x.q.w); }
    else split16_get4(make_uint2(x.q.x, x.q.y), make_uint2(x.q.z, x.q.w), qq);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      u[i] = dd[i] * v[i] * s_next;
      zb[i] = kBeta * (1.f - dd[i]) * qq[i] * v[i];
    }
  }
  // The NT tiles ring-store zbar over the staged sp' stash and ubar_next's split over the staged split of qt, or, at the
  // last linear, ubar_next's fp32 copy over both halves of qt (two boxes of 8 columns): not the copy and the split at
  // once.  Every extent is the padded width Np, whose padding gets zeros (zero sp' / qt padding, acc = 0 past N).  Into
  // a skip layer (N = 217 of a 256-wide ubar_next) that writes zeros to ubar_next's columns 217..223, which hold the
  // encoding half of the skip input's adjoint: backward() launches k_fill_gebar after this GEMM, and it rewrites columns
  // 217..255.
  using Out = tc::Outs<4, 4, 2, 2>;
  tc::OutOp out_op(int i, int) const {
    return i == 0 ? tc::OutOp{ZBAR, Np, Np} : i == 1 ? tc::OutOp{UNEXT, ldu, Np}
                                               : tc::OutOp{i == 2 ? u16.hi : u16.lo, u16.ld, Np};
  }
  __host__ __device__ static constexpr tc::Over over(int i) {
    return i == 0 ? tc::Over{0, 0, 1} : i == 1 ? tc::Over{1, 0, 2} : tc::Over{i - 1, 0, 1};
  }
  template <typename S>
  __device__ __forceinline__ void ring(int, int, float4 a, const Aux& x, const S& s) const {
    float u[4], zb[4];
    vals(a, x, u, zb);
    s.f32(0, zb); s.f32(1, u); s.split(2, u);
  }
  __device__ __forceinline__ void operator()(int row, int col, float4 a, const Aux& x) const {
    float u[4], zb[4];
    vals(a, x, u, zb);
    if (UNEXT) *reinterpret_cast<float4*>(UNEXT + (size_t)row * ldu + col) = make_float4(u[0], u[1], u[2], u[3]);
    split16_put4(u16, (size_t)row, col, u);
    *reinterpret_cast<float4*>(ZBAR + (size_t)row * Np + col) = make_float4(zb[0], zb[1], zb[2], zb[3]);
  }
  AVC_EPI_DIRECT
};

// value backward dgrad into layer l-1: abar = (acc [+ sdfbar[row] * wsdf[col]]) * s ;
//   zbar_prev[row][col] = sp'(z_prev) * abar + zbar_prev[row][col]   (col < Nprev);  D1prev = softplus'(z_prev) stash
struct EpiDgrad {
  static constexpr int kProbeId = 4;      // slot of the optional NT stall probe (avc_gemm_tc.cuh)
  int Nprev, Npp; float s; const float* D1prev; float* ZBARprev; const float* sdfbar; const float* wsdf;
  float sdf_inv_scale; Split16 z16; int store_f32;     // store_f32 = 0: only the split of the new zbar_prev is kept
  struct Aux { float4 d, zb; };
  __device__ __forceinline__ Aux prefetch(int row, int col) const {
    const size_t o = (size_t)row * Npp + clamp_group(col, Npp);
    return {*reinterpret_cast<const float4*>(D1prev + o), *reinterpret_cast<const float4*>(ZBARprev + o)};
  }
  using Stage = tc::Staged<4, 4>;             // the NT tiles stage D1prev and ZBARprev in shared memory
  tc::StageOp stage_op(int i) const {
    if (Npp % 4 || Nprev > Npp) return {nullptr, 0, 0};
    return {i == 0 ? D1prev : ZBARprev, Npp, Npp};
  }
  static __device__ __forceinline__ Aux from_stage(const uint4 (&r)[2]) {
    return {make_float4(__uint_as_float(r[0].x), __uint_as_float(r[0].y), __uint_as_float(r[0].z), __uint_as_float(r[0].w)),
            make_float4(__uint_as_float(r[1].x), __uint_as_float(r[1].y), __uint_as_float(r[1].z), __uint_as_float(r[1].w))};
  }
  // Both engines call with col < Nprev and col % 4 == 0, and Npp (a multiple of 8) >= Nprev: every group lies inside the
  // padded width, where the sp' stash and the zbar padding are zero, and so is the result.
  __device__ __forceinline__ void vals(int row, int col, float4 a, const Aux& x, float r[4]) const {
    AVC_EPI_UNPACK;
    float sb = sdfbar ? sdfbar[row] * sdf_inv_scale : 0.f;
    const float dd[4] = {x.d.x, x.d.y, x.d.z, x.d.w}, zo[4] = {x.zb.x, x.zb.y, x.zb.z, x.zb.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float ab = v[i];
      if (sdfbar) ab = fmaf(sb, wsdf[col + i], ab);
      r[i] = fmaf(dd[i], ab * s, zo[i]);
    }
  }
  // The NT tiles ring-store the new zbar_prev over the padded width Npp (its padding gets zeros): the split's hi and lo
  // boxes over the staged sp' stash, the fp32 copy (store_f32) over the staged old zbar_prev.
  using Out = tc::Outs<4, 2, 2>;
  tc::OutOp out_op(int i, int) const {
    return i == 0 ? tc::OutOp{store_f32 ? ZBARprev : nullptr, Npp, Npp} : tc::OutOp{i == 1 ? z16.hi : z16.lo, z16.ld, Npp};
  }
  __host__ __device__ static constexpr tc::Over over(int i) { return i == 0 ? tc::Over{1, 0, 1} : tc::Over{0, i - 1, 1}; }
  template <typename S>
  __device__ __forceinline__ void ring(int row, int col, float4 a, const Aux& x, const S& sk) const {
    float r[4];
    vals(row, col, a, x, r);
    sk.f32(0, r); sk.split(1, r);
  }
  __device__ __forceinline__ void operator()(int row, int col, float4 a, const Aux& x) const {
    float r[4];
    vals(row, col, a, x, r);
    if (store_f32) *reinterpret_cast<float4*>(ZBARprev + (size_t)row * Npp + col) = make_float4(r[0], r[1], r[2], r[3]);
    split16_put4(z16, (size_t)row, col, r);
  }
  AVC_EPI_DIRECT
};

// =============================================================================================
// Compositing (render_core, renderer.py:234-286).  One warp per ray; samples in blocks of 32.
// =============================================================================================
struct CompositeArgs {
  const float* rays_d;      // [Rc][3]
  const float* z_vals;      // [Rc][S]
  const float* sdf;         // [P]
  const float* cin;         // [P][8]
  const float* rgb6;        // [P][8]
  const float* background;  // NULL | [3] | [Rc]
  int bg_kind;
  const float* ctx;         // ctx[CTX_INV_S]
  float cos_anneal;
  float sample_dist;
  int S; int64_t Rc;
};

struct SampleTerms { float alpha, araw, Pp, Pn, ep, en, tc, dist, gn, relax; };

__device__ __forceinline__ SampleTerms sample_terms(const CompositeArgs& A, int64_t r, int j, float inv_s,
                                                    const float d[3]) {
  SampleTerms t;
  int64_t p = r * A.S + j;
  float z0 = A.z_vals[p];
  t.dist = (j + 1 < A.S) ? __fsub_rn(A.z_vals[p + 1], z0) : A.sample_dist;
  const float4 c0 = *reinterpret_cast<const float4*>(A.cin + (size_t)p * 8);
  const float4 c1 = *reinterpret_cast<const float4*>(A.cin + (size_t)p * 8 + 4);
  const float n0 = c0.w, n1 = c1.x, n2 = c1.y;
  float sdf = A.sdf[p];
  t.tc = d[0] * n0 + d[1] * n1 + d[2] * n2;                                   // renderer.py:237
  float ic = -(fmaxf(-t.tc * 0.5f + 0.5f, 0.f) * (1.0f - A.cos_anneal) + fmaxf(-t.tc, 0.f) * A.cos_anneal);
  t.en = sdf + ic * t.dist * 0.5f;                                            // :245-246
  t.ep = sdf - ic * t.dist * 0.5f;
  t.Pp = sigmoidf_acc(t.ep * inv_s);
  t.Pn = sigmoidf_acc(t.en * inv_s);
  t.araw = (t.Pp - t.Pn + 1e-5f) / (t.Pp + 1e-5f);                            // :251-254
  t.alpha = fminf(fmaxf(t.araw, 0.f), 1.f);
  t.gn = sqrtf(n0 * n0 + n1 * n1 + n2 * n2);
  float xn = sqrtf(c0.x * c0.x + c0.y * c0.y + c0.z * c0.z);
  t.relax = xn < 1.2f ? 1.f : 0.f;                                            // :258
  return t;
}

__device__ __forceinline__ float warp_excl_prod(float v, float* total) {
  // exclusive prefix product over lanes; *total = product of all lanes
  const int lane = threadIdx.x & 31;
  float inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc *= t;
  }
  *total = __shfl_sync(0xffffffffu, inc, 31);
  float ex = __shfl_up_sync(0xffffffffu, inc, 1);
  return lane == 0 ? 1.f : ex;
}

__global__ void __launch_bounds__(256)
k_composite_fwd(CompositeArgs A, float* __restrict__ color, float* __restrict__ extra, float* __restrict__ s_val,
                float* __restrict__ cdf, float* __restrict__ wsum_out, float* __restrict__ wmax_out,
                float* __restrict__ weights, float* __restrict__ ray_part) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= A.Rc) return;
  const int lane = threadIdx.x & 31;
  const float inv_s = A.ctx[CTX_INV_S];
  const float d[3] = {A.rays_d[r * 3], A.rays_d[r * 3 + 1], A.rays_d[r * 3 + 2]};
  float carry = 1.f;
  float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float wsum = 0.f, wmax = -1.f, eik_num = 0.f, eik_den = 0.f;
  for (int j0 = 0; j0 < A.S; j0 += 32) {
    const int j = j0 + lane;
    const bool ok = j < A.S;
    SampleTerms t;
    float one_m = 1.f;
    if (ok) {
      t = sample_terms(A, r, j, inv_s, d);
      one_m = 1.f - t.alpha + 1e-7f;                                          // :268
    }
    float total;
    float T = carry * warp_excl_prod(one_m, &total);
    carry *= total;
    if (ok) {
      const int64_t p = r * A.S + j;
      float w = t.alpha * T;
      weights[p] = w;
      cdf[p] = t.Pp;
      const float4 q0 = *reinterpret_cast<const float4*>(A.rgb6 + (size_t)p * 8);
      const float4 q1 = *reinterpret_cast<const float4*>(A.rgb6 + (size_t)p * 8 + 4);
      acc[0] += w * q0.x; acc[1] += w * q0.y; acc[2] += w * q0.z;
      acc[3] += w * q0.w; acc[4] += w * q1.x; acc[5] += w * q1.y;
      wsum += w;
      wmax = fmaxf(wmax, w);
      float e = t.gn - 1.f;
      eik_num += t.relax * e * e;                                             // :284-286
      eik_den += t.relax;
    }
  }
#pragma unroll
  for (int i = 0; i < 6; ++i) acc[i] = warp_sum(acc[i]);
  wsum = warp_sum(wsum); eik_num = warp_sum(eik_num); eik_den = warp_sum(eik_den);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) wmax = fmaxf(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
  if (lane == 0) {
    float bg[3] = {0.f, 0.f, 0.f};
    if (A.bg_kind == 1) { bg[0] = A.background[0]; bg[1] = A.background[1]; bg[2] = A.background[2]; }
    else if (A.bg_kind == 2) { bg[0] = bg[1] = bg[2] = A.background[r]; }
    color[r * 3 + 0] = acc[0]; color[r * 3 + 1] = acc[1]; color[r * 3 + 2] = acc[2];
    extra[r * 3 + 0] = acc[3] + bg[0] * (1.f - wsum);                          // :277-279 (extra_color=True)
    extra[r * 3 + 1] = acc[4] + bg[1] * (1.f - wsum);
    extra[r * 3 + 2] = acc[5] + bg[2] * (1.f - wsum);
    wsum_out[r] = wsum; wmax_out[r] = wmax;
    s_val[r] = 1.0f / inv_s;                                                   // :293, :383
    ray_part[r * 4 + 0] = eik_num; ray_part[r * 4 + 1] = eik_den;
  }
}

struct CompositeBwdArgs {
  const float* g_color; const float* g_extra; const float* g_wsum; const float* g_wmax;
  const float* g_w; const float* g_cdf; const float* g_n; const float* g_gerr;
  const float* weights;     // forward output [Rc][S] (for the argmax of weight_max)
  float* y6bar; float* sdfbar; float* nbar; float* ray_part;
};

__global__ void __launch_bounds__(256) k_composite_bwd(CompositeArgs A, CompositeBwdArgs G) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= A.Rc) return;
  const int lane = threadIdx.x & 31;
  const float inv_s = A.ctx[CTX_INV_S];
  const float eik_den_total = A.ctx[CTX_EIK_DEN];
  const float g_gerr = G.g_gerr ? G.g_gerr[0] : 0.f;
  const float d[3] = {A.rays_d[r * 3], A.rays_d[r * 3 + 1], A.rays_d[r * 3 + 2]};
  float gc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (G.g_color) { gc[0] = G.g_color[r * 3]; gc[1] = G.g_color[r * 3 + 1]; gc[2] = G.g_color[r * 3 + 2]; }
  if (G.g_extra) { gc[3] = G.g_extra[r * 3]; gc[4] = G.g_extra[r * 3 + 1]; gc[5] = G.g_extra[r * 3 + 2]; }
  float wbar_common = G.g_wsum ? G.g_wsum[r] : 0.f;
  if (A.bg_kind == 1) wbar_common -= gc[3] * A.background[0] + gc[4] * A.background[1] + gc[5] * A.background[2];
  else if (A.bg_kind == 2) wbar_common -= (gc[3] + gc[4] + gc[5]) * A.background[r];
  const int nb = (A.S + 31) >> 5;

  // argmax of the stored weights (first occurrence), only when weight_max has a cotangent
  int amax = -1;
  float g_wmax = 0.f;
  if (G.g_wmax) {
    g_wmax = G.g_wmax[r];
    float best = -1.f; int bi = 0x7fffffff;
    for (int j = lane; j < A.S; j += 32) {
      float w = G.weights[r * A.S + j];
      if (w > best) { best = w; bi = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float ob = __shfl_xor_sync(0xffffffffu, best, o);
      int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    amax = bi;
  }

  // pass A: recompute alpha, T, w and the total cotangent of w per sample
  SampleTerms tt[8];
  float Tj[8], wb[8], ww[8];
  float carry = 1.f;
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    if (b >= nb) break;
    const int j = b * 32 + lane;
    const bool ok = j < A.S;
    float one_m = 1.f;
    if (ok) { tt[b] = sample_terms(A, r, j, inv_s, d); one_m = 1.f - tt[b].alpha + 1e-7f; }
    float total;
    float T = carry * warp_excl_prod(one_m, &total);
    carry *= total;
    Tj[b] = T; wb[b] = 0.f; ww[b] = 0.f;
    if (ok) {
      const int64_t p = r * A.S + j;
      float w = tt[b].alpha * T;
      ww[b] = w;
      const float4 q0 = *reinterpret_cast<const float4*>(A.rgb6 + (size_t)p * 8);
      const float4 q1 = *reinterpret_cast<const float4*>(A.rgb6 + (size_t)p * 8 + 4);
      float wbar = wbar_common + (G.g_w ? G.g_w[p] : 0.f);
      wbar += gc[0] * q0.x + gc[1] * q0.y + gc[2] * q0.z + gc[3] * q0.w + gc[4] * q1.x + gc[5] * q1.y;
      if (j == amax) wbar += g_wmax;
      wb[b] = wbar;
      // colour heads: rgb6bar = w * g ; through the sigmoid
      float y[6] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y};
      float o6[8];
#pragma unroll
      for (int i = 0; i < 6; ++i) o6[i] = w * gc[i] * y[i] * (1.f - y[i]);
      o6[6] = o6[7] = 0.f;
      reinterpret_cast<float4*>(G.y6bar + (size_t)p * 8)[0] = make_float4(o6[0], o6[1], o6[2], o6[3]);
      reinterpret_cast<float4*>(G.y6bar + (size_t)p * 8)[1] = make_float4(o6[4], o6[5], 0.f, 0.f);
    }
  }
  // pass B: suffix sums  Asuf_j = sum_{t > j} wbar_t w_t   (reverse order over blocks and lanes)
  float invs_bar = 0.f;
  float suffix_carry = 0.f;
#pragma unroll
  for (int b = 7; b >= 0; --b) {
    if (b >= nb) continue;
    const int j = b * 32 + lane;
    const bool ok = j < A.S;
    float v = ok ? wb[b] * ww[b] : 0.f;
    float inc = v;   // inclusive suffix scan over lanes (lane 31 -> 0)
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      float t = __shfl_down_sync(0xffffffffu, inc, o);
      if (lane + o < 32) inc += t;
    }
    float block_total = __shfl_sync(0xffffffffu, inc, 0);
    float Asuf = inc - v + suffix_carry;
    suffix_carry += block_total;
    if (ok) {
      const SampleTerms& t = tt[b];
      const int64_t p = r * A.S + j;
      float abar = wb[b] * Tj[b] - Asuf / (1.f - t.alpha + 1e-7f);
      if (!(t.araw >= 0.f && t.araw <= 1.f)) abar = 0.f;                       // clip(0,1) (:254)
      float den = t.Pp + 1e-5f;
      float Ppbar = abar * t.Pn / (den * den) + (G.g_cdf ? G.g_cdf[p] : 0.f);
      float Pnbar = -abar / den;
      float dPp = t.Pp * (1.f - t.Pp), dPn = t.Pn * (1.f - t.Pn);
      float epbar = Ppbar * dPp * inv_s, enbar = Pnbar * dPn * inv_s;
      invs_bar += Ppbar * dPp * t.ep + Pnbar * dPn * t.en;
      G.sdfbar[p] = epbar + enbar;
      float icbar = (enbar - epbar) * t.dist * 0.5f;
      float tcbar = icbar * (0.5f * (1.f - A.cos_anneal) * (t.tc < 1.f ? 1.f : 0.f) + A.cos_anneal * (t.tc < 0.f ? 1.f : 0.f));
      const float4 c0 = *reinterpret_cast<const float4*>(A.cin + (size_t)p * 8);
      const float4 c1 = *reinterpret_cast<const float4*>(A.cin + (size_t)p * 8 + 4);
      float n[3] = {c0.w, c1.x, c1.y};
      float eik = (t.gn > 0.f) ? g_gerr * t.relax * 2.f * (t.gn - 1.f) / (eik_den_total + 1e-5f) / t.gn : 0.f;
      float nb3[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) nb3[a] = tcbar * d[a] + eik * n[a] + (G.g_n ? G.g_n[p * 3 + a] : 0.f);
      *reinterpret_cast<float4*>(G.nbar + (size_t)p * 4) = make_float4(nb3[0], nb3[1], nb3[2], 0.f);
    }
  }
  invs_bar = warp_sum(invs_bar);
  if (lane == 0) G.ray_part[r * 4 + 2] = invs_bar;
}

// Deterministic single-block reductions of the per-ray partials into ctx.
__global__ void __launch_bounds__(1024) k_reduce_ray_part(const float* __restrict__ ray_part, int64_t Rc, int comp,
                                                          float* __restrict__ dst) {
  __shared__ float red[32];
  float s = 0.f;
  for (int64_t r = threadIdx.x; r < Rc; r += blockDim.x) s += ray_part[r * 4 + comp];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) dst[0] += v;
  }
}

// Eikonal normaliser sum_p [ ||x_p|| < 1.2 ] recomputed from the geometry alone (renderer.py:258),
// so that the backward does not depend on scalars left in the workspace by the forward.
// One warp per ray, lanes <-> samples (a thread per ray walked its 128 samples serially: 22 us for 512 rays); the count is
// a sum of 0 / 1 terms, exact in any order.
__global__ void k_relax_count(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                              const float* __restrict__ z_vals, int S, int64_t Rc, float sample_dist,
                              float* __restrict__ ray_part) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= Rc) return;
  const int lane = threadIdx.x & 31;
  const float o0 = rays_o[r * 3 + 0], o1 = rays_o[r * 3 + 1], o2 = rays_o[r * 3 + 2];
  const float d0 = rays_d[r * 3 + 0], d1 = rays_d[r * 3 + 1], d2 = rays_d[r * 3 + 2];
  float cnt = 0.f;
  for (int j = lane; j < S; j += 32) {
    float z0 = z_vals[r * S + j];
    float dist = (j + 1 < S) ? __fsub_rn(z_vals[r * S + j + 1], z0) : sample_dist;
    float mid = __fadd_rn(z0, __fmul_rn(dist, 0.5f));
    float x0 = __fadd_rn(o0, __fmul_rn(d0, mid));
    float x1 = __fadd_rn(o1, __fmul_rn(d1, mid));
    float x2 = __fadd_rn(o2, __fmul_rn(d2, mid));
    cnt += sqrtf(x0 * x0 + x1 * x1 + x2 * x2) < 1.2f ? 1.f : 0.f;
  }
  cnt = warp_sum(cnt);
  if (lane == 0) ray_part[r * 4 + 1] = cnt;
}

__global__ void k_ctx_init(const float* __restrict__ params, int64_t off_var, float* __restrict__ ctx, int zero_sums) {
  if (threadIdx.x == 0) {
    float e = expf(params[off_var] * 10.0f);                                   // models/fields.py:276
    ctx[CTX_INV_S] = fminf(fmaxf(e, 1e-6f), 1e6f);                             // renderer.py:234
    if (zero_sums) { ctx[CTX_EIK_NUM] = 0.f; ctx[CTX_EIK_DEN] = 0.f; }
    ctx[CTX_INVS_BAR] = 0.f;
  }
}

__global__ void k_finalize_fwd(const float* __restrict__ ctx, float* __restrict__ gerr_out) {
  if (threadIdx.x == 0) gerr_out[0] = ctx[CTX_EIK_NUM] / (ctx[CTX_EIK_DEN] + 1e-5f);   // renderer.py:286
}

// variance gradient: inv_s = clip(exp(10 v)); s_val = 1/inv_s.
__global__ void __launch_bounds__(256)
k_variance_grad(const float* __restrict__ params, int64_t off_var, const float* __restrict__ ctx,
                const float* __restrict__ g_sval, int64_t R, float* __restrict__ grad_var) {
  __shared__ float red[8];
  float s = 0.f;
  if (g_sval) for (int64_t r = threadIdx.x; r < R; r += blockDim.x) s += g_sval[r];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f;
    for (int i = 0; i < 8; ++i) tot += red[i];
    float inv_s = ctx[CTX_INV_S];
    float e = expf(params[off_var] * 10.0f);
    float bar = ctx[CTX_INVS_BAR] - tot / (inv_s * inv_s);
    grad_var[0] = (e > 1e-6f && e < 1e6f) ? bar * 10.0f * inv_s : 0.f;
  }
}

// Fused Adam (torch.optim.Adam defaults; main.py:145,536-538).
__global__ void k_adam(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                       float* __restrict__ v, int64_t n, float lr, float b1, float b2, float eps, float bc1,
                       float bc2_sqrt, float gscale, float omb1, float omb2) {
  // omb1 / omb2 = (float)(1 - (double)beta): torch evaluates `1 - beta` in double before the cast (a float 1 - 0.999f is
  // 1.3e-5 off), lerp(m, g, 1 - b1) and v * b2 + (1 - b2) * g * g
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float gi = g[i] * gscale;
  float mi = m[i] = m[i] + omb1 * (gi - m[i]);
  float vi = v[i] = b2 * v[i] + omb2 * gi * gi;
  float denom = sqrtf(vi) / bc2_sqrt + eps;
  p[i] -= (lr / bc1) * (mi / denom);
}

// Device-state variant for CUDA-graph replay: state[0] = steps so far, state[1] = lr, state[2] = 1 - b1^t, state[3] =
// sqrt(1 - b2^t).
__global__ void k_adam_state(float* __restrict__ state, double b1d, double b2d) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    float t = state[0] + 1.0f;
    state[0] = t;
    state[2] = (float)(1.0 - pow((double)b1d, (double)t));
    state[3] = (float)sqrt(1.0 - pow((double)b2d, (double)t));
  }
}
__global__ void k_adam_dev(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                           float* __restrict__ v, int64_t n, const float* __restrict__ state, float b1, float b2,
                           float eps, float gscale, float omb1, float omb2) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float lr = state[1], bc1 = state[2], bc2_sqrt = state[3];
  float gi = g[i] * gscale;
  float mi = m[i] = m[i] + omb1 * (gi - m[i]);
  float vi = v[i] = b2 * v[i] + omb2 * gi * gi;
  float denom = sqrtf(vi) / bc2_sqrt + eps;
  p[i] -= (lr / bc1) * (mi / denom);
}

}  // namespace avc
