// avc_common.cuh -- shared helpers for the sm_90a kernels of libavc_b200.so.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/avc_b200.h"

#define AVC_CUDA_TRY(expr)                      \
  do {                                          \
    cudaError_t e__ = (expr);                   \
    if (e__ != cudaSuccess) return (int)e__;    \
  } while (0)
#define AVC_LAUNCH_TRY()                        \
  do {                                          \
    cudaError_t e__ = cudaGetLastError();       \
    if (e__ != cudaSuccess) return (int)e__;    \
  } while (0)
#define AVC_TRY(expr)                           \
  do {                                          \
    int r__ = (expr);                           \
    if (r__ != 0) return r__;                   \
  } while (0)

namespace avc {

constexpr float kSqrtHalf = 0.70710678118654752440f;
constexpr float kBeta = 100.0f;      // nn.Softplus(beta=100), models/fields.py:70
constexpr float kThresh = 20.0f;     // torch's default softplus threshold

// scalar slots of the per-call context block (workspace header)
enum { CTX_INV_S = 0, CTX_EIK_NUM = 1, CTX_EIK_DEN = 2, CTX_INVS_BAR = 3, CTX_FLOATS = 64 };

static inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }
static inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// softplus_beta with torch's threshold rule: beta*z > 20 -> identity.
__device__ __forceinline__ float softplus100(float z) {
  float bz = z * kBeta;
  return bz > kThresh ? z : log1pf(expf(bz)) / kBeta;
}
// first derivative (torch softplus_backward: e/(e+1) with e = exp(beta z); 1 above the threshold)
__device__ __forceinline__ float softplus100_d1(float z) {
  float bz = z * kBeta;
  if (bz > kThresh) return 1.0f;
  float e = expf(bz);
  return e / (e + 1.0f);
}
// SFU primitives with flush-to-zero: no denormal pre/post-scaling around the MUFU instruction (the non-ftz forms expand
// to a compare + two predicated multiplies each)
__device__ __forceinline__ float ex2_ftz(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float lg2_ftz(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_ftz(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// softplus and softplus' of the same argument, sharing the exponential; branch free (the selects discard the inf / NaN
// the discarded arm produces for large arguments).  FAST: SFU ex2 / lg2 / rcp;  else libm accuracy.
template <bool FAST>
__device__ __forceinline__ void softplus100_both(float z, float* h, float* d1) {
  if (FAST) {
    const float e = ex2_ftz(z * (kBeta * 1.4426950408889634f));
    const float t = 1.0f + e;
    const bool big = z * kBeta > kThresh;
    *h = big ? z : lg2_ftz(t) * (0.6931471805599453f / kBeta);
    *d1 = big ? 1.0f : e * rcp_ftz(t);
  } else {
    *h = softplus100(z);
    *d1 = softplus100_d1(z);
  }
}

// two floats -> packed bf16x2 bits (element 0 in the low half)
__device__ __forceinline__ uint32_t bf16x2_bits(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);       // one F2FP.BF16.F32.PACK_AB
  return *reinterpret_cast<uint32_t*>(&t);
}

__device__ __forceinline__ float sigmoidf_acc(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// x reduced over the CTA by op, the result in every thread: an xor tree in each warp, then the warp results folded onto
// init in warp order.  The fold order is fixed, so a floating-point sum is the same on every run; init decides the sign
// of a zero sum.  red holds blockDim.x / 32 values (blockDim.x a multiple of 32).
template <class T, class Op>
__device__ __forceinline__ T block_reduce(T x, T* red, Op op, T init) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x = op(x, __shfl_xor_sync(0xffffffffu, x, o));
  __syncthreads();                      // red may still be read by a previous call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = x;
  __syncthreads();
  for (int w = 0, nw = blockDim.x >> 5; w < nw; ++w) init = op(init, red[w]);
  return init;
}

// The exclusive prefix sum of x over the CTA's NT threads in thread order, and in total the CTA's sum.  warp_tot holds
// 33 ints.
template <int NT>
__device__ __forceinline__ int block_exclusive_scan(int x, int* warp_tot, int& total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int inc = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  __syncthreads();                      // warp_tot may still be read by a previous call
  if (lane == 31) warp_tot[w] = inc;
  __syncthreads();
  if (w == 0) {
    int t = lane < NT / 32 ? warp_tot[lane] : 0, ti = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, ti, o);
      if (lane >= o) ti += y;
    }
    if (lane < NT / 32) warp_tot[lane] = ti - t;
    if (lane == 31) warp_tot[32] = ti;
  }
  __syncthreads();
  total = warp_tot[32];
  return warp_tot[w] + inc - x;
}

// avc_scan.cu: the in-place exclusive scan of a[0, n) (n >= 1) in index order over the whole device, and the sum of a
// to *total (it must fit in an int32).  sums is a workspace of exclusive_scan_sums(n) ints; what it held is not read.
size_t exclusive_scan_sums(int n);
void exclusive_scan(int* a, int n, int* sums, int32_t* total, cudaStream_t st);

// float -> uint32 whose unsigned order is the float order; -0.0 maps to +0.0's bits, so the two zeros are equal
__device__ __forceinline__ unsigned ordered_bits(float f) {
  const unsigned u = __float_as_uint(f) == 0x80000000u ? 0u : __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// key = (ordered value bits, ~index): the larger key is the larger value, on ties the smaller index (a 64-bit atomicMax
// or max reduction selects the first argmax); sel_index decodes the index
__device__ __forceinline__ unsigned long long sel_key(float v, int i) {
  return ((unsigned long long)ordered_bits(v) << 32) | (unsigned)(0xffffffffu - (unsigned)i);
}
__device__ __forceinline__ int sel_index(unsigned long long key) {
  return (int)(0xffffffffu - (unsigned)(key & 0xffffffffu));
}

// key = (bits of z, id) for z >= +0 (a depth, a collapse cost): the smaller key is the smaller z, on ties the smaller
// id, so a 64-bit atomicMin keeps the nearest (a -0.0 z keys above every positive one)
__device__ __forceinline__ unsigned long long depth_key(float z, int id) {
  return ((unsigned long long)__float_as_uint(z) << 32) | (unsigned)id;
}

// A carve-out allocator over the caller-provided workspace (256-byte aligned pieces).
struct Carver {
  char* base;
  size_t off;
  explicit Carver(void* p) : base((char*)p), off(0) {}
  template <typename T>
  T* take(size_t count) {
    off = (off + 255) & ~(size_t)255;
    T* r = base ? (T*)(base + off) : nullptr;
    off += count * sizeof(T);
    return r;
  }
  size_t used() const { return (off + 255) & ~(size_t)255; }
};

}  // namespace avc
