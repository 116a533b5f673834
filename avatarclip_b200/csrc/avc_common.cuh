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
  if (FAST) {       // same operations as softplus100_both4 (bit-identical results whichever form an epilogue path uses)
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

// softplus and softplus' of four independent arguments.  FAST: staged so that the four SFU chains (ex2 -> lg2 / rcp)
// are issued side by side and without branches -- the ternary form of softplus100_both<true> compiles to a branch
// around each element's MUFUs, which serialises the four chains of an epilogue pass (ncu: stall_wait dominated).
template <bool FAST>
__device__ __forceinline__ void softplus100_both4(const float (&z)[4], float (&h)[4], float (&d1)[4]) {
  if (FAST) {
    constexpr float kLog2e = 1.4426950408889634f, kLn2 = 0.6931471805599453f;
    float e[4], lg[4], rc[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) e[i] = ex2_ftz(z[i] * (kBeta * kLog2e));
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float t = 1.0f + e[i]; lg[i] = lg2_ftz(t); rc[i] = rcp_ftz(t); }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const bool big = z[i] * kBeta > kThresh;        // the discarded arm may hold inf / NaN: selects, not arithmetic
      h[i] = big ? z[i] : lg[i] * (kLn2 / kBeta);
      d1[i] = big ? 1.0f : e[i] * rc[i];
    }
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) { h[i] = softplus100(z[i]); d1[i] = softplus100_d1(z[i]); }
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
