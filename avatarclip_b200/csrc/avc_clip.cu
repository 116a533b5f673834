// avc_clip.cu -- CLIP ViT-B/32 image tower forward + input-gradient backward and the cosine loss.
//
// Replaces openai/CLIP's VisionTransformer as called from AvatarGen/AppearanceGen/main.py:509-526
// (RandomResizedCrop(scale=(1,1)) == whole-image bilinear resize, Normalize, encode_image, cosine).
// Weights are frozen (main.py:260): no weight gradients exist, so the backward only needs the
// non-linearities' inputs (LayerNorm inputs, q/k/v, the c_fc pre-activation).
//
// Shapes: M = B*T token rows (T = 50), width 768.  Every GEMM here has M <= 128*k rows and streams its
// fp16 weight matrix exactly once: by bytes they are weight-bandwidth bound, in practice latency bound (~200 dependent
// kernels per step), so the tiles are small and split over K where N alone cannot fill the SMs, and every kernel issues
// all its global loads in one batch (DESIGN.md 3.3).  Every pass is one chain of stand-alone kernels linked by
// programmatic dependent launch.  Two GEMM kernels, chosen by M: k_gemm16_tc (M <= 128: TMA-fed wgmma tiles of
// 128 x 32, the constant weight tiles issued before the programmatic-dependency wait) and k_gemm16 (M > 128: mma.sync
// m16n8k16, 64 x 32 tiles, 6-stage cp.async).
#include <cuda_fp16.h>

#include "avc_common.cuh"
#include "avc_gemm_tc.cuh"

using namespace avc;

namespace {

// Programmatic dependent launch: the tower is a chain of ~230 tiny dependent kernels.  Every kernel lets its
// successor start launching at once (launch_dependents) and itself waits for its predecessor's completion and memory
// flush (griddepcontrol.wait) before touching global memory, so launch latency and tail drain overlap.
__device__ __forceinline__ void pdl_enter() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
}

template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// Each kernel reads its thread and block indices and the block size once into const locals at its top.  With
// blockDim.x read inside the strided loops instead, nvcc stops unrolling them.

// ------------------------------------------------------------------------------------------------
// fp16 tensor-core GEMM  C[M,N] = A[M,K] . W[N,K]^T  (mma.sync m16n8k16, fp32 accumulate).
// CTA: 128 threads, tile 64 x 32, BK = 64, 6-stage cp.async pipeline, grid (N/32, ceil(M/64), ksplit).
// Epilogue functor: pre = epi.prefetch(row, col, ksplit_index) before the main loop, then epi(row, col, v0, v1,
// ksplit_index, pre) for two consecutive columns.
// ------------------------------------------------------------------------------------------------
constexpr int GBM = 64, GBN = 32, GBK = 64, GST = 6, GPAD = 8;
constexpr int G_SMEM = GST * (GBM + GBN) * (GBK + GPAD) * 2;   // 82,944 B of dynamic shared memory

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

template <typename Epi>
__global__ void __launch_bounds__(128)
k_gemm16(const __half* __restrict__ A, int lda, const __half* __restrict__ Wt, int ldw, int M, int N, int K,
         int k_per_split, Epi epi) {
  extern __shared__ __align__(16) unsigned char g_smem[];
  __half (*sA)[GBM][GBK + GPAD] = reinterpret_cast<__half (*)[GBM][GBK + GPAD]>(g_smem);
  __half (*sW)[GBN][GBK + GPAD] =
      reinterpret_cast<__half (*)[GBN][GBK + GPAD]>(g_smem + (size_t)GST * GBM * (GBK + GPAD) * 2);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n0 = blockIdx.x * GBN, m0 = blockIdx.y * GBM, ks = blockIdx.z;
  const int kb = ks * k_per_split;
  const int ke = min(K, kb + k_per_split);
  const int nk = (ke - kb + GBK - 1) / GBK;

  auto issue_a = [&](int kt, int st) {
    const int k0 = kb + kt * GBK;
#pragma unroll
    for (int i = 0; i < 4; ++i) {        // A: 64 rows x 8 chunks
      int c = tid + i * 128;
      int r = c >> 3, ch = c & 7;
      bool ok = (m0 + r) < M;
      const __half* src = A + (size_t)(ok ? (m0 + r) : 0) * lda + k0 + ch * 8;
      cp_async16(&sA[st][r][ch * 8], src, ok);
    }
  };
  auto issue_w = [&](int kt, int st) {
    const int k0 = kb + kt * GBK;
#pragma unroll
    for (int i = 0; i < 2; ++i) {        // W: 32 rows x 8 chunks
      int c = tid + i * 128;
      int r = c >> 3, ch = c & 7;
      const __half* src = Wt + (size_t)(n0 + r) * ldw + k0 + ch * 8;
      cp_async16(&sW[st][r][ch * 8], src, true);
    }
  };
  auto issue = [&](int kt, int st) { issue_a(kt, st); issue_w(kt, st); };

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  // (Streaming the constant weight stages in before griddepcontrol.wait was measured: no gain forward, 0.1 ms slower
  // backward -- the first MMA then waits for five weight stages instead of one.)
  asm volatile("griddepcontrol.wait;" ::: "memory");
  for (int s = 0; s < GST - 1; ++s) {
    if (s < nk) issue(s, s);
    cp_async_commit();
  }
  // epilogue operands (bias, saved pre-activation, row scale) are fetched now, behind the operand stream, instead of as
  // a dependent load phase after the main loop
  const int er0 = m0 + warp * 16 + (lane >> 2);
  float2 epre[4][2];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int col = n0 + t * 8 + (lane & 3) * 2;
    epre[t][0] = (er0 < M) ? epi.prefetch(er0, col, ks) : make_float2(0.f, 0.f);
    epre[t][1] = (er0 + 8 < M) ? epi.prefetch(er0 + 8, col, ks) : make_float2(0.f, 0.f);
  }
  for (int kt = 0; kt < nk; ++kt) {
    cp_async_wait<GST - 2>();
    __syncthreads();
    if (kt + GST - 1 < nk) issue(kt + GST - 1, (kt + GST - 1) % GST);
    cp_async_commit();
    const int st = kt % GST;
#pragma unroll
    for (int kk = 0; kk < GBK; kk += 16) {
      unsigned a[4];
      {
        unsigned addr = (unsigned)__cvta_generic_to_shared(&sA[st][warp * 16 + (lane & 15)][kk + (lane >> 4) * 8]);
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                     : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3]) : "r"(addr));
      }
#pragma unroll
      for (int np = 0; np < 2; ++np) {   // two pairs of n8 tiles
        unsigned b[4];
        unsigned addr = (unsigned)__cvta_generic_to_shared(
            &sW[st][np * 16 + (lane & 7) + (lane >> 4) * 8][kk + ((lane >> 3) & 1) * 8]);
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                     : "=r"(b[0]), "=r"(b[1]), "=r"(b[2]), "=r"(b[3]) : "r"(addr));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float* c = acc[np * 2 + h];
          asm volatile(
              "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
              : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
              : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[h * 2]), "r"(b[h * 2 + 1]));
        }
      }
    }
  }
  cp_async_wait<0>();
  // the successor is released after the main loop, so that its CTAs (which only spin in griddepcontrol.wait) do not
  // take SM slots from this kernel's later waves
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int r0 = m0 + warp * 16 + (lane >> 2);
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    int col = n0 + t * 8 + (lane & 3) * 2;
    if (r0 < M) epi(r0, col, acc[t][0], acc[t][1], ks, epre[t][0]);
    if (r0 + 8 < M) epi(r0 + 8, col, acc[t][2], acc[t][3], ks, epre[t][1]);
  }
}

template <typename Epi>
int gemm16_tc(cudaStream_t st, const __half* A, int lda, const __half* Wt, int ldw, int M, int N, int K, int ksplit,
              const Epi& epi);

template <typename Epi>
int gemm16(cudaStream_t st, const __half* A, int lda, const __half* Wt, int ldw, int M, int N, int K, int ksplit,
           const Epi& epi) {
  if (N % GBN || K % GBK) return AVC_E_BADCFG;
  if (M <= 128) return gemm16_tc(st, A, lda, Wt, ldw, M, N, K, ksplit, epi);      // all rows in one wgmma tile
  int kper = (int)round_up(ceil_div(K, ksplit), GBK);
  ksplit = ceil_div(K, kper);
  dim3 grid(N / GBN, ceil_div(M, GBM), ksplit);
  static bool attr_set = false;      // per epilogue instantiation
  if (!attr_set) {
    AVC_CUDA_TRY(cudaFuncSetAttribute(k_gemm16<Epi>, cudaFuncAttributeMaxDynamicSharedMemorySize, G_SMEM));
    attr_set = true;
  }
  AVC_CUDA_TRY(launch_pdl(k_gemm16<Epi>, dim3(grid), dim3(128), G_SMEM, st, A, lda, Wt, ldw, M, N, K, kper, epi));
  AVC_LAUNCH_TRY();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// The same GEMM on the warpgroup MMA (every launch with M <= 128): all token rows of the
// batch (M = 100 at B = 2) are ONE 128-row tile, so a CTA owns a 128 x 32 output tile for its K range.
//   warps 0-7  two consumer warpgroups (rows 0-63 / 64-127): wgmma m64n32k16 (fp16 operands, fp32 accumulate) into
//              16 registers per thread, then the functor straight from the fragment (column pairs, as mma.sync gives);
//   warp 8     TMA producer: W tiles (constants) go out BEFORE griddepcontrol.wait, the A tiles right after it;
//              8-stage ring of (A 16 KB + W 4 KB), K-major SWIZZLE_128B.
// grid (N / 32, ksplit); rows >= M of the A box are zero-filled by TMA and never stored.
// ------------------------------------------------------------------------------------------------
constexpr int TBN = 32, TBK = 64, TST = 8;
constexpr int T_A_BYTES = 128 * TBK * 2, T_W_BYTES = TBN * TBK * 2, T_STAGE = T_A_BYTES + T_W_BYTES;
constexpr int T_SMEM = 1024 + TST * T_STAGE + 256;

template <typename Epi>
__global__ void __launch_bounds__(tc::kTcThreads, 1)
k_gemm16_tc(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapW, int M, int N, int K,
            int k_per_split, Epi epi) {
  using namespace avc::tc;
  extern __shared__ uint8_t t_smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)t_smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = (uint64_t*)(smem + TST * T_STAGE);
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t full0 = smem_u32(bars), empty0 = full0 + 8 * TST;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * TBN, ks = blockIdx.y;
  const int kb0 = ks * k_per_split, ke = min(K, kb0 + k_per_split);
  const int nk = (ke - kb0 + TBK - 1) / TBK;

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&mapA); tma_prefetch_desc(&mapW);
    for (int s = 0; s < TST; ++s) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, 2); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kProducerWarp) {
    if (lane == 0) {
      const int npre = nk < TST ? nk : TST;
      for (int s = 0; s < npre; ++s) {      // weights do not depend on the predecessor kernel
        mbar_expect_tx(full0 + 8 * s, T_STAGE);
        tma_load_2d(smem_base + s * T_STAGE + T_A_BYTES, &mapW, kb0 + s * TBK, n0, full0 + 8 * s);
      }
      asm volatile("griddepcontrol.wait;" ::: "memory");
      for (int s = 0; s < npre; ++s) tma_load_2d(smem_base + s * T_STAGE, &mapA, kb0 + s * TBK, 0, full0 + 8 * s);
      for (int kb = npre; kb < nk; ++kb) {
        const int s = kb % TST;
        mbar_wait(empty0 + 8 * s, ((kb / TST) & 1) ^ 1);
        mbar_expect_tx(full0 + 8 * s, T_STAGE);
        tma_load_2d(smem_base + s * T_STAGE + T_A_BYTES, &mapW, kb0 + kb * TBK, n0, full0 + 8 * s);
        tma_load_2d(smem_base + s * T_STAGE, &mapA, kb0 + kb * TBK, 0, full0 + 8 * s);
      }
    }
    return;
  }
  const int g = warp >> 2, wq = warp & 3;
  const bool leader = (threadIdx.x & 127) == 0;
  const int r0 = 64 * g + 16 * wq + (lane >> 2), cp = 2 * (lane & 3);
  asm volatile("griddepcontrol.wait;" ::: "memory");
  float2 pre[4][2];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      pre[j][h] = r0 + 8 * h < M ? epi.prefetch(r0 + 8 * h, n0 + 8 * j + cp, ks) : make_float2(0.f, 0.f);
  float acc[16];
  int prev = -1;
  for (int kb = 0; kb < nk; ++kb) {
    const int s = kb % TST;
    mbar_wait(full0 + 8 * s, (kb / TST) & 1);
    const uint64_t da = make_wgmma_desc(smem_base + s * T_STAGE + (uint32_t)g * 8192u, 16, 1024);
    const uint64_t db = make_wgmma_desc(smem_base + s * T_STAGE + T_A_BYTES, 16, 1024);
    wgmma_fence_acc(acc);
    wgmma_fence();
#pragma unroll
    for (int k4 = 0; k4 < TBK / 16; ++k4) wgmma_f16_n32<0, 0>(acc, da + 2 * k4, db + 2 * k4, (kb | k4) ? 1u : 0u);
    wgmma_commit();
    wgmma_fence_acc(acc);
    wgmma_wait<1>();
    if (prev >= 0 && leader) mbar_arrive(empty0 + 8 * prev);
    prev = s;
  }
  wgmma_wait<0>();
  wgmma_fence_acc(acc);
  // the dependent kernel is released after the main loop, like in the mma.sync kernel
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r0 + 8 * h;
      if (row < M) epi(row, n0 + 8 * j + cp, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], ks, pre[j][h]);
    }
}

template <typename Epi>
int gemm16_tc(cudaStream_t st, const __half* A, int lda, const __half* Wt, int ldw, int M, int N, int K, int ksplit,
              const Epi& epi) {
  int kper = (int)round_up(ceil_div(K, ksplit), TBK);
  ksplit = ceil_div(K, kper);
  CUtensorMap mA, mW;     // fp16 data through bf16-typed maps: TMA only moves bytes (and zero-fills out-of-range rows)
  AVC_TRY(tc::make_map_bf16_cached(&mA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, TBK, 128));
  AVC_TRY(tc::make_map_bf16_cached(&mW, Wt, (uint64_t)N, (uint64_t)K, (uint64_t)ldw, TBK, TBN));
  static bool attr_set = false;      // per epilogue instantiation
  if (!attr_set) {
    AVC_CUDA_TRY(cudaFuncSetAttribute(k_gemm16_tc<Epi>, cudaFuncAttributeMaxDynamicSharedMemorySize, T_SMEM));
    attr_set = true;
  }
  AVC_CUDA_TRY(launch_pdl(k_gemm16_tc<Epi>, dim3(N / TBN, ksplit), dim3(tc::kTcThreads), T_SMEM, st, mA, mW, M, N, K, kper, epi));
  AVC_LAUNCH_TRY();
  return 0;
}

// ---- epilogues -----------------------------------------------------------------------------------
struct EpiPatch {   // token row b*T + 1 + p  +=  acc   (rows pre-initialised with the positional embedding; split-K)
  float* x; int T, Wd, np;
  __device__ float2 prefetch(int, int, int) const { return make_float2(0.f, 0.f); }
  __device__ void operator()(int row, int col, float v0, float v1, int, float2) const {
    int b = row / np, p = row - b * np;
    size_t o = ((size_t)b * T + 1 + p) * Wd + col;
    atomicAdd(x + o, v0);
    atomicAdd(x + o + 1, v1);
  }
};
struct EpiBiasStore {   // out = acc + b
  float* out; int ld; const float* bias;
  __device__ float2 prefetch(int, int col, int) const { return make_float2(bias[col], bias[col + 1]); }
  __device__ void operator()(int row, int col, float v0, float v1, int, float2 p) const {
    out[(size_t)row * ld + col] = v0 + p.x;
    out[(size_t)row * ld + col + 1] = v1 + p.y;
  }
};
struct EpiResidual {    // x += acc (+ bias once): split-K partials meet in fp32 atomics
  float* x; int ld; const float* bias;
  __device__ float2 prefetch(int, int col, int ks) const {
    return ks == 0 ? make_float2(bias[col], bias[col + 1]) : make_float2(0.f, 0.f);
  }
  __device__ void operator()(int row, int col, float v0, float v1, int, float2 p) const {
    atomicAdd(x + (size_t)row * ld + col, v0 + p.x);
    atomicAdd(x + (size_t)row * ld + col + 1, v1 + p.y);
  }
};
struct EpiFc {          // pre = acc + b ; g = QuickGELU(pre) = pre * sigmoid(1.702 pre)
  float* pre; __half* g; int ld; const float* bias;
  __device__ float2 prefetch(int, int col, int) const { return make_float2(bias[col], bias[col + 1]); }
  __device__ void operator()(int row, int col, float v0, float v1, int, float2 p) const {
    float p0 = v0 + p.x, p1 = v1 + p.y;
    size_t o = (size_t)row * ld + col;
    pre[o] = p0; pre[o + 1] = p1;
    *reinterpret_cast<__half2*>(g + o) = __floats2half2_rn(p0 * sigmoidf_acc(1.702f * p0), p1 * sigmoidf_acc(1.702f * p1));
  }
};
struct EpiDfc {         // (row-scaled) dpre = acc * QuickGELU'(pre) -> fp16 operand of the next GEMM
  const float* pre; __half* out; int ld;
  __device__ float2 prefetch(int row, int col, int) const {
    return *reinterpret_cast<const float2*>(pre + (size_t)row * ld + col);
  }
  __device__ void operator()(int row, int col, float v0, float v1, int, float2 p) const {
    size_t o = (size_t)row * ld + col;
    float p0 = p.x, p1 = p.y;
    float s0 = sigmoidf_acc(1.702f * p0), s1 = sigmoidf_acc(1.702f * p1);
    float d0 = v0 * (s0 + 1.702f * p0 * s0 * (1.f - s0));
    float d1 = v1 * (s1 + 1.702f * p1 * s1 * (1.f - s1));
    *reinterpret_cast<__half2*>(out + o) = __floats2half2_rn(d0, d1);
  }
};
struct EpiAccumUnscale {  // dst += acc / rowscale   (split-K)
  float* dst; int ld; const float* rowscale;
  __device__ float2 prefetch(int row, int, int) const { return make_float2(rowscale[row], 0.f); }
  __device__ void operator()(int row, int col, float v0, float v1, int, float2 p) const {
    float inv = 1.0f / p.x;
    atomicAdd(dst + (size_t)row * ld + col, v0 * inv);
    atomicAdd(dst + (size_t)row * ld + col + 1, v1 * inv);
  }
};
struct EpiStoreUnscale {  // dst = acc / rowscale
  float* dst; int ld; const float* rowscale;
  __device__ float2 prefetch(int row, int, int) const { return make_float2(rowscale[row], 0.f); }
  __device__ void operator()(int row, int col, float v0, float v1, int, float2 p) const {
    float inv = 1.0f / p.x;
    dst[(size_t)row * ld + col] = v0 * inv;
    dst[(size_t)row * ld + col + 1] = v1 * inv;
  }
};

// ------------------------------------------------------------------------------------------------
// Pre-processing: bilinear resize (align_corners=False, no antialias) + Normalize, written directly as
// the im2col operand of the patch-embedding GEMM: row b*np + patch, column c*p*p + (y%p)*p + (x%p).
// ------------------------------------------------------------------------------------------------
__constant__ float kMean[3] = {0.48145466f, 0.4578275f, 0.40821073f};
__constant__ float kStd[3] = {0.26862954f, 0.26130258f, 0.27577711f};

struct ResizeTap { int i0, i1; float l; };
__device__ __forceinline__ ResizeTap resize_tap(int dst, float scale, int in) {
  float src = ((float)dst + 0.5f) * scale - 0.5f;    // area_pixel_compute_source_index, align_corners=False
  if (src < 0.f) src = 0.f;
  int i0 = (int)src;
  if (i0 > in - 1) i0 = in - 1;
  ResizeTap t;
  t.i0 = i0; t.i1 = i0 + ((i0 < in - 1) ? 1 : 0); t.l = src - (float)i0;
  return t;
}

__global__ void k_preprocess(const float* __restrict__ canvas, int H, int W, int B, int IS, int P,
                             __half* __restrict__ a0, int mode) {
  pdl_enter();
  const int bx = blockIdx.x, nt = blockDim.x, tid = threadIdx.x;
  int64_t i = (int64_t)bx * nt + tid;
  int64_t tot = (int64_t)B * 3 * IS * IS;
  if (i >= tot) return;
  int x = (int)(i % IS); int64_t r = i / IS;
  int y = (int)(r % IS); r /= IS;
  int c = (int)(r % 3); int b = (int)(r / 3);
  if (mode == 1) {     // already normalised NCHW image [B][3][IS][IS]: im2col only
    int g1 = IS / P;
    int patch1 = (y / P) * g1 + (x / P);
    int col1 = c * P * P + (y % P) * P + (x % P);
    a0[((size_t)b * g1 * g1 + patch1) * (3 * P * P) + col1] = __float2half_rn(canvas[i]);
    return;
  }
  ResizeTap ty = resize_tap(y, (float)H / (float)IS, H), tx = resize_tap(x, (float)W / (float)IS, W);
  const float* cv = canvas + (size_t)b * H * W * 3;
  auto px = [&](int yy, int xx) { return cv[((size_t)yy * W + xx) * 3 + c]; };
  float top = px(ty.i0, tx.i0) * (1.f - tx.l) + px(ty.i0, tx.i1) * tx.l;
  float bot = px(ty.i1, tx.i0) * (1.f - tx.l) + px(ty.i1, tx.i1) * tx.l;
  float v = (top * (1.f - ty.l) + bot * ty.l - kMean[c]) / kStd[c];
  int g = IS / P;
  int patch = (y / P) * g + (x / P);
  int col = c * P * P + (y % P) * P + (x % P);
  a0[((size_t)b * g * g + patch) * (3 * P * P) + col] = __float2half_rn(v);
}

// adjoint: d canvas += bilinear^T ( d img / std ), d img read from the im2col gradient
__global__ void k_preprocess_bwd(const float* __restrict__ dpatch, int H, int W, int B, int IS, int P,
                                 float* __restrict__ dcanvas, int mode) {
  pdl_enter();
  const int bx = blockIdx.x, nt = blockDim.x, tid = threadIdx.x;
  int64_t i = (int64_t)bx * nt + tid;
  int64_t tot = (int64_t)B * 3 * IS * IS;
  if (i >= tot) return;
  int x = (int)(i % IS); int64_t r = i / IS;
  int y = (int)(r % IS); r /= IS;
  int c = (int)(r % 3); int b = (int)(r / 3);
  int g = IS / P;
  int patch = (y / P) * g + (x / P);
  int col = c * P * P + (y % P) * P + (x % P);
  if (mode == 1) { dcanvas[i] = dpatch[((size_t)b * g * g + patch) * (3 * P * P) + col]; return; }
  float gv = dpatch[((size_t)b * g * g + patch) * (3 * P * P) + col] / kStd[c];
  ResizeTap ty = resize_tap(y, (float)H / (float)IS, H), tx = resize_tap(x, (float)W / (float)IS, W);
  float* dc = dcanvas + (size_t)b * H * W * 3;
  auto add = [&](int yy, int xx, float w) { atomicAdd(dc + ((size_t)yy * W + xx) * 3 + c, gv * w); };
  add(ty.i0, tx.i0, (1.f - ty.l) * (1.f - tx.l));
  add(ty.i0, tx.i1, (1.f - ty.l) * tx.l);
  add(ty.i1, tx.i0, ty.l * (1.f - tx.l));
  add(ty.i1, tx.i1, ty.l * tx.l);
}

// token buffer initialisation: row 0 = class_embedding + pos[0], rows 1.. = pos[t] (the patch GEMM adds onto them)
__global__ void k_cls_rows(const float* __restrict__ cls, const float* __restrict__ pos, int B, int T, int Wd,
                           float* __restrict__ x) {
  pdl_enter();
  const int bx = blockIdx.x, nt = blockDim.x, tid = threadIdx.x;
  int i = bx * nt + tid;
  if (i >= B * T * Wd) return;
  int c = i % Wd, t = (i / Wd) % T;
  x[i] = pos[(size_t)t * Wd + c] + (t == 0 ? cls[c] : 0.f);
}

// ------------------------------------------------------------------------------------------------
// LayerNorm (fp32 statistics, eps 1e-5): one warp per row.
// ------------------------------------------------------------------------------------------------
// Rows are cached in registers (Wd <= 32 * kLnMax): one round trip to memory per operand instead of one per pass.
constexpr int kLnMax = 32;

__global__ void __launch_bounds__(256)
k_layernorm(const float* __restrict__ x, int M, int Wd, const float* __restrict__ g, const float* __restrict__ b,
            float* __restrict__ y32, __half* __restrict__ y16, float* __restrict__ save_x) {
  pdl_enter();
  const int bx = blockIdx.x, nt = blockDim.x, tid = threadIdx.x;
  int row = bx * (nt >> 5) + (tid >> 5);
  if (row >= M) return;
  const int lane = tid & 31;
  const float* xr = x + (size_t)row * Wd;
  float xv[kLnMax], gv[kLnMax], bv[kLnMax];      // gamma / beta are fetched with the row, not after the reductions
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kLnMax; ++i) {
    int c = lane + 32 * i;
    bool ok = c < Wd;
    xv[i] = ok ? xr[c] : 0.f; gv[i] = ok ? g[c] : 0.f; bv[i] = ok ? b[c] : 0.f;
    s += xv[i];
  }
  float mean = warp_sum(s) / (float)Wd;
  float v = 0.f;
#pragma unroll
  for (int i = 0; i < kLnMax; ++i) { int c = lane + 32 * i; float d = (c < Wd) ? xv[i] - mean : 0.f; v += d * d; }
  float rstd = rsqrtf(warp_sum(v) / (float)Wd + 1e-5f);
#pragma unroll
  for (int i = 0; i < kLnMax; ++i) {
    int c = lane + 32 * i;
    if (c < Wd) {
      float yv = (xv[i] - mean) * rstd * gv[i] + bv[i];
      if (y32) y32[(size_t)row * Wd + c] = yv;
      if (y16) y16[(size_t)row * Wd + c] = __float2half_rn(yv);
      if (save_x) save_x[(size_t)row * Wd + c] = xv[i];
    }
  }
}

// dx (+)= LN'(x)^T dy :  dx = rstd * (dy*g - mean(dy*g) - xhat * mean(dy*g*xhat)); optionally also the row-scaled fp16
// copy of the updated dx row (operand of the next input-gradient GEMM)
__global__ void __launch_bounds__(256)
k_layernorm_bwd(const float* __restrict__ x, float* __restrict__ dy, int M, int Wd, const float* __restrict__ g,
                float* __restrict__ dx, int accumulate, int row_stride_x, int row_stride_dy, int row_stride_dx,
                __half* __restrict__ dx16, float* __restrict__ dx_scale, int zero_dy) {
  pdl_enter();
  const int bx = blockIdx.x, nt = blockDim.x, tid = threadIdx.x;
  int row = bx * (nt >> 5) + (tid >> 5);
  if (row >= M) return;
  const int lane = tid & 31;
  const float* xr = x + (size_t)row * row_stride_x;
  float* dr = dy + (size_t)row * row_stride_dy;
  float* o = dx + (size_t)row * row_stride_dx;
  float xv[kLnMax], dg[kLnMax], ov[kLnMax];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kLnMax; ++i) {
    int c = lane + 32 * i;
    bool ok = c < Wd;
    xv[i] = ok ? xr[c] : 0.f;
    dg[i] = ok ? dr[c] * g[c] : 0.f;
    ov[i] = (ok && accumulate) ? o[c] : 0.f;
    s += xv[i];
  }
  float mean = warp_sum(s) / (float)Wd;
  float v = 0.f;
#pragma unroll
  for (int i = 0; i < kLnMax; ++i) { int c = lane + 32 * i; float d = (c < Wd) ? xv[i] - mean : 0.f; v += d * d; }
  float rstd = rsqrtf(warp_sum(v) / (float)Wd + 1e-5f);
  float a = 0.f, bq = 0.f;
#pragma unroll
  for (int i = 0; i < kLnMax; ++i) {
    int c = lane + 32 * i;
    if (c < Wd) { a += dg[i]; bq += dg[i] * (xv[i] - mean) * rstd; }
  }
  a = warp_sum(a) / (float)Wd; bq = warp_sum(bq) / (float)Wd;
  float mx = 0.f;
#pragma unroll
  for (int i = 0; i < kLnMax; ++i) {
    int c = lane + 32 * i;
    if (c < Wd) {
      float xh = (xv[i] - mean) * rstd;
      float r = ov[i] + rstd * (dg[i] - a - xh * bq);
      ov[i] = r;
      o[c] = r;
      if (zero_dy) dr[c] = 0.f;          // dy is the split-K accumulator of the next GEMM: hand it back cleared
      mx = fmaxf(mx, fabsf(r));
    }
  }
  if (dx16) {
#pragma unroll
    for (int of = 16; of > 0; of >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, of));
    float sc = 1.f;
    if (mx > 0.f && isfinite(mx)) { int e; frexpf(mx, &e); sc = ldexpf(1.f, 1 - e); }
#pragma unroll
    for (int i = 0; i < kLnMax; ++i) {
      int c = lane + 32 * i;
      if (c < Wd) dx16[(size_t)row * Wd + c] = __float2half_rn(ov[i] * sc);
    }
    if (lane == 0) dx_scale[row] = sc;
  }
}

// fp32 -> fp16 with a per-row power-of-two scale so that max|row| lands in [1,2): keeps tiny
// gradients out of the fp16 subnormal range.  scale[row] is undone in the consuming GEMM's epilogue.
__global__ void __launch_bounds__(256)
k_to_half_rowscaled(const float* __restrict__ src, int M, int N, int ld_src, __half* __restrict__ dst,
                    float* __restrict__ scale, const int* __restrict__ row_map) {
  pdl_enter();
  const int bx = blockIdx.x, nt = blockDim.x, tid = threadIdx.x;
  int row = bx * (nt >> 5) + (tid >> 5);
  if (row >= M) return;
  const int lane = tid & 31;
  const float* s = src + (size_t)(row_map ? row_map[row] : row) * ld_src;
  // Rows up to 32 * 4 * kRsMax = 2304 floats (3 x 768, the widest operand) are held in registers: ONE batch of
  // independent 16-byte loads instead of a loop of dependent round trips, and no second pass over memory.
  constexpr int kRsMax = 18;
  const bool cached = (N <= 128 * kRsMax) && (N % 4 == 0) && (ld_src % 4 == 0);
  float4 rv[kRsMax];
  float mx = 0.f;
  if (cached) {
#pragma unroll
    for (int i = 0; i < kRsMax; ++i) {
      const int c = (lane + 32 * i) * 4;
      rv[i] = (c < N) ? *reinterpret_cast<const float4*>(s + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < kRsMax; ++i)
      mx = fmaxf(mx, fmaxf(fmaxf(fabsf(rv[i].x), fabsf(rv[i].y)), fmaxf(fabsf(rv[i].z), fabsf(rv[i].w))));
  } else {
    for (int c = lane; c < N; c += 32) mx = fmaxf(mx, fabsf(s[c]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sc = 1.f;
  if (mx > 0.f && isfinite(mx)) {
    int e;
    frexpf(mx, &e);               // mx = m * 2^e, m in [0.5, 1)
    sc = ldexpf(1.f, 1 - e);      // mx * sc in [1, 2)
  }
  if (cached) {
#pragma unroll
    for (int i = 0; i < kRsMax; ++i) {
      const int c = (lane + 32 * i) * 4;
      if (c < N) {
        __half2 h0 = __floats2half2_rn(rv[i].x * sc, rv[i].y * sc), h1 = __floats2half2_rn(rv[i].z * sc, rv[i].w * sc);
        uint2 pk;
        pk.x = *reinterpret_cast<unsigned*>(&h0); pk.y = *reinterpret_cast<unsigned*>(&h1);
        *reinterpret_cast<uint2*>(dst + (size_t)row * N + c) = pk;
      }
    }
  } else {
    for (int c = lane; c < N; c += 32) dst[(size_t)row * N + c] = __float2half_rn(s[c] * sc);
  }
  if (lane == 0) scale[row] = sc;
}

// ------------------------------------------------------------------------------------------------
// Attention, one CTA per (image, head): T <= 64 tokens, head dim 64.  fp32 throughout.
// qkv: [M][3W] fp32 (q | k | v).  o16: [M][W] fp16 operand of out_proj.
// ------------------------------------------------------------------------------------------------
constexpr int AT = 64;   // max tokens
constexpr int AD = 64;   // head dim
constexpr int AP = AD + 4;   // shared-memory row pitch: 16-byte aligned rows, LDS.128 conflict-free across 8 rows
constexpr int kAttnFwdSmem = (3 * AT * AP + AT * (AT + 1)) * (int)sizeof(float);       // q, k, v | S
constexpr int kAttnBwdSmem = (4 * AT * AP + 2 * AT * (AT + 1)) * (int)sizeof(float);   // q, k, v, dO | P, dS

// 64 x 64 x 64 tile product on the tensor cores for the attention kernels (16 warps): C(m, n) = sum_k A(m, k) B(k, n) with
// TF32 operands (mma.sync.m16n8k8, fp32 accumulate: the same 10-bit mantissa as the fp16 matmuls of the reference's CUDA
// path, fp32 range).  fa(m, k) / fb(k, n) fetch (guarded) elements from shared memory; warp w owns the 16-row tile w / 4 and
// the two 8-column tiles 2 (w % 4), 2 (w % 4) + 1:  c[j][0..3] = C(m0+g, n0+8j+2t), (.., +1), (m0+g+8, ..), (.., +1).
__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm volatile("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
template <class FA, class FB>
__device__ __forceinline__ void mma_tf32_64(float (&c)[2][4], int warp, int lane, FA&& fa, FB&& fb) {
  const int g = lane >> 2, t = lane & 3, m0 = (warp >> 2) * 16, n0 = (warp & 3) * 16;
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) c[j][i] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {
    const int k0 = ks * 8;
    const uint32_t a0 = to_tf32(fa(m0 + g, k0 + t)), a1 = to_tf32(fa(m0 + g + 8, k0 + t));
    const uint32_t a2 = to_tf32(fa(m0 + g, k0 + t + 4)), a3 = to_tf32(fa(m0 + g + 8, k0 + t + 4));
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint32_t b0 = to_tf32(fb(k0 + t, n0 + 8 * j + g)), b1 = to_tf32(fb(k0 + t + 4, n0 + 8 * j + g));
      asm volatile(
          "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
          : "+f"(c[j][0]), "+f"(c[j][1]), "+f"(c[j][2]), "+f"(c[j][3])
          : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
    }
  }
}

__global__ void __launch_bounds__(512)
k_attention(const float* __restrict__ qkv, int T, int Wd, int heads, __half* __restrict__ o16) {
  pdl_enter();
  extern __shared__ __align__(16) unsigned char dyn_smem[];
  const int bx = blockIdx.x, nt = blockDim.x, tid = threadIdx.x;
  float* sm = reinterpret_cast<float*>(dyn_smem);
  float* q = sm;                  // [T][AP]
  float* k = q + AT * AP;
  float* v = k + AT * AP;
  float* S = v + AT * AP;         // [T][AT+1]
  const int b = bx / heads, h = bx % heads;
  const float* base = qkv + (size_t)b * T * 3 * Wd;
  {   // all global loads of the thread first (one latency, not one per loop trip), then the shared-memory stores
    constexpr int NIT = (AT * (AD / 4) + 511) / 512;
    float4 rq[NIT], rk[NIT], rv[NIT];
#pragma unroll
    for (int j = 0; j < NIT; ++j) {
      const int i = tid + j * 512;
      if (i < T * (AD / 4)) {
        const int t = i / (AD / 4), d = (i % (AD / 4)) * 4;
        const float* r = base + (size_t)t * 3 * Wd + h * AD + d;
        rq[j] = *reinterpret_cast<const float4*>(r);
        rk[j] = *reinterpret_cast<const float4*>(r + Wd);
        rv[j] = *reinterpret_cast<const float4*>(r + 2 * Wd);
      }
    }
#pragma unroll
    for (int j = 0; j < NIT; ++j) {
      const int i = tid + j * 512;
      if (i < T * (AD / 4)) {
        const int t = i / (AD / 4), d = (i % (AD / 4)) * 4;
        *reinterpret_cast<float4*>(q + t * AP + d) = rq[j];
        *reinterpret_cast<float4*>(k + t * AP + d) = rk[j];
        *reinterpret_cast<float4*>(v + t * AP + d) = rv[j];
      }
    }
  }
  __syncthreads();
  const int lane = tid & 31, warp = tid >> 5;
  {   // S = q k^T / sqrt(64) on the tensor cores
    float c[2][4];
    mma_tf32_64(c, warp, lane, [&](int m, int kk) { return m < T ? q[m * AP + kk] : 0.f; },
                [&](int kk, int n) { return n < T ? k[n * AP + kk] : 0.f; });
    const int g = lane >> 2, t = lane & 3, m0 = (warp >> 2) * 16, n0 = (warp & 3) * 16;
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int m = m0 + g + 8 * (i >> 1), n = n0 + 8 * j + 2 * t + (i & 1);
        if (m < T && n < T) S[m * (AT + 1) + n] = c[j][i] * 0.125f;
      }
  }
  __syncthreads();
  for (int a = warp; a < T; a += (nt >> 5)) {
    float mx = -1e30f;
    for (int c = lane; c < T; c += 32) mx = fmaxf(mx, S[a * (AT + 1) + c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int c = lane; c < T; c += 32) { float e = expf(S[a * (AT + 1) + c] - mx); S[a * (AT + 1) + c] = e; sum += e; }
    sum = warp_sum(sum);
    float inv = 1.f / sum;
    for (int c = lane; c < T; c += 32) S[a * (AT + 1) + c] *= inv;
  }
  __syncthreads();
  {   // o = P v on the tensor cores -> fp16 operand of out_proj
    float c[2][4];
    mma_tf32_64(c, warp, lane, [&](int m, int kk) { return (m < T && kk < T) ? S[m * (AT + 1) + kk] : 0.f; },
                [&](int kk, int n) { return kk < T ? v[kk * AP + n] : 0.f; });
    const int g = lane >> 2, t = lane & 3, m0 = (warp >> 2) * 16, n0 = (warp & 3) * 16;
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int m = m0 + g + 8 * hh, n = n0 + 8 * j + 2 * t;
        if (m < T)
          *reinterpret_cast<__half2*>(o16 + ((size_t)b * T + m) * Wd + h * AD + n) = __floats2half2_rn(c[j][2 * hh], c[j][2 * hh + 1]);
      }
  }
}

// backward: recompute P; dqkv[M][3W] fp32 from dO[M][W] fp32
__global__ void __launch_bounds__(512)
k_attention_bwd(const float* __restrict__ qkv, const float* __restrict__ dO, int T, int Wd, int heads,
                float* __restrict__ dqkv) {
  pdl_enter();
  extern __shared__ __align__(16) unsigned char dyn_smem[];
  const int bx = blockIdx.x, nt = blockDim.x, tid = threadIdx.x;
  float* sm = reinterpret_cast<float*>(dyn_smem);
  float* q = sm;
  float* k = q + AT * AP;
  float* v = k + AT * AP;
  float* dO_s = v + AT * AP;
  float* Pm = dO_s + AT * AP;           // [T][AT+1]
  float* dS = Pm + AT * (AT + 1);
  const int b = bx / heads, h = bx % heads;
  const float* base = qkv + (size_t)b * T * 3 * Wd;
  {   // all global loads first, then the shared-memory stores (see k_attention)
    constexpr int NIT = (AT * (AD / 4) + 511) / 512;
    float4 rq[NIT], rk[NIT], rv[NIT], ro[NIT];
#pragma unroll
    for (int j = 0; j < NIT; ++j) {
      const int i = tid + j * 512;
      if (i < T * (AD / 4)) {
        const int t = i / (AD / 4), d = (i % (AD / 4)) * 4;
        const float* r = base + (size_t)t * 3 * Wd + h * AD + d;
        rq[j] = *reinterpret_cast<const float4*>(r);
        rk[j] = *reinterpret_cast<const float4*>(r + Wd);
        rv[j] = *reinterpret_cast<const float4*>(r + 2 * Wd);
        ro[j] = *reinterpret_cast<const float4*>(dO + ((size_t)b * T + t) * Wd + h * AD + d);
      }
    }
#pragma unroll
    for (int j = 0; j < NIT; ++j) {
      const int i = tid + j * 512;
      if (i < T * (AD / 4)) {
        const int t = i / (AD / 4), d = (i % (AD / 4)) * 4;
        *reinterpret_cast<float4*>(q + t * AP + d) = rq[j];
        *reinterpret_cast<float4*>(k + t * AP + d) = rk[j];
        *reinterpret_cast<float4*>(v + t * AP + d) = rv[j];
        *reinterpret_cast<float4*>(dO_s + t * AP + d) = ro[j];
      }
    }
  }
  __syncthreads();
  const int lane = tid & 31, warp = tid >> 5;
  const int fg = lane >> 2, ft = lane & 3, fm0 = (warp >> 2) * 16, fn0 = (warp & 3) * 16;      // C-fragment coordinates
  {   // S = q k^T / 8 and dP = dO v^T on the tensor cores
    float c[2][4], e[2][4];
    mma_tf32_64(c, warp, lane, [&](int m, int kk) { return m < T ? q[m * AP + kk] : 0.f; },
                [&](int kk, int n) { return n < T ? k[n * AP + kk] : 0.f; });
    mma_tf32_64(e, warp, lane, [&](int m, int kk) { return m < T ? dO_s[m * AP + kk] : 0.f; },
                [&](int kk, int n) { return n < T ? v[n * AP + kk] : 0.f; });
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int m = fm0 + fg + 8 * (i >> 1), n = fn0 + 8 * j + 2 * ft + (i & 1);
        if (m < T && n < T) { Pm[m * (AT + 1) + n] = c[j][i] * 0.125f; dS[m * (AT + 1) + n] = e[j][i]; }      // dP for now
      }
  }
  __syncthreads();
  for (int a = warp; a < T; a += (nt >> 5)) {
    float mx = -1e30f;
    for (int c = lane; c < T; c += 32) mx = fmaxf(mx, Pm[a * (AT + 1) + c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int c = lane; c < T; c += 32) { float e = expf(Pm[a * (AT + 1) + c] - mx); Pm[a * (AT + 1) + c] = e; sum += e; }
    sum = warp_sum(sum);
    float inv = 1.f / sum, dot = 0.f;
    for (int c = lane; c < T; c += 32) { float p = Pm[a * (AT + 1) + c] * inv; Pm[a * (AT + 1) + c] = p; dot += p * dS[a * (AT + 1) + c]; }
    dot = warp_sum(dot);
    for (int c = lane; c < T; c += 32) dS[a * (AT + 1) + c] = Pm[a * (AT + 1) + c] * (dS[a * (AT + 1) + c] - dot) * 0.125f;
  }
  __syncthreads();
  float* dbase = dqkv + (size_t)b * T * 3 * Wd;
  {   // dq = dS k, dk = dS^T q, dv = P^T dO on the tensor cores
    float cq[2][4], ck[2][4], cv[2][4];
    auto dS_at = [&](int a, int c) { return (a < T && c < T) ? dS[a * (AT + 1) + c] : 0.f; };
    auto P_at = [&](int a, int c) { return (a < T && c < T) ? Pm[a * (AT + 1) + c] : 0.f; };
    mma_tf32_64(cq, warp, lane, [&](int m, int kk) { return dS_at(m, kk); }, [&](int kk, int n) { return kk < T ? k[kk * AP + n] : 0.f; });
    mma_tf32_64(ck, warp, lane, [&](int m, int kk) { return dS_at(kk, m); }, [&](int kk, int n) { return kk < T ? q[kk * AP + n] : 0.f; });
    mma_tf32_64(cv, warp, lane, [&](int m, int kk) { return P_at(kk, m); }, [&](int kk, int n) { return kk < T ? dO_s[kk * AP + n] : 0.f; });
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int m = fm0 + fg + 8 * hh, n = fn0 + 8 * j + 2 * ft;
        if (m < T) {
          float* r = dbase + (size_t)m * 3 * Wd + h * AD + n;
          *reinterpret_cast<float2*>(r) = make_float2(cq[j][2 * hh], cq[j][2 * hh + 1]);
          *reinterpret_cast<float2*>(r + Wd) = make_float2(ck[j][2 * hh], ck[j][2 * hh + 1]);
          *reinterpret_cast<float2*>(r + 2 * Wd) = make_float2(cv[j][2 * hh], cv[j][2 * hh + 1]);
        }
      }
  }
}

// ------------------------------------------------------------------------------------------------
// Head: ln_post(x[b,0]) @ proj -> emb ; cosine with the text embedding.  One CTA per image.
// ------------------------------------------------------------------------------------------------
// ln_post(x[b,0]) @ proj: grid (B, OD/64); every CTA recomputes the (cheap) LayerNorm of the cls row and produces 64
// outputs, each from 4 partial dots over a quarter of the 768 inputs.
__global__ void __launch_bounds__(256)
k_head_proj(const float* __restrict__ x, int T, int Wd, const float* __restrict__ g, const float* __restrict__ bta,
            const float* __restrict__ proj, int OD, float* __restrict__ emb, float* __restrict__ ynorm) {
  pdl_enter();
  extern __shared__ __align__(16) unsigned char dyn_smem[];
  const int bx = blockIdx.x, by = blockIdx.y, nt = blockDim.x, tid = threadIdx.x;
  float* sm = reinterpret_cast<float*>(dyn_smem);
  float* y = sm;               // [Wd]
  float* part = y + Wd;        // [4][64]
  __shared__ float red[8];
  const int b = bx;
  const float* xr = x + (size_t)b * T * Wd;
  float s = 0.f;
  for (int c = tid; c < Wd; c += nt) s += xr[c];
  s = warp_sum(s);
  if ((tid & 31) == 0) red[tid >> 5] = s;
  __syncthreads();
  float mean = 0.f;
  for (int i = 0; i < 8; ++i) mean += red[i];
  mean /= (float)Wd;
  float v = 0.f;
  for (int c = tid; c < Wd; c += nt) { float d = xr[c] - mean; v += d * d; }
  v = warp_sum(v);
  __syncthreads();
  if ((tid & 31) == 0) red[tid >> 5] = v;
  __syncthreads();
  float var = 0.f;
  for (int i = 0; i < 8; ++i) var += red[i];
  float rstd = rsqrtf(var / (float)Wd + 1e-5f);
  for (int c = tid; c < Wd; c += nt) {
    float yy = (xr[c] - mean) * rstd * g[c] + bta[c];
    y[c] = yy;
    if (by == 0) ynorm[(size_t)b * Wd + c] = yy;
  }
  __syncthreads();
  const int ol = tid & 63, pt = tid >> 6;
  const int o = by * 64 + ol;
  const int c0 = pt * (Wd / 4), c1 = c0 + Wd / 4;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  if (o < OD) {
    int c = c0;
    for (; c + 3 < c1; c += 4) {
      a0 = fmaf(y[c], proj[(size_t)c * OD + o], a0);
      a1 = fmaf(y[c + 1], proj[(size_t)(c + 1) * OD + o], a1);
      a2 = fmaf(y[c + 2], proj[(size_t)(c + 2) * OD + o], a2);
      a3 = fmaf(y[c + 3], proj[(size_t)(c + 3) * OD + o], a3);
    }
    for (; c < c1; ++c) a0 = fmaf(y[c], proj[(size_t)c * OD + o], a0);
  }
  part[pt * 64 + ol] = (a0 + a1) + (a2 + a3);
  __syncthreads();
  if (pt == 0 && o < OD) emb[(size_t)b * OD + o] = (part[ol] + part[64 + ol]) + (part[128 + ol] + part[192 + ol]);
}

// cosine(emb[b], text[b]); torch.cosine_similarity: x.y / max(||x|| * ||y||, 1e-8)
__global__ void __launch_bounds__(256)
k_cosine(const float* __restrict__ emb, const float* __restrict__ text, int OD, float* __restrict__ cos_out) {
  pdl_enter();
  const int bx = blockIdx.x, nt = blockDim.x, tid = threadIdx.x;
  __shared__ float red[3][8];
  const int b = bx;
  float ee = 0.f, tt = 0.f, et = 0.f;
  for (int o = tid; o < OD; o += nt) {
    float a = emb[(size_t)b * OD + o], t = text[(size_t)b * OD + o];
    ee += a * a; tt += t * t; et += a * t;
  }
  ee = warp_sum(ee); tt = warp_sum(tt); et = warp_sum(et);
  if ((tid & 31) == 0) { red[0][tid >> 5] = ee; red[1][tid >> 5] = tt; red[2][tid >> 5] = et; }
  __syncthreads();
  if (tid == 0) {
    float a = 0.f, t = 0.f, c = 0.f;
    for (int i = 0; i < 8; ++i) { a += red[0][i]; t += red[1][i]; c += red[2][i]; }
    cos_out[b] = c / fmaxf(sqrtf(a) * sqrtf(t), 1e-8f);
  }
}

// d cos / d emb (+ g_emb) -> dy = proj . de, spread over (B, Wd/96) CTAs (one warp per row of proj: coalesced)
__global__ void __launch_bounds__(256)
k_head_bwd_dy(int Wd, const float* __restrict__ proj, int OD, const float* __restrict__ text,
              const float* __restrict__ emb, const float* __restrict__ g_cos, const float* __restrict__ g_emb,
              float* __restrict__ dy_out, int rows_per_cta) {
  pdl_enter();
  extern __shared__ __align__(16) unsigned char dyn_smem[];
  const int bx = blockIdx.x, by = blockIdx.y, nt = blockDim.x, tid = threadIdx.x;
  float* sm = reinterpret_cast<float*>(dyn_smem);
  float* de = sm;            // [OD]
  __shared__ float red[3][8];
  const int b = bx;
  float ee = 0.f, tt = 0.f, et = 0.f;
  for (int o = tid; o < OD; o += nt) {
    float a = emb[(size_t)b * OD + o], t = text[(size_t)b * OD + o];
    ee += a * a; tt += t * t; et += a * t;
  }
  ee = warp_sum(ee); tt = warp_sum(tt); et = warp_sum(et);
  if ((tid & 31) == 0) { red[0][tid >> 5] = ee; red[1][tid >> 5] = tt; red[2][tid >> 5] = et; }
  __syncthreads();
  float a2 = 0.f, t2 = 0.f, c = 0.f;
  for (int i = 0; i < 8; ++i) { a2 += red[0][i]; t2 += red[1][i]; c += red[2][i]; }
  float nrm_a = sqrtf(a2), nrm_t = sqrtf(t2);
  float gc = g_cos ? g_cos[b] : 0.f;
  for (int o = tid; o < OD; o += nt) {
    float a = emb[(size_t)b * OD + o], t = text[(size_t)b * OD + o];
    // d/d a [ a.t / (|a||t|) ] = t/(|a||t|) - (a.t) a / (|a|^3 |t|)
    float d = (g_cos && nrm_a > 0.f && nrm_t > 0.f) ? gc * (t / (nrm_a * nrm_t) - c * a / (nrm_a * nrm_a * nrm_a * nrm_t)) : 0.f;
    if (g_emb) d += g_emb[(size_t)b * OD + o];
    de[o] = d;
  }
  __syncthreads();
  const int r0 = by * rows_per_cta, r1 = min(Wd, r0 + rows_per_cta);
  for (int cc = r0 + (tid >> 5); cc < r1; cc += (nt >> 5)) {
    float s = 0.f;
    for (int o = tid & 31; o < OD; o += 32) s = fmaf(proj[(size_t)cc * OD + o], de[o], s);
    s = warp_sum(s);
    if ((tid & 31) == 0) dy_out[(size_t)b * Wd + cc] = s;
  }
}

// LayerNorm (ln_post) backward on the cls row; the other token rows receive no gradient from the head
__global__ void __launch_bounds__(256)
k_head_bwd_ln(const float* __restrict__ x, int T, int Wd, const float* __restrict__ g, const float* __restrict__ dy_in,
              float* __restrict__ dx) {
  pdl_enter();
  const int bx = blockIdx.x, nt = blockDim.x, tid = threadIdx.x;
  __shared__ float red[3][8];
  const int b = bx;
  const float* xr = x + (size_t)b * T * Wd;
  const float* dy = dy_in + (size_t)b * Wd;
  float s = 0.f;
  for (int cc = tid; cc < Wd; cc += nt) s += xr[cc];
  s = warp_sum(s);
  if ((tid & 31) == 0) red[0][tid >> 5] = s;
  __syncthreads();
  float mean = 0.f;
  for (int i = 0; i < 8; ++i) mean += red[0][i];
  mean /= (float)Wd;
  float v = 0.f;
  for (int cc = tid; cc < Wd; cc += nt) { float d = xr[cc] - mean; v += d * d; }
  v = warp_sum(v);
  __syncthreads();
  if ((tid & 31) == 0) red[0][tid >> 5] = v;
  __syncthreads();
  float var = 0.f;
  for (int i = 0; i < 8; ++i) var += red[0][i];
  float rstd = rsqrtf(var / (float)Wd + 1e-5f);
  float pa = 0.f, pb = 0.f;
  for (int cc = tid; cc < Wd; cc += nt) {
    float dg = dy[cc] * g[cc];
    pa += dg; pb += dg * (xr[cc] - mean) * rstd;
  }
  pa = warp_sum(pa); pb = warp_sum(pb);
  if ((tid & 31) == 0) { red[1][tid >> 5] = pa; red[2][tid >> 5] = pb; }
  __syncthreads();
  float A = 0.f, Bq = 0.f;
  for (int i = 0; i < 8; ++i) { A += red[1][i]; Bq += red[2][i]; }
  A /= (float)Wd; Bq /= (float)Wd;
  for (int cc = tid; cc < Wd; cc += nt) {
    float xh = (xr[cc] - mean) * rstd;
    dx[(size_t)b * T * Wd + cc] = rstd * (dy[cc] * g[cc] - A - xh * Bq);
  }
  for (int64_t i = tid; i < (int64_t)(T - 1) * Wd; i += nt) dx[(size_t)b * T * Wd + Wd + i] = 0.f;
}

__global__ void k_patch_row_map(int B, int T, int* __restrict__ map) {
  pdl_enter();
  const int bx = blockIdx.x, nt = blockDim.x, tid = threadIdx.x;
  int i = bx * nt + tid;
  int np = T - 1;
  if (i >= B * np) return;
  int b = i / np, p = i - b * np;
  map[i] = b * T + 1 + p;
}

// ------------------------------------------------------------------------------------------------
struct ClipWs {
  __half* a0;        // [B*np][3pp] im2col operand
  float* x;          // [M][W] residual stream
  float* tok_pre;    // [M][W] tokens before ln_pre
  float* xs;         // [2*layers][M][W] LayerNorm inputs (ln_1, ln_2 per block)
  float* x_final;    // [M][W]
  __half* h16;       // [M][W]
  float* qkv;        // [layers][M][3W]
  __half* o16;       // [M][W]
  float* fc_pre;     // [layers][M][mlp]
  __half* g16;       // [M][mlp]
  float* emb;        // [B][OD] (copy for the backward)
  float* ynorm;      // [B][W]
  // backward
  float* dx;         // [M][W]
  float* dtmp;       // [M][W]
  float* dO;         // [M][W]
  float* dqkv;       // [M][3W]
  __half* d16a;      // [M][max(W,3W,mlp)]
  __half* d16b;      // [M][mlp]
  float* scale;      // [M]
  float* dpatch;     // [B*np][3pp]
  int* rowmap;       // [B*np]
  size_t bytes;
};

int clip_dims(const avc_clip_cfg* c, int* T, int* np, int* pp3) {
  if (!c) return AVC_E_NULL;
  if (c->image_size <= 0 || c->patch <= 0 || c->image_size % c->patch) return AVC_E_BADCFG;
  int g = c->image_size / c->patch;
  *np = g * g; *T = *np + 1; *pp3 = 3 * c->patch * c->patch;
  if (*T > AT) return AVC_E_BADCFG;
  if (c->width % 64 || c->heads <= 0 || c->width / c->heads != AD || c->width % c->heads) return AVC_E_BADCFG;
  if (c->width > 32 * kLnMax) return AVC_E_BADCFG;
  if (c->mlp % 64 || *pp3 % 64 || c->layers < 1 || c->layers > AVC_CLIP_MAX_LAYERS || c->out_dim < 1) return AVC_E_BADCFG;
  return 0;
}

void carve_clip(const avc_clip_cfg& c, int B, int T, int np, int pp3, void* base, ClipWs* w) {
  Carver cv(base);
  const int64_t M = (int64_t)B * T, Wd = c.width;
  w->a0 = cv.take<__half>((int64_t)B * np * pp3);
  w->x = cv.take<float>(M * Wd);
  w->tok_pre = cv.take<float>(M * Wd);
  w->xs = cv.take<float>((int64_t)2 * c.layers * M * Wd);
  w->x_final = cv.take<float>(M * Wd);
  w->h16 = cv.take<__half>(M * Wd);
  w->qkv = cv.take<float>((int64_t)c.layers * M * 3 * Wd);
  w->o16 = cv.take<__half>(M * Wd);
  w->fc_pre = cv.take<float>((int64_t)c.layers * M * c.mlp);
  w->g16 = cv.take<__half>(M * c.mlp);
  w->emb = cv.take<float>((int64_t)B * c.out_dim);
  w->ynorm = cv.take<float>((int64_t)B * Wd);
  w->dx = cv.take<float>(M * Wd);
  w->dtmp = cv.take<float>(M * Wd);
  w->dO = cv.take<float>(M * Wd);
  w->dqkv = cv.take<float>(M * 3 * Wd);
  int64_t mx = c.mlp > 3 * Wd ? c.mlp : 3 * Wd;
  w->d16a = cv.take<__half>(M * mx);
  w->d16b = cv.take<__half>(M * mx);
  w->scale = cv.take<float>(M);
  w->dpatch = cv.take<float>((int64_t)B * np * pp3);
  w->rowmap = cv.take<int>((int64_t)B * np);
  w->bytes = cv.used();
}

int set_attn_smem() {
  AVC_CUDA_TRY(cudaFuncSetAttribute(k_attention, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnFwdSmem));
  AVC_CUDA_TRY(cudaFuncSetAttribute(k_attention_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnBwdSmem));
  return 0;
}

}  // namespace

extern "C" {

int avc_clip_workspace_bytes(const avc_clip_cfg* cfg, int32_t B, size_t* bytes) {
  if (!cfg || !bytes) return AVC_E_NULL;
  if (B < 1) return AVC_E_SIZE;
  int T, np, pp3;
  AVC_TRY(clip_dims(cfg, &T, &np, &pp3));
  ClipWs w;
  carve_clip(*cfg, B, T, np, pp3, nullptr, &w);
  *bytes = w.bytes;
  return 0;
}

int avc_clip_loss_fwd(const avc_clip_cfg* cfg, const avc_clip_weights* wt, const float* canvases, int32_t H,
                      int32_t W, int32_t B, int32_t input_mode, const float* text_emb, float* emb_out,
                      float* cos_out, void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!cfg || !wt || !canvases || !text_emb || !emb_out || !cos_out || !workspace) return AVC_E_NULL;
  if (B < 1 || H < 1 || W < 1) return AVC_E_SIZE;
  if (input_mode != 0 && input_mode != 1) return AVC_E_BADCFG;
  if (input_mode == 1 && (H != cfg->image_size || W != cfg->image_size)) return AVC_E_SIZE;
  int T, np, pp3;
  AVC_TRY(clip_dims(cfg, &T, &np, &pp3));
  if (((uintptr_t)workspace & 15u)) return AVC_E_ALIGN;
  ClipWs w;
  carve_clip(*cfg, B, T, np, pp3, workspace, &w);
  if (w.bytes > workspace_bytes) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  const int Wd = cfg->width, M = B * T, IS = cfg->image_size;
  AVC_TRY(set_attn_smem());

  int64_t npx = (int64_t)B * 3 * IS * IS;
  AVC_CUDA_TRY(launch_pdl(k_preprocess, dim3((int)((npx + 255) / 256)), dim3(256), 0, st, canvases, H, W, B, IS, cfg->patch, w.a0, input_mode));
  AVC_CUDA_TRY(launch_pdl(k_cls_rows, dim3((B * T * Wd + 255) / 256), dim3(256), 0, st, wt->cls, wt->pos, B, T, Wd, w.tok_pre));
  AVC_LAUNCH_TRY();
  {
    EpiPatch e{w.tok_pre, T, Wd, np};
    AVC_TRY(gemm16(st, w.a0, pp3, (const __half*)wt->w_patch, pp3, B * np, Wd, pp3, 4, e));
  }
  AVC_CUDA_TRY(launch_pdl(k_layernorm, dim3(ceil_div(M, 8)), dim3(256), 0, st, w.tok_pre, M, Wd, wt->ln_pre_g, wt->ln_pre_b, w.x, nullptr, nullptr));
  AVC_LAUNCH_TRY();
  for (int l = 0; l < cfg->layers; ++l) {
    const avc_clip_layer_weights& lw = wt->layer[l];
    float* xs1 = w.xs + (size_t)(2 * l) * M * Wd;
    float* xs2 = w.xs + (size_t)(2 * l + 1) * M * Wd;
    float* qkv = w.qkv + (size_t)l * M * 3 * Wd;
    float* fcp = w.fc_pre + (size_t)l * M * cfg->mlp;
    AVC_CUDA_TRY(launch_pdl(k_layernorm, dim3(ceil_div(M, 8)), dim3(256), 0, st, w.x, M, Wd, lw.ln1_g, lw.ln1_b, nullptr, w.h16, xs1));
    AVC_LAUNCH_TRY();
    { EpiBiasStore e{qkv, 3 * Wd, lw.b_qkv};
      AVC_TRY(gemm16(st, w.h16, Wd, (const __half*)lw.w_qkv, Wd, M, 3 * Wd, Wd, 1, e)); }
    AVC_CUDA_TRY(launch_pdl(k_attention, dim3(B * cfg->heads), dim3(512), kAttnFwdSmem, st, qkv, T, Wd, cfg->heads, w.o16));
    AVC_LAUNCH_TRY();
    { EpiResidual e{w.x, Wd, lw.b_out};
      AVC_TRY(gemm16(st, w.o16, Wd, (const __half*)lw.w_out, Wd, M, Wd, Wd, 2, e)); }
    AVC_CUDA_TRY(launch_pdl(k_layernorm, dim3(ceil_div(M, 8)), dim3(256), 0, st, w.x, M, Wd, lw.ln2_g, lw.ln2_b, nullptr, w.h16, xs2));
    AVC_LAUNCH_TRY();
    { EpiFc e{fcp, w.g16, cfg->mlp, lw.b_fc};
      AVC_TRY(gemm16(st, w.h16, Wd, (const __half*)lw.w_fc, Wd, M, cfg->mlp, Wd, 1, e)); }
    { EpiResidual e{w.x, Wd, lw.b_proj};
      AVC_TRY(gemm16(st, w.g16, cfg->mlp, (const __half*)lw.w_proj, cfg->mlp, M, Wd, cfg->mlp, 4, e)); }
  }
  AVC_CUDA_TRY(cudaMemcpyAsync(w.x_final, w.x, sizeof(float) * (size_t)M * Wd, cudaMemcpyDeviceToDevice, st));
  AVC_CUDA_TRY(launch_pdl(k_head_proj, dim3(dim3(B, (cfg->out_dim + 63) / 64)), dim3(256), (Wd + 256) * sizeof(float), st, 
      w.x_final, T, Wd, wt->ln_post_g, wt->ln_post_b, wt->proj, cfg->out_dim, w.emb, w.ynorm));
  AVC_CUDA_TRY(launch_pdl(k_cosine, dim3(B), dim3(256), 0, st, w.emb, text_emb, cfg->out_dim, cos_out));
  AVC_LAUNCH_TRY();
  AVC_CUDA_TRY(cudaMemcpyAsync(emb_out, w.emb, sizeof(float) * (size_t)B * cfg->out_dim, cudaMemcpyDeviceToDevice, st));
  return 0;
}

int avc_clip_loss_bwd(const avc_clip_cfg* cfg, const avc_clip_weights* wt, int32_t H, int32_t W, int32_t B,
                      int32_t input_mode, const float* text_emb, const float* g_cos, const float* g_emb,
                      float* d_canvases, void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!cfg || !wt || !text_emb || !d_canvases || !workspace) return AVC_E_NULL;
  if (!g_cos && !g_emb) return AVC_E_NULL;
  if (B < 1 || H < 1 || W < 1) return AVC_E_SIZE;
  if (input_mode != 0 && input_mode != 1) return AVC_E_BADCFG;
  int T, np, pp3;
  AVC_TRY(clip_dims(cfg, &T, &np, &pp3));
  ClipWs w;
  carve_clip(*cfg, B, T, np, pp3, workspace, &w);
  if (w.bytes > workspace_bytes) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  const int Wd = cfg->width, M = B * T, IS = cfg->image_size, mlp = cfg->mlp;
  AVC_TRY(set_attn_smem());

  {
    const int rows = 96;
    AVC_CUDA_TRY(launch_pdl(k_head_bwd_dy, dim3(dim3(B, ceil_div(Wd, rows))), dim3(256), cfg->out_dim * sizeof(float), st, 
        Wd, wt->proj, cfg->out_dim, text_emb, w.emb, g_cos, g_emb, w.dO, rows));      // w.dO[0 .. B*Wd) as scratch
    AVC_CUDA_TRY(launch_pdl(k_head_bwd_ln, dim3(B), dim3(256), 0, st, w.x_final, T, Wd, wt->ln_post_g, w.dO, w.dx));
  }
  AVC_LAUNCH_TRY();
  // w.dtmp is the split-K accumulator of the two Wd-wide input-gradient GEMMs of a layer; it is cleared once here and
  // then by the LayerNorm backward that consumes it (no memset nodes inside the dependent-launch chain)
  AVC_CUDA_TRY(cudaMemsetAsync(w.dtmp, 0, sizeof(float) * (size_t)M * Wd, st));
  for (int l = cfg->layers - 1; l >= 0; --l) {
    const avc_clip_layer_weights& lw = wt->layer[l];
    const float* xs1 = w.xs + (size_t)(2 * l) * M * Wd;
    const float* xs2 = w.xs + (size_t)(2 * l + 1) * M * Wd;
    const float* qkv = w.qkv + (size_t)l * M * 3 * Wd;
    const float* fcp = w.fc_pre + (size_t)l * M * mlp;
    // ---- MLP branch: x_out = x_mid + c_proj(QuickGELU(c_fc(ln_2(x_mid))))
    if (l == cfg->layers - 1) {     // later layers get this conversion fused into the previous LayerNorm backward
      AVC_CUDA_TRY(launch_pdl(k_to_half_rowscaled, dim3(ceil_div(M, 8)), dim3(256), 0, st, w.dx, M, Wd, Wd, w.d16a, w.scale, nullptr));
      AVC_LAUNCH_TRY();
    }
    { EpiDfc e{fcp, w.d16b, mlp};
      AVC_TRY(gemm16(st, w.d16a, Wd, (const __half*)lw.w_proj_t, Wd, M, mlp, Wd, 1, e)); }
    { EpiAccumUnscale e{w.dtmp, Wd, w.scale};
      AVC_TRY(gemm16(st, w.d16b, mlp, (const __half*)lw.w_fc_t, mlp, M, Wd, mlp, 4, e)); }
    AVC_CUDA_TRY(launch_pdl(k_layernorm_bwd, dim3(ceil_div(M, 8)), dim3(256), 0, st, xs2, w.dtmp, M, Wd, lw.ln2_g, w.dx, 1, Wd, Wd, Wd, w.d16a, w.scale, 1));
    AVC_LAUNCH_TRY();
    // ---- attention branch: x_mid = x_in + out_proj(attn(in_proj(ln_1(x_in))))
    { EpiStoreUnscale e{w.dO, Wd, w.scale};
      AVC_TRY(gemm16(st, w.d16a, Wd, (const __half*)lw.w_out_t, Wd, M, Wd, Wd, 1, e)); }
    AVC_CUDA_TRY(launch_pdl(k_attention_bwd, dim3(B * cfg->heads), dim3(512), kAttnBwdSmem, st, qkv, w.dO, T, Wd, cfg->heads, w.dqkv));
    AVC_LAUNCH_TRY();
    AVC_CUDA_TRY(launch_pdl(k_to_half_rowscaled, dim3(ceil_div(M, 8)), dim3(256), 0, st, w.dqkv, M, 3 * Wd, 3 * Wd, w.d16a, w.scale, nullptr));
    AVC_LAUNCH_TRY();
    { EpiAccumUnscale e{w.dtmp, Wd, w.scale};
      AVC_TRY(gemm16(st, w.d16a, 3 * Wd, (const __half*)lw.w_qkv_t, 3 * Wd, M, Wd, 3 * Wd, 3, e)); }
    AVC_CUDA_TRY(launch_pdl(k_layernorm_bwd, dim3(ceil_div(M, 8)), dim3(256), 0, st, xs1, w.dtmp, M, Wd, lw.ln1_g, w.dx, 1, Wd, Wd, Wd, w.d16a, w.scale, 1));
    AVC_LAUNCH_TRY();
  }
  // ln_pre, patch embedding, pre-processing
  AVC_CUDA_TRY(launch_pdl(k_layernorm_bwd, dim3(ceil_div(M, 8)), dim3(256), 0, st, w.tok_pre, w.dx, M, Wd, wt->ln_pre_g, w.dtmp, 0, Wd, Wd, Wd, nullptr,
                                                  nullptr, 0));
  AVC_CUDA_TRY(launch_pdl(k_patch_row_map, dim3(ceil_div(B * np, 128)), dim3(128), 0, st, B, T, w.rowmap));
  AVC_CUDA_TRY(launch_pdl(k_to_half_rowscaled, dim3(ceil_div(B * np, 8)), dim3(256), 0, st, w.dtmp, B * np, Wd, Wd, w.d16a, w.scale, w.rowmap));
  AVC_LAUNCH_TRY();
  { EpiStoreUnscale e{w.dpatch, pp3, w.scale};
    AVC_TRY(gemm16(st, w.d16a, Wd, (const __half*)wt->w_patch_t, Wd, B * np, pp3, Wd, 1, e)); }
  AVC_CUDA_TRY(cudaMemsetAsync(d_canvases, 0, sizeof(float) * (size_t)B * H * W * 3, st));
  int64_t npx = (int64_t)B * 3 * IS * IS;
  AVC_CUDA_TRY(launch_pdl(k_preprocess_bwd, dim3((int)((npx + 255) / 256)), dim3(256), 0, st, w.dpatch, H, W, B, IS, cfg->patch, d_canvases, input_mode));
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"

// ================================================================================================
// CLIP text tower forward (openai/CLIP `CLIP.encode_text`, called from main.py:276,282,288).  Forward only: the text
// weights are frozen and the reference detaches the embedding.  The same pre-LN residual blocks as the image tower,
// built from its kernels (k_layernorm, gemm16 with EpiBiasStore / EpiResidual / EpiFc, k_head_proj) plus three new
// ones: the token-embedding gather, causal attention over up to 128 tokens and the end-of-text row gather.  Every
// position of the context runs (no truncation at the end-of-text token): the tower runs once per training run.
// ================================================================================================
namespace {

constexpr int kTextMaxT = 128;     // max context
constexpr int kTextAP = AD + 1;    // shared-memory row pitch of q / k / v: row j's element d sits in bank (j + d) % 32
constexpr int kTextAttnThreads = 256;
constexpr int kTextAttnSmem = (3 * kTextMaxT * kTextAP + (kTextAttnThreads / 32) * kTextMaxT) * (int)sizeof(float);

// x[b,t] = token_embedding[tok[b,t]] + positional_embedding[t] (fp32).  An id outside [0, vocab) is clamped so that
// the gather never leaves the table; the Python wrapper rejects such ids before the call.
__global__ void k_text_embed(const int32_t* __restrict__ tok, const float* __restrict__ emb,
                             const float* __restrict__ pos, int B, int T, int Wd, int vocab, float* __restrict__ x) {
  pdl_enter();
  const int bx = blockIdx.x, nt = blockDim.x, tid = threadIdx.x;
  const int64_t i = (int64_t)bx * nt + tid;
  if (i >= (int64_t)B * T * Wd) return;
  const int c = (int)(i % Wd);
  const int64_t row = i / Wd;
  const int t = (int)(row % T);
  const int id = min(max(tok[row], 0), vocab - 1);
  x[i] = emb[(size_t)id * Wd + c] + pos[(size_t)t * Wd + c];
}

// Causal self-attention, one CTA per (sequence, head): T <= 128 tokens, head dim 64, scale 1/8, fp32 FFMA and softmax.
// Query row a attends to keys 0..a (build_attention_mask: -inf above the diagonal), so no row is ever fully masked.
// qkv: [B*T][3W] fp32 (q | k | v).  o16: [B*T][W] fp16 operand of out_proj.  Warp w owns the query rows w, w + 8, ...:
// lanes split the keys for the scores and the head dimension for the output.
__global__ void __launch_bounds__(kTextAttnThreads)
k_causal_attention(const float* __restrict__ qkv, int T, int Wd, int heads, __half* __restrict__ o16) {
  pdl_enter();
  extern __shared__ __align__(16) unsigned char dyn_smem[];
  const int bx = blockIdx.x, nt = blockDim.x, tid = threadIdx.x;
  float* q = reinterpret_cast<float*>(dyn_smem);   // [T][kTextAP]
  float* k = q + kTextMaxT * kTextAP;
  float* v = k + kTextMaxT * kTextAP;
  float* pw = v + kTextMaxT * kTextAP;              // [warps][kTextMaxT] probabilities of the warp's current row
  const int b = bx / heads, h = bx % heads;
  const float* base = qkv + (size_t)b * T * 3 * Wd + h * AD;
  for (int i = tid; i < T * (AD / 4); i += nt) {
    const int t = i / (AD / 4), d = (i % (AD / 4)) * 4;
    const float* r = base + (size_t)t * 3 * Wd + d;
    const float4 a = *reinterpret_cast<const float4*>(r);
    const float4 c = *reinterpret_cast<const float4*>(r + Wd);
    const float4 e = *reinterpret_cast<const float4*>(r + 2 * Wd);
    float* qs = q + t * kTextAP + d; float* ks = k + t * kTextAP + d; float* vs = v + t * kTextAP + d;
    qs[0] = a.x; qs[1] = a.y; qs[2] = a.z; qs[3] = a.w;
    ks[0] = c.x; ks[1] = c.y; ks[2] = c.z; ks[3] = c.w;
    vs[0] = e.x; vs[1] = e.y; vs[2] = e.z; vs[3] = e.w;
  }
  __syncthreads();
  const int lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
  float* p = pw + warp * kTextMaxT;
  for (int a = warp; a < T; a += nw) {
    const float* qa = q + a * kTextAP;
    float mx = -INFINITY;
    for (int j = lane; j <= a; j += 32) {
      const float* kj = k + j * kTextAP;
      float s = 0.f;
#pragma unroll 16
      for (int d = 0; d < AD; ++d) s = fmaf(qa[d], kj[d], s);
      s *= 0.125f;
      p[j] = s;
      mx = fmaxf(mx, s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int j = lane; j <= a; j += 32) { const float e = expf(p[j] - mx); p[j] = e; sum += e; }
    const float inv = 1.f / warp_sum(sum);
    __syncwarp();
    float o0 = 0.f, o1 = 0.f;
    for (int j = 0; j <= a; ++j) {
      const float pj = p[j];
      o0 = fmaf(pj, v[j * kTextAP + lane], o0);
      o1 = fmaf(pj, v[j * kTextAP + lane + 32], o1);
    }
    __half* out = o16 + ((size_t)b * T + a) * Wd + h * AD;
    out[lane] = __float2half_rn(o0 * inv);
    out[lane + 32] = __float2half_rn(o1 * inv);
    __syncwarp();      // p is rewritten for the warp's next row
  }
}

// End-of-text pooling: eot[b] = x[b, argmax_t tok[b,t]] (the first maximum, as torch.argmax; <|endoftext|> is the
// largest id).  One CTA (one warp) per sequence.
__global__ void k_text_eot_rows(const int32_t* __restrict__ tok, const float* __restrict__ x, int T, int Wd,
                                float* __restrict__ eot) {
  pdl_enter();
  const int b = blockIdx.x, lane = threadIdx.x;
  int best = INT_MIN, at = 0;
  for (int t = lane; t < T; t += 32) {
    const int v = tok[(size_t)b * T + t];
    if (v > best) { best = v; at = t; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const int ob = __shfl_xor_sync(0xffffffffu, best, o), oa = __shfl_xor_sync(0xffffffffu, at, o);
    if (ob > best || (ob == best && oa < at)) { best = ob; at = oa; }
  }
  const float* src = x + ((size_t)b * T + at) * Wd;
  for (int c = lane; c < Wd; c += 32) eot[(size_t)b * Wd + c] = src[c];
}

struct ClipTextWs {
  float* x;          // [M][W] residual stream
  __half* h16;       // [M][W] LayerNorm output, operand of qkv / c_fc
  float* qkv;        // [M][3W] (one layer)
  __half* o16;       // [M][W] attention output, operand of out_proj
  float* fc_pre;     // [M][mlp] c_fc pre-activation (one layer; written by EpiFc, not read)
  __half* g16;       // [M][mlp] QuickGELU output, operand of c_proj
  float* eot;        // [B][W] end-of-text rows
  float* ynorm;      // [B][W] ln_final of those rows (written by k_head_proj)
  size_t bytes;
};

int text_dims(const avc_clip_text_cfg* c) {
  if (!c) return AVC_E_NULL;
  if (c->context < 1 || c->context > kTextMaxT || c->vocab < 1 || c->out_dim < 1) return AVC_E_BADCFG;
  if (c->heads <= 0 || c->width % c->heads || c->width / c->heads != AD || c->width > 32 * kLnMax) return AVC_E_BADCFG;
  if (c->mlp < 64 || c->mlp % 64 || c->layers < 1 || c->layers > AVC_CLIP_MAX_LAYERS) return AVC_E_BADCFG;
  return 0;
}

void carve_text(const avc_clip_text_cfg& c, int B, void* base, ClipTextWs* w) {
  Carver cv(base);
  const int64_t M = (int64_t)B * c.context, Wd = c.width;
  w->x = cv.take<float>(M * Wd);
  w->h16 = cv.take<__half>(M * Wd);
  w->qkv = cv.take<float>(M * 3 * Wd);
  w->o16 = cv.take<__half>(M * Wd);
  w->fc_pre = cv.take<float>(M * c.mlp);
  w->g16 = cv.take<__half>(M * c.mlp);
  w->eot = cv.take<float>((int64_t)B * Wd);
  w->ynorm = cv.take<float>((int64_t)B * Wd);
  w->bytes = cv.used();
}

}  // namespace

extern "C" {

int avc_clip_text_workspace_bytes(const avc_clip_text_cfg* cfg, int32_t B, size_t* bytes) {
  if (!cfg || !bytes) return AVC_E_NULL;
  if (B < 1) return AVC_E_SIZE;
  AVC_TRY(text_dims(cfg));
  ClipTextWs w;
  carve_text(*cfg, B, nullptr, &w);
  *bytes = w.bytes;
  return 0;
}

int avc_clip_encode_text(const avc_clip_text_cfg* cfg, const avc_clip_text_weights* wt, const int32_t* tokens, int32_t B,
                         float* emb_out, void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!cfg || !wt || !tokens || !emb_out || !workspace) return AVC_E_NULL;
  if (B < 1) return AVC_E_SIZE;
  AVC_TRY(text_dims(cfg));
  if (((uintptr_t)workspace & 15u)) return AVC_E_ALIGN;
  ClipTextWs w;
  carve_text(*cfg, B, workspace, &w);
  if (w.bytes > workspace_bytes) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  const int Wd = cfg->width, T = cfg->context, M = B * T, mlp = cfg->mlp;
  AVC_CUDA_TRY(cudaFuncSetAttribute(k_causal_attention, cudaFuncAttributeMaxDynamicSharedMemorySize, kTextAttnSmem));

  AVC_CUDA_TRY(launch_pdl(k_text_embed, dim3(ceil_div((int64_t)M * Wd, 256)), dim3(256), 0, st, tokens, wt->token_emb, wt->pos, B, T, Wd,
                          cfg->vocab, w.x));
  AVC_LAUNCH_TRY();
  for (int l = 0; l < cfg->layers; ++l) {
    const avc_clip_layer_weights& lw = wt->layer[l];
    AVC_CUDA_TRY(launch_pdl(k_layernorm, dim3(ceil_div(M, 8)), dim3(256), 0, st, w.x, M, Wd, lw.ln1_g, lw.ln1_b, nullptr, w.h16, nullptr));
    AVC_LAUNCH_TRY();
    { EpiBiasStore e{w.qkv, 3 * Wd, lw.b_qkv};
      AVC_TRY(gemm16(st, w.h16, Wd, (const __half*)lw.w_qkv, Wd, M, 3 * Wd, Wd, 1, e)); }
    AVC_CUDA_TRY(launch_pdl(k_causal_attention, dim3(B * cfg->heads), dim3(kTextAttnThreads), kTextAttnSmem, st, w.qkv, T, Wd, cfg->heads,
                            w.o16));
    AVC_LAUNCH_TRY();
    { EpiResidual e{w.x, Wd, lw.b_out};
      AVC_TRY(gemm16(st, w.o16, Wd, (const __half*)lw.w_out, Wd, M, Wd, Wd, 2, e)); }
    AVC_CUDA_TRY(launch_pdl(k_layernorm, dim3(ceil_div(M, 8)), dim3(256), 0, st, w.x, M, Wd, lw.ln2_g, lw.ln2_b, nullptr, w.h16, nullptr));
    AVC_LAUNCH_TRY();
    { EpiFc e{w.fc_pre, w.g16, mlp, lw.b_fc};
      AVC_TRY(gemm16(st, w.h16, Wd, (const __half*)lw.w_fc, Wd, M, mlp, Wd, 1, e)); }
    { EpiResidual e{w.x, Wd, lw.b_proj};
      AVC_TRY(gemm16(st, w.g16, mlp, (const __half*)lw.w_proj, mlp, M, Wd, mlp, 4, e)); }
  }
  AVC_CUDA_TRY(launch_pdl(k_text_eot_rows, dim3(B), dim3(32), 0, st, tokens, w.x, T, Wd, w.eot));
  // ln_final(eot) @ text_projection: the image tower's head with one token per sequence
  AVC_CUDA_TRY(launch_pdl(k_head_proj, dim3(B, ceil_div(cfg->out_dim, 64)), dim3(256), (Wd + 256) * sizeof(float), st, w.eot, 1, Wd,
                          wt->ln_final_g, wt->ln_final_b, wt->proj, cfg->out_dim, emb_out, w.ynorm));
  AVC_LAUNCH_TRY();
  return 0;
}

// One CLIP kernel on caller buffers, launched the way the towers launch it (argument roles in include/avc_b200.h).
int avc_clip_kernel_test(int32_t kind, const int32_t* d, const void* const* in, void* const* out, avc_stream_t stream) {
  if (!d || !in || !out) return AVC_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  const auto H16 = [](const void* p) { return (const __half*)p; };
  const auto F32 = [](const void* p) { return (const float*)p; };
  if (kind >= 0 && kind <= 6) {
    const int M = d[0], N = d[1], K = d[2], ks = d[3];
    if (M < 1 || N < 1 || K < 1 || ks < 1) return AVC_E_SIZE;
    const __half *A = H16(in[0]), *W = H16(in[1]);
    switch (kind) {
      case 0: return gemm16(st, A, K, W, K, M, N, K, ks, EpiBiasStore{(float*)out[0], N, F32(in[2])});
      case 1: return gemm16(st, A, K, W, K, M, N, K, ks, EpiResidual{(float*)out[0], N, F32(in[2])});
      case 2: return gemm16(st, A, K, W, K, M, N, K, ks, EpiFc{(float*)out[0], (__half*)out[1], N, F32(in[2])});
      case 3: return gemm16(st, A, K, W, K, M, N, K, ks, EpiDfc{F32(in[2]), (__half*)out[1], N});
      case 4: return gemm16(st, A, K, W, K, M, N, K, ks, EpiAccumUnscale{(float*)out[0], N, F32(in[2])});
      case 5: return gemm16(st, A, K, W, K, M, N, K, ks, EpiStoreUnscale{(float*)out[0], N, F32(in[2])});
      default: {
        const int np = d[4];
        if (np < 1) return AVC_E_SIZE;
        return gemm16(st, A, K, W, K, M, N, K, ks, EpiPatch{(float*)out[0], np + 1, N, np});
      }
    }
  }
  switch (kind) {
    case 7: {       // k_layernorm
      const int M = d[0], Wd = d[1];
      if (M < 1 || Wd < 1 || Wd > 32 * kLnMax) return AVC_E_SIZE;
      AVC_CUDA_TRY(launch_pdl(k_layernorm, dim3(ceil_div(M, 8)), dim3(256), 0, st, F32(in[0]), M, Wd, F32(in[1]), F32(in[2]),
                              (float*)out[0], (__half*)out[1], (float*)out[2]));
      break;
    }
    case 8: {       // k_layernorm_bwd
      const int M = d[0], Wd = d[1];
      if (M < 1 || Wd < 1 || Wd > 32 * kLnMax) return AVC_E_SIZE;
      AVC_CUDA_TRY(launch_pdl(k_layernorm_bwd, dim3(ceil_div(M, 8)), dim3(256), 0, st, F32(in[0]), (float*)out[0], M, Wd, F32(in[1]),
                              (float*)out[1], d[2], Wd, Wd, Wd, (__half*)out[2], (float*)out[3], d[3]));
      break;
    }
    case 9: {       // k_to_half_rowscaled
      const int M = d[0], N = d[1];
      if (M < 1 || N < 1 || d[2] < N) return AVC_E_SIZE;
      AVC_CUDA_TRY(launch_pdl(k_to_half_rowscaled, dim3(ceil_div(M, 8)), dim3(256), 0, st, F32(in[0]), M, N, d[2], (__half*)out[0],
                              (float*)out[1], (const int*)in[1]));
      break;
    }
    case 10:        // k_attention
    case 11: {      // k_attention_bwd
      const int B = d[0], T = d[1], Wd = d[2], heads = d[3];
      if (B < 1 || T < 1 || T > AT || heads < 1 || Wd != heads * AD) return AVC_E_SIZE;
      AVC_TRY(set_attn_smem());
      if (kind == 10)
        AVC_CUDA_TRY(launch_pdl(k_attention, dim3(B * heads), dim3(512), kAttnFwdSmem, st, F32(in[0]), T, Wd, heads, (__half*)out[0]));
      else
        AVC_CUDA_TRY(launch_pdl(k_attention_bwd, dim3(B * heads), dim3(512), kAttnBwdSmem, st, F32(in[0]), F32(in[1]), T, Wd, heads,
                                (float*)out[0]));
      break;
    }
    case 12: {      // k_causal_attention
      const int B = d[0], T = d[1], Wd = d[2], heads = d[3];
      if (B < 1 || T < 1 || T > kTextMaxT || heads < 1 || Wd != heads * AD) return AVC_E_SIZE;
      AVC_CUDA_TRY(cudaFuncSetAttribute(k_causal_attention, cudaFuncAttributeMaxDynamicSharedMemorySize, kTextAttnSmem));
      AVC_CUDA_TRY(launch_pdl(k_causal_attention, dim3(B * heads), dim3(kTextAttnThreads), kTextAttnSmem, st, F32(in[0]), T, Wd, heads,
                              (__half*)out[0]));
      break;
    }
    case 13:        // k_preprocess
    case 14: {      // k_preprocess_bwd (d canvas is overwritten, as avc_clip_loss_bwd does)
      const int H = d[0], W = d[1], B = d[2], IS = d[3], P = d[4], mode = d[5];
      if (H < 1 || W < 1 || B < 1 || P < 1 || IS < P || IS % P || (mode != 0 && mode != 1)) return AVC_E_SIZE;
      if (mode == 1 && (H != IS || W != IS)) return AVC_E_SIZE;
      const int64_t npx = (int64_t)B * 3 * IS * IS;
      if (kind == 13) {
        AVC_CUDA_TRY(launch_pdl(k_preprocess, dim3((int)((npx + 255) / 256)), dim3(256), 0, st, F32(in[0]), H, W, B, IS, P,
                                (__half*)out[0], mode));
      } else {
        AVC_CUDA_TRY(cudaMemsetAsync(out[0], 0, sizeof(float) * (size_t)B * H * W * 3, st));
        AVC_CUDA_TRY(launch_pdl(k_preprocess_bwd, dim3((int)((npx + 255) / 256)), dim3(256), 0, st, F32(in[0]), H, W, B, IS, P,
                                (float*)out[0], mode));
      }
      break;
    }
    case 15: {      // k_head_proj
      const int B = d[0], T = d[1], Wd = d[2], OD = d[3];
      if (B < 1 || T < 1 || Wd < 4 || Wd % 4 || OD < 1) return AVC_E_SIZE;
      AVC_CUDA_TRY(launch_pdl(k_head_proj, dim3(B, ceil_div(OD, 64)), dim3(256), (Wd + 256) * sizeof(float), st, F32(in[0]), T, Wd,
                              F32(in[1]), F32(in[2]), F32(in[3]), OD, (float*)out[0], (float*)out[1]));
      break;
    }
    case 16: {      // k_cosine
      const int B = d[0], OD = d[1];
      if (B < 1 || OD < 1) return AVC_E_SIZE;
      AVC_CUDA_TRY(launch_pdl(k_cosine, dim3(B), dim3(256), 0, st, F32(in[0]), F32(in[1]), OD, (float*)out[0]));
      break;
    }
    case 17: {      // k_head_bwd_dy
      const int B = d[0], Wd = d[1], OD = d[2], rows = 96;
      if (B < 1 || Wd < 1 || OD < 1 || (!in[3] && !in[4])) return AVC_E_SIZE;
      AVC_CUDA_TRY(launch_pdl(k_head_bwd_dy, dim3(B, ceil_div(Wd, rows)), dim3(256), OD * sizeof(float), st, Wd, F32(in[0]), OD,
                              F32(in[1]), F32(in[2]), F32(in[3]), F32(in[4]), (float*)out[0], rows));
      break;
    }
    case 18: {      // k_head_bwd_ln
      const int B = d[0], T = d[1], Wd = d[2];
      if (B < 1 || T < 1 || Wd < 1) return AVC_E_SIZE;
      AVC_CUDA_TRY(launch_pdl(k_head_bwd_ln, dim3(B), dim3(256), 0, st, F32(in[0]), T, Wd, F32(in[1]), F32(in[2]), (float*)out[0]));
      break;
    }
    case 19: {      // k_text_eot_rows
      const int B = d[0], T = d[1], Wd = d[2];
      if (B < 1 || T < 1 || Wd < 1) return AVC_E_SIZE;
      AVC_CUDA_TRY(launch_pdl(k_text_eot_rows, dim3(B), dim3(32), 0, st, (const int32_t*)in[0], F32(in[1]), T, Wd, (float*)out[0]));
      break;
    }
    default: return AVC_E_BADCFG;
  }
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"
