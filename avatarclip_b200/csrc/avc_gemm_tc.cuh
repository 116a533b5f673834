// avc_gemm_tc.cuh -- Hopper (sm_90a) warpgroup-MMA GEMM tiles with TMA-fed operands; engine 1 of the NeuS MLP
// contractions.
//
// Precision: the NeuS SDF trunk cannot run on single-pass 16-bit tensor-core math (SURVEY.md Appendix C:
// inv_s ~ 500 amplifies SDF error; bf16 gives 2.6e-2 RGB error, TF32 3e-3).  Operands are therefore kept as
// TWO-TERM bf16 splits  x = hi + lo  (hi = bf16(x), lo = bf16(x - hi), ~16 mantissa bits) and every product is
// three MMAs  hi*hi + hi*lo + lo*hi  accumulated in fp32 (the dropped lo*lo term is ~2^-16 relative).
//
//   gemm_tc_nt : C[m,n] = sum_k A[m,k] B[n,k]     A:[M,lda] B:[N,ldb], both K-contiguous (K-major operands)
//   gemm_tc_tn : C[i,j] += sum_p A[p,i] B[p,j]    reduction over rows (weight gradients; MN-major operands)
//
// Kernel shape (288 threads): warps 0-7 are two consumer warpgroups, warpgroup g owning rows [64 g, 64 g + 64) of the
// 128-row tile: it issues wgmma.mma_async m64nBNk16 on shared-memory descriptors, keeps its fp32 accumulator in
// registers and runs the epilogue straight from that fragment; warp 8 is the TMA producer.  K step 64 (one 128-byte
// swizzle atom), shared-memory ring with full (TMA transaction count) / empty (one arrival per consumer warpgroup)
// mbarriers.  NT: persistent, one column tile per CTA, B panel resident in shared memory when K <= 256.  TN: one tile
// per CTA, split over the reduction dimension.
#pragma once
#include <type_traits>
#include <cuda.h>
#include <cuda_bf16.h>

#include <cstdlib>

#include "avc_common.cuh"
#include "avc_wgmma.cuh"

namespace avc {
namespace tc {

// ------------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Bounded spin: a protocol bug must trap (CUDA error) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  for (uint32_t spins = 0; !done; ++spins) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (spins > (1u << 26)) __trap();      // ~seconds: far beyond any legitimate wait, short of the driver's watchdog
  }
}
// Optional stall probe of the NT kernel (compile with -DAVC_NT_PROBE=1, see tools/nt_probe.py): cycles the TMA warp waits
// for a free stage, consumer warpgroup 0 waits for operands, and each role's total loop time, summed over the CTAs of
// every launch, per epilogue functor (Epi::kProbeId).
#ifdef AVC_NT_PROBE
static __device__ unsigned long long g_nt_probe[16][8];
#define AVC_PROBE_WAIT(acc, bar, par) do { long long t__ = clock64(); mbar_wait(bar, par); (acc) += clock64() - t__; } while (0)
#define AVC_PROBE_DECL(name) long long name = 0
#define AVC_PROBE_START(name) const long long name = clock64()
#define AVC_PROBE_NOW() clock64()
#define AVC_PROBE_ADD(id, slot, v) atomicAdd(&g_nt_probe[id][slot], (unsigned long long)(v))
#else
#define AVC_PROBE_WAIT(acc, bar, par) mbar_wait(bar, par)
#define AVC_PROBE_DECL(name)
#define AVC_PROBE_START(name)
#define AVC_PROBE_NOW() 0
#define AVC_PROBE_ADD(id, slot, v)
#endif
template <typename E, typename = void>
struct EpiNoAPf { static constexpr bool value = false; };
template <typename E>
struct EpiNoAPf<E, std::void_t<decltype(E::kNoATilePrefetch)>> { static constexpr bool value = E::kNoATilePrefetch; };
template <typename E, typename = void>
struct EpiProbeId { static constexpr int value = 0; };
template <typename E>
struct EpiProbeId<E, std::void_t<decltype(E::kProbeId)>> { static constexpr int value = E::kProbeId; };

// Programmatic dependent launch (the GEMM kernels of a step run back to back in one stream / graph): a kernel launched
// with launch_pdl may start while its predecessor is still running -- as SMs free up its CTAs do their set-up (barriers,
// tensor-map prefetch) and load what does NOT depend on the predecessor (the packed weights) -- and calls
// pdl_wait() before it touches anything the predecessor may have written.  pdl_trigger() lets the NEXT kernel do the same;
// it is only issued after this kernel's own pdl_wait(), so everything older than the predecessor is complete by induction.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  const char* e = getenv("AVC_TC_PDL");      // AVC_TC_PDL=0: plain stream-ordered launches (A-B knob; read on every call:
  const int on = (e && atoi(e) == 0) ? 0 : 1;      // bench.py takes its per-kernel durations with plain launches)
  cfg.attrs = at; cfg.numAttrs = on ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// bar.sync on a named barrier: the 128 threads of one consumer warpgroup (ids 1 + g; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"((uint64_t)map), "r"(bar), "r"(x), "r"(y) : "memory");
}
// TMA prefetch of one box into L2 (no shared memory, no barrier): decouples the HBM latency of the A stream from the
// depth of the shared-memory ring
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* map, int x, int y) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"((uint64_t)map), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)map) : "memory");
}

// ------------------------------------------------------------------------------------------------ host: tensor maps
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && p) fn = (PFN_encodeTiled)p;
  }
  return fn;
}

// 2-D bf16 tensor [rows][cols] with row pitch ld (elements); box = box_cols x box_rows, 128-byte swizzle.
// Encoding a tensor map costs a few microseconds of host time and a step issues ~400 of them with a few dozen
// distinct (pointer, shape) keys: keep a small direct-mapped cache (host-only, one host thread per device).
struct MapCacheEntry { const void* base; uint64_t rows, cols, ld; uint32_t bc, br; CUtensorMap map; };
static inline int make_map_bf16(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                                uint32_t box_cols, uint32_t box_rows);
static inline int make_map_bf16_cached(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                                       uint32_t box_cols, uint32_t box_rows) {
  static thread_local MapCacheEntry cache[256];      // one host thread per device: every thread has its own cache
  uint64_t h = ((uintptr_t)base >> 8) * 0x9E3779B97F4A7C15ull ^ (rows * 31 + cols * 131 + ld * 7 + box_cols + 3 * box_rows);
  MapCacheEntry& e = cache[(h >> 32) & 255];
  if (e.base == base && e.rows == rows && e.cols == cols && e.ld == ld && e.bc == box_cols && e.br == box_rows) {
    *m = e.map;
    return 0;
  }
  int r = make_map_bf16(m, base, rows, cols, ld, box_cols, box_rows);
  if (r == 0) { e.base = base; e.rows = rows; e.cols = cols; e.ld = ld; e.bc = box_cols; e.br = box_rows; e.map = *m; }
  return r;
}
static inline int make_map_bf16(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                                uint32_t box_cols, uint32_t box_rows) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return AVC_E_BADCFG;
  if (((uintptr_t)base & 15u) || (ld * 2) % 16) return AVC_E_ALIGN;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : AVC_E_BADCFG;
}

struct SplitPtr {            // two-term bf16 split of an fp32 matrix, both [rows][ld]
  const __nv_bfloat16* hi;
  const __nv_bfloat16* lo;
  int ld;
};

constexpr int kBM = 128, kBK = 64;
constexpr int kConsumerThreads = 256;                      // two consumer warpgroups
constexpr int kTcThreads = kConsumerThreads + 32;          // + the TMA producer warp
constexpr int kProducerWarp = kConsumerThreads / 32;
constexpr int kSmemMax = 232448;                           // 227 KB of shared memory per CTA

// RESB: the CTA keeps its whole B panel (BN rows x up to kResK k-blocks, hi and lo) resident in shared memory and only
// streams A: re-fetched for every 128-row tile, the B panel would double the L2 -> SM operand traffic of a tile.
constexpr int kResK = 4;          // k-blocks (of 64) a resident panel holds: K <= 256
template <int BN, int NPROD, bool RESB = false>
struct TcCfg {
  static constexpr int A_BYTES = kBM * kBK * 2;                    // one (hi or lo) A slab: 16 KB
  static constexpr int B_BYTES = BN * kBK * 2;
  static constexpr int NOP = (NPROD == 3) ? 2 : 1;                 // slabs per operand (hi, lo)
  static constexpr int BRES_BYTES = RESB ? kResK * NOP * B_BYTES : 0;
  static constexpr int STAGE_BYTES = RESB ? NOP * A_BYTES : NOP * (A_BYTES + B_BYTES);
  static constexpr int kBudget = kSmemMax - 1024 /*align*/ - 256 /*barriers*/ - BRES_BYTES;
  static constexpr int STAGES = kBudget / STAGE_BYTES >= 4 ? 4 : kBudget / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + BRES_BYTES + 1024 + 256;
  static_assert(STAGES >= 2, "tile too large for shared memory");
  static_assert(SMEM_BYTES <= kSmemMax, "exceeds the 227 KB of shared memory per CTA");
};

// Epilogue functor interface (see avc_neus_kernels.cuh): functors with a nested `Aux` type split into
// prefetch(row, col) -> Aux and operator()(row, col, acc, aux); plain functors only have operator()(row, col, acc).
struct NoAux {};
template <typename E, typename = void>
struct EpiTraits {
  using Aux = NoAux;
  static __device__ __forceinline__ Aux prefetch(const E&, int, int) { return {}; }
  static __device__ __forceinline__ void apply(const E& e, int r, int c, float4 a, const Aux&) { e(r, c, a); }
};
template <typename E>
struct EpiTraits<E, std::void_t<typename E::Aux>> {
  using Aux = typename E::Aux;
  static __device__ __forceinline__ Aux prefetch(const E& e, int r, int c) { return e.prefetch(r, c); }
  static __device__ __forceinline__ void apply(const E& e, int r, int c, float4 a, const Aux& x) { e(r, c, a, x); }
};
// The epilogue's own global operands (stashes written passes ago: always DRAM misses) are loaded right before use.
// Functors with `l2_prefetch(m0, n0, bn, M, et, nth)` get the chance to pull the NEXT row tile's operand lines into L2 a
// whole tile ahead (thread et of nth epilogue threads).
template <int ES>   // element size in bytes; [rows][ld] row-major array, tile rows [m0, m0 + 128) x columns [n0, n0 + bn)
__device__ __forceinline__ void l2_prefetch_tile(const void* base, int ld, int ncols, int m0, int n0, int bn, int M,
                                                 int et, int nth) {
  constexpr int kPerLine = 128 / ES;
  const int lpr = (bn + kPerLine - 1) / kPerLine;
  for (int i = et; i < kBM * lpr; i += nth) {
    const int row = m0 + i / lpr, col = n0 + (i % lpr) * kPerLine;
    if (row < M && col < ncols)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(base) + ((size_t)row * ld + col) * ES));
  }
}
template <typename E, typename = void>
struct EpiL2 {
  static __device__ __forceinline__ void run(const E&, int, int, int, int, int, int) {}
};
template <typename E>
struct EpiL2<E, std::void_t<decltype(&E::l2_prefetch)>> {
  static __device__ __forceinline__ void run(const E& e, int m0, int n0, int bn, int M, int et, int nth) {
    if (m0 < M) e.l2_prefetch(m0, n0, bn, M, et, nth);
  }
};

// ------------------------------------------------------------------------------------------------ NT kernel
// The accumulator fragment gives a thread column PAIRS of two rows r and r + 8 (avc_wgmma.cuh).  One exchange with the
// neighbouring lane (lane ^ 1) turns them into one group of 4 consecutive columns per 8-column group -- even lanes take
// row r, odd lanes row r + 8 -- so the functors see (row, col..col+3) with col % 4 == 0, as from the fp32 engine.  A warp
// covers 16 rows x 32 bytes per group: every global access of a functor is whole 32-byte sectors.
template <int BN, typename Epi>
__device__ __forceinline__ void epilogue_nt(const Epi& epi, const float (&acc)[BN / 2], int row, int col0, int M, int N,
                                            int lane) {
  using Tr = EpiTraits<Epi>;
  const bool odd = lane & 1;
  constexpr int kB = 4;      // groups whose functor operands are loaded together, ahead of the arithmetic
#pragma unroll
  for (int j0 = 0; j0 < BN / 8; j0 += kB) {
    float4 v[kB];
    typename Tr::Aux aux[kB];
#pragma unroll
    for (int u = 0; u < kB; ++u) {
      const int j = j0 + u;
      const float s0 = odd ? acc[4 * j] : acc[4 * j + 2], s1 = odd ? acc[4 * j + 1] : acc[4 * j + 3];
      const float r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
      v[u] = odd ? make_float4(r0, r1, acc[4 * j + 2], acc[4 * j + 3]) : make_float4(acc[4 * j], acc[4 * j + 1], r0, r1);
      const int col = col0 + 8 * j;
      if (row < M && col < N) aux[u] = Tr::prefetch(epi, row, col);
    }
#pragma unroll
    for (int u = 0; u < kB; ++u) {
      const int col = col0 + 8 * (j0 + u);
      if (row < M && col < N) Tr::apply(epi, row, col, v[u], aux[u]);
    }
  }
}

// Persistent: gridDim.x CTAs (<= one per SM, a multiple of the number of column tiles); a CTA keeps one column tile
// and walks the row tiles m_first, +m_stride, ...  While the consumers run the epilogue of tile i the producer already
// fills the ring with the first k-blocks of tile i + 1.
template <int BN, int NPROD, bool RESB, typename Epi>
__global__ void __launch_bounds__(kTcThreads, 1)
gemm_tc_nt_kernel(const __grid_constant__ CUtensorMap mapAhi, const __grid_constant__ CUtensorMap mapAlo,
                  const __grid_constant__ CUtensorMap mapBhi, const __grid_constant__ CUtensorMap mapBlo,
                  int M, int N, int K, Epi epi, int l2pf, int b_const) {
  using Cfg = TcCfg<BN, NPROD, RESB>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);   // SWIZZLE_128B wants 1024-B tiles
  constexpr int kOpBytes = Cfg::STAGES * Cfg::STAGE_BYTES + Cfg::BRES_BYTES;     // stages, then the resident B panel
  uint64_t* bars = (uint64_t*)(smem + kOpBytes);
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bres_base = smem_base + Cfg::STAGES * Cfg::STAGE_BYTES;
  const uint32_t full0 = smem_u32(bars), empty0 = full0 + 8 * Cfg::STAGES, bfull = empty0 + 8 * Cfg::STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_n = (N + BN - 1) / BN;
  const int tiles_m = (M + kBM - 1) / kBM;
  const int nk = (K + kBK - 1) / kBK;
  // A CTA owns ONE column tile (n0 fixed: its B panel can stay resident) and walks the row tiles m_first, +m_stride, ..;
  // neighbouring CTAs work on the same row tile at the same time (A is read from HBM once, from L2 after that).
  // The host makes gridDim.x a multiple of tiles_n.
  const int n0 = (int)(blockIdx.x % tiles_n) * BN;
  const int m_first = (int)(blockIdx.x / tiles_n), m_stride = (int)(gridDim.x / tiles_n);

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&mapAhi); tma_prefetch_desc(&mapBhi);
    if (NPROD == 3) { tma_prefetch_desc(&mapAlo); tma_prefetch_desc(&mapBlo); }
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, 2); }
    for (int kb = 0; kb < kResK; ++kb) mbar_init(bfull + 8 * kb, 1);     // one per k-block of the resident B panel
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kProducerWarp) {
    if (lane == 0) {
      // b_const: B holds constants of the step (the packed weights, written many kernels ago): its resident panel is
      // loaded while the predecessor kernel may still be running
      if (!b_const) pdl_wait();
      if (RESB && m_first < tiles_m) {
        for (int kb = 0; kb < nk; ++kb) {
          const uint32_t dst = bres_base + kb * (Cfg::NOP * Cfg::B_BYTES);
          mbar_expect_tx(bfull + 8 * kb, (uint32_t)(Cfg::NOP * Cfg::B_BYTES));
          tma_load_2d(dst, &mapBhi, kb * kBK, n0, bfull + 8 * kb);
          if (NPROD == 3) tma_load_2d(dst + Cfg::B_BYTES, &mapBlo, kb * kBK, n0, bfull + 8 * kb);
        }
      }
      if (b_const) pdl_wait();
      pdl_trigger();
      // l2pf (see the launcher): pull the A boxes of the NEXT row tile into L2 while this one is loaded, so that the
      // ring's loads see L2 latency.
      if (l2pf && m_first < tiles_m)
        for (int kb = 0; kb < nk; ++kb) {
          tma_prefetch_2d(&mapAhi, kb * kBK, m_first * kBM);
          if (NPROD == 3) tma_prefetch_2d(&mapAlo, kb * kBK, m_first * kBM);
        }
      int it = 0;
      AVC_PROBE_DECL(w_empty);
      AVC_PROBE_START(t_tma0);
      for (int mt = m_first; mt < tiles_m; mt += m_stride) {
        const int m0 = mt * kBM;
        const bool pf = l2pf && (mt + m_stride < tiles_m);
        for (int kb = 0; kb < nk; ++kb, ++it) {
          if (pf) {
            tma_prefetch_2d(&mapAhi, kb * kBK, m0 + m_stride * kBM);
            if (NPROD == 3) tma_prefetch_2d(&mapAlo, kb * kBK, m0 + m_stride * kBM);
          }
          const int s = it % Cfg::STAGES;
          AVC_PROBE_WAIT(w_empty, empty0 + 8 * s, ((it / Cfg::STAGES) & 1) ^ 1);
          const uint32_t st = smem_base + s * Cfg::STAGE_BYTES;
          mbar_expect_tx(full0 + 8 * s, Cfg::STAGE_BYTES);
          tma_load_2d(st, &mapAhi, kb * kBK, m0, full0 + 8 * s);
          if (NPROD == 3) tma_load_2d(st + Cfg::A_BYTES, &mapAlo, kb * kBK, m0, full0 + 8 * s);
          if (!RESB) {
            tma_load_2d(st + Cfg::NOP * Cfg::A_BYTES, &mapBhi, kb * kBK, n0, full0 + 8 * s);
            if (NPROD == 3) tma_load_2d(st + Cfg::NOP * Cfg::A_BYTES + Cfg::B_BYTES, &mapBlo, kb * kBK, n0, full0 + 8 * s);
          }
        }
      }
      AVC_PROBE_ADD(EpiProbeId<Epi>::value, 0, w_empty);
      AVC_PROBE_ADD(EpiProbeId<Epi>::value, 1, AVC_PROBE_NOW() - t_tma0);
      AVC_PROBE_ADD(EpiProbeId<Epi>::value, 7, 1);
    }
  } else {
    const int g = warp >> 2, wq = warp & 3;      // consumer warpgroup, warp within it
    const bool leader = (threadIdx.x & 127) == 0;
    const int row_in = 64 * g + 16 * wq + (lane >> 2) + 8 * (lane & 1), col_in = 4 * ((lane >> 1) & 1);
    pdl_wait();      // the functor's operands and outputs belong to predecessor kernels
    float acc[BN / 2];
    int it = 0, lt = 0;
    AVC_PROBE_DECL(w_full);
    AVC_PROBE_START(t_mma0);
    EpiL2<Epi>::run(epi, m_first * kBM, n0, BN, M, (int)threadIdx.x, kConsumerThreads);
    for (int mt = m_first; mt < tiles_m; mt += m_stride, ++lt) {
      const int m0 = mt * kBM;
      EpiL2<Epi>::run(epi, (mt + m_stride) * kBM, n0, BN, M, (int)threadIdx.x, kConsumerThreads);   // a tile ahead
      int prev = -1;
      for (int kb = 0; kb < nk; ++kb, ++it) {
        const int s = it % Cfg::STAGES;
        if (RESB && lt == 0) mbar_wait(bfull + 8 * kb, 0);      // this k-block of the B panel has landed (first tile only)
        AVC_PROBE_WAIT(w_full, full0 + 8 * s, (it / Cfg::STAGES) & 1);
        const uint32_t a_hi = smem_base + s * Cfg::STAGE_BYTES + (uint32_t)g * (64 * 128);   // this warpgroup's 64 rows
        const uint32_t b_hi = RESB ? bres_base + kb * (Cfg::NOP * Cfg::B_BYTES) : smem_base + s * Cfg::STAGE_BYTES + Cfg::NOP * Cfg::A_BYTES;
        const uint64_t da = make_wgmma_desc(a_hi, 16, 1024), db = make_wgmma_desc(b_hi, 16, 1024);
        constexpr uint64_t kLoA = (uint64_t)(Cfg::A_BYTES >> 4), kLoB = (uint64_t)(Cfg::B_BYTES >> 4);
        wgmma_fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int k4 = 0; k4 < kBK / 16; ++k4) {
          wgmma_bf16<BN, 0, 0>(acc, da + 2 * k4, db + 2 * k4, (kb | k4) ? 1u : 0u);
          if (NPROD == 3) {
            wgmma_bf16<BN, 0, 0>(acc, da + 2 * k4, db + kLoB + 2 * k4, 1u);
            wgmma_bf16<BN, 0, 0>(acc, da + kLoA + 2 * k4, db + 2 * k4, 1u);
          }
        }
        wgmma_commit();
        wgmma_fence_acc(acc);
        wgmma_wait<1>();                      // the previous k-block's MMAs are done: its stage can be refilled
        if (prev >= 0 && leader) mbar_arrive(empty0 + 8 * prev);
        prev = s;
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (leader) mbar_arrive(empty0 + 8 * prev);
      epilogue_nt<BN>(epi, acc, m0 + row_in, n0 + col_in, M, N, lane);
    }
    if (threadIdx.x == 0) {
      AVC_PROBE_ADD(EpiProbeId<Epi>::value, 3, w_full);
      AVC_PROBE_ADD(EpiProbeId<Epi>::value, 4, AVC_PROBE_NOW() - t_mma0);
    }
  }
}

template <int BN, int NPROD, bool RESB, typename Epi>
static inline int launch_gemm_tc_nt_bn(cudaStream_t st, int64_t M, int N, int K, const SplitPtr& A, const SplitPtr& B,
                                       const Epi& epi, bool b_const) {
  using Cfg = TcCfg<BN, NPROD, RESB>;
  CUtensorMap mAh, mAl, mBh, mBl;
  AVC_TRY(make_map_bf16_cached(&mAh, A.hi, (uint64_t)M, (uint64_t)K, (uint64_t)A.ld, kBK, kBM));
  AVC_TRY(make_map_bf16_cached(&mBh, B.hi, (uint64_t)N, (uint64_t)K, (uint64_t)B.ld, kBK, BN));
  if (NPROD == 3) {
    AVC_TRY(make_map_bf16_cached(&mAl, A.lo, (uint64_t)M, (uint64_t)K, (uint64_t)A.ld, kBK, kBM));
    AVC_TRY(make_map_bf16_cached(&mBl, B.lo, (uint64_t)N, (uint64_t)K, (uint64_t)B.ld, kBK, BN));
  } else {
    mAl = mAh; mBl = mBh;
  }
  auto kern = gemm_tc_nt_kernel<BN, NPROD, RESB, Epi>;
  static thread_local bool attr_set = false;    // per template instantiation and host thread (= device)
  if (!attr_set) {
    AVC_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_set = true;
  }
  static thread_local int num_sms = 0;
  if (!num_sms) {
    int dev = 0;
    AVC_CUDA_TRY(cudaGetDevice(&dev));
    AVC_CUDA_TRY(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  const int tiles_n = ceil_div(N, BN);
  const int ntiles = ceil_div(M, kBM) * tiles_n;
  int g = ntiles < num_sms ? ntiles : num_sms;         // persistent: at most one CTA per SM ...
  g = (g / tiles_n) * tiles_n;                         // ... and a whole number of CTAs per column tile
  if (g < tiles_n) return AVC_E_BADCFG;
  dim3 grid(g);
  // TMA-prefetch of the next row tile's A boxes into L2, so that the ring's loads see L2 rather than DRAM latency.
  // Launches whose epilogue pulls its own operands into L2 (Epi::kNoATilePrefetch) keep it off.
  // AVC_NT_L2PF=0 / 1 forces it off / on everywhere.
  static int l2pf_env = -2;
  if (l2pf_env == -2) { const char* e = getenv("AVC_NT_L2PF"); l2pf_env = e ? (atoi(e) != 0 ? 1 : 0) : -1; }
  const int l2pf = l2pf_env >= 0 ? l2pf_env : (EpiNoAPf<Epi>::value ? 0 : 1);
  AVC_CUDA_TRY(launch_pdl(kern, dim3(grid), dim3(kTcThreads), (size_t)Cfg::SMEM_BYTES, st, mAh, mAl, mBh, mBl, (int)M, N, K, epi, l2pf, b_const ? 1 : 0));
  AVC_LAUNCH_TRY();
  return 0;
}

// N <= 64 -> one 64-wide tile, else 128-wide tiles (a 65536-row GEMM then has 1024 tiles = 7.8 waves over 132
// persistent CTAs instead of 3.9 with 256-wide tiles: a smaller tail).
template <int NPROD, typename Epi>
static inline int launch_gemm_tc_nt(cudaStream_t st, int64_t M, int N, int K, const SplitPtr& A, const SplitPtr& B,
                                    const Epi& epi, bool b_const = false) {
  if (M <= 0 || N <= 0) return 0;
  // K <= 256: the B panel stays resident in shared memory (RESB); longer reductions stream both operands.
  static int resb = -1;       // AVC_NT_RESB=0 forces the streaming variant (tuning knob)
  if (resb < 0) { const char* e = getenv("AVC_NT_RESB"); resb = (e && atoi(e) == 0) ? 0 : 1; }
  if (resb && K <= kResK * kBK) {
    if (N <= 64) return launch_gemm_tc_nt_bn<64, NPROD, true, Epi>(st, M, N, K, A, B, epi, b_const);
    return launch_gemm_tc_nt_bn<128, NPROD, true, Epi>(st, M, N, K, A, B, epi, b_const);
  }
  if (N <= 64) return launch_gemm_tc_nt_bn<64, NPROD, false, Epi>(st, M, N, K, A, B, epi, b_const);
  return launch_gemm_tc_nt_bn<128, NPROD, false, Epi>(st, M, N, K, A, B, epi, b_const);
}

// ------------------------------------------------------------------------------------------------ TN kernel
// C[i*ldc + j] += sum_{p in slice} A[p,i] * B[p,j]   (i < N1, j < N2): weight gradients.  Both operands are read
// "MN-major": the reduction index p is the row of the global arrays.  TMA boxes are 64 (i or j) x 64 (p); in shared
// memory one box is an MN block [64 p][128 B] (SWIZZLE_128B); a 128-wide M tile is 2 blocks (one per consumer
// warpgroup), a BN-wide N tile BN/64 blocks.  Descriptor: LBO = 8192 B (next 64-wide block), SBO = 1024 B (8 p-rows), a K
// step of 16 p-rows is +2048 B.  Split over p across blockIdx.z; partial tiles meet in fp32 red.global.add.
template <int BN, int NPROD>
struct TcTnCfg {
  static constexpr int BLK = kBK * 128;                             // one 64 x 64 bf16 block: 8 KB
  static constexpr int A_BYTES = (kBM / 64) * BLK;                  // 16 KB
  static constexpr int B_BYTES = (BN / 64) * BLK;
  static constexpr int NOP = (NPROD == 3) ? 2 : 1;
  static constexpr int STAGE_BYTES = NOP * (A_BYTES + B_BYTES);
  static constexpr int kBudget = kSmemMax - 1024 /*align*/ - 1024 /*ones*/ - 256 /*barriers*/;
  static constexpr int STAGES = kBudget / STAGE_BYTES >= 4 ? 4 : kBudget / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 1024 + 256;
  static_assert(SMEM_BYTES <= kSmemMax, "exceeds the 227 KB of shared memory per CTA");
  static_assert(STAGES >= 2, "tile too large for shared memory");
};

template <int BN, int NPROD>
__global__ void __launch_bounds__(kTcThreads, 1)
gemm_tc_tn_kernel(const __grid_constant__ CUtensorMap mapAhi, const __grid_constant__ CUtensorMap mapAlo,
                  const __grid_constant__ CUtensorMap mapBhi, const __grid_constant__ CUtensorMap mapBlo,
                  int P, int N1, int N2, int rows_per_split, float* __restrict__ C, int ldc,
                  float* __restrict__ colsum /* += sum_p A[p,i]; nullptr: off */) {
  using Cfg = TcTnCfg<BN, NPROD>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  // 1 KB of bf16 1.0: the K-major B operand of the column-sum MMA (any layout of an all-ones tile is the all-ones tile)
  uint8_t* ones_tile = smem + Cfg::STAGES * Cfg::STAGE_BYTES;
  uint64_t* bars = (uint64_t*)(ones_tile + 1024);
  const bool do_colsum = (colsum != nullptr) && (blockIdx.y == 0);
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t full0 = smem_u32(bars), empty0 = full0 + 8 * Cfg::STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i0 = blockIdx.x * kBM, j0 = blockIdx.y * BN;
  const int p_begin = blockIdx.z * rows_per_split;
  const int p_end = min(P, p_begin + rows_per_split);
  const int nk = (p_end - p_begin + kBK - 1) / kBK;     // host guarantees rows_per_split % 64 == 0 and nk >= 1

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&mapAhi); tma_prefetch_desc(&mapBhi);
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, 2); }
    fence_barrier_init();
  }
  if (do_colsum) {
    for (int i = threadIdx.x; i < 1024 / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(ones_tile)[i] = 0x3F803F80u;
    fence_proxy_async();
  }
  __syncthreads();

  if (warp == kProducerWarp) {
    if (lane == 0) {
      pdl_wait();         // both operands are activations of predecessor kernels
      pdl_trigger();
      for (int kb = 0; kb < nk; ++kb) {
        const int s = kb % Cfg::STAGES;
        mbar_wait(empty0 + 8 * s, ((kb / Cfg::STAGES) & 1) ^ 1);
        const uint32_t st = smem_base + s * Cfg::STAGE_BYTES;
        const int p0 = p_begin + kb * kBK;
        mbar_expect_tx(full0 + 8 * s, Cfg::STAGE_BYTES);
        // rows beyond p_end inside the last box belong to the next split: they must not be counted twice, so the
        // tensor maps are built with `rows = P` and the host makes every split a multiple of 64 rows.
#pragma unroll
        for (int a = 0; a < kBM / 64; ++a) {
          tma_load_2d(st + a * Cfg::BLK, &mapAhi, i0 + 64 * a, p0, full0 + 8 * s);
          if (NPROD == 3) tma_load_2d(st + Cfg::A_BYTES + a * Cfg::BLK, &mapAlo, i0 + 64 * a, p0, full0 + 8 * s);
        }
#pragma unroll
        for (int b = 0; b < BN / 64; ++b) {
          tma_load_2d(st + Cfg::NOP * Cfg::A_BYTES + b * Cfg::BLK, &mapBhi, j0 + 64 * b, p0, full0 + 8 * s);
          if (NPROD == 3)
            tma_load_2d(st + Cfg::NOP * Cfg::A_BYTES + Cfg::B_BYTES + b * Cfg::BLK, &mapBlo, j0 + 64 * b, p0, full0 + 8 * s);
        }
      }
    }
  } else {
    const int g = warp >> 2, wq = warp & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    const uint64_t dones = make_wgmma_desc(smem_u32(ones_tile), 16, 1024);
    float acc[BN / 2], cs[4];
    int prev = -1;
    for (int kb = 0; kb < nk; ++kb) {
      const int s = kb % Cfg::STAGES;
      mbar_wait(full0 + 8 * s, (kb / Cfg::STAGES) & 1);
      const uint32_t a_hi = smem_base + s * Cfg::STAGE_BYTES + (uint32_t)g * Cfg::BLK;   // this warpgroup's 64 columns i
      const uint32_t b_hi = smem_base + s * Cfg::STAGE_BYTES + Cfg::NOP * Cfg::A_BYTES;
      const uint64_t da = make_wgmma_desc(a_hi, Cfg::BLK, 1024), db = make_wgmma_desc(b_hi, Cfg::BLK, 1024);
      constexpr uint64_t kLoA = (uint64_t)(Cfg::A_BYTES >> 4), kLoB = (uint64_t)(Cfg::B_BYTES >> 4);
      wgmma_fence_acc(acc);
      wgmma_fence_acc(cs);
      // the column-sum switch is decided outside the batch: a branch between the MMAs of a batch would make the compiler
      // serialise them
      auto batch = [&](auto with_colsum) {
        wgmma_fence();
#pragma unroll
        for (int k4 = 0; k4 < kBK / 16; ++k4) {
          wgmma_bf16<BN, 1, 1>(acc, da + 128 * k4, db + 128 * k4, (kb | k4) ? 1u : 0u);
          if (NPROD == 3) {
            wgmma_bf16<BN, 1, 1>(acc, da + 128 * k4, db + kLoB + 128 * k4, 1u);
            wgmma_bf16<BN, 1, 1>(acc, da + kLoA + 128 * k4, db + 128 * k4, 1u);
          }
          if constexpr (decltype(with_colsum)::value) {      // cs[64 x 8] += A^T . ones: every column is A's column sum
            wgmma_bf16<8, 1, 0>(cs, da + 128 * k4, dones, (kb | k4) ? 1u : 0u);
            if (NPROD == 3) wgmma_bf16<8, 1, 0>(cs, da + kLoA + 128 * k4, dones, 1u);
          }
        }
        wgmma_commit();
      };
      if (do_colsum) batch(std::true_type{});
      else batch(std::false_type{});
      wgmma_fence_acc(acc);
      wgmma_fence_acc(cs);
      wgmma_wait<1>();
      if (prev >= 0 && leader) mbar_arrive(empty0 + 8 * prev);
      prev = s;
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    wgmma_fence_acc(cs);
    if (leader) mbar_arrive(empty0 + 8 * prev);
    pdl_wait();           // C is accumulated with atomics: not before the predecessors have drained
    const int r0 = i0 + 64 * g + 16 * wq + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = j0 + 8 * j + 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h;
        if (r < N1) {
          if (c < N2) atomicAdd(C + (size_t)r * ldc + c, acc[4 * j + 2 * h]);
          if (c + 1 < N2) atomicAdd(C + (size_t)r * ldc + c + 1, acc[4 * j + 2 * h + 1]);
        }
      }
    }
    if (do_colsum && (lane & 3) == 0) {
      if (r0 < N1) atomicAdd(colsum + r0, cs[0]);
      if (r0 + 8 < N1) atomicAdd(colsum + r0 + 8, cs[2]);
    }
  }
}

// A: [P][N1] (ld A.ld), B: [P][N2] (ld B.ld); C[N1][ldc] += A^T B.
template <int NPROD>
static inline int launch_gemm_tc_tn(cudaStream_t st, int64_t P, int N1, int N2, const SplitPtr& A, const SplitPtr& B,
                                    float* C, int ldc, float* colsum = nullptr) {
  if (P <= 0 || N1 <= 0 || N2 <= 0) return 0;
  CUtensorMap mAh, mAl, mBh, mBl;
  AVC_TRY(make_map_bf16_cached(&mAh, A.hi, (uint64_t)P, (uint64_t)N1, (uint64_t)A.ld, 64, kBK));
  AVC_TRY(make_map_bf16_cached(&mBh, B.hi, (uint64_t)P, (uint64_t)N2, (uint64_t)B.ld, 64, kBK));
  if (NPROD == 3) {
    AVC_TRY(make_map_bf16_cached(&mAl, A.lo, (uint64_t)P, (uint64_t)N1, (uint64_t)A.ld, 64, kBK));
    AVC_TRY(make_map_bf16_cached(&mBl, B.lo, (uint64_t)P, (uint64_t)N2, (uint64_t)B.ld, 64, kBK));
  } else {
    mAl = mAh; mBl = mBh;
  }
  const int t1 = ceil_div(N1, kBM);
  auto go = [&](auto kern, int BN, int smem) -> int {
    AVC_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const int t2 = ceil_div(N2, BN);
    static thread_local int sms = 0;
    if (!sms) { int dev = 0; AVC_CUDA_TRY(cudaGetDevice(&dev)); AVC_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)); }
    int splits = (sms + t1 * t2 - 1) / (t1 * t2);
    int rows = (int)round_up(ceil_div(P, splits), kBK);
    splits = ceil_div(P, rows);
    dim3 grid(t1, t2, splits);
    AVC_CUDA_TRY(launch_pdl(kern, grid, dim3(kTcThreads), (size_t)smem, st, mAh, mAl, mBh, mBl, (int)P, N1, N2, rows, C, ldc, colsum));
    AVC_LAUNCH_TRY();
    return 0;
  };
  if (N2 <= 64) return go(gemm_tc_tn_kernel<64, NPROD>, 64, TcTnCfg<64, NPROD>::SMEM_BYTES);
  if (N2 <= 128) return go(gemm_tc_tn_kernel<128, NPROD>, 128, TcTnCfg<128, NPROD>::SMEM_BYTES);
  return go(gemm_tc_tn_kernel<256, NPROD>, 256, TcTnCfg<256, NPROD>::SMEM_BYTES);
}

// ------------------------------------------------------------------------------------------------ split helper
// fp32 [rows][ld_src] -> bf16 hi/lo [rows][ld_dst] (columns >= cols zero-filled up to ld_dst)
static __global__ void k_split_bf16(const float* __restrict__ src, int64_t rows, int cols, int ld_src,
                             __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int ld_dst) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * ld_dst) return;
  int64_t r = i / ld_dst;
  int c = (int)(i - r * ld_dst);
  float v = c < cols ? src[(size_t)r * ld_src + c] : 0.f;
  __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[i] = h;
  lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
}

}  // namespace tc
}  // namespace avc
