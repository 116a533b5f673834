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
// Consumer warpgroups issue wgmma.mma_async m64nBNk16 on shared-memory descriptors, keep their fp32 accumulator in
// registers and run the epilogue straight from that fragment; a TMA producer fills a shared-memory ring (K step 64, one
// 128-byte swizzle atom; 32 for TN) guarded by full (TMA transaction count) / empty mbarriers.
//   NT (384 threads): persistent ping-pong.  A producer warpgroup and two consumer warpgroups that take turns at the
//      tensor pipe, one 64-row tile each, so that one's epilogue runs under the other's MMAs; one column tile per CTA,
//      B panel resident in shared memory when K <= 256.
//   TN (288 threads): warps 0-7 are two consumer warpgroups, warpgroup g owning rows [64 g, 64 g + 64) of the 128-row
//      tile, warp 8 the producer; one tile per CTA, split over the reduction dimension.
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
// Optional stall probe of the NT kernel (compile with -DAVC_NT_PROBE=1, see tools/nt_probe.py).  Cycles summed over the
// CTAs of every launch, per epilogue functor (Epi::kProbeId), in the slots
//   0 producer waits for a free stage   1 producer loop          2 consumers wait for operands   3 consumers wait for turn
//   4 consumers' MMAs (turn to done)    5 consumers' epilogues   6 consumers' loops              7 CTAs
//   8 consumers wait for staged epilogue operands     9 consumers wait for their TMA stores to release a ring slot
// (the consumer slots add up both consumer warpgroups).  AVC_PROBE(...) code only exists in the probe build.
constexpr int kNtProbeSlots = 10;
#ifdef AVC_NT_PROBE
static __device__ unsigned long long g_nt_probe[16][kNtProbeSlots];
#define AVC_PROBE(...) __VA_ARGS__
#define AVC_PROBE_WAIT(acc, bar, par) do { long long t__ = clock64(); mbar_wait(bar, par); (acc) += clock64() - t__; } while (0)
#define AVC_PROBE_ADD(id, slot, v) atomicAdd(&g_nt_probe[id][slot], (unsigned long long)(v))
#else
#define AVC_PROBE(...)
#define AVC_PROBE_WAIT(acc, bar, par) mbar_wait(bar, par)
#define AVC_PROBE_ADD(id, slot, v)
#endif
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
// bar.sync / bar.arrive on a named barrier (id >= 1; 0 is __syncthreads) over `count` threads
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"((uint64_t)map), "r"(bar), "r"(x), "r"(y) : "memory");
}
// C[0] += a, C[1] += b as one 8-byte reduction (C 8-byte aligned)
__device__ __forceinline__ void red_add_v2(float* C, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(C), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)map) : "memory");
}
// TMA bulk store of a box from shared memory; elements outside the map's extents are not written
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int x, int y) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"((uint64_t)map), "r"(src), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's bulk groups still read their shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// all of this thread's bulk groups have completed their writes
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

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

// 2-D fp32 (es = 4) or bf16 (es = 2) tensor [rows][cols], row pitch ld elements, box = box_cols x box_rows; the swizzle
// spans one box row (box_cols * es = 32, 64 or 128 bytes).  Columns >= cols and rows >= rows of a box read as zero.
// Cached like make_map_bf16_cached.
static inline int make_map_rows_cached(CUtensorMap* m, int es, const void* base, uint64_t rows, uint64_t cols,
                                       uint64_t ld, uint32_t box_cols, uint32_t box_rows) {
  static thread_local MapCacheEntry cache[256];
  const uint64_t h = ((uintptr_t)base >> 8) * 0x9E3779B97F4A7C15ull ^ (rows * 31 + cols * 131 + ld * 7 + box_cols + 3 * box_rows + es);
  MapCacheEntry& e = cache[(h >> 32) & 255];
  const uint32_t bc = box_cols | ((uint32_t)es << 16);      // the element size is part of the key
  if (e.base == base && e.rows == rows && e.cols == cols && e.ld == ld && e.bc == bc && e.br == box_rows) {
    *m = e.map;
    return 0;
  }
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return AVC_E_BADCFG;
  if (((uintptr_t)base & 15u) || (ld * es) % 16) return AVC_E_ALIGN;
  const uint32_t span = box_cols * es;
  const CUtensorMapSwizzle sw = span == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : span == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                                                     : CU_TENSOR_MAP_SWIZZLE_32B;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * es};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, es == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base),
                  dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return AVC_E_BADCFG;
  e.base = base; e.rows = rows; e.cols = cols; e.ld = ld; e.bc = bc; e.br = box_rows; e.map = *m;
  return 0;
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

// NT kernel: a producer warpgroup and two consumer warpgroups; its work unit is one warpgroup's m64 row block.
constexpr int kNtBM = 64;
constexpr int kNtThreads = 384;
constexpr int kNtTurnBar = 1;     // named barrier kNtTurnBar + c: consumer warpgroup c may issue its next tile's MMAs

// RESB: the CTA keeps its whole B panel (BN rows x up to kResK k-blocks, hi and lo) resident in shared memory and only
// streams A: re-fetched for every row tile, the B panel would multiply the L2 -> SM operand traffic of a tile.
constexpr int kResK = 4;          // k-blocks (of 64) a resident panel holds: K <= 256
// Functors with epilogue rings (staged operands, EpiStage, or ring-stored outputs, EpiOut, below) give the A ring
// kEpiAStages stages and the rest of the shared memory to the rings, at most kEpiSlotsMax slots per consumer warpgroup.
constexpr int kEpiAStages = 3, kEpiSlotsMax = 8;
// EPI_SLOT: bytes of one epilogue ring slot (0: the functor stages nothing, no rings)
template <int BN, int NPROD, bool RESB = false, int EPI_SLOT = 0>
struct TcCfg {
  static constexpr int A_BYTES = kNtBM * kBK * 2;                  // one (hi or lo) A slab: 8 KB
  static constexpr int B_BYTES = BN * kBK * 2;
  static constexpr int NOP = (NPROD == 3) ? 2 : 1;                 // slabs per operand (hi, lo)
  static constexpr int BRES_BYTES = RESB ? kResK * NOP * B_BYTES : 0;
  static constexpr int STAGE_BYTES = RESB ? NOP * A_BYTES : NOP * (A_BYTES + B_BYTES);
  static constexpr int BAR_BYTES = EPI_SLOT ? 512 : 256;
  static constexpr int kBudget = kSmemMax - 1024 /*align*/ - BAR_BYTES - BRES_BYTES;
  static constexpr int STAGES = EPI_SLOT ? kEpiAStages : kBudget / STAGE_BYTES >= 8 ? 8 : kBudget / STAGE_BYTES;
  static constexpr int kEpiFit = EPI_SLOT ? (kBudget - STAGES * STAGE_BYTES) / (2 * EPI_SLOT) : 0;
  static constexpr int EPI_SLOTS = kEpiFit > kEpiSlotsMax ? kEpiSlotsMax : kEpiFit;      // per consumer warpgroup
  static constexpr int SLOT_BYTES = EPI_SLOT;
  static constexpr int EPI_BYTES = 2 * EPI_SLOTS * EPI_SLOT;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + BRES_BYTES + EPI_BYTES + 1024 + BAR_BYTES;
  static_assert(STAGES >= 2, "tile too large for shared memory");
  static_assert(!EPI_SLOT || EPI_SLOTS >= 2, "no room for two epilogue slots per consumer");
  static_assert(8 * (2 * STAGES + kResK + 4 * EPI_SLOTS) <= BAR_BYTES, "mbarriers overflow their area");
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
  template <typename S>
  static __device__ __forceinline__ void ring(const E& e, int r, int c, float4 a, const Aux&, const S& s) { e.ring(r, c, a, s); }
};
template <typename E>
struct EpiTraits<E, std::void_t<typename E::Aux>> {
  using Aux = typename E::Aux;
  static __device__ __forceinline__ Aux prefetch(const E& e, int r, int c) { return e.prefetch(r, c); }
  static __device__ __forceinline__ void apply(const E& e, int r, int c, float4 a, const Aux& x) { e(r, c, a, x); }
  template <typename S>
  static __device__ __forceinline__ void ring(const E& e, int r, int c, float4 a, const Aux& x, const S& s) { e.ring(r, c, a, x, s); }
};
template <typename E, typename = void>
struct HasStage : std::false_type {};
template <typename E>
struct HasStage<E, std::void_t<typename E::Stage>> : std::true_type {};
// groups of 8 columns per epilogue batch: two batches of global operands are live beside the accumulator; with 32-byte
// operands (EpiChainBwd, EpiDgrad) batches of 4 need more registers than ptxas grants a 384-thread kernel and spill
// (RING: outputs stored through the epilogue ring, EpiOut below: batches of 2, so that two slots per consumer fit beside
// the B panel; staged functors, whose outputs are ring-stored over their staged operands, too: with batches of 4 the
// ring stores of EpiChain spill)
template <typename E, bool RING = false>
struct EpiBatch {
  static constexpr int kB = (RING || HasStage<E>::value || sizeof(typename EpiTraits<E>::Aux) > 16) ? 2 : 4;
  static constexpr int kCols = 8 * kB;
};

// Staged epilogue operands.  A functor with a nested `using Stage = tc::Staged<ES0[, ES1[, ES2]]>` (element sizes in bytes:
// 4 fp32, 2 bf16) has the per-tile global operands of its epilogue loaded by TMA into shared memory ahead of the tile:
//   tc::StageOp stage_op(int i) const                 (host) operand i: [rows][ld] array, column extent = padded width
//   static Aux from_stage(const uint4 (&raw)[kN])      4 consecutive elements of each operand (bf16: raw.x, raw.y) -> Aux
// A ring slot holds one batch (EpiBatch::kCols columns x 64 rows) of every operand.  Columns past the extent and rows past
// M read as zero (TMA out-of-bounds fill).
template <int E0, int E1 = 0, int E2 = 0>
struct Staged {
  static constexpr int kN = 1 + (E1 > 0) + (E2 > 0);
  static constexpr int kColBytes = E0 + E1 + E2;
  __host__ __device__ static constexpr int es(int i) { return i == 0 ? E0 : i == 1 ? E1 : E2; }
  __host__ __device__ static constexpr int before(int i) { return i == 0 ? 0 : i == 1 ? E0 : E0 + E1; }
};
struct StageOp { const void* base; int ld; int cols; };
template <typename E, typename = void>
struct EpiStage {
  static constexpr int kN = 0, kSlotBytes = 0;
};
template <typename E>
struct EpiStage<E, std::void_t<typename E::Stage>> {
  using S = typename E::Stage;
  static constexpr int kN = S::kN, kSlotBytes = kNtBM * EpiBatch<E>::kCols * S::kColBytes;
};
template <int N>
struct EpiMaps { CUtensorMap m[N]; };
template <>
struct EpiMaps<0> {};
// Address of the 4 elements at (r, c) of a [rows][COLS] box as TMA reads and writes it: rows of span = COLS * ES bytes,
// swizzled over the span (16-byte unit bits 4.. ^= address bits 7..; the box starts at a multiple of 8 rows' bytes)
__device__ __forceinline__ uint32_t box_addr(uint32_t slab, int r, int c, int es, int span) {
  const uint32_t lin = (uint32_t)(r * span + c * es);
  return slab + (lin ^ (((lin >> 7) & (span / 16 - 1)) << 4));
}
template <int ES, int COLS>
__device__ __forceinline__ uint32_t box_addr(uint32_t slab, int r, int c) {
  static_assert(COLS * ES == 32 || COLS * ES == 64 || COLS * ES == 128, "swizzle span");
  return box_addr(slab, r, c, ES, COLS * ES);
}
// 4 elements at (r, c) of a [64][cols] box as TMA wrote it
// (volatile: stays behind the slot's full-barrier wait)
template <int ES, int COLS>
__device__ __forceinline__ uint4 stage_read(uint32_t slab, int r, int c) {
  const uint32_t addr = box_addr<ES, COLS>(slab, r, c);
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if constexpr (ES == 4)
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  else
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
  return v;
}

// Ring-stored epilogue outputs.  A functor with a nested `using Out = tc::Outs<ES0, ES1, ...>` (element sizes in bytes: 4
// fp32, 2 bf16) has the NT tiles send its outputs through the consumer's epilogue ring and TMA bulk stores instead of
// register stores:
//   tc::OutOp out_op(int i, int N) const       (host) output i of a GEMM N columns wide: [rows][ld] array and column
//                                              extent; base nullptr: not stored
//   void ring(row, col, acc[, aux], const S& s) const    operator()'s arithmetic, handing the values of the 4 columns
//                                              to s.f32(i, v) or s.split(i, v) (bf16 hi to output i, lo to output i + 1)
// Each warp owns 16 rows of the 64-row tile and its own part of every slot, [output][16 rows][kCols], and stores it
// with boxes of 16 rows x kCols.  Rows >= M and columns past an output's extent are not written (TMA bounds), so the
// extents restate which columns the functor's global path writes.  Columns < N go through ring(), groups wholly at
// columns >= N are zeros.
// A staged functor (EpiStage) writes its outputs in place over its staged operands, so its slots need no extra bytes:
//   static constexpr tc::Over over(int i)      output i overwrites the warp's 16 rows of staged operand `op`, `off` of
//                                              its own boxes into them; with pieces = 2 it is stored as two boxes of
//                                              kCols / 2 columns, over the warp's rows of operands op and op + 1
// Outputs that would overlap cannot be stored by one launch: the host rejects them (AVC_E_BADCFG).
struct Over { int op, off, pieces; };
template <int... ES>
struct Outs {
  static constexpr int kN = sizeof...(ES);
  static constexpr int kColBytes = (ES + ...);
  __host__ __device__ static constexpr int es(int i) { int k = 0, r = 0; ((r = (k++ == i ? ES : r)), ...); return r; }
  __host__ __device__ static constexpr int before(int i) { int k = 0, r = 0; ((r += (k++ < i ? ES : 0)), ...); return r; }
};
struct OutOp { const void* base; int ld; int cols; };
template <typename E, typename = void>
struct EpiOut {
  static constexpr int kN = 0, kSlotBytes = 0;
};
template <typename E>
struct EpiOut<E, std::void_t<typename E::Out>> {
  using O = typename E::Out;
  static constexpr int kN = O::kN;
  static constexpr int kSlotBytes = EpiStage<E>::kN ? EpiStage<E>::kSlotBytes : kNtBM * EpiBatch<E, true>::kCols * O::kColBytes;
};
// Where the boxes of the ring-stored outputs lie in a slot: output i is stored as pieces(i) boxes of 16 rows x cols(i),
// piece p of warp wq at byte at(i, p, wq) of the slot.
template <typename E, bool STAGED = (EpiStage<E>::kN > 0)>
struct OutLayout {      // store-only functors: [warp][output][16 rows][kCols]
  using O = typename E::Out;
  static constexpr int kCols = EpiBatch<E, true>::kCols;
  __host__ __device__ static constexpr int pieces(int) { return 1; }
  __host__ __device__ static constexpr int cols(int) { return kCols; }
  __host__ __device__ static constexpr int at(int i, int, int wq) { return 16 * kCols * (wq * O::kColBytes + O::before(i)); }
};
template <typename E>
struct OutLayout<E, true> {      // staged functors: in place over the staged operands, [operand][4 warps][16 rows][kCols]
  using O = typename E::Out;
  using St = typename E::Stage;
  static constexpr int kCols = EpiBatch<E>::kCols;
  __host__ __device__ static constexpr int pieces(int i) { return E::over(i).pieces; }
  __host__ __device__ static constexpr int cols(int i) { return kCols / pieces(i); }
  __host__ __device__ static constexpr int box_bytes(int i) { return 16 * cols(i) * O::es(i); }
  __host__ __device__ static constexpr int part(int k) { return 16 * kCols * St::es(k); }      // a warp's rows of operand k
  __host__ __device__ static constexpr int at(int i, int p, int wq) {
    const int k = E::over(i).op + p;
    return kNtBM * kCols * St::before(k) + wq * part(k) + E::over(i).off * box_bytes(i);
  }
  // every box inside the warp's rows of its operand and on its swizzle period (8 rows of its span): box_addr's swizzle
  // is the one TMA applies
  static constexpr bool fits() {
    for (int i = 0; i < O::kN; ++i) {
      const int span = cols(i) * O::es(i), period = 8 * span;
      if (span != 32 && span != 64 && span != 128) return false;
      for (int p = 0; p < pieces(i); ++p) {
        const int k = E::over(i).op + p;
        if (k >= St::kN || (E::over(i).off + 1) * box_bytes(i) > part(k)) return false;
        if ((kNtBM * kCols * St::before(k)) % period || part(k) % period || (E::over(i).off * box_bytes(i)) % period) return false;
      }
    }
    return true;
  }
  static constexpr bool overlap(int i, int j) {
    for (int p = 0; p < pieces(i); ++p)
      for (int q = 0; q < pieces(j); ++q) {
        const int a = at(i, p, 0), b = at(j, q, 0);
        if (a < b + box_bytes(j) && b < a + box_bytes(i)) return true;
      }
    return false;
  }
};
// TMA bounds the columns of a store in whole 16-byte units (it writes past an extent up to the next 16 bytes), so a
// launch whose stored outputs do not all end on 16 bytes keeps the functor's register stores (RING = false).
// (measured on an H100: with an extent of 217 bf16 columns, a store box wrote through column 223, and with 217 fp32
// columns through column 219)
template <int N>
struct EpiOutMaps { CUtensorMap m[N]; };      // per output: its tensor map (box 16 rows x OutLayout::cols)
template <>
struct EpiOutMaps<0> {};
// A thread's view of its warp's part of a ring slot: row r (0..15) of the warp's boxes, columns c..c+3 of the batch.
// Outputs whose bit in `mask` is clear are not stored, so they are not written here either.
template <typename L>
struct RingSink {
  using O = typename L::O;
  uint32_t slot; int wq, r, c; uint32_t mask;
  __device__ __forceinline__ uint32_t at(int i) const {
    const int p = L::pieces(i) == 1 ? 0 : c / L::cols(i);
    return box_addr(slot + L::at(i, p, wq), r, c - p * L::cols(i), O::es(i), L::cols(i) * O::es(i));
  }
  __device__ __forceinline__ void f32(int i, const float v[4]) const {
    if (!((mask >> i) & 1u)) return;
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(at(i)), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]) : "memory");
  }
  // the two-term bf16 split of v, rounded as split16_put4 rounds it
  __device__ __forceinline__ void split(int i, const float v[4]) const {
    if (!((mask >> i) & 3u)) return;
    const uint32_t h01 = bf16x2_bits(v[0], v[1]), h23 = bf16x2_bits(v[2], v[3]);
    const float r0 = v[0] - __uint_as_float(h01 << 16), r1 = v[1] - __uint_as_float(h01 & 0xffff0000u);
    const float r2 = v[2] - __uint_as_float(h23 << 16), r3 = v[3] - __uint_as_float(h23 & 0xffff0000u);
    if ((mask >> i) & 1u) asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(at(i)), "r"(h01), "r"(h23) : "memory");
    if ((mask >> (i + 1)) & 1u)
      asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(at(i + 1)), "r"(bf16x2_bits(r0, r1)), "r"(bf16x2_bits(r2, r3)) : "memory");
  }
  // a group wholly at columns >= N: zeros (they land only where an extent reaches past N, in a stash's padding)
  __device__ __forceinline__ void zero() const {
#pragma unroll
    for (int i = 0; i < O::kN; ++i) {
      if (!((mask >> i) & 1u)) continue;
      if (O::es(i) == 4) asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(at(i)), "r"(0u) : "memory");
      else asm volatile("st.shared.v2.u32 [%0], {%1, %1};" ::"r"(at(i)), "r"(0u) : "memory");
    }
  }
};
// (lane 0 of a warp) one TMA bulk store per piece of every stored output from the warp's boxes in `slot`, as one bulk
// group; (x, y) = the global column and row of the boxes
template <typename L, int N>
__device__ __forceinline__ void ring_store(const EpiOutMaps<N>& omaps, uint32_t mask, uint32_t slot, int wq, int x, int y) {
#pragma unroll
  for (int i = 0; i < N; ++i) {
    if (!((mask >> i) & 1u)) continue;
#pragma unroll
    for (int p = 0; p < L::pieces(i); ++p) tma_store_2d(&omaps.m[i], slot + L::at(i, p, wq), x + p * L::cols(i), y);
  }
  bulk_commit();
}

// ------------------------------------------------------------------------------------------------ NT kernel
// The accumulator fragment gives a thread column PAIRS of two rows r and r + 8 (avc_wgmma.cuh).  One exchange with the
// neighbouring lane (lane ^ 1) turns them into one group of 4 consecutive columns per 8-column group -- even lanes take
// row r, odd lanes row r + 8 -- so the functors see (row, col..col+3) with col % 4 == 0, as from the fp32 engine.  A warp
// covers 16 rows x 32 bytes per group: every global access of a functor is whole 32-byte sectors.
// The functor operands (prefetch) are loaded in batches of kB groups, one batch ahead of the arithmetic: the first batch
// before `mma_done()` (which waits for the accumulator), every later one before the previous batch's arithmetic and
// stores, so that a memory round trip is always in flight under other work.
// Staged functors (EpiStage) read their operands from the consumer's epilogue ring instead: batch b is chunk q0 + b of the
// ring (one slot per batch), waited for on its full barrier.  Each warp writes its outputs over its own 16 rows of the
// operands it has just read (OutLayout) and stores them with TMA.  A slot goes back to its loader (one empty-barrier
// arrival per warp) once the warp's stores have read it: after committing batch b, lane 0 waits until only that batch's
// stores may still read (`wait_group.read 1`) and releases batch b - 1's slot; the tile's last slot after `read 0`.
// Functors with ring-stored outputs (EpiOut) write batch b into chunk q0 + b of the ring, and each warp sends its part
// of the slot out with TMA bulk stores (one bulk group per batch).  Before a warp rewrites a slot, its lane 0 waits
// until the stores issued from that slot SLOTS batches ago have read it (`wait_group.read SLOTS - 1`): no barrier.
struct EpiRing {
  uint32_t base;               // slot 0 of this consumer's ring (shared-memory address)
  uint32_t full0, empty0;      // mbarriers of slot 0 (8 bytes apart)
  int q0;                      // ring chunk counter of the tile's first batch
  int r, c;                    // this thread's row / first column inside a chunk
  int m0, n0, wq;              // the tile's origin, the warp within the consumer warpgroup
  uint32_t omask;              // ring-stored outputs that are stored (bit i: output i)
};
template <int BN, int SLOTS, bool RING, typename Epi, typename OMaps, typename MmaDone>
__device__ __forceinline__ void epilogue_nt(const Epi& epi, const float (&acc)[BN / 2], int row, int col0, int M, int N,
                                            int lane, MmaDone&& mma_done, const EpiRing& ring, const OMaps& omaps,
                                            long long& w_stage, long long& w_drain) {
  using Tr = EpiTraits<Epi>;
  const bool odd = lane & 1;
  constexpr int kB = EpiBatch<Epi, RING>::kB, kNB = BN / 8 / kB;
  auto group = [&](int j) {      // the 4-column group j of this thread's row (one exchange with lane ^ 1)
    const float s0 = odd ? acc[4 * j] : acc[4 * j + 2], s1 = odd ? acc[4 * j + 1] : acc[4 * j + 3];
    const float r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
    return odd ? make_float4(r0, r1, acc[4 * j + 2], acc[4 * j + 3]) : make_float4(acc[4 * j], acc[4 * j + 1], r0, r1);
  };
  if constexpr (EpiStage<Epi>::kN > 0) {
    using St = typename Epi::Stage;
    using L = OutLayout<Epi>;
    constexpr int kCols = EpiBatch<Epi>::kCols, kSlot = EpiStage<Epi>::kSlotBytes;
    mma_done();
#pragma unroll
    for (int b = 0; b < kNB; ++b) {
      const int q = ring.q0 + b, s = q % SLOTS;
      AVC_PROBE_WAIT(w_stage, ring.full0 + 8 * s, (q / SLOTS) & 1);
      const uint32_t slot = ring.base + s * kSlot;
      typename Tr::Aux aux[kB];
#pragma unroll
      for (int u = 0; u < kB; ++u) {
        uint4 raw[St::kN];
#pragma unroll
        for (int i = 0; i < St::kN; ++i) {
          const uint32_t slab = slot + kNtBM * kCols * St::before(i);
          raw[i] = St::es(i) == 4 ? stage_read<4, kCols>(slab, ring.r, ring.c + 8 * u)
                                  : stage_read<2, kCols>(slab, ring.r, ring.c + 8 * u);
        }
        aux[u] = Epi::from_stage(raw);
      }
      __syncwarp();      // the warp has read its operands before any lane writes its outputs over them
#pragma unroll
      for (int u = 0; u < kB; ++u) {
        const int j = kB * b + u;
        const float4 v = group(j);
        const int col = col0 + 8 * j;
        const RingSink<L> sink{slot, ring.wq, ring.r - 16 * ring.wq, ring.c + 8 * u, ring.omask};
        if (row < M) {
          if (col < N) Tr::ring(epi, row, col, v, aux[u], sink);
          else sink.zero();
        }
      }
      fence_proxy_async();      // the generic-proxy writes above, before the async proxy reads them
      __syncwarp();
      if (lane == 0) {
        ring_store<L>(omaps, ring.omask, slot, ring.wq, ring.n0 + b * kCols, ring.m0 + 16 * ring.wq);
        // one arrival per warp: the previous batch's slot may be refilled once its stores have read it
        if (b > 0) {
          AVC_PROBE(const long long t0 = clock64());
          bulk_wait_read<1>();
          AVC_PROBE(w_drain += clock64() - t0);
          mbar_arrive(ring.empty0 + 8 * ((q - 1) % SLOTS));
        }
      }
    }
    if (lane == 0) {      // the last slot goes back before the next tile's MMAs, during which its loader refills
      AVC_PROBE(const long long t0 = clock64());
      bulk_wait_read<0>();
      AVC_PROBE(w_drain += clock64() - t0);
      mbar_arrive(ring.empty0 + 8 * ((ring.q0 + kNB - 1) % SLOTS));
    }
  } else if constexpr (RING) {
    using L = OutLayout<Epi>;
    constexpr int kCols = EpiBatch<Epi, true>::kCols, kSlot = EpiOut<Epi>::kSlotBytes;
    typename Tr::Aux aux[2][kB];
    auto load = [&](int b) {
#pragma unroll
      for (int u = 0; u < kB; ++u) {
        const int col = col0 + 8 * (kB * b + u);
        if (row < M && col < N) aux[b & 1][u] = Tr::prefetch(epi, row, col);
      }
    };
    load(0);
    mma_done();
#pragma unroll
    for (int b = 0; b < kNB; ++b) {
      if (b + 1 < kNB) load(b + 1);
      // the warp's part of the slot: its boxes at L::at(i, 0, 0) from there
      const uint32_t box = ring.base + ((ring.q0 + b) % SLOTS) * kSlot + L::at(0, 0, ring.wq);
      if (lane == 0) {
        AVC_PROBE(const long long t0 = clock64());
        bulk_wait_read<SLOTS - 1>();
        AVC_PROBE(w_drain += clock64() - t0);
      }
      __syncwarp();
#pragma unroll
      for (int u = 0; u < kB; ++u) {
        const int j = kB * b + u;
        const float4 v = group(j);
        const int col = col0 + 8 * j;
        const RingSink<L> sink{box, 0, ring.r - 16 * ring.wq, ring.c + 8 * u, ring.omask};
        if (row < M) {
          if (col < N) Tr::ring(epi, row, col, v, aux[b & 1][u], sink);
          else sink.zero();
        }
      }
      fence_proxy_async();      // the generic-proxy writes above, before the async proxy reads them
      __syncwarp();
      if (lane == 0) ring_store<L>(omaps, ring.omask, box, 0, ring.n0 + b * kCols, ring.m0 + 16 * ring.wq);
    }
  } else {
    typename Tr::Aux aux[2][kB];
    auto load = [&](int b) {
#pragma unroll
      for (int u = 0; u < kB; ++u) {
        const int col = col0 + 8 * (kB * b + u);
        if (row < M && col < N) aux[b & 1][u] = Tr::prefetch(epi, row, col);
      }
    };
    load(0);
    mma_done();
#pragma unroll
    for (int b = 0; b < kNB; ++b) {
      if (b + 1 < kNB) load(b + 1);
#pragma unroll
      for (int u = 0; u < kB; ++u) {
        const int j = kB * b + u;
        const float s0 = odd ? acc[4 * j] : acc[4 * j + 2], s1 = odd ? acc[4 * j + 1] : acc[4 * j + 3];
        const float r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
        const float4 v = odd ? make_float4(r0, r1, acc[4 * j + 2], acc[4 * j + 3]) : make_float4(acc[4 * j], acc[4 * j + 1], r0, r1);
        const int col = col0 + 8 * j;
        if (row < M && col < N) Tr::apply(epi, row, col, v, aux[b & 1][u]);
      }
    }
  }
}

// Persistent ping-pong: gridDim.x CTAs (<= one per SM, a multiple of the number of column tiles); a CTA keeps one column
// tile and walks the 64-row tiles m_first, +m_stride, ...; its j-th tile belongs to consumer warpgroup j % 2.
//   warpgroup 0      producer: one thread issues the TMA (resident B panel, then the A ring); 40 registers
//   warpgroups 1, 2  consumers: MMAs of a tile into a register accumulator, then its epilogue; 232 registers
// The consumers take strict turns at issuing MMAs (named barriers kNtTurnBar + c).  A consumer passes the turn as soon as
// its last k-block is issued, then waits for its MMAs and runs the epilogue while the other one issues: the tensor pipe
// works under the epilogues.  Turns make the ring's consumption follow the tile order, so the k-block counter j * nk + kb
// gives every role the stage and its parity, and each stage is released by the one warpgroup that read it.
// Staged functors (EpiStage): threads 32 and 64 of the producer warpgroup are the epilogue operand loaders of consumer
// warpgroups 0 and 1.  Each walks its consumer's tiles and issues, batch by batch, one chunk of every staged operand
// (TMA, box kCols x 64) into the consumer's epilogue ring (EPI_SLOTS slots, full / empty mbarriers), so that the
// operands of a tile land while its MMAs run.  The ring chunk counter (tile j: (j / 2) * batches + b) gives both sides the
// slot and its parity.  Their outputs are stored with TMA from the same slots, written over the operands.
// Store-only functors with ring-stored outputs (EpiOut) use the same rings, without loaders or mbarriers: the consumers'
// warps write their outputs into them and store them with TMA (omaps: one tensor map per output, omask: the outputs
// stored).
template <int BN, int NPROD, bool RESB, typename Epi, bool RING = false>
__global__ void __launch_bounds__(kNtThreads, 1)
gemm_tc_nt_kernel(const __grid_constant__ CUtensorMap mapAhi, const __grid_constant__ CUtensorMap mapAlo,
                  const __grid_constant__ CUtensorMap mapBhi, const __grid_constant__ CUtensorMap mapBlo,
                  int M, int N, int K, Epi epi, int b_const, const __grid_constant__ EpiMaps<EpiStage<Epi>::kN> emaps,
                  const __grid_constant__ EpiOutMaps<EpiOut<Epi>::kN> omaps, uint32_t omask) {
  static_assert(!RING || EpiOut<Epi>::kN > 0, "only functors with an Out ring-store");
  static_assert(RING || EpiStage<Epi>::kN == 0, "staged functors ring-store their outputs");
  using Cfg = TcCfg<BN, NPROD, RESB, RING ? EpiOut<Epi>::kSlotBytes : 0>;
  constexpr int kStaged = EpiStage<Epi>::kN;
  constexpr int kEpiCols = EpiBatch<Epi, RING>::kCols, kEpiNB = BN / kEpiCols;      // ring chunks per tile
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);   // SWIZZLE_128B wants 1024-B tiles
  // stages, then the resident B panel, then the two epilogue rings
  constexpr int kOpBytes = Cfg::STAGES * Cfg::STAGE_BYTES + Cfg::BRES_BYTES + Cfg::EPI_BYTES;
  uint64_t* bars = (uint64_t*)(smem + kOpBytes);
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bres_base = smem_base + Cfg::STAGES * Cfg::STAGE_BYTES;
  const uint32_t full0 = smem_u32(bars), empty0 = full0 + 8 * Cfg::STAGES, bfull = empty0 + 8 * Cfg::STAGES;
  // epilogue ring of consumer c: slots at epi_off + c * EPI_SLOTS * EPI_SLOT, barriers efull0 / eempty0 + 8 * (c * EPI_SLOTS + s)
  constexpr int kEpiOff = Cfg::STAGES * Cfg::STAGE_BYTES + Cfg::BRES_BYTES;
  const uint32_t efull0 = bfull + 8 * kResK, eempty0 = efull0 + 16 * Cfg::EPI_SLOTS;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_n = (N + BN - 1) / BN;
  const int tiles_m = (M + kNtBM - 1) / kNtBM;
  const int nk = (K + kBK - 1) / kBK;
  // A CTA owns ONE column tile (n0 fixed: its B panel can stay resident) and walks the row tiles m_first, +m_stride, ..;
  // neighbouring CTAs work on the same row tile at the same time (A is read from HBM once, from L2 after that).
  // The host makes gridDim.x a multiple of tiles_n.
  const int n0 = (int)(blockIdx.x % tiles_n) * BN;
  const int m_first = (int)(blockIdx.x / tiles_n), m_stride = (int)(gridDim.x / tiles_n);
  const int n_tiles = m_first < tiles_m ? (tiles_m - m_first + m_stride - 1) / m_stride : 0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapAhi); tma_prefetch_desc(&mapBhi);
    if (NPROD == 3) { tma_prefetch_desc(&mapAlo); tma_prefetch_desc(&mapBlo); }
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, 1); }
    for (int kb = 0; kb < kResK; ++kb) mbar_init(bfull + 8 * kb, 1);     // one per k-block of the resident B panel
    if constexpr (kStaged > 0) {
      for (int i = 0; i < kStaged; ++i) tma_prefetch_desc(&emaps.m[i]);
      for (int s = 0; s < 2 * Cfg::EPI_SLOTS; ++s) { mbar_init(efull0 + 8 * s, 1); mbar_init(eempty0 + 8 * s, 4); }
    }
    if constexpr (RING) {
      for (int i = 0; i < EpiOut<Epi>::kN; ++i)
        if ((omask >> i) & 1u) tma_prefetch_desc(&omaps.m[i]);
    }
    fence_barrier_init();
  }
  __syncthreads();      // the last CTA-wide barrier: after the role split only mbarriers and named barriers 1, 2

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if constexpr (kStaged > 0) {
      if (threadIdx.x == 32 || threadIdx.x == 64) {      // epilogue operand loader of consumer warpgroup c
        const int c = warp - 1;
        pdl_wait();      // the stashes belong to predecessor kernels
        int q = 0;
        for (int j = c; j < n_tiles; j += 2) {
          const int m0 = (m_first + j * m_stride) * kNtBM;
#pragma unroll 1
          for (int b = 0; b < kEpiNB; ++b, ++q) {      // rolled: this warpgroup runs on 40 registers
            const int s = c * Cfg::EPI_SLOTS + q % Cfg::EPI_SLOTS;
            mbar_wait(eempty0 + 8 * s, ((q / Cfg::EPI_SLOTS) & 1) ^ 1);
            const uint32_t dst = smem_base + kEpiOff + s * Cfg::SLOT_BYTES;
            mbar_expect_tx(efull0 + 8 * s, (uint32_t)Cfg::SLOT_BYTES);     // out-of-bounds fill counts as well
#pragma unroll
            for (int i = 0; i < kStaged; ++i)
              tma_load_2d(dst + kNtBM * kEpiCols * Epi::Stage::before(i), &emaps.m[i], n0 + b * kEpiCols, m0, efull0 + 8 * s);
          }
        }
        return;
      }
    }
    if (threadIdx.x == 0) {
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
      int it = 0;
      AVC_PROBE(long long w_empty = 0; const long long t_tma0 = clock64());
      for (int mt = m_first; mt < tiles_m; mt += m_stride) {
        const int m0 = mt * kNtBM;
        for (int kb = 0; kb < nk; ++kb, ++it) {
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
      AVC_PROBE_ADD(EpiProbeId<Epi>::value, 1, clock64() - t_tma0);
      AVC_PROBE_ADD(EpiProbeId<Epi>::value, 7, 1);
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int c = (warp >> 2) - 1, wq = warp & 3;      // consumer warpgroup, warp within it
  const int tw = threadIdx.x & 127;
  const bool leader = tw == 0;
  const int row_in = 16 * wq + (lane >> 2) + 8 * (lane & 1), col_in = 4 * ((lane >> 1) & 1);
  pdl_wait();      // the functor's operands and outputs belong to predecessor kernels
  float acc[BN / 2];
  long long w_stage = 0, w_drain = 0;      // (probe build) waits on the epilogue ring, on the TMA stores' reads
  EpiRing ring{smem_base + kEpiOff + c * Cfg::EPI_SLOTS * Cfg::SLOT_BYTES, efull0 + 8 * c * Cfg::EPI_SLOTS,
               eempty0 + 8 * c * Cfg::EPI_SLOTS, 0, row_in, col_in, 0, n0, wq, omask};
  AVC_PROBE(long long w_full = 0, w_turn = 0, t_mma = 0, t_epi = 0; const long long t_loop0 = clock64());
  for (int j = c; j < n_tiles; j += 2) {
    const int m0 = (m_first + j * m_stride) * kNtBM;
    AVC_PROBE(const long long t_turn0 = clock64());
    if (j > 0) named_bar_sync(kNtTurnBar + c, 256);      // the other warpgroup has issued tile j - 1
    AVC_PROBE(const long long t_mma0 = clock64(); w_turn += t_mma0 - t_turn0);
    int prev = -1, last = 0;
    for (int kb = 0; kb < nk; ++kb) {
      const int it = j * nk + kb, s = it % Cfg::STAGES;
      if (RESB && j < 2) mbar_wait(bfull + 8 * kb, 0);      // this k-block of the B panel has landed (first tile only)
      AVC_PROBE_WAIT(w_full, full0 + 8 * s, (it / Cfg::STAGES) & 1);
      const uint32_t a_hi = smem_base + s * Cfg::STAGE_BYTES;
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
      last = s;
      if (kb + 1 < nk) {
        wgmma_wait<1>();                      // the previous k-block's MMAs are done: its stage can be refilled
        if (prev >= 0 && leader) mbar_arrive(empty0 + 8 * prev);
        prev = s;
      }
    }
    if (j + 1 < n_tiles) named_bar_arrive(kNtTurnBar + (c ^ 1), 256);      // all k-blocks issued: the other's turn
    ring.q0 = (j >> 1) * kEpiNB;
    ring.m0 = m0;
    epilogue_nt<BN, Cfg::EPI_SLOTS, RING>(epi, acc, m0 + row_in, n0 + col_in, M, N, lane, [&] {
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (leader) {
        if (prev >= 0) mbar_arrive(empty0 + 8 * prev);
        mbar_arrive(empty0 + 8 * last);
      }
      AVC_PROBE(t_mma += clock64() - t_mma0);
    }, ring, omaps, w_stage, w_drain);
    AVC_PROBE(t_epi += clock64() - t_mma0);
  }
  if constexpr (RING) {
    if (lane == 0) bulk_wait_all();      // the outputs are written before the CTA exits (and its shared memory goes)
  }
  (void)w_stage; (void)w_drain;
  AVC_PROBE(if (leader) {
    AVC_PROBE_ADD(EpiProbeId<Epi>::value, 8, w_stage);
    AVC_PROBE_ADD(EpiProbeId<Epi>::value, 9, w_drain);
    AVC_PROBE_ADD(EpiProbeId<Epi>::value, 2, w_full);
    AVC_PROBE_ADD(EpiProbeId<Epi>::value, 3, w_turn);
    AVC_PROBE_ADD(EpiProbeId<Epi>::value, 4, t_mma);
    AVC_PROBE_ADD(EpiProbeId<Epi>::value, 5, t_epi - t_mma);
    AVC_PROBE_ADD(EpiProbeId<Epi>::value, 6, clock64() - t_loop0);
  })
}

// 1: the last NT launch of this host thread stored its outputs through the ring, 0: from registers (read by the tests)
inline thread_local int g_nt_last_ring = -1;
// Test hooks (avc_tc_nt_set_max_ctas, avc_tc_nt_last_grid): a cap on the persistent grid of this host thread's NT
// launches (0: none), so that a small launch walks many row tiles per CTA, and the grid of its last NT launch (-1: none)
inline thread_local int g_nt_max_ctas = 0;
inline thread_local int g_nt_last_grid = -1;

template <int BN, int NPROD, bool RESB, typename Epi, bool RING>
static inline int launch_gemm_tc_nt_kern(cudaStream_t st, int64_t M, int N, int K, const CUtensorMap (&mab)[4],
                                         const Epi& epi, bool b_const, const EpiMaps<EpiStage<Epi>::kN>& emaps,
                                         const EpiOutMaps<EpiOut<Epi>::kN>& omaps, uint32_t omask) {
  using Cfg = TcCfg<BN, NPROD, RESB, RING ? EpiOut<Epi>::kSlotBytes : 0>;
  auto kern = gemm_tc_nt_kernel<BN, NPROD, RESB, Epi, RING>;
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
  const int ntiles = ceil_div(M, kNtBM) * tiles_n;
  int g = ntiles < num_sms ? ntiles : num_sms;         // persistent: at most one CTA per SM ...
  g = (g / tiles_n) * tiles_n;                         // ... and a whole number of CTAs per column tile
  if (g < tiles_n) return AVC_E_BADCFG;
  if (g_nt_max_ctas > 0) {                             // the test cap, in whole CTAs per column tile, at least one
    const int cap = g_nt_max_ctas / tiles_n > 1 ? g_nt_max_ctas / tiles_n * tiles_n : tiles_n;
    g = cap < g ? cap : g;
  }
  g_nt_last_grid = g;
  dim3 grid(g);
  AVC_CUDA_TRY(launch_pdl(kern, dim3(grid), dim3(kNtThreads), (size_t)Cfg::SMEM_BYTES, st, mab[0], mab[1], mab[2], mab[3],
                          (int)M, N, K, epi, b_const ? 1 : 0, emaps, omaps, omask));
  AVC_LAUNCH_TRY();
  return 0;
}

template <int BN, int NPROD, bool RESB, typename Epi>
static inline int launch_gemm_tc_nt_bn(cudaStream_t st, int64_t M, int N, int K, const SplitPtr& A, const SplitPtr& B,
                                       const Epi& epi, bool b_const) {
  EpiMaps<EpiStage<Epi>::kN> emaps;
  if constexpr (EpiStage<Epi>::kN > 0) {
    for (int i = 0; i < EpiStage<Epi>::kN; ++i) {
      const StageOp op = epi.stage_op(i);
      if (!op.base) return AVC_E_BADCFG;
      AVC_TRY(make_map_rows_cached(&emaps.m[i], Epi::Stage::es(i), op.base, (uint64_t)M, (uint64_t)op.cols,
                                   (uint64_t)op.ld, EpiBatch<Epi>::kCols, kNtBM));
    }
  }
  EpiOutMaps<EpiOut<Epi>::kN> omaps{};
  uint32_t omask = 0;
  bool ring = false;
  constexpr bool kStaged = EpiStage<Epi>::kN > 0;
  if constexpr (EpiOut<Epi>::kN > 0) {
    ring = true;
    for (int i = 0; i < EpiOut<Epi>::kN; ++i) {
      const OutOp op = epi.out_op(i, N);
      if (!op.base) continue;
      const int es = Epi::Out::es(i);      // TMA addresses whole 16 bytes: base, row pitch and extent
      if (((uintptr_t)op.base & 15u) || (op.ld * es) % 16 || (op.cols * es) % 16) {
        if (kStaged) return AVC_E_BADCFG;      // staged functors have no register stores
        ring = false;
        break;
      }
      AVC_TRY(make_map_rows_cached(&omaps.m[i], Epi::Out::es(i), op.base, (uint64_t)M, (uint64_t)op.cols,
                                   (uint64_t)op.ld, OutLayout<Epi>::cols(i), 16));      // one warp's box
      omask |= 1u << i;
    }
    if constexpr (kStaged) {      // outputs written in place over the staged operands must not overlap each other
      static_assert(OutLayout<Epi>::fits(), "the outputs do not fit over the staged operands");
      for (int i = 0; i < EpiOut<Epi>::kN; ++i)
        for (int j = i + 1; j < EpiOut<Epi>::kN; ++j)
          if (((omask >> i) & (omask >> j) & 1u) && OutLayout<Epi>::overlap(i, j)) return AVC_E_BADCFG;
    }
  }
  static_assert(!kStaged || EpiOut<Epi>::kN > 0, "a staged functor ring-stores its outputs");
  CUtensorMap mab[4];
  AVC_TRY(make_map_bf16_cached(&mab[0], A.hi, (uint64_t)M, (uint64_t)K, (uint64_t)A.ld, kBK, kNtBM));
  AVC_TRY(make_map_bf16_cached(&mab[2], B.hi, (uint64_t)N, (uint64_t)K, (uint64_t)B.ld, kBK, BN));
  if (NPROD == 3) {
    AVC_TRY(make_map_bf16_cached(&mab[1], A.lo, (uint64_t)M, (uint64_t)K, (uint64_t)A.ld, kBK, kNtBM));
    AVC_TRY(make_map_bf16_cached(&mab[3], B.lo, (uint64_t)N, (uint64_t)K, (uint64_t)B.ld, kBK, BN));
  } else {
    mab[1] = mab[0]; mab[3] = mab[2];
  }
  g_nt_last_ring = ring ? 1 : 0;
  if constexpr (kStaged) {
    return launch_gemm_tc_nt_kern<BN, NPROD, RESB, Epi, true>(st, M, N, K, mab, epi, b_const, emaps, omaps, omask);
  } else {
    if constexpr (EpiOut<Epi>::kN > 0) {
      if (ring) return launch_gemm_tc_nt_kern<BN, NPROD, RESB, Epi, true>(st, M, N, K, mab, epi, b_const, emaps, omaps, omask);
    }
    return launch_gemm_tc_nt_kern<BN, NPROD, RESB, Epi, false>(st, M, N, K, mab, epi, b_const, emaps, omaps, 0);
  }
}

// N <= 64 -> one 64-wide tile, else 128-wide tiles (a 65536-row GEMM then has 1024 tiles = 7.8 waves over 132
// persistent CTAs instead of 3.9 with 256-wide tiles: a smaller tail).
template <int NPROD, typename Epi>
static inline int launch_gemm_tc_nt(cudaStream_t st, int64_t M, int N, int K, const SplitPtr& A, const SplitPtr& B,
                                    const Epi& epi, bool b_const = false) {
  if (M <= 0 || N <= 0) return 0;
  // K <= 256: the B panel stays resident in shared memory (RESB); longer reductions stream both operands.
  if (K <= kResK * kBK) {
    if (N <= 64) return launch_gemm_tc_nt_bn<64, NPROD, true, Epi>(st, M, N, K, A, B, epi, b_const);
    return launch_gemm_tc_nt_bn<128, NPROD, true, Epi>(st, M, N, K, A, B, epi, b_const);
  }
  if (N <= 64) return launch_gemm_tc_nt_bn<64, NPROD, false, Epi>(st, M, N, K, A, B, epi, b_const);
  return launch_gemm_tc_nt_bn<128, NPROD, false, Epi>(st, M, N, K, A, B, epi, b_const);
}

// ------------------------------------------------------------------------------------------------ TN kernel
// C[i*ldc + j] += sum_{p in slice} A[p,i] * B[p,j]   (i < N1, j < N2): weight gradients.  Both operands are read
// "MN-major": the reduction index p is the row of the global arrays.  TMA boxes are 64 (i or j) x kTnBK = 32 (p); in
// shared memory one box is an MN block [32 p][128 B] (SWIZZLE_128B); a 128-wide M tile is 2 blocks (one per consumer
// warpgroup), a BN-wide N tile BN/64 blocks.  Descriptor: LBO = 4096 B (next 64-wide block), SBO = 1024 B (8 p-rows), a K
// step of 16 p-rows is +2048 B, two K steps per stage.  Split over p across blockIdx.z; partial tiles meet in fp32
// red.global.add, two columns per reduction where the host found C and ldc 8-byte aligned (red_v2): that halves the
// flush, 4.2 M scalar reductions for a 256 x 256 output split 64 ways.
// A stage is 32 p-rows rather than kBK = 64: at BN = 256 with split operands a 64-row stage is 96 KB and only two fit, and
// as a consumer frees a stage only after it has issued the next one's MMAs, a single load was in flight; 48 KB stages
// give four, and two or three loads stay in flight.
constexpr int kTnBK = 32;
template <int BN, int NPROD>
struct TcTnCfg {
  static constexpr int BLK = kTnBK * 128;                           // one 64-wide x 32-row bf16 block: 4 KB
  static constexpr int A_BYTES = (kBM / 64) * BLK;                  // 8 KB
  static constexpr int B_BYTES = (BN / 64) * BLK;
  static constexpr int NOP = (NPROD == 3) ? 2 : 1;
  static constexpr int STAGE_BYTES = NOP * (A_BYTES + B_BYTES);
  static constexpr int kBudget = kSmemMax - 1024 /*align*/ - 1024 /*ones*/ - 256 /*barriers*/;
  static constexpr int STAGES = kBudget / STAGE_BYTES >= 8 ? 8 : kBudget / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 1024 + 256;
  static_assert(SMEM_BYTES <= kSmemMax, "exceeds the 227 KB of shared memory per CTA");
  static_assert(STAGES >= 4, "tile too large for a four-stage ring");
  static_assert(16 * STAGES <= 256, "mbarriers overflow their area");
};

template <int BN, int NPROD>
__global__ void __launch_bounds__(kTcThreads, 1)
gemm_tc_tn_kernel(const __grid_constant__ CUtensorMap mapAhi, const __grid_constant__ CUtensorMap mapAlo,
                  const __grid_constant__ CUtensorMap mapBhi, const __grid_constant__ CUtensorMap mapBlo,
                  int P, int N1, int N2, int rows_per_split, float* __restrict__ C, int ldc,
                  float* __restrict__ colsum /* += sum_p A[p,i]; nullptr: off */, int red_v2) {
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
  const int nk = (p_end - p_begin + kTnBK - 1) / kTnBK;     // host guarantees rows_per_split % 64 == 0 and nk >= 1

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
        const int p0 = p_begin + kb * kTnBK;
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
        for (int k4 = 0; k4 < kTnBK / 16; ++k4) {
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
      const int c = j0 + 8 * j + 2 * (lane & 3);      // even: with red_v2, C + r * ldc + c is 8-byte aligned
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h;
        float* q = C + (size_t)r * ldc + c;
        if (r < N1) {
          if (red_v2 && c + 1 < N2) {
            red_add_v2(q, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          } else {
            if (c < N2) atomicAdd(q, acc[4 * j + 2 * h]);
            if (c + 1 < N2) atomicAdd(q + 1, acc[4 * j + 2 * h + 1]);
          }
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
  AVC_TRY(make_map_bf16_cached(&mAh, A.hi, (uint64_t)P, (uint64_t)N1, (uint64_t)A.ld, 64, kTnBK));
  AVC_TRY(make_map_bf16_cached(&mBh, B.hi, (uint64_t)P, (uint64_t)N2, (uint64_t)B.ld, 64, kTnBK));
  if (NPROD == 3) {
    AVC_TRY(make_map_bf16_cached(&mAl, A.lo, (uint64_t)P, (uint64_t)N1, (uint64_t)A.ld, 64, kTnBK));
    AVC_TRY(make_map_bf16_cached(&mBl, B.lo, (uint64_t)P, (uint64_t)N2, (uint64_t)B.ld, 64, kTnBK));
  } else {
    mAl = mAh; mBl = mBh;
  }
  // 8-byte reductions when every even column of C starts on 8 bytes
  const int red_v2 = ((uintptr_t)C & 7u) == 0 && ldc % 2 == 0;
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
    AVC_CUDA_TRY(launch_pdl(kern, grid, dim3(kTcThreads), (size_t)smem, st, mAh, mAl, mBh, mBl, (int)P, N1, N2, rows, C, ldc,
                            colsum, red_v2));
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
