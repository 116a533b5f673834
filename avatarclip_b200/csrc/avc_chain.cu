// avc_chain.cu -- the SDF value chain (models/fields.py:72-88: embed -> [Linear -> Softplus] x L -> sdf head) of a tile
// of 128 points as ONE kernel: the layer's activations never leave the SM.
//
// Used by the sample-placement passes of NeuSRenderer.render (renderer.py:336-352: coarse SDF + the up-sampling rounds,
// under no_grad) and by SDFNetwork.sdf queries (extract_fields / validate_mesh) -- everywhere the chain runs without a
// stash for the backward.  Per CTA (persistent, one per SM, tiles of 128 points):
//
//   shared memory   A: the current layer's input as a two-term bf16 split, K-major SWIZZLE_128B, 4 k-blocks x (hi, lo)
//                      x 16 KB = 128 KB -- written in place by the epilogue of the previous layer (layer 0: by TMA);
//                   W: 3-stage ring of 32 KB slabs ([256 rows][64 k] of W_l hi or lo, rows >= N zero-filled by TMA),
//                      streamed by TMA from L2 (the whole 1.6-3.2 MB model is L2 resident), running ahead across layers
//                      and tiles
//   warps 0-7       two consumer warpgroups, warpgroup g owning points [64 g, 64 g + 64) of the tile: wgmma m64n256k16
//                   (hi*hi + lo*hi on the W_hi slab, hi*lo on the W_lo slab) into a 64 x 256 fp32 register accumulator,
//                   then the epilogue from that fragment: bias + softplus_100 (SFU) + 1/sqrt(2) skip scaling, bf16
//                   (hi, lo) split, st.shared into the swizzled A tile of the NEXT layer (its own 64 rows only: the two
//                   warpgroups never wait for each other); the last hidden layer instead folds its columns into the sdf
//                   head (fp32 dot with row 0 of the last linear, reduced over the 4 lanes that share a row)
//   warps 8-11      TMA producer (one thread), registers handed to the consumers with setmaxnreg
//
// HBM traffic per point: 160 B in (the encoded pair) + 4 B out, against 2 x 1 KB per layer and direction for the
// unfused launches (8 launches per pass); L2 -> SM: 256 KB of weights per layer and 128-point tile.
// Synchronisation: wfull/wempty (W ring; one empty arrival per warpgroup), a0full (TMA tile input), afree (both
// warpgroups' last-layer MMAs are done: the A buffer may take the next tile's input).
#include <cuda.h>

#include <cstdlib>

#include "avc_chain.h"
#include "avc_gemm_tc.cuh"

namespace avc {
namespace chain {

using namespace avc::tc;

constexpr int kCM = 128;
constexpr int kASlab = kCM * 128;                 // [128 rows][64 bf16]: 16 KB
constexpr int kAKB = 4;                           // K <= 256
constexpr int kABytes = kAKB * 2 * kASlab;        // 131072
constexpr int kWRows = 256;                       // the MMA is always 256 wide; rows >= N of a slab are zeros
constexpr int kWSlab = kWRows * 128;              // [256 rows][64 bf16]: 32 KB
constexpr int kWStages = 3;
// a whole producer warpgroup (one thread issues the TMA): setmaxnreg works per warpgroup, and the consumers need the
// registers it gives up (a 64 x 256 fp32 accumulator is 128 registers per thread)
constexpr int kThreads = kConsumerThreads + 128;
constexpr int kBarBytes = 256;
constexpr int kSmemBytes = 1024 + kABytes + kWStages * kWSlab + kBarBytes;
static_assert(kSmemBytes <= kSmemMax, "exceeds the 227 KB of shared memory per CTA");

struct DevLayer {
  int N, K, nkb;
  const float* bias;
  float oscale;
  int next_skip_cols;
};
struct DevArgs {
  int L;
  DevLayer lay[kMaxHidden];
  const __nv_bfloat16* skip_hi;
  const __nv_bfloat16* skip_lo;
  int skip_ld, skip_col0;
  const float* w_sdf;
  const float* b_sdf;
  int head_skip_cols;
  float inv_scale;
  float* sdf_out;
  int nz, pitch;
  long long P;
  int tiles;
  long long* dbg;     // profiling aid (AVC_CHAIN_DEBUG=1): cycle counters of block 0, see launch()
};
struct Maps {
  CUtensorMap a0hi, a0lo;
  CUtensorMap whi[kMaxHidden], wlo[kMaxHidden];
};

__device__ __forceinline__ void st_shared_b16(uint32_t addr, uint16_t v) {
  asm volatile("st.shared.b16 [%0], %1;" ::"r"(addr), "h"(v) : "memory");
}
__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// byte offset of element (row, col) in the A buffer's hi slab (the lo slab is kASlab further)
__device__ __forceinline__ uint32_t a_offset(int row, int col) {
  return (uint32_t)((col >> 6) * 2) * kASlab + (uint32_t)((row >> 3) * 1024 + (row & 7) * 128) +
         (((uint32_t)((col & 63) >> 3) ^ (uint32_t)(row & 7)) << 4) + (uint32_t)(col & 7) * 2u;
}

__global__ void __launch_bounds__(kThreads, 1)
k_sdf_chain(const __grid_constant__ Maps maps, const __grid_constant__ DevArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const uint32_t sA = smem_u32(smem);
  const uint32_t sW = sA + kABytes;
  uint64_t* bars = (uint64_t*)(smem + kABytes + kWStages * kWSlab);
  const uint32_t wfull0 = smem_u32(bars), wempty0 = wfull0 + 8 * kWStages, a0full = wempty0 + 8 * kWStages,
                 afree = a0full + 8;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int L = a.L;

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&maps.a0hi); tma_prefetch_desc(&maps.a0lo);
    for (int s = 0; s < kWStages; ++s) { mbar_init(wfull0 + 8 * s, 1); mbar_init(wempty0 + 8 * s, 2); }
    mbar_init(a0full, 1);
    mbar_init(afree, 2);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kProducerWarp) {
    // ------------------------------------------------------------------------------------------ TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == kProducerWarp && lane == 0) {
      int it = 0, lt = 0;
      pdl_wait();            // the encoded points are the predecessor kernel's output (launched with launch_pdl: this
      pdl_trigger();         // CTA's set-up ran while that kernel was still draining)
      const int nkb0 = a.lay[0].nkb;
      for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x, ++lt) {
        // the A buffer is free for the next tile's input once both warpgroups' last-layer MMAs of the previous tile are done
        if (lt > 0) mbar_wait(afree, (uint32_t)((lt - 1) & 1));
        mbar_expect_tx(a0full, (uint32_t)(nkb0 * 2 * kASlab));
        for (int kb = 0; kb < nkb0; ++kb) {
          tma_load_2d(sA + (uint32_t)(kb * 2) * kASlab, &maps.a0hi, kb * 64, tile * kCM, a0full);
          tma_load_2d(sA + (uint32_t)(kb * 2 + 1) * kASlab, &maps.a0lo, kb * 64, tile * kCM, a0full);
        }
        for (int l = 0; l < L; ++l) {
          for (int kb = 0; kb < a.lay[l].nkb; ++kb)
            for (int h = 0; h < 2; ++h, ++it) {
              const int s = it % kWStages;
              mbar_wait(wempty0 + 8 * s, ((it / kWStages) & 1) ^ 1);
              mbar_expect_tx(wfull0 + 8 * s, (uint32_t)kWSlab);
              tma_load_2d(sW + s * kWSlab, h == 0 ? &maps.whi[l] : &maps.wlo[l], kb * 64, 0, wfull0 + 8 * s);
            }
        }
      }
    }
    return;
  }
  // ------------------------------------------------------------------------------------------ consumer warpgroups
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int g = warp >> 2, wq = warp & 3;
  const int tw = threadIdx.x & 127;
  const bool leader = tw == 0;
  const int row0 = 64 * g + 16 * wq + (lane >> 2);      // this thread's tile rows: row0 and row0 + 8
  const int cq = 2 * (lane & 3);                         // and columns 8 j + cq, + 1
  const bool prof = a.dbg != nullptr && blockIdx.x == 0 && threadIdx.x == 0;
  long long t_wa = 0, t_ww = 0, e_work = 0, t_all0 = prof ? clock64() : 0;
  pdl_wait();                             // skip-concat columns in, sdf out: predecessor kernels' buffers
  float acc[128];
  int it = 0, lt = 0;
  for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x, ++lt) {
    for (int l = 0; l < L; ++l) {
      const DevLayer& ly = a.lay[l];
      const bool last = (l == L - 1);
      long long t0 = prof ? clock64() : 0;
      if (l == 0) mbar_wait(a0full, (uint32_t)(lt & 1));
      if (prof) t_wa += clock64() - t0;
      int prev = -1;
      for (int kb = 0; kb < ly.nkb; ++kb)
        for (int h = 0; h < 2; ++h, ++it) {
          const int s = it % kWStages;
          long long t1 = prof ? clock64() : 0;
          mbar_wait(wfull0 + 8 * s, (uint32_t)((it / kWStages) & 1));
          if (prof) t_ww += clock64() - t1;
          const uint64_t da_hi = make_wgmma_desc(sA + (uint32_t)(kb * 2) * kASlab + (uint32_t)g * 8192u, 16, 1024);
          const uint64_t da_lo = make_wgmma_desc(sA + (uint32_t)(kb * 2 + 1) * kASlab + (uint32_t)g * 8192u, 16, 1024);
          const uint64_t db = make_wgmma_desc(sW + s * kWSlab, 16, 1024);
          wgmma_fence_acc(acc);
          wgmma_fence();
          if (h == 0) {
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4) {
              wgmma_bf16<256, 0, 0>(acc, da_hi + 2 * k4, db + 2 * k4, (kb | k4) ? 1u : 0u);
              wgmma_bf16<256, 0, 0>(acc, da_lo + 2 * k4, db + 2 * k4, 1u);
            }
          } else {
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4) wgmma_bf16<256, 0, 0>(acc, da_hi + 2 * k4, db + 2 * k4, 1u);
          }
          wgmma_commit();
          wgmma_fence_acc(acc);
          wgmma_wait<1>();
          if (prev >= 0 && leader) mbar_arrive(wempty0 + 8 * prev);
          prev = s;
        }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (leader) mbar_arrive(wempty0 + 8 * prev);
      if (last && leader) mbar_arrive(afree);       // this warpgroup no longer reads the A buffer in this tile
      // every warp of the warpgroup is past its MMAs before anyone overwrites the A rows they read
      named_bar_sync(1 + g, 128);
      const long long e1 = prof ? clock64() : 0;
      // branch-free: 4 values per 8-column group (two rows x two columns), bias pairs loaded one group ahead, columns
      // >= N zeroed by a select
      float dot0 = 0.f, dot1 = 0.f;
      auto load_b = [&](int c) {
        return make_float2(c < ly.N ? __ldg(ly.bias + c) : 0.f, c + 1 < ly.N ? __ldg(ly.bias + c + 1) : 0.f);
      };
      float2 bnext = load_b(cq);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int c = 8 * j + cq;
        const float2 b = bnext;
        if (j < 31) bnext = load_b(c + 8);
        const float bb[2] = {b.x, b.y};
        float hv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float z = acc[4 * j + i] + bb[i & 1];
          const float bz = z * kBeta;
          const float sp = __logf(1.0f + __expf(bz)) * (1.0f / kBeta);
          const float hh = (bz > kThresh ? z : sp) * ly.oscale;
          hv[i] = (c + (i & 1) < ly.N) ? hh : 0.f;
        }
        if (last) {
          if (c < ly.N) {
            const float w0 = __ldg(a.w_sdf + c), w1 = c + 1 < ly.N ? __ldg(a.w_sdf + c + 1) : 0.f;
            dot0 = fmaf(hv[0], w0, fmaf(hv[1], w1, dot0));
            dot1 = fmaf(hv[2], w0, fmaf(hv[3], w1, dot1));
          }
        } else {
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const float* v = hv + 2 * rr;
            const uint32_t hp = bf16x2_bits(v[0], v[1]);
            const uint32_t lp = bf16x2_bits(v[0] - __uint_as_float(hp << 16), v[1] - __uint_as_float(hp & 0xffff0000u));
            const uint32_t o = sA + a_offset(row0 + 8 * rr, c);
            st_shared_b32(o, hp);
            st_shared_b32(o + kASlab, lp);
          }
        }
      }
      if (!last) {
        if (ly.next_skip_cols > 0) {
          // cat([h, enc]) / sqrt(2): the enc / sqrt(2) columns come from the pair k_encode_* wrote for this layer.  They
          // overwrite zeros other threads of the warpgroup wrote above: wait for those first.
          named_bar_sync(1 + g, 128);
          const int E = ly.next_skip_cols;
          for (int e = tw; e < 64 * E; e += 128) {
            const int rr = 64 * g + e / E, c = ly.N + (e % E);
            const long long pp = (long long)tile * kCM + rr;
            uint16_t vh = 0, vl = 0;
            if (pp < a.P) {
              const size_t o = (size_t)pp * a.skip_ld + a.skip_col0 + (c - ly.N);
              vh = reinterpret_cast<const uint16_t*>(a.skip_hi)[o];
              vl = reinterpret_cast<const uint16_t*>(a.skip_lo)[o];
            }
            const uint32_t base = sA + a_offset(rr, c);
            st_shared_b16(base, vh);
            st_shared_b16(base + kASlab, vl);
          }
        }
        fence_proxy_async();            // generic-proxy smem writes -> visible to the tensor core (async proxy)
        named_bar_sync(1 + g, 128);     // the whole next A (this warpgroup's rows) is written before its MMAs
      } else {
        // sdf head: the 4 lanes of a row hold interleaved column pairs; their partial dots meet in a FIXED butterfly, so
        // the result does not depend on scheduling (sample placement is discontinuous in the sdf: bit-stable runs)
        dot0 += __shfl_xor_sync(0xffffffffu, dot0, 1);
        dot1 += __shfl_xor_sync(0xffffffffu, dot1, 1);
        dot0 += __shfl_xor_sync(0xffffffffu, dot0, 2);
        dot1 += __shfl_xor_sync(0xffffffffu, dot1, 2);
        if ((lane & 3) == 0) {
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const long long p = (long long)tile * kCM + row0 + 8 * rr;
            if (p < a.P) {
              float s = rr == 0 ? dot0 : dot1;
              for (int c = 0; c < a.head_skip_cols; ++c) {      // head takes the skip concat itself (skip_in has n_layers)
                const size_t o = (size_t)p * a.skip_ld + a.skip_col0 + c;
                s = fmaf(__bfloat162float(a.skip_hi[o]) + __bfloat162float(a.skip_lo[o]), __ldg(a.w_sdf + ly.N + c), s);
              }
              const long long o = a.nz > 0 ? (p / a.nz) * a.pitch + (p % a.nz) : p;
              a.sdf_out[o] = (s + __ldg(a.b_sdf)) * a.inv_scale;
            }
          }
        }
      }
      if (prof) e_work += clock64() - e1;
    }
  }
  if (prof) { a.dbg[0] = t_wa; a.dbg[1] = t_ww; a.dbg[2] = clock64() - t_all0; a.dbg[3] = (long long)lt * L; a.dbg[5] = e_work; }
}

static long long* g_dbg = nullptr;

bool supported(const Args& a) {
  if (a.L < 1 || a.L > kMaxHidden) return false;
  for (int l = 0; l < a.L; ++l) {
    const Layer& y = a.lay[l];
    if (y.N < 1 || y.N > 256 || y.K < 1 || y.K > 256 || (y.ldw % 8) != 0) return false;
    if (l + 1 < a.L && y.N + y.next_skip_cols != a.lay[l + 1].K) return false;
  }
  if (a.lay[a.L - 1].N + a.head_skip_cols != a.K_head) return false;
  if (a.ld0 % 8) return false;
  return true;
}

int launch(const Args& a, cudaStream_t st) {
  if (a.P <= 0) return 0;
  if (!supported(a)) return AVC_E_BADCFG;
  Maps m;
  DevArgs d;
  d.L = a.L;
  AVC_TRY(make_map_bf16_cached(&m.a0hi, a.a0_hi, (uint64_t)a.P, (uint64_t)a.lay[0].K, (uint64_t)a.ld0, 64, kCM));
  AVC_TRY(make_map_bf16_cached(&m.a0lo, a.a0_lo, (uint64_t)a.P, (uint64_t)a.lay[0].K, (uint64_t)a.ld0, 64, kCM));
  for (int l = 0; l < a.L; ++l) {
    const Layer& y = a.lay[l];
    DevLayer& o = d.lay[l];
    o.N = y.N; o.K = y.K; o.nkb = (y.K + 63) / 64;
    o.bias = y.bias; o.oscale = y.oscale; o.next_skip_cols = y.next_skip_cols;
    AVC_TRY(make_map_bf16_cached(&m.whi[l], y.w_hi, (uint64_t)y.N, (uint64_t)y.K, (uint64_t)y.ldw, 64, kWRows));
    AVC_TRY(make_map_bf16_cached(&m.wlo[l], y.w_lo, (uint64_t)y.N, (uint64_t)y.K, (uint64_t)y.ldw, 64, kWRows));
  }
  for (int l = a.L; l < kMaxHidden; ++l) { m.whi[l] = m.whi[0]; m.wlo[l] = m.wlo[0]; d.lay[l] = d.lay[0]; }
  d.skip_hi = a.skip_hi; d.skip_lo = a.skip_lo; d.skip_ld = a.skip_ld; d.skip_col0 = a.skip_col0;
  d.w_sdf = a.w_sdf; d.b_sdf = a.b_sdf; d.head_skip_cols = a.head_skip_cols;
  d.inv_scale = a.inv_scale; d.sdf_out = a.sdf_out; d.nz = a.nz; d.pitch = a.pitch; d.P = a.P;
  d.tiles = (int)((a.P + kCM - 1) / kCM);
  static thread_local bool attr_set = false;
  if (!attr_set) {
    AVC_CUDA_TRY(cudaFuncSetAttribute(k_sdf_chain, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    attr_set = true;
  }
  static thread_local int num_sms = 0;
  if (!num_sms) {
    int dev = 0;
    AVC_CUDA_TRY(cudaGetDevice(&dev));
    AVC_CUDA_TRY(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  const int grid = d.tiles < num_sms ? d.tiles : num_sms;
  d.dbg = nullptr;
  static long long* dbg_buf = nullptr;
  const char* dbg_env = getenv("AVC_CHAIN_DEBUG");      // profiling aid: cycle counters of block 0 -> avc_chain_debug_read
  if (dbg_env && atoi(dbg_env) == 1) {
    if (!dbg_buf) AVC_CUDA_TRY(cudaMalloc(&dbg_buf, 16 * sizeof(long long)));
    AVC_CUDA_TRY(cudaMemsetAsync(dbg_buf, 0, 16 * sizeof(long long), st));
    d.dbg = dbg_buf;
    g_dbg = dbg_buf;
  }
  AVC_CUDA_TRY(launch_pdl(k_sdf_chain, dim3(grid), dim3(kThreads), (size_t)kSmemBytes, st, m, d));
  AVC_LAUNCH_TRY();
  return 0;
}

// thread 0 of block 0: [0] waiting for the tile input (a0full), [1] waiting for weight slabs (wfull), [2] total,
// [3] tile-layers processed, [5] epilogue work
int debug_read(long long out[8]) {
  if (!g_dbg) return AVC_E_NULL;
  AVC_CUDA_TRY(cudaDeviceSynchronize());
  AVC_CUDA_TRY(cudaMemcpy(out, g_dbg, 8 * sizeof(long long), cudaMemcpyDeviceToHost));
  return 0;
}

}  // namespace chain
}  // namespace avc

extern "C" int avc_chain_debug_read(long long* out8) { return avc::chain::debug_read(out8); }
