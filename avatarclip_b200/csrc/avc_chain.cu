// avc_chain.cu -- the SDF value chain (models/fields.py:72-88: embed -> [Linear -> Softplus] x L -> sdf head) of a tile
// of 64 points as ONE kernel: the layer's activations never leave the SM.
//
// Used by the sample-placement passes of NeuSRenderer.render (renderer.py:336-352: coarse SDF + the up-sampling rounds,
// under no_grad) and by SDFNetwork.sdf queries (extract_fields / validate_mesh) -- everywhere the chain runs without a
// stash for the backward.  Persistent CTAs (at most one per SM) walk tiles of 64 points: tile t belongs to CTA
// t % gridDim.x, and a CTA's j-th tile to consumer warpgroup j % 2, so the tiles are dealt over every SM before any
// CTA's second warpgroup gets one.  Per CTA:
//
//   shared memory   A0, A1: consumer warpgroup g's current layer input as a two-term bf16 split, K-major SWIZZLE_128B,
//                      4 k-blocks x (hi, lo) x 8 KB = 64 KB each -- written in place by the warpgroup's epilogue of the
//                      previous layer (layer 0: by TMA)
//                   W: 3-stage ring of 32 KB slabs ([256 rows][64 k] of W_l hi or lo, rows >= N zero-filled by TMA),
//                      streamed by TMA from L2 (the whole 1.6-3.2 MB model is L2 resident), running ahead across layers
//                      and tiles
//   warps 0-7       two consumer warpgroups, each on its own tile: wgmma m64n256k16 (hi*hi + lo*hi on the W_hi slab,
//                   hi*lo on the W_lo slab) into a 64 x 256 fp32 register accumulator, then the epilogue from that
//                   fragment: bias + softplus_100 (SFU) + 1/sqrt(2) skip scaling, bf16 (hi, lo) split, st.shared into
//                   the swizzled A tile of the NEXT layer; the last hidden layer instead folds its columns into the sdf
//                   head (fp32 dot with row 0 of the last linear, reduced over the 4 lanes that share a row)
//   warps 8-11      producers, registers handed to the consumers with setmaxnreg: warp 8 streams the W ring, warps 9
//                   and 10 load the layer-0 tiles of consumer warpgroups 0 and 1 (one thread each)
//
// Ping-pong: the consumers take strict turns at issuing a layer's MMAs (named barriers kTurnBar + g).  A warpgroup
// passes the turn as soon as its last k-block is issued, then waits for its MMAs and runs the epilogue while the other
// warpgroup's MMAs keep the tensor pipe busy.  MMA steps of a tile pair (CTA tiles 2q, 2q + 1) run as
// (2q, layer 0), (2q + 1, layer 0), (2q, layer 1), ...; a last odd tile runs its layers alone.  The producer streams W_l
// once per step in that order (the second warpgroup's slabs are fetched from L2 again), so every ring stage is read by
// one warpgroup and released by it.  A row's MMAs, epilogue and head are those of the 64-row fragment of any other
// placement: the sdf bits do not depend on the tile, warpgroup, CTA or grid (sample placement is discontinuous in them).
//
// HBM traffic per point: 160 B in (the encoded pair) + 4 B out, against 2 x 1 KB per layer and direction for the
// unfused launches (8 launches per pass); L2 -> SM: 256 KB of weights per layer and 64-point tile.
// Synchronisation: wfull/wempty (W ring; one empty arrival, from the warpgroup that read the stage), a0full[g] (TMA
// tile input), afree[g] (warpgroup g's last-layer MMAs are done: its A buffer may take its next tile's input).
#include <cuda.h>

#include <cstdlib>

#include "avc_chain.h"
#include "avc_gemm_tc.cuh"

namespace avc {
namespace chain {

using namespace avc::tc;

constexpr int kCM = 64;                           // points per tile: one consumer warpgroup's wgmma M
constexpr int kASlab = kCM * 128;                 // [64 rows][64 bf16]: 8 KB
constexpr int kAKB = 4;                           // K <= 256
constexpr int kABytes = kAKB * 2 * kASlab;        // 65536 per consumer warpgroup
constexpr int kWRows = 256;                       // the MMA is always 256 wide; rows >= N of a slab are zeros
constexpr int kWSlab = kWRows * 128;              // [256 rows][64 bf16]: 32 KB
constexpr int kWStages = 3;
// a whole producer warpgroup: setmaxnreg works per warpgroup, and the consumers need the registers it gives up (a
// 64 x 256 fp32 accumulator is 128 registers per thread)
constexpr int kThreads = kConsumerThreads + 128;
constexpr int kBarBytes = 256;
constexpr int kSmemBytes = 1024 + 2 * kABytes + kWStages * kWSlab + kBarBytes;
static_assert(kSmemBytes <= kSmemMax, "exceeds the 227 KB of shared memory per CTA");
constexpr int kTurnBar = 3;       // named barrier kTurnBar + g: warpgroup g may issue its next MMAs (1 + g: in-warpgroup)

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
  long long* dbg;     // profiling aid (AVC_CHAIN_DEBUG=1): cycle counters of block 0, see debug_read()
};
struct Maps {
  CUtensorMap a0hi, a0lo;
  CUtensorMap whi[kMaxHidden], wlo[kMaxHidden];
};

__device__ __forceinline__ void st_shared_b16(uint32_t addr, uint16_t v) {
  asm volatile("st.shared.b16 [%0], %1;" ::"r"(addr), "h"(v) : "memory");
}
// st.shared without a memory clobber: the epilogue's stores into the A tile, ordered against its readers by the
// fence and named barrier that follow them, so the compiler may keep loads and values in registers across them
__device__ __forceinline__ void st_shared_b32_nc(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v));
}
// softplus_100's log branch, log(1 + exp(bz)) / 100, with the bits of __logf(1.0f + __expf(bz)) * (1.0f / kBeta):
// __expf is ex2.approx of bz * log2(e) and __logf lg2.approx times ln 2.  The flush-to-zero forms skip the denormal
// fix-ups: ex2 of an argument below -126 is below 2^-126, and 1 + it rounds to 1 either way; 1 + e >= 1 is never
// denormal.
__device__ __forceinline__ float softplus_tail(float bz) {
  float e, l;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(bz * 1.44269502162933349609f));
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(1.0f + e));
  return (l * 0.693147182464599609375f) * (1.0f / kBeta);
}
// byte offset of element (row, col) in a warpgroup's A buffer's hi slab (the lo slab is kASlab further)
__device__ __forceinline__ uint32_t a_offset(int row, int col) {
  return (uint32_t)((col >> 6) * 2) * kASlab + (uint32_t)((row >> 3) * 1024 + (row & 7) * 128) +
         (((uint32_t)((col & 63) >> 3) ^ (uint32_t)(row & 7)) << 4) + (uint32_t)(col & 7) * 2u;
}

// PROF: the profiling instantiation (AVC_CHAIN_DEBUG=1), see debug_read()
template <bool PROF>
__global__ void __launch_bounds__(kThreads, 1)
k_sdf_chain(const __grid_constant__ Maps maps, const __grid_constant__ DevArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const uint32_t sA0 = smem_u32(smem);
  const uint32_t sW = sA0 + 2 * kABytes;
  uint64_t* bars = (uint64_t*)(smem + 2 * kABytes + kWStages * kWSlab);
  const uint32_t wfull0 = smem_u32(bars), wempty0 = wfull0 + 8 * kWStages, a0full0 = wempty0 + 8 * kWStages,
                 afree0 = a0full0 + 16;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int L = a.L;
  // this CTA's tiles: blockIdx.x + j * gridDim.x, j < n_tiles
  const int n_tiles = (a.tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&maps.a0hi); tma_prefetch_desc(&maps.a0lo);
    for (int s = 0; s < kWStages; ++s) { mbar_init(wfull0 + 8 * s, 1); mbar_init(wempty0 + 8 * s, 1); }
    for (int g = 0; g < 2; ++g) { mbar_init(a0full0 + 8 * g, 1); mbar_init(afree0 + 8 * g, 1); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kProducerWarp) {
    // ------------------------------------------------------------------------------------------ TMA producers
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == kProducerWarp && lane == 0) {
      // the W ring, in the order of the MMA steps
      long long w_empty = 0;      // (profiling) waiting for a free stage
      pdl_wait();            // the encoded points are the predecessor kernel's output (launched with launch_pdl: this
      pdl_trigger();         // CTA's set-up ran while that kernel was still draining)
      int it = 0;
      for (int j = 0; j < n_tiles; j += 2) {
        const int duo = j + 1 < n_tiles ? 2 : 1;
        for (int l = 0; l < L; ++l)
          for (int w = 0; w < duo; ++w)
            for (int kb = 0; kb < a.lay[l].nkb; ++kb)
              for (int h = 0; h < 2; ++h, ++it) {
                const int s = it % kWStages;
                const long long t0 = PROF ? clock64() : 0;
                mbar_wait(wempty0 + 8 * s, ((it / kWStages) & 1) ^ 1);
                if (PROF) w_empty += clock64() - t0;
                mbar_expect_tx(wfull0 + 8 * s, (uint32_t)kWSlab);
                tma_load_2d(sW + s * kWSlab, h == 0 ? &maps.whi[l] : &maps.wlo[l], kb * 64, 0, wfull0 + 8 * s);
              }
      }
      if (PROF && blockIdx.x == 0) a.dbg[7] = w_empty;
    } else if ((warp == kProducerWarp + 1 || warp == kProducerWarp + 2) && lane == 0) {
      // the layer-0 input of consumer warpgroup g's tiles
      const int g = warp - kProducerWarp - 1;
      const uint32_t sA = sA0 + (uint32_t)g * kABytes, full = a0full0 + 8 * g;
      const int nkb0 = a.lay[0].nkb;
      pdl_wait();
      for (int j = g, lt = 0; j < n_tiles; j += 2, ++lt) {
        const int row = ((int)blockIdx.x + j * (int)gridDim.x) * kCM;
        if (lt > 0) mbar_wait(afree0 + 8 * g, (uint32_t)((lt - 1) & 1));      // the previous tile's MMAs are done
        mbar_expect_tx(full, (uint32_t)(nkb0 * 2 * kASlab));
        for (int kb = 0; kb < nkb0; ++kb) {
          tma_load_2d(sA + (uint32_t)(kb * 2) * kASlab, &maps.a0hi, kb * 64, row, full);
          tma_load_2d(sA + (uint32_t)(kb * 2 + 1) * kASlab, &maps.a0lo, kb * 64, row, full);
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
  const uint32_t sA = sA0 + (uint32_t)g * kABytes;
  const int row0 = 16 * wq + (lane >> 2);                // this thread's tile rows: row0 and row0 + 8
  const int cq = 2 * (lane & 3);                         // and columns 8 j + cq, + 1
  // profiling: thread 0 adds up cycles in shared memory, so that the counters hold no registers across the loop; lap(k)
  // adds the cycles since the previous lap to counter k
  const bool prof = PROF && threadIdx.x == 0;
  long long* sdbg = (long long*)(smem + 2 * kABytes + kWStages * kWSlab + 128);
  uint32_t tp = 0;
  auto lap = [&](int k) {
    if (prof) { const uint32_t t = (uint32_t)clock(); sdbg[k] += (long long)(t - tp); tp = t; }
  };
  if (prof) {
    for (int k = 0; k < 8; ++k) sdbg[k] = 0;
    tp = (uint32_t)clock();
  }
  pdl_wait();                             // skip-concat columns in, sdf out: predecessor kernels' buffers
  float acc[128];
  int it = 0, lt = 0;
  for (int j = g; j < n_tiles; j += 2, ++lt) {
    const long long tile = (long long)blockIdx.x + (long long)j * gridDim.x;
    const bool duo = (j | 1) < n_tiles;          // the other warpgroup has a tile of this pair: turns alternate
    for (int l = 0; l < L; ++l) {
      const DevLayer& ly = a.lay[l];
      const bool last = (l == L - 1);
      const int nsl = 2 * ly.nkb;                // ring slabs of one MMA step of layer l
      if (g == 1) it += nsl;                     // warpgroup 0's step of this layer came first
      lap(2);
      // the turn: every step but the CTA's first waits for the other warpgroup's previous step, except the layers
      // after the first of a last odd tile, whose previous step is its own
      if (duo ? (j | l) != 0 : (l == 0 && j > 0)) named_bar_sync(kTurnBar + g, 256);
      lap(4);
      if (l == 0) mbar_wait(a0full0 + 8 * g, (uint32_t)(lt & 1));
      lap(0);
      int prev = -1;
      for (int kb = 0; kb < ly.nkb; ++kb)
        for (int h = 0; h < 2; ++h, ++it) {
          const int s = it % kWStages;
          lap(6);
          mbar_wait(wfull0 + 8 * s, (uint32_t)((it / kWStages) & 1));
          lap(1);
          const uint64_t da_hi = make_wgmma_desc(sA + (uint32_t)(kb * 2) * kASlab, 16, 1024);
          const uint64_t da_lo = make_wgmma_desc(sA + (uint32_t)(kb * 2 + 1) * kASlab, 16, 1024);
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
      // all k-blocks issued: the other warpgroup's turn, unless this was the CTA's last step
      if (duo && !(g == 1 && last && j + 1 >= n_tiles)) named_bar_arrive(kTurnBar + (g ^ 1), 256);
      if (g == 0 && duo) it += nsl;              // warpgroup 1's step of this layer comes next
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (leader) mbar_arrive(wempty0 + 8 * prev);
      if (last && leader) mbar_arrive(afree0 + 8 * g);    // this warpgroup no longer reads its A buffer in this tile
      // every warp of the warpgroup is past its MMAs before anyone overwrites the A rows they read
      named_bar_sync(1 + g, 128);
      lap(6);
      // 4 values per 8-column group (two rows x two columns), bias pairs loaded one group ahead, columns >= N zeroed by
      // a select; one loop for the hidden layers, one for the head, so that no group branches.  The layer's fields are
      // read once: the stores below do not clobber memory for the compiler, so nothing is reloaded between groups.
      const int N = ly.N;
      const float osc = ly.oscale;
      const float* bias = ly.bias;
      auto load_b = [&](int c) {
        return make_float2(c < N ? __ldg(bias + c) : 0.f, c + 1 < N ? __ldg(bias + c + 1) : 0.f);
      };
      // the 4 values of group jc: z + bias -> softplus_100 -> skip scaling, columns >= N zeroed
      auto act = [&](int jc, float2 b, float (&hv)[4]) {
        const int c = 8 * jc + cq;
        const float bb[2] = {b.x, b.y};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float z = acc[4 * jc + i] + bb[i & 1];
          const float bz = z * kBeta;
          const float sp = softplus_tail(bz);
          const float hh = (bz > kThresh ? z : sp) * osc;
          hv[i] = (c + (i & 1) < N) ? hh : 0.f;
        }
      };
      float dot0 = 0.f, dot1 = 0.f;
      float2 bnext = load_b(cq);
      if (last) {
#pragma unroll
        for (int jc = 0; jc < 32; ++jc) {
          const int c = 8 * jc + cq;
          const float2 b = bnext;
          if (jc < 31) bnext = load_b(c + 8);
          float hv[4];
          act(jc, b, hv);
          if (c < N) {
            const float w0 = __ldg(a.w_sdf + c), w1 = c + 1 < N ? __ldg(a.w_sdf + c + 1) : 0.f;
            dot0 = fmaf(hv[0], w0, fmaf(hv[1], w1, dot0));
            dot1 = fmaf(hv[2], w0, fmaf(hv[3], w1, dot1));
          }
        }
      } else {
#pragma unroll
        for (int jc = 0; jc < 32; ++jc) {
          const int c = 8 * jc + cq;
          const float2 b = bnext;
          if (jc < 31) bnext = load_b(c + 8);
          float hv[4];
          act(jc, b, hv);
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const float* v = hv + 2 * rr;
            const uint32_t hp = bf16x2_bits(v[0], v[1]);
            const uint32_t lp = bf16x2_bits(v[0] - __uint_as_float(hp << 16), v[1] - __uint_as_float(hp & 0xffff0000u));
            const uint32_t o = sA + a_offset(row0 + 8 * rr, c);
            st_shared_b32_nc(o, hp);
            st_shared_b32_nc(o + kASlab, lp);
          }
        }
        if (ly.next_skip_cols > 0) {
          // cat([h, enc]) / sqrt(2): the enc / sqrt(2) columns come from the pair k_encode_* wrote for this layer.  They
          // overwrite zeros other threads of the warpgroup wrote above: wait for those first.
          named_bar_sync(1 + g, 128);
          const int E = ly.next_skip_cols;
          for (int e = tw; e < kCM * E; e += 128) {
            const int rr = e / E, c = N + (e % E);
            const long long pp = tile * kCM + rr;
            uint16_t vh = 0, vl = 0;
            if (pp < a.P) {
              const size_t o = (size_t)pp * a.skip_ld + a.skip_col0 + (c - N);
              vh = reinterpret_cast<const uint16_t*>(a.skip_hi)[o];
              vl = reinterpret_cast<const uint16_t*>(a.skip_lo)[o];
            }
            const uint32_t base = sA + a_offset(rr, c);
            st_shared_b16(base, vh);
            st_shared_b16(base + kASlab, vl);
          }
        }
        fence_proxy_async();            // generic-proxy smem writes -> visible to the tensor core (async proxy)
        named_bar_sync(1 + g, 128);     // the whole next A is written before this warpgroup's MMAs
      }
      if (last) {
        // sdf head: the 4 lanes of a row hold interleaved column pairs; their partial dots meet in a FIXED butterfly, so
        // the result does not depend on scheduling (sample placement is discontinuous in the sdf: bit-stable runs)
        dot0 += __shfl_xor_sync(0xffffffffu, dot0, 1);
        dot1 += __shfl_xor_sync(0xffffffffu, dot1, 1);
        dot0 += __shfl_xor_sync(0xffffffffu, dot0, 2);
        dot1 += __shfl_xor_sync(0xffffffffu, dot1, 2);
        if ((lane & 3) == 0) {
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const long long p = tile * kCM + row0 + 8 * rr;
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
      lap(5);
    }
  }
  if (prof && blockIdx.x == 0) {
    lap(2);
    // [2] collected the time outside the counted phases: the loop total is the sum of all of them
    sdbg[2] += sdbg[0] + sdbg[1] + sdbg[4] + sdbg[5] + sdbg[6];
    sdbg[3] = (long long)lt * L;
    for (int k = 0; k < 7; ++k) a.dbg[k] = sdbg[k];
  }
}

static long long* g_dbg = nullptr;
// Test hooks (avc_chain_set_max_ctas, avc_chain_last_grid): a cap on the persistent grid of this host thread's launches
// (0: none), so that a small launch walks many tiles per CTA on both warpgroups, and the grid of its last launch
static thread_local int g_max_ctas = 0;
static thread_local int g_last_grid = -1;

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
  const int64_t tiles = (a.P + kCM - 1) / kCM;
  if (tiles > INT32_MAX) return AVC_E_SIZE;
  d.tiles = (int)tiles;
  static thread_local bool attr_set = false;
  if (!attr_set) {
    AVC_CUDA_TRY(cudaFuncSetAttribute(k_sdf_chain<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    AVC_CUDA_TRY(cudaFuncSetAttribute(k_sdf_chain<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    attr_set = true;
  }
  static thread_local int num_sms = 0;
  if (!num_sms) {
    int dev = 0;
    AVC_CUDA_TRY(cudaGetDevice(&dev));
    AVC_CUDA_TRY(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  // one CTA per SM at most, and every CTA has a tile: a launch of up to num_sms tiles runs each on its own SM
  int grid = d.tiles < num_sms ? d.tiles : num_sms;
  if (g_max_ctas > 0 && g_max_ctas < grid) grid = g_max_ctas;
  g_last_grid = grid;
  d.dbg = nullptr;
  static long long* dbg_buf = nullptr;
  const char* dbg_env = getenv("AVC_CHAIN_DEBUG");      // profiling aid: cycle counters of block 0 -> avc_chain_debug_read
  if (dbg_env && atoi(dbg_env) == 1) {
    if (!dbg_buf) AVC_CUDA_TRY(cudaMalloc(&dbg_buf, 16 * sizeof(long long)));
    AVC_CUDA_TRY(cudaMemsetAsync(dbg_buf, 0, 16 * sizeof(long long), st));
    d.dbg = dbg_buf;
    g_dbg = dbg_buf;
  }
  AVC_CUDA_TRY(launch_pdl(d.dbg ? k_sdf_chain<true> : k_sdf_chain<false>, dim3(grid), dim3(kThreads), (size_t)kSmemBytes,
                          st, m, d));
  AVC_LAUNCH_TRY();
  return 0;
}

// block 0, consumer warpgroup 0 (thread 0): [0] waiting for its layer-0 input (a0full), [1] waiting for weight slabs
// (wfull), [2] total, [3] tile-layers processed, [4] waiting for the MMA turn, [5] epilogue work, [6] MMAs (turn taken
// to accumulator ready, [1] included); the W producer of block 0: [7] waiting for a free ring stage (wempty)
int debug_read(long long out[8]) {
  if (!g_dbg) return AVC_E_NULL;
  AVC_CUDA_TRY(cudaDeviceSynchronize());
  AVC_CUDA_TRY(cudaMemcpy(out, g_dbg, 8 * sizeof(long long), cudaMemcpyDeviceToHost));
  return 0;
}

}  // namespace chain
}  // namespace avc

extern "C" int avc_chain_debug_read(long long* out8) { return avc::chain::debug_read(out8); }

// Caps the persistent grid of the calling host thread's fused value-chain launches at n CTAs (0: no cap); returns the
// previous cap.
extern "C" int avc_chain_set_max_ctas(int32_t n) {
  const int prev = avc::chain::g_max_ctas;
  avc::chain::g_max_ctas = n > 0 ? n : 0;
  return prev;
}

// gridDim.x of the calling host thread's last fused value-chain launch, -1: none yet.
extern "C" int avc_chain_last_grid(void) { return avc::chain::g_last_grid; }
