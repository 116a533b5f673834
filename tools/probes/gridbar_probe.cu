// gridbar_probe.cu -- latency of grid-wide barrier variants on a cooperative launch (one 512-thread CTA per SM).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/probes/gridbar_probe tools/probes/gridbar_probe.cu
#include <cooperative_groups.h>
#include <cstdio>
#include <cuda_runtime.h>
namespace cg = cooperative_groups;

__device__ __forceinline__ unsigned ld_acq(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// (a) one counter: arrive with atomicAdd, poll the same word
__device__ void bar_single(unsigned* c, unsigned& gen) {
  __syncthreads();
  if (threadIdx.x == 0) {
    ++gen;
    __threadfence();
    atomicAdd(c, 1u);
    while (ld_acq(c) < gen * gridDim.x) {}
    __threadfence();
  }
  __syncthreads();
}
// (b) 8 leaf counters (128 B apart) + root counter + separate flag word that only the last arriver writes
__device__ void bar_tree(unsigned* base, unsigned& gen) {
  __syncthreads();
  if (threadIdx.x == 0) {
    ++gen;
    const unsigned G = 8, g = blockIdx.x % G;
    const unsigned members = gridDim.x / G + (g < gridDim.x % G ? 1 : 0);
    unsigned* leaf = base + 32 * (1 + g);
    unsigned* root = base + 32 * 10;
    unsigned* flag = base + 32 * 12;
    __threadfence();
    if (atomicAdd(leaf, 1u) + 1 == gen * members) {
      if (atomicAdd(root, 1u) + 1 == gen * G) { __threadfence(); atomicExch(flag, gen); }
    }
    while (ld_acq(flag) < gen) {}
    __threadfence();
  }
  __syncthreads();
}
// (c) red.release + polling with nanosleep-free ld.relaxed then one acquire fence
__device__ void bar_red(unsigned* c, unsigned& gen) {
  __syncthreads();
  if (threadIdx.x == 0) {
    ++gen;
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(c) : "memory");
    unsigned v;
    do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(c) : "memory"); } while (v < gen * gridDim.x);
    asm volatile("fence.acq_rel.gpu;" ::: "memory");
  }
  __syncthreads();
}

template <int MODE>
__global__ void __launch_bounds__(512, 1) k_probe(unsigned* bars, int iters, long long* cycles) {
  cg::grid_group grid = cg::this_grid();
  unsigned gen = 0;
  long long t0 = clock64();
  for (int i = 0; i < iters; ++i) {
    if (MODE == 0) bar_single(bars, gen);
    else if (MODE == 1) bar_tree(bars, gen);
    else if (MODE == 2) bar_red(bars, gen);
    else grid.sync();
  }
  long long t1 = clock64();
  if (blockIdx.x == 0 && threadIdx.x == 0) *cycles = t1 - t0;
}

template <int MODE>
float run(int grid, int iters, unsigned* bars, long long* cyc) {
  cudaMemset(bars, 0, 4096);
  void* args[3] = {&bars, &iters, &cyc};
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaLaunchCooperativeKernel((const void*)k_probe<MODE>, dim3(grid), dim3(512), args, 0, 0);   // warm-up
  cudaMemset(bars, 0, 4096);
  cudaEventRecord(e0);
  cudaLaunchCooperativeKernel((const void*)k_probe<MODE>, dim3(grid), dim3(512), args, 0, 0);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) printf("error: %s\n", cudaGetErrorString(err));
  return ms * 1000.f / iters;
}

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  unsigned* bars; long long* cyc;
  cudaMalloc(&bars, 4096); cudaMalloc(&cyc, 8);
  const int iters = 2000;
  printf("{\"sms\": %d, \"single_counter_us\": %.3f, \"tree_flag_us\": %.3f, \"red_relaxed_us\": %.3f, \"cg_grid_sync_us\": %.3f}\n", sms,
         run<0>(sms, iters, bars, cyc), run<1>(sms, iters, bars, cyc), run<2>(sms, iters, bars, cyc), run<3>(sms, iters, bars, cyc));
  return 0;
}
