// avc_scan.cu -- the device-wide ordered exclusive scan of ints shared by the mesh kernels (avc_common.cuh):
//   k_scan_reduce   per tile of SCAN_TILE elements its sum
//   k_scan_top      one block: the exclusive scan of the tile sums, SCAN_TOP at a time with a running carry, and the total
//   k_scan_down     per tile: the block scan of its elements from the tile's offset
#include "avc_common.cuh"

using namespace avc;

namespace {

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8, SCAN_TILE = SCAN_THREADS * SCAN_ITEMS, SCAN_TOP = 1024;

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_reduce(const int* __restrict__ a, int n, int* __restrict__ sums) {
  __shared__ int wt[33];
  const long long base = (long long)blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  int s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; ++k) s += base + k < n ? a[base + k] : 0;
  int total;
  block_exclusive_scan<SCAN_THREADS>(s, wt, total);
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(SCAN_TOP) k_scan_top(int* sums, int nb, int32_t* total_out) {
  __shared__ int wt[33];
  int carry = 0;
  for (int c0 = 0; c0 < nb; c0 += SCAN_TOP) {
    const int i = c0 + threadIdx.x;
    const int x = i < nb ? sums[i] : 0;
    int total;
    const int ex = block_exclusive_scan<SCAN_TOP>(x, wt, total);
    if (i < nb) sums[i] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) *total_out = carry;
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_down(int* a, int n, const int* __restrict__ sums) {
  __shared__ int wt[33];
  const long long base = (long long)blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  int x[SCAN_ITEMS], s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; ++k) { x[k] = base + k < n ? a[base + k] : 0; s += x[k]; }
  int total;
  int run = sums[blockIdx.x] + block_exclusive_scan<SCAN_THREADS>(s, wt, total);
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; ++k) {
    if (base + k < n) a[base + k] = run;
    run += x[k];
  }
}

}  // namespace

namespace avc {

size_t exclusive_scan_sums(int n) { return (size_t)ceil_div(n, SCAN_TILE); }

void exclusive_scan(int* a, int n, int* sums, int32_t* total, cudaStream_t st) {
  const int nb = ceil_div(n, SCAN_TILE);
  k_scan_reduce<<<nb, SCAN_THREADS, 0, st>>>(a, n, sums);
  k_scan_top<<<1, SCAN_TOP, 0, st>>>(sums, nb, total);
  k_scan_down<<<nb, SCAN_THREADS, 0, st>>>(a, n, sums);
}

}  // namespace avc
