// avc_common_test.cu -- the shared pieces of avc_common.cuh and avc_scan.cu on caller buffers, each kernel calling
// exactly one of them, for tests/test_prims_gpu.py (argument roles in include/avc_b200.h, avc_common_kernel_test):
//   k_reduce3        three back-to-back block_reduce calls on one red, as k_rows_cos and k_pose_score make them
//   k_block_scan     block_exclusive_scan<NT> in a loop with a running carry, as k_scan_top calls it
//   k_keys           ordered_bits, sel_key, sel_index and depth_key of every element
//   k_select         64-bit atomicMax of sel_key and atomicMin of depth_key from every thread of many CTAs
// and the device-wide exclusive_scan itself.
#include "avc_common.cuh"

using namespace avc;

namespace {

struct AddOp {
  template <class T>
  __device__ __forceinline__ T operator()(T a, T b) const { return a + b; }
};
struct MinOp {
  template <class T>
  __device__ __forceinline__ T operator()(T a, T b) const { return a < b ? a : b; }
};
struct MaxOp {
  template <class T>
  __device__ __forceinline__ T operator()(T a, T b) const { return a > b ? a : b; }
};

// x and r are [3][n], n = gridDim.x blockDim.x; every thread writes the three results it received
template <class T, class Op>
__global__ void __launch_bounds__(1024) k_reduce3(const T* __restrict__ x, size_t n, Op op, T init, T* __restrict__ r) {
  __shared__ T red[32];
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const T a = block_reduce(x[i], red, op, init);
  const T b = block_reduce(x[n + i], red, op, init);
  const T c = block_reduce(x[2 * n + i], red, op, init);
  r[i] = a;
  r[n + i] = b;
  r[2 * n + i] = c;
}

template <class T, class Op>
void launch_reduce3(const void* x, int threads, int blocks, Op op, T init, void* r, cudaStream_t st) {
  k_reduce3<T, Op><<<blocks, threads, 0, st>>>((const T*)x, (size_t)blocks * threads, op, init, (T*)r);
}

// per CTA rounds consecutive slices of NT elements; total[b][t] is thread t's carry after the last round
template <int NT>
__global__ void __launch_bounds__(NT) k_block_scan(const int* __restrict__ x, int rounds, int* __restrict__ ex,
                                                   int* __restrict__ total) {
  __shared__ int wt[33];
  const size_t base = (size_t)blockIdx.x * rounds * NT + threadIdx.x;
  int carry = 0;
  for (int r = 0; r < rounds; ++r) {
    int t;
    const int e = block_exclusive_scan<NT>(x[base + (size_t)r * NT], wt, t);
    ex[base + (size_t)r * NT] = carry + e;
    carry += t;
  }
  total[(size_t)blockIdx.x * NT + threadIdx.x] = carry;
}

template <int NT>
void launch_block_scan(int blocks, int rounds, const void* x, void* ex, void* total, cudaStream_t st) {
  k_block_scan<NT><<<blocks, NT, 0, st>>>((const int*)x, rounds, (int*)ex, (int*)total);
}

__global__ void k_keys(const float* __restrict__ v, int n, unsigned* __restrict__ ob, unsigned long long* __restrict__ sk,
                       int* __restrict__ si, unsigned long long* __restrict__ dk) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = sel_key(v[i], i);
  ob[i] = ordered_bits(v[i]);
  sk[i] = k;
  si[i] = sel_index(k);
  dk[i] = depth_key(v[i], i);
}

__global__ void k_select(const float* __restrict__ v, const float* __restrict__ z, int n, unsigned long long* mx,
                         unsigned long long* mn) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    atomicMax(mx, sel_key(v[i], i));
    if (z) atomicMin(mn, depth_key(z[i], i));
  }
}

__global__ void k_select_index(const unsigned long long* __restrict__ mx, int* __restrict__ best) {
  *best = sel_index(*mx);
}

}  // namespace

extern "C" {

int avc_common_kernel_test(int32_t kind, const int64_t* d, const void* const* in, void* const* out,
                           avc_stream_t stream) {
  if (!d || !in || !out) return AVC_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  switch (kind) {
    case 0: {       // block_reduce
      const int64_t op = d[0], threads = d[1], blocks = d[2];
      if (threads < 32 || threads > 1024 || threads % 32 || blocks < 1 || blocks > 65535) return AVC_E_SIZE;
      if (!in[0] || !out[0]) return AVC_E_NULL;
      const int t = (int)threads, b = (int)blocks;
      switch (op) {
        case 0: launch_reduce3<double>(in[0], t, b, AddOp{}, 0.0, out[0], st); break;
        case 1: launch_reduce3<int>(in[0], t, b, AddOp{}, 0, out[0], st); break;
        case 2: launch_reduce3<unsigned long long>(in[0], t, b, MinOp{}, ~0ull, out[0], st); break;
        case 3: launch_reduce3<unsigned long long>(in[0], t, b, MaxOp{}, 0ull, out[0], st); break;
        default: return AVC_E_BADCFG;
      }
      break;
    }
    case 1: {       // block_exclusive_scan<NT>
      const int64_t NT = d[0], blocks = d[1], rounds = d[2];
      if (blocks < 1 || blocks > 65535 || rounds < 1) return AVC_E_SIZE;
      if (!in[0] || !out[0] || !out[1]) return AVC_E_NULL;
      const int b = (int)blocks, r = (int)rounds;
      switch (NT) {
        case 32: launch_block_scan<32>(b, r, in[0], out[0], out[1], st); break;
        case 128: launch_block_scan<128>(b, r, in[0], out[0], out[1], st); break;
        case 256: launch_block_scan<256>(b, r, in[0], out[0], out[1], st); break;
        case 1024: launch_block_scan<1024>(b, r, in[0], out[0], out[1], st); break;
        default: return AVC_E_BADCFG;
      }
      break;
    }
    case 2: {       // keys
      const int64_t n = d[0];
      if (n < 1 || n > (1LL << 30)) return AVC_E_SIZE;
      if (!in[0] || !out[0] || !out[1] || !out[2] || !out[3]) return AVC_E_NULL;
      k_keys<<<ceil_div(n, 256), 256, 0, st>>>((const float*)in[0], (int)n, (unsigned*)out[0],
                                                (unsigned long long*)out[1], (int*)out[2], (unsigned long long*)out[3]);
      break;
    }
    case 3: {       // contended selection
      const int64_t n = d[0], threads = d[1], blocks = d[2];
      if (n < 1 || n > (1LL << 30) || threads < 1 || threads > 1024 || blocks < 1 || blocks > 65535) return AVC_E_SIZE;
      if (!in[0] || !out[0] || !out[1] || !out[2]) return AVC_E_NULL;
      AVC_CUDA_TRY(cudaMemsetAsync(out[0], 0, sizeof(unsigned long long), st));
      AVC_CUDA_TRY(cudaMemsetAsync(out[1], 0xff, sizeof(unsigned long long), st));
      k_select<<<(int)blocks, (int)threads, 0, st>>>((const float*)in[0], (const float*)in[1], (int)n,
                                                     (unsigned long long*)out[0], (unsigned long long*)out[1]);
      k_select_index<<<1, 1, 0, st>>>((const unsigned long long*)out[0], (int*)out[2]);
      break;
    }
    case 4: {       // exclusive_scan
      const int64_t n = d[0];
      if (n < 1 || n > INT32_MAX) return AVC_E_SIZE;
      if (!out[0] || !out[1] || !out[2]) return AVC_E_NULL;
      exclusive_scan((int*)out[0], (int)n, (int*)out[1], (int32_t*)out[2], st);
      break;
    }
    case 5: {       // exclusive_scan's workspace
      const int64_t n = d[0];
      if (n < 1 || n > INT32_MAX) return AVC_E_SIZE;
      if (!out[0]) return AVC_E_NULL;
      *(int64_t*)out[0] = (int64_t)exclusive_scan_sums((int)n);
      return 0;
    }
    default: return AVC_E_BADCFG;
  }
  AVC_LAUNCH_TRY();
  return 0;
}

}  // extern "C"
