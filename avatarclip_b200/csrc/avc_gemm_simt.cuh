// avc_gemm_simt.cuh -- fp32 CUDA-core (FFMA) GEMM tiles with pluggable epilogues.
//
// This is the correctness anchor of the MLP contractions (engine 0): exact fp32 products and
// fp32 accumulation, so parity against the reference's fp32 SGEMM path is round-off only.
// The tensor-core engine (avc_gemm_tc.cuh) reuses the same epilogue functors.
//
//   gemm_nt : C[m,n] = sum_k A[m,k] * B[n,k]        (A: [M,lda], B: [N,ldb], both K-contiguous)
//   gemm_tn : C[i,j] += sum_p A[p,i] * B[p,j]       (reduction over rows: weight gradients)
//
// Requirements: lda, ldb multiples of 4 floats, 16-byte aligned bases, K a multiple of 4 with the
// padding columns of BOTH operands finite and at least one of them zero.
#pragma once
#include "avc_common.cuh"

namespace avc {

// ------------------------------------------------------------------------------------------
// NT: 256 threads, tile 128 x (16*TN), K step 16, register-prefetch double buffering.
// Thread (tx = tid & 15, ty = tid >> 4) owns rows {ty*4+i, 64+ty*4+i} and, for TN = 8, columns
// {tx*4+j, 64+tx*4+j}; for TN = 4 columns {tx*4+j}.
// Epilogue: epi(row, col, float4 acc) with col % 4 == 0, called only for row < M and col < N.
// ------------------------------------------------------------------------------------------
template <int TN, typename Epi>
__global__ void __launch_bounds__(256)
gemm_nt_kernel(int M, int N, int K, const float* __restrict__ A, int lda,
               const float* __restrict__ B, int ldb, Epi epi) {
  constexpr int BM = 128, BN = 16 * TN, BK = 16, PAD = 4;
  __shared__ __align__(16) float As[2][BK][BM + PAD];
  __shared__ __align__(16) float Bs[2][BK][BN + PAD];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

  // global -> register staging: A tile = 128 rows x 4 float4; B tile = BN rows x 4 float4
  constexpr int A_F4 = BM * BK / 4 / 256;  // 2
  constexpr int B_F4 = (BN * BK / 4 + 255) / 256;  // 2 (TN=8) or 1 (TN=4)
  float4 ra[A_F4], rb[B_F4];

  auto load_tiles = [&](int k0) {
#pragma unroll
    for (int s = 0; s < A_F4; ++s) {
      int i = tid + s * 256;
      int r = i >> 2, kq = (i & 3) * 4;
      int gr = m0 + r, gk = k0 + kq;
      ra[s] = (gr < M && gk < K) ? *reinterpret_cast<const float4*>(A + (size_t)gr * lda + gk)
                                 : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int s = 0; s < B_F4; ++s) {
      int i = tid + s * 256;
      int r = i >> 2, kq = (i & 3) * 4;
      int gr = n0 + r, gk = k0 + kq;
      bool ok = (BN * BK / 4 >= 256 || i < BN * BK / 4) && gr < N && gk < K;
      rb[s] = ok ? *reinterpret_cast<const float4*>(B + (size_t)gr * ldb + gk)
                 : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int s = 0; s < A_F4; ++s) {
      int i = tid + s * 256;
      int r = i >> 2, kq = (i & 3) * 4;
      As[buf][kq + 0][r] = ra[s].x; As[buf][kq + 1][r] = ra[s].y;
      As[buf][kq + 2][r] = ra[s].z; As[buf][kq + 3][r] = ra[s].w;
    }
#pragma unroll
    for (int s = 0; s < B_F4; ++s) {
      int i = tid + s * 256;
      if (BN * BK / 4 >= 256 || i < BN * BK / 4) {
        int r = i >> 2, kq = (i & 3) * 4;
        Bs[buf][kq + 0][r] = rb[s].x; Bs[buf][kq + 1][r] = rb[s].y;
        Bs[buf][kq + 2][r] = rb[s].z; Bs[buf][kq + 3][r] = rb[s].w;
      }
    }
  };

  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int nk = (K + BK - 1) / BK;
  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tiles((kt + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[8], b[TN];
      *reinterpret_cast<float4*>(&a[0]) = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      *reinterpret_cast<float4*>(&a[4]) = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
      *reinterpret_cast<float4*>(&b[0]) = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      if (TN == 8)
        *reinterpret_cast<float4*>(&b[TN - 4]) = *reinterpret_cast<const float4*>(&Bs[buf][kk][(BN / 2) + tx * 4]);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int row = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (row >= M) continue;
#pragma unroll
    for (int jg = 0; jg < TN / 4; ++jg) {
      int col = n0 + (jg == 0 ? tx * 4 : (BN / 2) + tx * 4);
      if (col >= N) continue;
      epi(row, col, make_float4(acc[i][jg * 4 + 0], acc[i][jg * 4 + 1], acc[i][jg * 4 + 2], acc[i][jg * 4 + 3]));
    }
  }
}

template <typename Epi>
static inline int launch_gemm_nt(cudaStream_t st, int64_t M, int N, int K, const float* A, int lda,
                                 const float* B, int ldb, const Epi& epi) {
  if (M <= 0 || N <= 0) return 0;
  if (N > 64) {
    dim3 grid(ceil_div(N, 128), ceil_div(M, 128));
    gemm_nt_kernel<8, Epi><<<grid, 256, 0, st>>>((int)M, N, K, A, lda, B, ldb, epi);
  } else {
    dim3 grid(ceil_div(N, 64), ceil_div(M, 128));
    gemm_nt_kernel<4, Epi><<<grid, 256, 0, st>>>((int)M, N, K, A, lda, B, ldb, epi);
  }
  AVC_LAUNCH_TRY();
  return 0;
}

// ------------------------------------------------------------------------------------------
// TN with split over the reduction (rows p): C[i*ldc + j] += sum_{p in slice} A[p,i] * B[p,j].
// 256 threads, tile 128 x 128, p step 16.  Results are accumulated with red.global.add.f32.
// Columns beyond N1/N2 may be read (up to lda/ldb) but never contribute to a stored output.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gemm_tn_kernel(int P, int N1, int N2, const float* __restrict__ A, int lda,
               const float* __restrict__ B, int ldb, float* __restrict__ C, int ldc, int rows_per_split) {
  constexpr int BM = 128, BN = 128, BK = 16;
  __shared__ __align__(16) float As[2][BK][BM];
  __shared__ __align__(16) float Bs[2][BK][BN];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int i0 = blockIdx.y * BM, j0 = blockIdx.x * BN;
  const int p_begin = blockIdx.z * rows_per_split;
  const int p_end = min(P, p_begin + rows_per_split);
  if (p_begin >= p_end) return;

  float4 ra[2], rb[2];
  auto load_tiles = [&](int p0) {
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      int i = tid + s * 256;        // 512 float4 = 16 rows x 32 float4
      int r = i >> 5, c4 = (i & 31) * 4;
      int gp = p0 + r;
      ra[s] = (gp < p_end && i0 + c4 < lda) ? *reinterpret_cast<const float4*>(A + (size_t)gp * lda + i0 + c4)
                                            : make_float4(0.f, 0.f, 0.f, 0.f);
      rb[s] = (gp < p_end && j0 + c4 < ldb) ? *reinterpret_cast<const float4*>(B + (size_t)gp * ldb + j0 + c4)
                                            : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      int i = tid + s * 256;
      int r = i >> 5, c4 = (i & 31) * 4;
      *reinterpret_cast<float4*>(&As[buf][r][c4]) = ra[s];
      *reinterpret_cast<float4*>(&Bs[buf][r][c4]) = rb[s];
    }
  };
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  const int nk = (p_end - p_begin + BK - 1) / BK;
  load_tiles(p_begin);
  store_tiles(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tiles(p_begin + (kt + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[8], b[8];
      *reinterpret_cast<float4*>(&a[0]) = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      *reinterpret_cast<float4*>(&a[4]) = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
      *reinterpret_cast<float4*>(&b[0]) = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      *reinterpret_cast<float4*>(&b[4]) = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int gi = i0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (gi >= N1) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int gj = j0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (gj < N2) atomicAdd(C + (size_t)gi * ldc + gj, acc[i][j]);
    }
  }
}

static inline int launch_gemm_tn(cudaStream_t st, int64_t P, int N1, int N2, const float* A, int lda,
                                 const float* B, int ldb, float* C, int ldc) {
  if (P <= 0 || N1 <= 0 || N2 <= 0) return 0;
  int tiles = ceil_div(N1, 128) * ceil_div(N2, 128);
  static thread_local int sms = 0;
  if (!sms) { int dev = 0; AVC_CUDA_TRY(cudaGetDevice(&dev)); AVC_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)); }
  int splits = (2 * sms + tiles - 1) / tiles;      // two CTAs per SM
  int rows_per_split = (int)round_up(ceil_div(P, splits), 16);
  splits = ceil_div(P, rows_per_split);
  dim3 grid(ceil_div(N2, 128), ceil_div(N1, 128), splits);
  gemm_tn_kernel<<<grid, 256, 0, st>>>((int)P, N1, N2, A, lda, B, ldb, C, ldc, rows_per_split);
  AVC_LAUNCH_TRY();
  return 0;
}

}  // namespace avc
