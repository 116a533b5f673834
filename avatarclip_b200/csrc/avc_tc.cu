// avc_tc.cu -- self-test entry points of the wgmma GEMM tiles (used by tests/test_tc_gemm_gpu.py).
#include "avc_gemm_tc.cuh"

using namespace avc;

namespace {
struct EpiPlainStore {
  float* C; int ldc; int N;
  __device__ void operator()(int row, int col, float4 a) const {
    float v[4] = {a.x, a.y, a.z, a.w};
    for (int i = 0; i < 4 && col + i < N; ++i) C[(size_t)row * ldc + col + i] = v[i];
  }
  // ring-stored when C's rows are whole 16 bytes (N % 4 == 0), else from registers
  using Out = tc::Outs<4>;
  tc::OutOp out_op(int, int) const { return {C, ldc, N}; }
  template <typename S>
  __device__ void ring(int, int, float4 a, const S& s) const {
    const float v[4] = {a.x, a.y, a.z, a.w};
    s.f32(0, v);
  }
};
}  // namespace

extern "C" {

// C[M][N] = A[M][K] . B[N][K]^T through the wgmma NT tiles.  nprod = 1 (single bf16 product) or 3 (two-term split).
// workspace >= 4 * (M + N) * round_up(K, 8) bytes.
int avc_tc_gemm_nt_test(const float* A, const float* B, int64_t M, int32_t N, int32_t K, int32_t nprod, float* C,
                        void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!A || !B || !C || !workspace) return AVC_E_NULL;
  if (M <= 0 || N <= 0 || K <= 0 || (nprod != 1 && nprod != 3)) return AVC_E_SIZE;
  const int ld = (int)round_up(K, 8);
  Carver cv(workspace);
  __nv_bfloat16* ah = cv.take<__nv_bfloat16>(M * ld);
  __nv_bfloat16* al = cv.take<__nv_bfloat16>(M * ld);
  __nv_bfloat16* bh = cv.take<__nv_bfloat16>((int64_t)N * ld);
  __nv_bfloat16* bl = cv.take<__nv_bfloat16>((int64_t)N * ld);
  if (cv.used() > workspace_bytes) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  tc::k_split_bf16<<<(int)((M * ld + 255) / 256), 256, 0, st>>>(A, M, K, K, ah, al, ld);
  tc::k_split_bf16<<<(int)(((int64_t)N * ld + 255) / 256), 256, 0, st>>>(B, N, K, K, bh, bl, ld);
  AVC_LAUNCH_TRY();
  tc::SplitPtr a{ah, al, ld}, b{bh, bl, ld};
  EpiPlainStore e{C, N, N};
  if (nprod == 3) return tc::launch_gemm_tc_nt<3, EpiPlainStore>(st, M, N, K, a, b, e);
  return tc::launch_gemm_tc_nt<1, EpiPlainStore>(st, M, N, K, a, b, e);
}

// C[N1][N2] += A[P][N1]^T . B[P][N2] through the wgmma TN (MN-major) tiles.  C must be initialised by the caller.
// workspace >= 4 * P * (round_up(N1,8) + round_up(N2,8)) + 2048 bytes.
int avc_tc_gemm_tn_test(const float* A, const float* B, int64_t P, int32_t N1, int32_t N2, int32_t nprod, float* C,
                        float* colsum, void* workspace, size_t workspace_bytes, avc_stream_t stream) {
  if (!A || !B || !C || !workspace) return AVC_E_NULL;
  if (P <= 0 || N1 <= 0 || N2 <= 0 || (nprod != 1 && nprod != 3)) return AVC_E_SIZE;
  const int l1 = (int)round_up(N1, 8), l2 = (int)round_up(N2, 8);
  Carver cv(workspace);
  __nv_bfloat16* ah = cv.take<__nv_bfloat16>(P * l1);
  __nv_bfloat16* al = cv.take<__nv_bfloat16>(P * l1);
  __nv_bfloat16* bh = cv.take<__nv_bfloat16>(P * l2);
  __nv_bfloat16* bl = cv.take<__nv_bfloat16>(P * l2);
  if (cv.used() > workspace_bytes) return AVC_E_SIZE;
  cudaStream_t st = (cudaStream_t)stream;
  tc::k_split_bf16<<<(int)((P * l1 + 255) / 256), 256, 0, st>>>(A, P, N1, N1, ah, al, l1);
  tc::k_split_bf16<<<(int)((P * l2 + 255) / 256), 256, 0, st>>>(B, P, N2, N2, bh, bl, l2);
  AVC_LAUNCH_TRY();
  tc::SplitPtr a{ah, al, l1}, b{bh, bl, l2};
  if (nprod == 3) return tc::launch_gemm_tc_tn<3>(st, P, N1, N2, a, b, C, N2, colsum);
  return tc::launch_gemm_tc_tn<1>(st, P, N1, N2, a, b, C, N2, colsum);
}

// 1: the last wgmma NT launch of the calling host thread stored its outputs with TMA through the epilogue ring, 0: from
// registers, -1: none yet.
int avc_tc_nt_last_ring(void) { return tc::g_nt_last_ring; }

}  // extern "C"
