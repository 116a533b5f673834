// avc_chain.h -- host interface of the fused SDF value-chain kernel (avc_chain.cu).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace avc {
namespace chain {

constexpr int kMaxHidden = 10;      // fused hidden linears (softplus layers): SDF nets up to n_layers = 10

struct Layer {
  const __nv_bfloat16* w_hi;   // effective (weight-normed) W_l as a bf16 (hi, lo) pair, [N][ldw] row-major, K-contiguous
  const __nv_bfloat16* w_lo;
  int ldw;                     // leading dimension (elements) of W_l
  int N, K;                    // output / input width of linear l (K includes the skip columns)
  const float* bias;           // [>= N] fp32
  float oscale;                // 1/sqrt(2) when the NEXT linear takes the skip concat (fields.py:79-80), else 1
  int next_skip_cols;          // E when the next linear's input is cat([h, enc]) / sqrt(2) (columns [N, N + E)), else 0
};

struct Args {
  int L;                       // number of hidden linears; linear L is the thin sdf head
  Layer lay[kMaxHidden];
  // layer-0 operand: encoded points [P][ld0] as a bf16 pair (k_encode_* wrote it), K_0 valid columns
  const __nv_bfloat16* a0_hi;
  const __nv_bfloat16* a0_lo;
  int ld0;
  // source of the skip columns: pair buffer [P][skip_ld]; columns [skip_col0, skip_col0 + E) hold enc / sqrt(2)
  const __nv_bfloat16* skip_hi;
  const __nv_bfloat16* skip_lo;
  int skip_ld, skip_col0;
  // sdf head (row 0 of the last linear): w_sdf [K_L] fp32, bias scalar, 1 / scale
  const float* w_sdf;
  const float* b_sdf;
  int K_head;                  // input width of the head = K of linear L
  int head_skip_cols;          // E when the head itself takes the skip concat (skip_in contains n_layers), else 0
  float inv_scale;
  float* sdf_out;              // point p -> sdf_out[nz > 0 ? (p / nz) * pitch + p % nz : p]
  int nz, pitch;
  int64_t P;
};

// true when the fused kernel covers this network shape: 1 <= L <= kMaxHidden; every hidden linear has 1 <= N, K <= 256
// and ldw % 8 == 0; the widths chain (N_l + next_skip_cols_l = K_{l+1}, N_{L-1} + head_skip_cols = K_head); ld0 % 8 == 0
bool supported(const Args& a);
int launch(const Args& a, cudaStream_t st);

}  // namespace chain
}  // namespace avc
