// Causal self-attention on wgmma (forward + backward), reading q/k/v in place from the packed projection output.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rb {

// qkv: bf16 [B*T, 3*nh*hd] (q | k | v, heads contiguous inside each third, RoPE already applied), row stride ld_qkv.
// out: bf16 [B*T, nh*hd] (row stride ld_out).  lse: fp32 [B, nh, T], log2-domain log-sum-exp of the scaled scores
//      (p = exp2(s * scale * log2(e) - lse)), consumed by the backward kernels.
// Requirements: hd % 8 == 0, hd <= 64 (a 64-wide TMA box over a narrower head is zero filled).
struct AttnDesc {
  const void* qkv = nullptr;
  long long ld_qkv = 0;
  void* out = nullptr;
  long long ld_out = 0;
  float* lse = nullptr;
  int B = 0, T = 0, nh = 0, hd = 0;
  float scale = 1.0f;  // 1/sqrt(hd)
};
void attention_fwd(const AttnDesc& d, cudaStream_t stream);

// Backward: dqkv bf16 [B*T, 3*nh*hd] receives dq | dk | dv in the layout of qkv (gradient w.r.t. the post-RoPE q / k).
// delta: fp32 workspace [B, nh, T] (row sums of dO * O), filled by this call.
struct AttnBwdDesc {
  const void* qkv = nullptr;
  long long ld_qkv = 0;
  const void* out = nullptr;   // forward output
  long long ld_out = 0;
  const void* dout = nullptr;  // gradient of the forward output, same layout as out
  long long ld_dout = 0;
  const float* lse = nullptr;
  float* delta = nullptr;
  void* dqkv = nullptr;
  long long ld_dqkv = 0;
  int B = 0, T = 0, nh = 0, hd = 0;
  float scale = 1.0f;
  // optional bf16 workspace of attention_ds_workspace_elems(B, T, nh) elements; not read by the sm_90 kernels (the dQ kernel
  // recomputes S and dP), kept so callers that size it need no change
  void* ds_workspace = nullptr;
};
void attention_bwd(const AttnBwdDesc& d, cudaStream_t stream);
long long attention_ds_pitch(int T);
long long attention_ds_workspace_elems(int B, int T, int nh);

}  // namespace rb
