// Causal self-attention on wgmma (forward + backward), reading q/k/v in place from the packed projection output.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rb {

// qkv: bf16 [B*T, (nh + 2*nkv)*hd] (q: nh heads | k: nkv heads | v: nkv heads, heads contiguous inside each part, RoPE already
//      applied), row stride ld_qkv.  Query head h attends with KV head h / (nh / nkv): grouped-query attention when nkv < nh.
// out: bf16 [B*T, nh*hd] (row stride ld_out).  lse: fp32 [B, nh, T], log2-domain log-sum-exp of the scaled scores
//      (p = exp2(s * scale * log2(e) - lse)), consumed by the backward kernels.
// Requirements: hd % 8 == 0, hd <= 256.  A head is read as ceil(hd / 64) TMA boxes 64 columns wide; the columns of the last box
// past hd are zero filled.
struct AttnDesc {
  const void* qkv = nullptr;
  long long ld_qkv = 0;
  void* out = nullptr;
  long long ld_out = 0;
  float* lse = nullptr;
  int B = 0, T = 0, nh = 0, hd = 0;
  int nkv = 0;         // KV heads, nh % nkv == 0 (nkv == nh: multi-head attention)
  float scale = 1.0f;  // 1/sqrt(hd)
  // false: qkv is [q | k | v] per row (above).  true: [nh, (q|k|v), hd] per row, the head-interleaved layout of GPT-NeoX's
  // query_key_value projection (q, k, v of head h at head-columns 3h, 3h+1, 3h+2); needs nkv == nh.
  bool interleaved = false;
};
void attention_fwd(const AttnDesc& d, cudaStream_t stream);

// Backward: dqkv bf16 [B*T, (nh + 2*nkv)*hd] receives dq | dk | dv in the layout of qkv (gradient w.r.t. the post-RoPE q / k).
// dK / dV of a KV head sum over its group's query heads inside one CTA (no atomics).
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
  int nkv = 0;  // see AttnDesc
  float scale = 1.0f;
  bool interleaved = false;  // layout of qkv and dqkv (see AttnDesc)
  // optional bf16 workspace of attention_ds_workspace_elems(B, T, nh) elements; not read by the sm_90 kernels (the dQ kernel
  // recomputes S and dP), kept so callers that size it need no change
  void* ds_workspace = nullptr;
};
void attention_bwd(const AttnBwdDesc& d, cudaStream_t stream);
long long attention_ds_pitch(int T);
// dynamic shared memory per CTA of the largest attention kernel launched for head size hd (bytes)
int attention_smem_bytes(int hd);
long long attention_ds_workspace_elems(int B, int T, int nh);

}  // namespace rb
