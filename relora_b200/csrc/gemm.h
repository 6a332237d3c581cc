// Host API of the wgmma GEMM family (implemented in gemm_wgmma.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rb {

// A bf16 matrix operand in global memory.
//   K-major  (mn_major = false): element (i, k) at ptr[i * ld + k]   (i = row of A / row of B = output column)
//   MN-major (mn_major = true) : element (i, k) at ptr[k * ld + i]
struct Operand {
  const void* ptr = nullptr;
  long long ld = 0;      // leading dimension in elements (must be a multiple of 8)
  bool mn_major = false;
};

// D[M,N] = alpha * ( A1[M,K1] · B1[N,K1]ᵀ  +  A2[M,K2] · B2[N,K2]ᵀ )  (+ residual)  (+ D if accumulate)
//
// Grouping (fused LoRA): output columns are split into groups of `n_per_group`; for a tile in group g the
// K-window of A1 starts at g*a1_group_kofs and the K-window of A2 at g*a2_group_kofs (B rows are the output
// columns themselves).  With a2_group_kofs = r this evaluates, per group,
//     y_g = x · W_gᵀ + u_g · B_gᵀ        (u = [u_0 | u_1 | ...] holds the down-projections side by side)
// in one pass over x and one write of y.  When both A1 and B1 take per-group K windows, K1 must be a multiple of the
// k-block (64 elements, fp8: 128).
struct GemmDesc {
  Operand a1, b1, a2, b2;
  int M = 0, N = 0, K1 = 0, K2 = 0;
  int n_per_group = 0;  // 0 => N (single group)
  int a1_group_kofs = 0, a2_group_kofs = 0;
  // B1 addressing for the backward GEMMs: K-window offset per N-group, MN coordinate taken relative to the group,
  // and an extra MN offset chosen by the group of the M-tile (stacked weight-gradient GEMMs dA_cat / dB_cat).
  int b1_group_kofs = 0;
  bool b1_local_n = false;
  int m_per_group = 0, b1_mn_ofs_per_mgroup = 0;
  void* out = nullptr;
  long long ldc = 0;
  bool out_f32 = false;     // output dtype: bf16 (default) or fp32
  bool accumulate = false;  // out += result (fp32 outputs: gradient accumulation)
  // residual and bias: bf16 outputs only (refused with an fp32 output)
  const void* residual = nullptr;  // bf16 [M, N], added in fp32 before rounding
  long long ldr = 0;
  const void* bias = nullptr;      // bf16 [N], added in fp32 (after alpha, before the residual)
  float alpha = 1.0f;
  const float* alpha_dev = nullptr;  // optional device scalar multiplied into alpha
  bool fp8_a_e5m2 = false;  // with fp8: A1 is E5M2 (gradients), B1 stays E4M3
  bool fp8 = false;  // A1 / B1 hold E4M3 bytes (K-major, leading dimensions in bytes); A2 / B2 (the LoRA branch) stay bf16
  int block_n = 0;  // 0 = auto (gemm_block_n), else 128, 192 or 256
  int split_k = 1;  // 1 = off, 0 = auto, >1 = fixed (fp32 accumulate outputs only: partial sums via atomics)
  int pair = -1;    // CTA pairs sharing the B tile (gemm_pairs): -1 = auto, 0 = off, 1 = wherever the call form allows
  // dropout-combine epilogue (backward of the LoRA branch): if n_lora_acc > 0 the A2/B2 products of
  // the first n_lora_acc K2-windows (each of width lora_r) are kept in separate accumulators and combined as
  //     out = acc0 + sum_g keep_g(row, col) * acc_{1+g} * inv_keep
  int n_lora_acc = 0;
  int lora_r = 0;
  uint32_t drop_threshold24 = 0;
  float inv_keep = 1.0f;
  const uint32_t* seed_ptr = nullptr;  // device: base seed of this step
  uint32_t seed_key[4] = {0, 0, 0, 0}; // per-accumulator stream keys
};

void gemm_bf16(const GemmDesc& d, cudaStream_t stream);
// The stored [rows, cols] (cols contiguous) of each operand that gemm_bf16's tensor maps span: [mn, k] K-major, [k, mn]
// MN-major, with the per-group K windows and M-group offsets included; fp8 extents are in bytes.  A2 / B2 are empty when K2 = 0.
struct GemmExtent {
  long long rows = 0, cols = 0;
};
struct GemmExtents {
  GemmExtent a1, b1, a2, b2;
};
GemmExtents gemm_operand_extents(const GemmDesc& d);
// Schedule choices of gemm_bf16 (host side): the tile width, whether the epilogue stores through shared memory with TMA,
// and the dynamic shared memory of a tile width.
// sms: the SM count the wave rule fills (0: this device's)
int gemm_block_n(const GemmDesc& d, int sms = 0);
bool gemm_uses_tma_store(const GemmDesc& d, int block_n, int split_k);
int gemm_smem_bytes(int block_n);
// whether the call runs as CTA pairs: 128-wide tiles, at least two M tiles, M groups of whole pairs; auto: long reductions
// into wide outputs
bool gemm_pairs(const GemmDesc& d, int block_n);

// Input gradient of a stacked LoRA group with the dropout mask applied in the epilogue:
//   out[M,N] = dy[M,Kb]·W[Kb,N] + inv_keep · Σ_g keep(seed_g; row, col) ⊙ (du_g[M,r]·A_g[r,N]),  g < groups <= 3
// dy/du are K-major activations (du = [du_0 | du_1 | ...]); W [Kb, N] and A = [A_0; A_1; ...] ([groups·r, N]) are the
// parameters as stored (read MN-major in place).  seed_g = mix_seed(*seed_ptr, seed_key[g]).
struct LoraDxDesc {
  const void *dy = nullptr, *w = nullptr, *du = nullptr, *a = nullptr;
  long long ld_dy = 0, ld_w = 0, ld_du = 0, ld_a = 0;
  void* out = nullptr;
  long long ldc = 0;
  int M = 0, N = 0, Kb = 0, r = 0, groups = 1;
  // Kb == 0: `base` [M, N] bf16 already holds dy·W (computed by a separate GEMM); this kernel then only adds the masked
  // low-rank terms
  const void* base = nullptr;
  long long ld_base = 0;
  uint32_t drop_threshold16 = 0;  // round(p * 65536); 0 = keep everything (no dropout)
  float inv_keep = 1.0f;
  const uint32_t* seed_ptr = nullptr;
  uint32_t seed_key[3] = {0, 0, 0};
  int pair = -1;  // CTA pairs sharing the A / W tile: -1 = auto (gemm_pairs' rule), 0 = off, 1 = on when M has two tiles or more
  int block_n = 0;  // output tile width: 0 = auto (the GEMM's wave rule), 128 or 192 (192 never pairs)
};
void lora_dx(const LoraDxDesc& d, cudaStream_t stream);
bool lora_dx_pairs(const LoraDxDesc& d);
int lora_dx_block_n(const LoraDxDesc& d);
// the output leaves through shared memory and TMA stores unless a row is not a whole number of 16-byte chunks
bool lora_dx_uses_tma_store(const LoraDxDesc& d);

// Drop cached TMA descriptors (call when buffers are freed / reallocated).
void gemm_clear_descriptor_cache();

}  // namespace rb
