// Host API of the bandwidth-bound kernels (elementwise.cu, optim.cu, loss.cu).  All tensors are bf16 unless noted.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "fp8out.h"

namespace rb {

// ---- norms ---------------------------------------------------------------------------------
// y = w * bf16(x * rstd),  rstd = rsqrt(mean(x^2) + eps).  Optionally also writes G dropout-masked copies
// xd[m, g*H + k] = keep(seed_g, m, k) ? y[m,k] / (1-p) : 0   (inputs of the LoRA down-projections).
void rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int M, int H, float eps, void* xd, int G,
                 const uint32_t* seed_ptr, const uint32_t* keys, uint32_t thr16, float inv_keep, Fp8Out f8, cudaStream_t s);
// dx = rstd * (g - xhat * mean(g * xhat)) with g = dy * w (+ dx_add);  dw_f32[H] += sum_m dy * bf16(xhat)
// `ws` (fp32 [rmsnorm_bwd_ws_blocks(), H]) + `ticket` (zeroed uint32) enable the warp-per-row kernel (H <= 2048); without
// them the block-per-row fallback with global atomics on dw is used.
void rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dx_add, void* dx, float* dw,
                 int M, int H, float* ws, unsigned int* ticket, cudaStream_t s);
int rmsnorm_bwd_ws_blocks();
bool rmsnorm_fwd_warp(const void* x, const void* w, void* y, float* rstd, int M, int H, float eps, void* xd, int G,
                      const uint32_t* seed_ptr, uint4 keys, uint32_t thr16, float inv_keep, Fp8Out f8, cudaStream_t s);
bool rmsnorm_bwd_warp(const void* dy, const void* x, const void* w, const float* rstd, const void* dx_add, void* dx, float* dw, int M,
                      int H, float* ws, unsigned int* ticket, cudaStream_t s);

// xd[m, g*H + k] = keep(seed_g, m, k) ? x[m,k] / (1-p) : 0
void dropout_expand(const void* x, void* xd, int M, int H, int G, const uint32_t* seed_ptr, const uint32_t* keys,
                    uint32_t thr16, float inv_keep, Fp8Out f8, cudaStream_t s);
// out[m,k] = base[m,k] + sum_g keep(seed_g, m, k) * part_g[m,k] / (1-p)        (backward through the LoRA dropout)
// part_g[m,k] = parts[g*part_stride + m*ld_parts + k]
void dropout_combine(const void* base, const void* parts, long long part_stride, long long ld_parts, void* out, int M, int H, int G,
                     const uint32_t* seed_ptr, const uint32_t* keys, uint32_t thr16, float inv_keep, cudaStream_t s);

// ---- rotary --------------------------------------------------------------------------------
// In-place rotation of the first `n_rot_heads` heads of every row of buf [M, ld] (head h at columns h*hd..),
// rotary_dim <= hd leading dims of each head; position of row m is (m % T) + pos0.  cos/sin: bf16 [*, rotary_dim].
void rope_inplace(void* buf, long long ld, int M, int T, int n_rot_heads, int hd, int rotary_dim, const void* cos,
                  const void* sin, bool backward, int pos0, cudaStream_t s);

bool rope_inplace_vec(void* buf, long long ld, int M, int T, int n_rot_heads, int hd, int rotary_dim, const void* cos,
                      const void* sin, bool backward, int pos0, cudaStream_t s);
// dqkv[b*T+t, which*nh*hd + h*hd + d] <- inverse-rotated dq / dk and dv, each [B, nh, T, hd] with strides (sB, sH, sT, 1)
void rope_pack_bwd(const void* dq, const void* dk, const void* dv, long long sB, long long sH, long long sT, void* out,
                   long long ldo, int B, int T, int nh, int hd, int rotary_dim, const void* cos, const void* sin, int pos0,
                   cudaStream_t s);

// ---- SwiGLU --------------------------------------------------------------------------------
// gu: [M, 2F] (gate | up) -> h[M, F] = silu(gate) * up
// optional hd[M, F] = keep(mix(seed, key); row, col) ⊙ h / (1-p): the dropout-expanded copy for the next LoRA down-projection
void swiglu_fwd(const void* gu, long long ldgu, void* h, long long ldh, int M, int F, void* hd, long long ldhd,
                const uint32_t* seed_ptr, uint32_t key, uint32_t thr16, float inv_keep, Fp8Out f8, cudaStream_t s);
void swiglu_bwd(const void* dh, long long lddh, const void* gu, long long ldgu, void* dgu, long long lddgu, int M, int F,
                cudaStream_t s);

// ---- GPT-NeoX / Pythia block (neox.cu) -------------------------------------------------------
// nn.LayerNorm (affine weight + optional bias), bf16 in/out, fp32 row statistics saved for the backward; false = shape not handled
bool layernorm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, int M, int H, float eps, cudaStream_t s);
// dw / db (fp32, may be nullptr for db) are accumulated (+=)
bool layernorm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, void* dx, float* dw, float* db, int M,
                   int H, cudaStream_t s);
void gelu_fwd(const void* z, void* a, long long n, bool tanh_approx, cudaStream_t s);
void gelu_bwd(const void* da, const void* z, void* dz, long long n, bool tanh_approx, cudaStream_t s);
// partial rotary embedding in place on the fused query_key_value output [rows, nh, 3*hd] (q | k | v per head); fp32 tables [n_pos, rot]
// holding the cos / sin of the first rot/2 frequencies twice (HF layout: emb = cat(freqs, freqs)); inverse = backward direction
void neox_rope(void* qkv, long long ld, long long rows, int T, int nh, int hd, int rot, const float* cos, const float* sin, int pos0,
               bool inverse, cudaStream_t s);

// ---- block-scaled MXFP8 path (gemm_mx.cu) ------------------------------------------------------
// Scale factors live in [row block of 128][group of 128 reduction elements][512 bytes] blocks (the layout the MX GEMM stages per k-block).
long long mx_sf_bytes(long long rows, long long k_elems);
// x bf16 [M, K] (pitch ldx) -> E4M3 q [M, Kpad] (pitch ldq >= Kpad = K rounded up to 128, padding written as zero) + UE8M0 scales per (row, 32 cols)
void mx_quantize_rows(const void* x, long long ldx, void* q, long long ldq, void* sf, int M, int K, cudaStream_t s);
// W [N, K] -> E4M3 q (pitch ldq >= Kpad, Npad rows allocated) with ONE scale per 32 x 32 tile, written in the forward layout (rows N, reduction K)
// and in the backward layout (rows K, reduction N).  Source: bf16 `w` (pitch ldw), or -- w == nullptr -- the packed q_old / sf_old (may
// alias q / sf_fwd: requantisation in place); `delta` (fp32 [N, K], pitch ldd, nullable) is added before quantising (the ReLoRA merge).
void mx_quantize_weight_2d(const void* w, long long ldw, const void* q_old, const void* sf_old, const float* delta, long long ldd, void* q,
                           long long ldq, void* sf_fwd, void* sf_bwd, int N, int K, cudaStream_t s);
void mx_dequantize_weight(const void* q, long long ldq, const void* sf_fwd, void* out, long long ldo, int N, int K, cudaStream_t s);
// out[M,N] (bf16) = A8[M,K]·B8ᵀ (block-scaled E4M3, kind::mxf8f6f4) + A2[M,K2]·B2[N,K2]ᵀ (bf16, same accumulator) (+ residual)
struct MxGemmDesc {
  const void *a = nullptr, *b = nullptr;   // fp8 bytes; a [M, Kpad] K-major; b [N, Kpad] K-major, or (b_mn_major) [Kpad rows, N] as stored
  long long lda = 0, ldb = 0;
  const void *sfa = nullptr, *sfb = nullptr;
  bool b_mn_major = false;
  const void *a2 = nullptr, *b2 = nullptr; // bf16 K-major LoRA segment (optional)
  long long lda2 = 0, ldb2 = 0;
  int M = 0, N = 0, K = 0, K2 = 0;
  void* out = nullptr;
  long long ldc = 0;
  const void* residual = nullptr;
  long long ldr = 0;
};
void gemm_mx(const MxGemmDesc& d, cudaStream_t stream);

// ---- embedding -----------------------------------------------------------------------------
void embedding_fwd(const int64_t* ids, const void* table, void* out, int M, int H, cudaStream_t s);
// dtable_f32[ids[m], :] += dout[m, :]   (skips padding_idx)
void embedding_bwd(const int64_t* ids, const void* dout, float* dtable, int M, int H, long long padding_idx, cudaStream_t s);
// deterministic: ids sorted ascending (stable) with their source positions; one writer per table row, fixed summation order
void embedding_bwd_sorted(const int64_t* sorted_ids, const int64_t* perm, const void* dout, float* dtable, int M, int H,
                          long long padding_idx, cudaStream_t s);

// ---- loss ----------------------------------------------------------------------------------
// Row-wise softmax cross-entropy over logits [M, ld] (V valid columns), in place:
//   loss_sum += sum_m nll(m);  count += #valid rows;  logits <- (softmax - onehot) * grad_scale  (0 for ignored rows)
void cross_entropy_fwd_bwd(void* logits, long long ld, const int64_t* labels, int M, int V, float grad_scale,
                           long long ignore_index, float* loss_sum, float* count, cudaStream_t s);

// ---- misc ----------------------------------------------------------------------------------
void transpose_bf16(const void* in, long long ld_in, void* out, long long ld_out, int R, int C, cudaStream_t s);  // out[C,R]
void add_bf16(const void* a, const void* b, void* out, long long n, cudaStream_t s);
void cast_f32_to_bf16(const float* in, void* out, long long n, float scale, cudaStream_t s);
void fill_uniform_hash(void* out, int R, int C, long long ld, uint32_t seed, float bound, cudaStream_t s);  // kaiming re-init
void seed_advance(uint32_t* seed, cudaStream_t s);  // *seed = lowbias32(*seed + 0x9E3779B9)

// ---- optimizer -----------------------------------------------------------------------------
// AdamW on flat buffers.  grad may be bf16 or fp32; state bf16 or fp32.  grad_scale / skip are device scalars
// (may be null => 1 / false).  lr comes from the host (scheduler).  step_dev (nullable): device-resident step count that
// replaces `step` in the bias corrections (it only advances on updates that were not NaN-skipped).
void adamw_flat(void* param, const void* grad, bool grad_f32, void* exp_avg, void* exp_avg_sq, bool state_f32, long long n,
                float lr, float beta1, float beta2, float eps, float weight_decay, int step, const float* grad_scale,
                float grad_scale_host, const float* skip, const float* step_dev, cudaStream_t s);
// out[0] += sum(x^2)  (fp32 accumulate; x bf16 or fp32)
void sumsq(const void* x, bool is_f32, long long n, float* out, cudaStream_t s);
void random_prune(void* x, bool is_f32, long long n, float ratio, uint32_t seed, long long col_offset, cudaStream_t s);
// zero every |x| <= thr[0]
void threshold_prune(void* x, bool is_f32, long long n, const float* thr, cudaStream_t s);
// magnitude histogram select: thr[0] = approx quantile(|x|, ratio) refined to an exact element value
void magnitude_quantile(const void* x, bool is_f32, long long n, float ratio, float* thr, void* workspace, cudaStream_t s);
size_t magnitude_quantile_workspace_bytes();

// ---- fp8 (E4M3) quantisation for the frozen-weight tensor-core path (fp8.cu) ---------------------------
// weights: amax -> scale -> quantise (scale / inv_scale are device scalars)
// w8t (optional): E4M3 copy of the transpose [C, R] for the input-gradient GEMM
void fp8_quantize_weight(const void* w, long long ld, void* w8, long long ld8, void* w8t, long long ld8t, int R, int C,
                         float* amax_scratch, float* scale, float* inv_scale, cudaStream_t s);
// activations: x8 = sat_e4m3(x * *inv_scale); |x| amax recorded into *amax_cur (may be null)
void fp8_quantize_act(const void* x, long long ld, void* x8, long long ld8, int R, int C, const float* inv_scale, float* amax_cur,
                      bool e5m2, cudaStream_t s);
// once per micro-step: rotate the per-site amax state and derive 1/s_x, s_x*s_w and 1/(s_x*s_w)
// sites [0, n_e4m3) are E4M3 activations, the rest E5M2 gradients
void fp8_prep(float* state, const float* w_scale, float* inv_sx, float* alpha_main, float* alpha_inv, int n, float margin,
              int n_e4m3, cudaStream_t s);

}  // namespace rb
