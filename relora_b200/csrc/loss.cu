// Softmax cross-entropy over one chunk of LM-head logits, forward and backward in a single pass, in place.
// The [tokens, V] logits of the whole batch are never materialised (reference: modeling_llama.py:692-708 builds
// the full bf16 [B,T,V] tensor, a shifted contiguous copy and fp32 gradients): the LM-head GEMM produces a chunk of
// rows, this kernel turns it into d(logits) and the following GEMMs consume it.
#include "common.cuh"
#include "kernels.h"

namespace rb {

// One block per row.  The row (V <= 64K bf16) is staged in shared memory once: max, sum(exp), then gradients.
__global__ void __launch_bounds__(512) ce_kernel(bf16* __restrict__ logits, long long ld, const int64_t* __restrict__ labels, int V,
                                                 float grad_scale, long long ignore_index, float* __restrict__ loss_sum,
                                                 float* __restrict__ count) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ __align__(16) uint8_t ce_smem[];
  bf16* row_s = reinterpret_cast<bf16*>(ce_smem);
  __shared__ float scratch[32];
  const int row = blockIdx.x;
  bf16* rp = logits + (long long)row * ld;
  const long long label = labels[row];
  const int nvec = V / 8;  // vector part; tail handled scalar
  const bool ignored = (label == ignore_index);

  if (ignored) {
    for (int c = threadIdx.x; c < nvec; c += blockDim.x) reinterpret_cast<uint4*>(rp)[c] = make_uint4(0, 0, 0, 0);
    for (int c = nvec * 8 + threadIdx.x; c < V; c += blockDim.x) rp[c] = __float2bfloat16_rn(0.f);
    return;
  }
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < nvec; c += blockDim.x) {
    const bf16x8 t = reinterpret_cast<const bf16x8*>(rp)[c];
    reinterpret_cast<bf16x8*>(row_s)[c] = t;
    float f[8];
    unpack8(t, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) mx = fmaxf(mx, f[j]);
  }
  for (int c = nvec * 8 + threadIdx.x; c < V; c += blockDim.x) {
    row_s[c] = rp[c];
    mx = fmaxf(mx, __bfloat162float(rp[c]));
  }
  mx = block_max(mx, scratch);
  float se = 0.f;
  for (int c = threadIdx.x; c < nvec; c += blockDim.x) {
    float f[8];
    unpack8(reinterpret_cast<const bf16x8*>(row_s)[c], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) se += __expf(f[j] - mx);
  }
  for (int c = nvec * 8 + threadIdx.x; c < V; c += blockDim.x) se += __expf(__bfloat162float(row_s[c]) - mx);
  se = block_sum(se, scratch);
  const float inv = 1.f / se;
  if (threadIdx.x == 0) {
    const float xl = __bfloat162float(row_s[label]);
    atomicAdd(loss_sum, logf(se) + mx - xl);
    atomicAdd(count, 1.f);
  }
  for (int c = threadIdx.x; c < nvec; c += blockDim.x) {
    float f[8];
    unpack8(reinterpret_cast<const bf16x8*>(row_s)[c], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float pr = __expf(f[j] - mx) * inv;
      if (c * 8 + j == label) pr -= 1.f;
      f[j] = pr * grad_scale;
    }
    reinterpret_cast<bf16x8*>(rp)[c] = pack8(f);
  }
  for (int c = nvec * 8 + threadIdx.x; c < V; c += blockDim.x) {
    float pr = __expf(__bfloat162float(row_s[c]) - mx) * inv;
    if (c == label) pr -= 1.f;
    rp[c] = __float2bfloat16_rn(pr * grad_scale);
  }
}

void cross_entropy_fwd_bwd(void* logits, long long ld, const int64_t* labels, int M, int V, float grad_scale, long long ignore_index,
                           float* loss_sum, float* count, cudaStream_t s) {
  const size_t smem = ((size_t)V * 2 + 15) & ~size_t(15);
  if (smem > 200 * 1024) throw std::runtime_error("cross_entropy: vocabulary too large for the single-pass kernel");
  static size_t configured = 0;
  if (smem > configured) {
    check(cudaFuncSetAttribute(ce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute(ce)");
    configured = smem;
  }
  launch_k(ce_kernel, M, 512, smem, s, (bf16*)logits, ld, labels, V, grad_scale, ignore_index, loss_sum, count);
  RB_CHECK_LAUNCH("cross_entropy");
}

}  // namespace rb
