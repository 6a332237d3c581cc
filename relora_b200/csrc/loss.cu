// Softmax cross-entropy over one chunk of LM-head logits, forward and backward in a single pass, in place.
// The [tokens, V] logits of the whole batch are never materialised (reference: modeling_llama.py:692-708 builds
// the full bf16 [B,T,V] tensor, a shifted contiguous copy and fp32 gradients): the LM-head GEMM produces a chunk of
// rows, this kernel turns it into d(logits) and the following GEMMs consume it.
#include "common.cuh"
#include "kernels.h"

namespace rb {

// One block per row.  The row (V <= 102,400 bf16) is staged in shared memory once: max, sum(exp), then gradients.
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

// Rows longer than the staging buffer (V > 102,400, e.g. Llama-3's 128,256) are streamed from global memory instead: one block
// per row reads it three times (max, sum(exp), gradients) with the same per-element arithmetic as ce_kernel.  Each thread
// reads and writes the same vectors in every pass, so a thread overwrites only elements no other thread reads; the label's
// logit is read in pass 1, before the block barriers that precede every write.  1024 threads and at most 64 registers keep
// one block per SM, so the rows in flight (132 x 256 KB at V = 128,256) fit in L2 and passes 2 and 3 find part of them there.
constexpr int kCeStreamThreads = 1024;
constexpr int kCeStreamUnroll = 4;  // 16-byte loads each thread keeps in flight

// Calls f(c, v) for this thread's vectors c = threadIdx.x + k·blockDim.x < nvec in increasing order (the order ce_kernel
// visits them), loading kCeStreamUnroll of them before using any.
template <typename F>
__device__ __forceinline__ void ce_row_vectors(const bf16x8* rv, int nvec, F&& f) {
  constexpr int U = kCeStreamUnroll;
  const int nt = blockDim.x;
  int c = threadIdx.x;
  for (; c + (U - 1) * nt < nvec; c += U * nt) {
    bf16x8 t[U];
#pragma unroll
    for (int u = 0; u < U; ++u) t[u] = rv[c + u * nt];
#pragma unroll
    for (int u = 0; u < U; ++u) f(c + u * nt, t[u]);
  }
  for (; c < nvec; c += nt) f(c, rv[c]);
}

__global__ void __launch_bounds__(kCeStreamThreads, 1) ce_stream_kernel(bf16* __restrict__ logits, long long ld,
                                                                        const int64_t* __restrict__ labels, int V, float grad_scale,
                                                                        long long ignore_index, float* __restrict__ loss_sum,
                                                                        float* __restrict__ count) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float scratch[32];
  bf16* rp = logits + (long long)blockIdx.x * ld;
  bf16x8* rv = reinterpret_cast<bf16x8*>(rp);
  const long long label = labels[blockIdx.x];
  const int nvec = V / 8;                 // vector part
  const int tail = nvec * 8 + threadIdx.x;  // the last V % 8 columns, one per thread

  if (label == ignore_index) {
    for (int c = threadIdx.x; c < nvec; c += blockDim.x) rv[c] = make_uint4(0, 0, 0, 0);
    if (tail < V) rp[tail] = __float2bfloat16_rn(0.f);
    return;
  }
  // pass 1: max, and the label's logit before anything is overwritten
  float mx = -INFINITY;
  ce_row_vectors(rv, nvec, [&](int, const bf16x8& v) {
    float f[8];
    unpack8(v, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) mx = fmaxf(mx, f[j]);
  });
  if (tail < V) mx = fmaxf(mx, __bfloat162float(rp[tail]));
  const float xl = threadIdx.x == 0 ? __bfloat162float(rp[label]) : 0.f;
  mx = block_max(mx, scratch);
  // pass 2: sum(exp(x - max))
  float se = 0.f;
  ce_row_vectors(rv, nvec, [&](int, const bf16x8& v) {
    float f[8];
    unpack8(v, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) se += __expf(f[j] - mx);
  });
  if (tail < V) se += __expf(__bfloat162float(rp[tail]) - mx);
  se = block_sum(se, scratch);
  const float inv = 1.f / se;
  if (threadIdx.x == 0) {
    atomicAdd(loss_sum, logf(se) + mx - xl);
    atomicAdd(count, 1.f);
  }
  // pass 3: gradients, each written over the vector it was computed from
  ce_row_vectors(rv, nvec, [&](int c, const bf16x8& v) {
    float f[8];
    unpack8(v, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float pr = __expf(f[j] - mx) * inv;
      if (c * 8 + j == label) pr -= 1.f;
      f[j] = pr * grad_scale;
    }
    rv[c] = pack8(f);
  });
  if (tail < V) {
    float pr = __expf(__bfloat162float(rp[tail]) - mx) * inv;
    if (tail == label) pr -= 1.f;
    rp[tail] = __float2bfloat16_rn(pr * grad_scale);
  }
}

// Longest row ce_kernel stages in shared memory; longer rows take ce_stream_kernel.
constexpr size_t kCeStageBytes = 200 * 1024;

void cross_entropy_fwd_bwd(void* logits, long long ld, const int64_t* labels, int M, int V, float grad_scale, long long ignore_index,
                           float* loss_sum, float* count, cudaStream_t s) {
  const size_t smem = ((size_t)V * 2 + 15) & ~size_t(15);
  if (smem > kCeStageBytes) {
    launch_k(ce_stream_kernel, M, kCeStreamThreads, 0, s, (bf16*)logits, ld, labels, V, grad_scale, ignore_index, loss_sum, count);
    RB_CHECK_LAUNCH("cross_entropy");
    return;
  }
  static size_t configured = 0;
  if (smem > configured) {
    check(cudaFuncSetAttribute(ce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute(ce)");
    configured = smem;
  }
  launch_k(ce_kernel, M, 512, smem, s, (bf16*)logits, ld, labels, V, grad_scale, ignore_index, loss_sum, count);
  RB_CHECK_LAUNCH("cross_entropy");
}

}  // namespace rb
