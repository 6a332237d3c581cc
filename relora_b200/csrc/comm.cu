// Hand-written NVLink collectives for the data-parallel update (sm_90a, NVLink 4 / NVSwitch).
//
// The reference all-reduces every gradient bucket through NCCL on every micro-batch (DDP without no_sync,
// torchrun_main.py:616-622, 796-800) and then runs clip_grad_norm_ and torch.optim.AdamW as separate passes.
// Here one kernel chain per *update* does: bf16 cast -> peer-memory reduce-scatter (128-bit P2P loads, or
// multimem.ld_reduce when an NVLS multicast mapping exists) with fp32 accumulation and sum(g^2) -> norm exchange ->
// AdamW on the owned shard -> broadcast of the new bf16 parameters into every peer's parameter buffer
// (P2P stores or multimem.st).  Cross-GPU ordering uses release/acquire flags in symmetric memory.
#include "comm.h"

#include "common.cuh"

namespace rb {

// ---------------------------------------------------------------------------------------------- flag primitives
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t gtimer() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// Signal every peer and wait for every peer (threads 0..world-1 of one block).  Flags are monotonically increasing
// epochs, so no reset (and no reset race) is needed.  A 20 s watchdog turns a lost peer into a trap, not a hang.
__device__ __forceinline__ void barrier_threads(const CommCtx& c, int set, uint32_t epoch) {
  const int t = threadIdx.x;
  if (t < c.world) {
    __threadfence_system();
    uint32_t* remote = reinterpret_cast<uint32_t*>(c.flags.ptr[t]) + set * kMaxPeers + c.rank;
    st_release_sys(remote, epoch);
    const uint32_t* mine = reinterpret_cast<const uint32_t*>(c.flags.ptr[c.rank]) + set * kMaxPeers + t;
    const uint64_t t0 = gtimer();
    while (ld_acquire_sys(mine) < epoch) {
      if (gtimer() - t0 > 20000000000ull) {
        printf("xgpu barrier timeout: rank %d waiting for rank %d (set %d epoch %u)\n", c.rank, t, set, epoch);
        __trap();
      }
    }
  }
  __syncthreads();
}

__global__ void barrier_kernel(const CommCtx c, int set, uint32_t epoch) { barrier_threads(c, set, epoch); }

void xgpu_barrier(const CommCtx& c, int set, uint32_t epoch, cudaStream_t s) {
  barrier_kernel<<<1, 32, 0, s>>>(c, set, epoch);
  RB_CHECK_LAUNCH("xgpu_barrier");
}

// ---------------------------------------------------------------------------------------------- data movement
__device__ __forceinline__ uint4 ld_peer(const void* p) {  // L1 is clean at kernel entry; bypass it anyway for peer data
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_peer(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// in-switch reduction of 8 bf16 over all ranks of the multicast group (fp32 accumulation inside the switch)
__device__ __forceinline__ uint4 mc_ld_reduce_bf16x8(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ void mc_st(void* mc, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// All `WORLD` peer loads of one 16-byte vector are issued before the first add (the loop is fully unrolled), so a thread keeps
// WORLD x U requests in flight across the ~2 us NVLink round trip instead of one.
template <int WORLD>
__device__ __forceinline__ void reduce_vec_p2p(const PeerPtrs& bufs, int rank, long long vec_index, float (&acc)[8]) {
  uint4 raw[WORLD];
#pragma unroll
  for (int k = 0; k < WORLD; ++k) {
    const int p = (rank + k) % WORLD;  // start with the local copy, spread the first remote requests over peers
    raw[k] = ld_peer(reinterpret_cast<const uint4*>(bufs.ptr[p]) + vec_index);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
  for (int k = 0; k < WORLD; ++k) {
    float f[8];
    unpack8(raw[k], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += f[j];
  }
}
__device__ __forceinline__ void reduce_vec(const PeerPtrs& bufs, const void* mc, int world, int rank, long long vec_index, float (&acc)[8]) {
  if (mc != nullptr) {
    unpack8(mc_ld_reduce_bf16x8(reinterpret_cast<const uint4*>(mc) + vec_index), acc);
    return;
  }
  switch (world) {
    case 2: reduce_vec_p2p<2>(bufs, rank, vec_index, acc); break;
    case 3: reduce_vec_p2p<3>(bufs, rank, vec_index, acc); break;
    case 4: reduce_vec_p2p<4>(bufs, rank, vec_index, acc); break;
    case 5: reduce_vec_p2p<5>(bufs, rank, vec_index, acc); break;
    case 6: reduce_vec_p2p<6>(bufs, rank, vec_index, acc); break;
    case 7: reduce_vec_p2p<7>(bufs, rank, vec_index, acc); break;
    case 8: reduce_vec_p2p<8>(bufs, rank, vec_index, acc); break;
    default: reduce_vec_p2p<1>(bufs, rank, vec_index, acc); break;
  }
}
__device__ __forceinline__ void broadcast_vec(const PeerPtrs& bufs, void* mc, int world, long long vec_index, const uint4& v) {
  if (mc != nullptr) {
    mc_st(reinterpret_cast<uint4*>(mc) + vec_index, v);
    return;
  }
#pragma unroll 1
  for (int p = 0; p < world; ++p) st_peer(reinterpret_cast<uint4*>(bufs.ptr[p]) + vec_index, v);
}

// ---------------------------------------------------------------------------------------------- plain all-reduce
// Block 0 runs the entry barrier and releases the other blocks through `local_go`; the last block to finish runs
// the exit barrier (ticket in local_go[1]).
__global__ void __launch_bounds__(512) allreduce_kernel(const CommCtx c, const PeerPtrs bufs, void* mc, long long off_vec, long long n_vec,
                                                        uint32_t epoch0) {
  if (blockIdx.x == 0) {
    barrier_threads(c, 0, epoch0);
    if (threadIdx.x == 0) {
      __threadfence();
      atomicExch(c.local_go, epoch0);
    }
  } else {
    if (threadIdx.x == 0) {
      while (atomicAdd(c.local_go, 0u) < epoch0) {}
    }
    __syncthreads();
  }
  const long long per = (n_vec + c.world - 1) / c.world;
  const long long lo = off_vec + per * c.rank;
  const long long hi = min(off_vec + n_vec, lo + per);
  // four independent vectors per thread per trip keep enough loads in flight to cover the ~2 us NVLink round trip
  constexpr int U = 4;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i0 = lo + blockIdx.x * (long long)blockDim.x + threadIdx.x; i0 < hi; i0 += stride * U) {
    float acc[U][8];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + u * stride;
      if (i < hi) reduce_vec(bufs, mc, c.world, c.rank, i, acc[u]);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + u * stride;
      if (i < hi) broadcast_vec(bufs, mc, c.world, i, pack8(acc[u]));
    }
  }
  __threadfence_system();
  __syncthreads();
  __shared__ bool last;
  if (threadIdx.x == 0) last = (atomicAdd(c.local_go + 1, 1u) == gridDim.x - 1);
  __syncthreads();
  if (last) {
    if (threadIdx.x == 0) c.local_go[1] = 0u;
    barrier_threads(c, 1, epoch0);
  }
}

void allreduce_bf16(const CommCtx& c, const PeerPtrs& bufs, void* mc, long long off_elems, long long n, uint32_t epoch0, int max_blocks,
                    cudaStream_t s) {
  if (n % 8 || off_elems % 8) throw std::runtime_error("allreduce: element counts must be multiples of 8");
  const long long n_vec = n / 8;
  const long long per = (n_vec + c.world - 1) / c.world;
  int grid = (int)std::min<long long>((per + 511) / 512, (long long)max_blocks);
  if (grid < 1) grid = 1;
  allreduce_kernel<<<grid, 512, 0, s>>>(c, bufs, mc, off_elems / 8, n_vec, epoch0);
  RB_CHECK_LAUNCH("allreduce_bf16");
}

// ---------------------------------------------------------------------------------------------- fused update
__global__ void __launch_bounds__(512) cast_to_symm_kernel(const float* __restrict__ g, bf16* __restrict__ out, long long n_vec) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
    const float4 a = reinterpret_cast<const float4*>(g)[2 * i], b = reinterpret_cast<const float4*>(g)[2 * i + 1];
    const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    reinterpret_cast<uint4*>(out)[i] = pack8(f);
  }
}

__global__ void __launch_bounds__(512) reduce_scatter_kernel(const CommCtx c, const PeerPtrs bufs, const void* mc, long long chunk_vec,
                                                             float* __restrict__ gred, float* __restrict__ sq_accum) {
  __shared__ float scratch[32];
  const long long lo = chunk_vec * c.rank;
  float sq = 0.f;
  constexpr int U = 2;  // independent vectors per thread per trip (x world peer loads each)
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i0 = blockIdx.x * (long long)blockDim.x + threadIdx.x; i0 < chunk_vec; i0 += stride * U) {
    float acc[U][8];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + u * stride;
      if (i < chunk_vec) reduce_vec(bufs, mc, c.world, c.rank, lo + i, acc[u]);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + u * stride;
      if (i < chunk_vec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) sq += acc[u][j] * acc[u][j];
        reinterpret_cast<float4*>(gred)[2 * i] = make_float4(acc[u][0], acc[u][1], acc[u][2], acc[u][3]);
        reinterpret_cast<float4*>(gred)[2 * i + 1] = make_float4(acc[u][4], acc[u][5], acc[u][6], acc[u][7]);
      }
    }
  }
  sq = block_sum(sq, scratch);
  if (threadIdx.x == 0) atomicAdd(sq_accum, sq);
}

// one block: publish this rank's sum(g^2) -- and its mean loss / NaN flag, the reference's `loss_info` all-reduce (torchrun_main.py:810)
// -- to every peer, barrier, combine -> clip coefficient, mean loss over ranks, "skip if any rank saw a NaN loss"
__global__ void norm_exchange_kernel(const CommCtx c, const float* __restrict__ sq_accum, float max_norm, float inv_world, uint32_t epoch,
                                     float* __restrict__ grad_scale, float* __restrict__ norm_out, const float* __restrict__ loss_in,
                                     const float* __restrict__ skip_in, float* __restrict__ loss_out, float* __restrict__ skip_out) {
  const int t = threadIdx.x;
  if (t < c.world) {
    float* slot = reinterpret_cast<float*>(reinterpret_cast<uint32_t*>(c.flags.ptr[t]) + 4 * kMaxPeers) + c.rank;
    *reinterpret_cast<volatile float*>(slot) = *sq_accum;
    *reinterpret_cast<volatile float*>(slot + kMaxPeers) = loss_in != nullptr ? *loss_in : 0.f;
    *reinterpret_cast<volatile float*>(slot + 2 * kMaxPeers) = skip_in != nullptr ? *skip_in : 0.f;
  }
  barrier_threads(c, 2, epoch);
  if (t == 0) {
    const volatile float* mine = reinterpret_cast<const volatile float*>(reinterpret_cast<const uint32_t*>(c.flags.ptr[c.rank]) + 4 * kMaxPeers);
    float tot = 0.f, loss = 0.f, skip = 0.f;
    for (int p = 0; p < c.world; ++p) {
      tot += mine[p];
      loss += mine[kMaxPeers + p];
      skip += (mine[2 * kMaxPeers + p] != 0.f) ? 1.f : 0.f;  // fixed order: bit-identical on every rank
    }
    const float norm = sqrtf(tot) * inv_world;  // norm of the rank-averaged gradient
    float coef = 1.f;
    if (max_norm > 0.f) coef = fminf(1.f, max_norm / (norm + 1e-6f));
    // a non-finite gradient norm poisons the scale on purpose: the Adam stage skips the update (see adam_allgather_kernel)
    *grad_scale = (norm < INFINITY) ? coef * inv_world : __int_as_float(0x7fc00000);
    *norm_out = norm;
    if (loss_out != nullptr) *loss_out = loss * inv_world;
    *skip_out = skip;
  }
}

__global__ void __launch_bounds__(512) adam_allgather_kernel(const CommCtx c, const PeerPtrs params, void* param_mc, long long chunk_vec,
                                                             const float* __restrict__ gred, bf16* __restrict__ m, bf16* __restrict__ v,
                                                             float lr, float b1, float b2, float eps, float wd, float bc1_inv, float bc2_rsqrt,
                                                             const float* __restrict__ grad_scale, const float* __restrict__ skip,
                                                             const float* __restrict__ step_dev) {
  if (skip != nullptr && *skip != 0.f) return;
  if (step_dev != nullptr) {
    const float t = fmaxf(*step_dev, 1.f);
    bc1_inv = 1.f / (1.f - powf(b1, t));
    bc2_rsqrt = 1.f / sqrtf(1.f - powf(b2, t));
  }
  const float gs = *grad_scale;
  if (!(fabsf(gs) < INFINITY)) return;  // non-finite gradient norm: leave parameters and moments untouched on every rank
  const float decay = 1.f - lr * wd, step_size = lr * bc1_inv;
  const long long lo = chunk_vec * c.rank;
  const uint4* plocal = reinterpret_cast<const uint4*>(params.ptr[c.rank]);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < chunk_vec; i += (long long)gridDim.x * blockDim.x) {
    float pf[8], mf[8], vf[8];
    unpack8(plocal[lo + i], pf);
    unpack8(reinterpret_cast<const uint4*>(m)[i], mf);
    unpack8(reinterpret_cast<const uint4*>(v)[i], vf);
    const float4 g0 = reinterpret_cast<const float4*>(gred)[2 * i], g1 = reinterpret_cast<const float4*>(gred)[2 * i + 1];
    const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float gr = g[j] * gs;
      mf[j] = b1 * mf[j] + (1.f - b1) * gr;
      vf[j] = b2 * vf[j] + (1.f - b2) * gr * gr;
      pf[j] = pf[j] * decay - step_size * (mf[j] / (sqrtf(vf[j]) * bc2_rsqrt + eps));
    }
    reinterpret_cast<uint4*>(m)[i] = pack8(mf);
    reinterpret_cast<uint4*>(v)[i] = pack8(vf);
    broadcast_vec(params, param_mc, c.world, lo + i, pack8(pf));
  }
}

void fused_update(const CommCtx& c, const FusedUpdateArgs& a, uint32_t epoch0, cudaStream_t s) {
  if (a.n % (8LL * c.world)) throw std::runtime_error("fused_update: n must be a multiple of 8 * world");
  const long long n_vec = a.n / 8, chunk_vec = n_vec / c.world;
  const int blocks = std::max(1, std::min<int>(a.max_blocks, (int)((chunk_vec + 511) / 512)));
  check(cudaMemsetAsync(a.sq_accum, 0, sizeof(float), s), "memset(sq_accum)");
  if (a.grads_f32 != nullptr) {  // null: the bf16 gradients already live in the symmetric buffer (module path: .grad views)
    const int cast_blocks = (int)std::min<long long>((n_vec + 511) / 512, (long long)num_sms() * 4);
    cast_to_symm_kernel<<<cast_blocks, 512, 0, s>>>(a.grads_f32, reinterpret_cast<bf16*>(a.grad_bufs.ptr[c.rank]), n_vec);
    RB_CHECK_LAUNCH("cast_to_symm");
  }
  xgpu_barrier(c, 0, epoch0, s);  // every rank's bf16 gradients are in place
  reduce_scatter_kernel<<<blocks, 512, 0, s>>>(c, a.grad_bufs, a.grad_mc, chunk_vec, a.gred, a.sq_accum);
  RB_CHECK_LAUNCH("reduce_scatter");
  float* grad_scale = a.sq_accum + 1;
  float* skip_all = a.sq_accum + 2;  // "some rank saw a NaN loss" (or the caller's already-global flag)
  norm_exchange_kernel<<<1, 32, 0, s>>>(c, a.sq_accum, a.max_norm, a.inv_world, epoch0, grad_scale, a.norm_out, a.loss_in, a.skip, a.loss_out,
                                        skip_all);
  RB_CHECK_LAUNCH("norm_exchange");
  const float bc1_inv = 1.f / (1.f - powf(a.beta1, (float)a.step));
  const float bc2_rsqrt = 1.f / sqrtf(1.f - powf(a.beta2, (float)a.step));
  adam_allgather_kernel<<<blocks, 512, 0, s>>>(c, a.param_bufs, a.param_mc, chunk_vec, a.gred, reinterpret_cast<bf16*>(a.exp_avg),
                                               reinterpret_cast<bf16*>(a.exp_avg_sq), a.lr, a.beta1, a.beta2, a.eps, a.weight_decay, bc1_inv,
                                               bc2_rsqrt, grad_scale, skip_all, a.step_dev);
  RB_CHECK_LAUNCH("adam_allgather");
  xgpu_barrier(c, 1, epoch0, s);  // every replica holds the new parameters before the next forward starts
}

}  // namespace rb
