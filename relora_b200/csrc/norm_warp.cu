// Warp-per-row RMSNorm forward / backward for H <= 2048 (one 128-bit vector per lane per step, no block barriers).
// Reference op: LlamaRMSNorm, peft_pretraining/modeling_llama.py:74-91 (normalise in fp32, round to bf16, then multiply by the
// bf16 weight -- the rounding order is kept); the dropout-expanded copies feed relora.py:321 (nn.Dropout on the LoRA input).
//
// forward : y = w * bf16(x * rstd) (+ G dropout-expanded copies for the LoRA down-projections), rstd saved
// backward: dx = rstd * (g - xhat * mean(g * xhat)) + dx_add,  g = dy * w
//           dw += sum_rows dy * bf16(xhat): per-lane fp32 partials -> block partial (smem) -> red.global.add.v4.f32
#include "common.cuh"
#include "kernels.h"

namespace rb {

constexpr int kWarpsPerBlock = 8;

template <int VPL>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) rmsnorm_fwd_warp_kernel(
    const bf16* __restrict__ x, const bf16* __restrict__ w, bf16* __restrict__ y, float* __restrict__ rstd_out, int M, int H, float eps,
    bf16* __restrict__ xd, int G, const uint32_t* __restrict__ seed_ptr, uint4 keys, uint32_t thr16, float inv_keep, Fp8Out f8, MxOut mo) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int row = blockIdx.x * kWarpsPerBlock + warp;
  if (row >= M) return;
  const int nvec = H / 8;
  const uint4* xr = reinterpret_cast<const uint4*>(x + (long long)row * H);
  uint4 xv[VPL];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c = lane + i * 32;
    if (c < nvec) {
      xv[i] = xr[c];
      float f[8];
      unpack8(xv[i], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) ss += f[j] * f[j];
    }
  }
  ss = warp_sum(ss);
  const float rstd = rsqrtf(ss / (float)H + eps);
  if (lane == 0) rstd_out[row] = rstd;
  uint32_t s0 = 0, s1 = 0, s2 = 0, s3 = 0;
  if (G > 0) {
    const uint32_t base = seed_ptr ? *seed_ptr : 0u;
    s0 = mix_seed(base, keys.x); s1 = mix_seed(base, keys.y); s2 = mix_seed(base, keys.z); s3 = mix_seed(base, keys.w);
  }
  const uint4* wr = reinterpret_cast<const uint4*>(w);
  uint4* yr = reinterpret_cast<uint4*>(y + (long long)row * H);
  const float q_inv = f8.q != nullptr ? *f8.inv_scale : 0.f;
  float q_max = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c = lane + i * 32;
    if (c < nvec) {
      float f[8], wf[8], o[8];
      unpack8(xv[i], f);
      unpack8(wr[c], wf);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = bf16_round(wf[j] * bf16_round(f[j] * rstd));
      yr[c] = pack8(o);
      if (mo.q != nullptr) mx_emit8(mo, row, c * 8, o, mx_group_mask());  // H % 128 == 0: whole 4-lane groups are active
      if (f8.q != nullptr) {
        *reinterpret_cast<uint2*>(f8.q + (long long)row * f8.ld + c * 8) = pack8_e4m3(o, q_inv);
        q_max = fmaxf(q_max, absmax8(o));
      }
#pragma unroll 1
      for (int g = 0; g < G; ++g) {
        const uint32_t sd = g == 0 ? s0 : (g == 1 ? s1 : (g == 2 ? s2 : s3));
        float d[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) d[j] = keep_drop(sd, (uint32_t)row, (uint32_t)(c * 8 + j), thr16) ? o[j] * inv_keep : 0.f;
        reinterpret_cast<uint4*>(xd + ((long long)row * G + g) * H)[c] = pack8(d);
      }
    }
  }
  if (f8.q != nullptr) amax_commit(q_max, f8.amax);
}

template <int VPL>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) rmsnorm_bwd_warp_kernel(
    const bf16* __restrict__ dy, const bf16* __restrict__ x, const bf16* __restrict__ w, const float* __restrict__ rstd,
    const bf16* __restrict__ dx_add, bf16* __restrict__ dx, float* __restrict__ dw, int M, int H) {
  extern __shared__ float sdw[];  // [H] block partial of dw
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nvec = H / 8;
  for (int c = threadIdx.x; c < H; c += blockDim.x) sdw[c] = 0.f;
  __syncthreads();
  uint4 wv[VPL];
  float dwacc[VPL][8];
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c = lane + i * 32;
    wv[i] = (c < nvec) ? reinterpret_cast<const uint4*>(w)[c] : make_uint4(0, 0, 0, 0);
#pragma unroll
    for (int j = 0; j < 8; ++j) dwacc[i][j] = 0.f;
  }
  const int stride = gridDim.x * kWarpsPerBlock;
  int row = blockIdx.x * kWarpsPerBlock + warp;
  // software pipeline: the loads of the next row are in flight while the current one is reduced and written
  uint4 ndy[VPL], nx[VPL], nadd[VPL];
  float nrs = 0.f;
  auto fetch = [&](int r) {
    if (r < M) {
      nrs = rstd[r];
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        const int c = lane + i * 32;
        if (c < nvec) {
          ndy[i] = reinterpret_cast<const uint4*>(dy + (long long)r * H)[c];
          nx[i] = reinterpret_cast<const uint4*>(x + (long long)r * H)[c];
          if (dx_add != nullptr) nadd[i] = reinterpret_cast<const uint4*>(dx_add + (long long)r * H)[c];
        }
      }
    }
  };
  constexpr bool kPrefetch = VPL <= 4;  // double-buffering 8 vectors per lane would spill
  if (kPrefetch) fetch(row);
  for (; row < M; row += stride) {
    uint4 dyv[VPL], xv[VPL], addv[VPL];
    if (!kPrefetch) fetch(row);
    const float rs = nrs;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      dyv[i] = ndy[i];
      xv[i] = nx[i];
      addv[i] = nadd[i];
    }
    if (kPrefetch) fetch(row + stride);
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int c = lane + i * 32;
      if (c < nvec) {
        float dyf[8], xf[8], wf[8];
        unpack8(dyv[i], dyf);
        unpack8(xv[i], xf);
        unpack8(wv[i], wf);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xh = xf[j] * rs;
          dot += dyf[j] * wf[j] * xh;
          dwacc[i][j] += dyf[j] * bf16_round(xh);
        }
      }
    }
    dot = warp_sum(dot) / (float)H;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int c = lane + i * 32;
      if (c < nvec) {
        float dyf[8], xf[8], wf[8], o[8];
        unpack8(dyv[i], dyf);
        unpack8(xv[i], xf);
        unpack8(wv[i], wf);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rs * (dyf[j] * wf[j] - xf[j] * rs * dot);
        if (dx_add != nullptr) {
          float a[8];
          unpack8(addv[i], a);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += a[j];
        }
        reinterpret_cast<uint4*>(dx + (long long)row * H)[c] = pack8(o);
      }
    }
  }
  // ---- dw: lanes -> block partial in shared memory -> one 16-byte vector reduction per 4 columns per block
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c = lane + i * 32;
    if (c < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) atomicAdd(&sdw[c * 8 + j], dwacc[i][j]);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x * 4; c < H; c += blockDim.x * 4) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dw + c), "f"(sdw[c]), "f"(sdw[c + 1]), "f"(sdw[c + 2]), "f"(sdw[c + 3])
                 : "memory");
  }
}

static int pick_vpl(int nvec) {
  const int need = (nvec + 31) / 32;
  for (int v : {1, 2, 3, 4, 8}) if (need <= v) return v;
  return 0;
}

bool rmsnorm_fwd_warp(const void* x, const void* w, void* y, float* rstd, int M, int H, float eps, void* xd, int G,
                      const uint32_t* seed_ptr, uint4 keys, uint32_t thr16, float inv_keep, Fp8Out f8, MxOut mo, cudaStream_t s) {
  const int vpl = pick_vpl(H / 8);
  if (vpl == 0) return false;
  const int grid = ceil_div(M, kWarpsPerBlock);
  const bf16 *xp = (const bf16*)x, *wp = (const bf16*)w;
  bf16 *yp = (bf16*)y, *xdp = (bf16*)xd;
#define L(V) launch_k(rmsnorm_fwd_warp_kernel<V>, grid, kWarpsPerBlock * 32, 0, s, xp, wp, yp, rstd, M, H, eps, xdp, G, seed_ptr, keys, thr16, inv_keep, f8, mo)
  switch (vpl) {
    case 1: L(1); break;
    case 2: L(2); break;
    case 3: L(3); break;
    case 4: L(4); break;
    default: L(8); break;
  }
#undef L
  RB_CHECK_LAUNCH("rmsnorm_fwd_warp");
  return true;
}

int rmsnorm_bwd_ws_blocks() { return 2 * num_sms(); }

bool rmsnorm_bwd_warp(const void* dy, const void* x, const void* w, const float* rstd, const void* dx_add, void* dx, float* dw, int M,
                      int H, float* ws, unsigned int* ticket, cudaStream_t s) {
  const int vpl = pick_vpl(H / 8);
  (void)ws; (void)ticket;  // kept in the signature for the workspace-based variant; dw now uses vector reductions
  if (vpl == 0 || (reinterpret_cast<uintptr_t>(dw) & 15) != 0) return false;
  const size_t smem = (size_t)H * sizeof(float);
  // exactly one resident wave: a second wave would pay the per-block prologue / dw reduction again for ~2 rows per warp
  static int occ[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (occ[vpl] == 0) {
    int n = 0;
#define O(V) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, rmsnorm_bwd_warp_kernel<V>, kWarpsPerBlock * 32, smem)
    switch (vpl) {
      case 1: O(1); break;
      case 2: O(2); break;
      case 3: O(3); break;
      case 4: O(4); break;
      default: O(8); break;
    }
#undef O
    occ[vpl] = n > 0 ? n : 1;
  }
  const int grid = std::min(ceil_div(M, kWarpsPerBlock), occ[vpl] * num_sms());
  const bf16 *a = (const bf16*)dy, *b = (const bf16*)x, *c = (const bf16*)w, *d = (const bf16*)dx_add;
#define L(V) launch_k(rmsnorm_bwd_warp_kernel<V>, grid, kWarpsPerBlock * 32, smem, s, a, b, c, rstd, d, (bf16*)dx, dw, M, H)
  switch (vpl) {
    case 1: L(1); break;
    case 2: L(2); break;
    case 3: L(3); break;
    case 4: L(4); break;
    default: L(8); break;
  }
#undef L
  RB_CHECK_LAUNCH("rmsnorm_bwd_warp");
  return true;
}

}  // namespace rb
