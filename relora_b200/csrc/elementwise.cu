// Bandwidth-bound fused kernels of the Llama hot path: RMSNorm fwd/bwd (+LoRA dropout expansion), rotary,
// SwiGLU, embedding, dropout combine, transpose, re-init.  128-bit accesses, fp32 math, one rounding at the end.
// Reference expressions being replaced: modeling_llama.py:83-91 (RMSNorm), :126-141 (rotary), :157-158 (SwiGLU),
// relora.py:244,321 (LoRA dropout), relora.py:303 (kaiming re-init).
#include "common.cuh"
#include "kernels.h"

namespace rb {

// ============================================================================================ RMSNorm
// one warp per row when H <= 1024*?; general: one block (256 threads) per row, row cached in registers
template <int VPT>  // bf16x8 vectors per thread
__global__ void __launch_bounds__(256) rmsnorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, bf16* __restrict__ y,
                                                          float* __restrict__ rstd_out, int M, int H, float eps, bf16* __restrict__ xd,
                                                          int G, const uint32_t* __restrict__ seed_ptr, uint4 keys, uint32_t thr16,
                                                          float inv_keep, MxOut mo) {
  __shared__ float scratch[32];
  const int row = blockIdx.x;
  const int nvec = H / 8;
  const bf16x8* xr = reinterpret_cast<const bf16x8*>(x + (long long)row * H);
  float v[VPT][8];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = threadIdx.x + i * 256;
    if (c < nvec) {
      unpack8(xr[c], v[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) ss += v[i][j] * v[i][j];
    }
  }
  ss = block_sum(ss, scratch);
  const float rstd = rsqrtf(ss / (float)H + eps);
  if (threadIdx.x == 0) rstd_out[row] = rstd;
  uint32_t seeds[4] = {0, 0, 0, 0};
  if (G > 0) {
    const uint32_t base = seed_ptr ? *seed_ptr : 0u;
    seeds[0] = mix_seed(base, keys.x); seeds[1] = mix_seed(base, keys.y);
    seeds[2] = mix_seed(base, keys.z); seeds[3] = mix_seed(base, keys.w);
  }
  const bf16x8* wr = reinterpret_cast<const bf16x8*>(w);
  bf16x8* yr = reinterpret_cast<bf16x8*>(y + (long long)row * H);
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = threadIdx.x + i * 256;
    if (c < nvec) {
      float wf[8], o[8];
      unpack8(wr[c], wf);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = bf16_round(wf[j] * bf16_round(v[i][j] * rstd));
      yr[c] = pack8(o);
      if (mo.q != nullptr) mx_emit8(mo, row, c * 8, o, mx_group_mask());  // H % 128 == 0: whole 4-thread groups are active
      for (int g = 0; g < G; ++g) {
        float d[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) d[j] = keep_drop(seeds[g], (uint32_t)row, (uint32_t)(c * 8 + j), thr16) ? o[j] * inv_keep : 0.f;
        reinterpret_cast<bf16x8*>(xd + ((long long)row * G + g) * H)[c] = pack8(d);
      }
    }
  }
}

void rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int M, int H, float eps, void* xd, int G,
                 const uint32_t* seed_ptr, const uint32_t* keys, uint32_t thr16, float inv_keep, Fp8Out f8, MxOut mo, cudaStream_t s) {
  if (H % 8 != 0 || H > 8 * 256 * 4) throw std::runtime_error("rmsnorm: H must be a multiple of 8 and <= 8192");
  if (mo.q != nullptr && H % 128) throw std::runtime_error("rmsnorm: the MX output needs H to be a multiple of 128");
  uint4 k = make_uint4(0, 0, 0, 0);
  if (G > 0) k = make_uint4(keys[0], G > 1 ? keys[1] : 0, G > 2 ? keys[2] : 0, G > 3 ? keys[3] : 0);
  if (rmsnorm_fwd_warp(x, w, y, rstd, M, H, eps, xd, G, seed_ptr, k, thr16, inv_keep, f8, mo, s)) return;
  if (f8.q != nullptr) throw std::runtime_error("rmsnorm: the fused fp8 output needs the warp-per-row kernel (H <= 2048)");
  const int nvec = H / 8;
  const bf16 *xp = (const bf16*)x, *wp = (const bf16*)w;
  bf16 *yp = (bf16*)y, *xdp = (bf16*)xd;
  if (nvec <= 256) rmsnorm_fwd_kernel<1><<<M, 256, 0, s>>>(xp, wp, yp, rstd, M, H, eps, xdp, G, seed_ptr, k, thr16, inv_keep, mo);
  else if (nvec <= 512) rmsnorm_fwd_kernel<2><<<M, 256, 0, s>>>(xp, wp, yp, rstd, M, H, eps, xdp, G, seed_ptr, k, thr16, inv_keep, mo);
  else rmsnorm_fwd_kernel<4><<<M, 256, 0, s>>>(xp, wp, yp, rstd, M, H, eps, xdp, G, seed_ptr, k, thr16, inv_keep, mo);
  RB_CHECK_LAUNCH("rmsnorm_fwd");
}

// Backward.  Each block handles a strip of rows; dw partials are reduced in registers over the strip and
// flushed with one fp32 atomic per column per block.
template <int VPT>
__global__ void __launch_bounds__(256) rmsnorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                          const float* __restrict__ rstd, const bf16* __restrict__ dx_add,
                                                          bf16* __restrict__ dx, float* __restrict__ dw, int M, int H, int rows_per_block) {
  __shared__ float scratch[32];
  const int nvec = H / 8;
  float wf[VPT][8], dwacc[VPT][8];
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = threadIdx.x + i * 256;
#pragma unroll
    for (int j = 0; j < 8; ++j) dwacc[i][j] = 0.f;
    if (c < nvec) unpack8(reinterpret_cast<const bf16x8*>(w)[c], wf[i]);
  }
  const int r0 = blockIdx.x * rows_per_block;
  const int r1 = min(M, r0 + rows_per_block);
  for (int row = r0; row < r1; ++row) {
    const float rs = rstd[row];
    float g[VPT][8], xh[VPT][8];
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = threadIdx.x + i * 256;
      if (c < nvec) {
        float dyf[8], xf[8];
        unpack8(reinterpret_cast<const bf16x8*>(dy + (long long)row * H)[c], dyf);
        unpack8(reinterpret_cast<const bf16x8*>(x + (long long)row * H)[c], xf);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[i][j] = xf[j] * rs;
          g[i][j] = dyf[j] * wf[i][j];
          dot += g[i][j] * xh[i][j];
          dwacc[i][j] += dyf[j] * bf16_round(xh[i][j]);
        }
      }
    }
    dot = block_sum(dot, scratch) / (float)H;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = threadIdx.x + i * 256;
      if (c < nvec) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rs * (g[i][j] - xh[i][j] * dot);
        if (dx_add != nullptr) {
          float a[8];
          unpack8(reinterpret_cast<const bf16x8*>(dx_add + (long long)row * H)[c], a);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += a[j];
        }
        reinterpret_cast<bf16x8*>(dx + (long long)row * H)[c] = pack8(o);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = threadIdx.x + i * 256;
    if (c < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) atomicAdd(dw + c * 8 + j, dwacc[i][j]);
    }
  }
}

void rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dx_add, void* dx, float* dw, int M,
                 int H, float* ws, unsigned int* ticket, cudaStream_t s) {
  if (H % 8 != 0 || H > 8192) throw std::runtime_error("rmsnorm_bwd: H must be a multiple of 8 and <= 8192");
  if (rmsnorm_bwd_warp(dy, x, w, rstd, dx_add, dx, dw, M, H, ws, ticket, s)) return;
  const int nvec = H / 8;
  const int blocks = min(M, num_sms() * 4);
  const int rpb = ceil_div(M, blocks);
  const int grid = ceil_div(M, rpb);
  const bf16 *a = (const bf16*)dy, *b = (const bf16*)x, *c = (const bf16*)w, *d = (const bf16*)dx_add;
  if (nvec <= 256) rmsnorm_bwd_kernel<1><<<grid, 256, 0, s>>>(a, b, c, rstd, d, (bf16*)dx, dw, M, H, rpb);
  else if (nvec <= 512) rmsnorm_bwd_kernel<2><<<grid, 256, 0, s>>>(a, b, c, rstd, d, (bf16*)dx, dw, M, H, rpb);
  else rmsnorm_bwd_kernel<4><<<grid, 256, 0, s>>>(a, b, c, rstd, d, (bf16*)dx, dw, M, H, rpb);
  RB_CHECK_LAUNCH("rmsnorm_bwd");
}

// ============================================================================================ LoRA dropout
__global__ void __launch_bounds__(256) dropout_expand_kernel(const bf16* __restrict__ x, bf16* __restrict__ xd, long long n_vec, int H,
                                                             int G, const uint32_t* __restrict__ seed_ptr, uint4 keys, uint32_t thr16,
                                                             float inv_keep, Fp8Out f8) {
  pdl_wait();
  pdl_launch_dependents();
  const float q_inv = f8.q != nullptr ? *f8.inv_scale : 0.f;
  float q_max = 0.f;
  const uint32_t base = seed_ptr ? *seed_ptr : 0u;
  const uint32_t seeds[4] = {mix_seed(base, keys.x), mix_seed(base, keys.y), mix_seed(base, keys.z), mix_seed(base, keys.w)};
  const int hv = H / 8;
  const long long stride = (long long)gridDim.x * blockDim.x;
  // two independent 16-byte loads in flight per thread (a single one leaves HBM half idle, Little's law)
  for (long long i0 = blockIdx.x * (long long)blockDim.x + threadIdx.x; i0 < n_vec; i0 += 2 * stride) {
    const long long i1 = i0 + stride;
    const bool has1 = i1 < n_vec;
    const bf16x8 v0 = reinterpret_cast<const bf16x8*>(x)[i0];
    const bf16x8 v1 = has1 ? reinterpret_cast<const bf16x8*>(x)[i1] : v0;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (u == 1 && !has1) break;
      const long long i = u ? i1 : i0;
      const long long row = i / hv;
      const int c = int(i % hv);
      float f[8];
      unpack8(u ? v1 : v0, f);
      if (f8.q != nullptr) {  // E4M3 copy of the (un-dropped) input for the frozen-weight GEMM
        *reinterpret_cast<uint2*>(f8.q + row * f8.ld + c * 8) = pack8_e4m3(f, q_inv);
        q_max = fmaxf(q_max, absmax8(f));
      }
      for (int g = 0; g < G; ++g) {
        float d[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) d[j] = keep_drop(seeds[g], (uint32_t)row, (uint32_t)(c * 8 + j), thr16) ? f[j] * inv_keep : 0.f;
        reinterpret_cast<bf16x8*>(xd + (row * G + g) * H)[c] = pack8(d);
      }
    }
  }
  if (f8.q != nullptr) amax_commit(q_max, f8.amax);
}

void dropout_expand(const void* x, void* xd, int M, int H, int G, const uint32_t* seed_ptr, const uint32_t* keys, uint32_t thr16,
                    float inv_keep, Fp8Out f8, cudaStream_t s) {
  if (H % 8 != 0) throw std::runtime_error("dropout_expand: H must be a multiple of 8");
  uint4 k = make_uint4(keys[0], G > 1 ? keys[1] : 0, G > 2 ? keys[2] : 0, G > 3 ? keys[3] : 0);
  const long long n_vec = (long long)M * H / 8;
  const int grid = (int)std::min<long long>((n_vec + 255) / 256, (long long)num_sms() * 8);
  launch_k(dropout_expand_kernel, grid, 256, 0, s, (const bf16*)x, (bf16*)xd, n_vec, H, G, seed_ptr, k, thr16, inv_keep, f8);
  RB_CHECK_LAUNCH("dropout_expand");
}

__global__ void __launch_bounds__(256) dropout_combine_kernel(const bf16* __restrict__ basep, const bf16* __restrict__ parts,
                                                              long long part_stride, long long ld_parts, bf16* __restrict__ out,
                                                              long long n_vec, int H, int G,
                                                              const uint32_t* __restrict__ seed_ptr, uint4 keys, uint32_t thr16,
                                                              float inv_keep) {
  const uint32_t base = seed_ptr ? *seed_ptr : 0u;
  const uint32_t seeds[4] = {mix_seed(base, keys.x), mix_seed(base, keys.y), mix_seed(base, keys.z), mix_seed(base, keys.w)};
  const int hv = H / 8;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / hv;
    const int c = int(i % hv);
    float acc[8];
    if (basep != nullptr) unpack8(reinterpret_cast<const bf16x8*>(basep)[i], acc);
    else {
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    }
    for (int g = 0; g < G; ++g) {
      float f[8];
      unpack8(*reinterpret_cast<const bf16x8*>(parts + g * part_stride + row * ld_parts + c * 8), f);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (keep_drop(seeds[g], (uint32_t)row, (uint32_t)(c * 8 + j), thr16)) acc[j] += f[j] * inv_keep;
    }
    reinterpret_cast<bf16x8*>(out)[i] = pack8(acc);
  }
}

void dropout_combine(const void* base, const void* parts, long long part_stride, long long ld_parts, void* out, int M, int H, int G,
                     const uint32_t* seed_ptr, const uint32_t* keys, uint32_t thr16, float inv_keep, cudaStream_t s) {
  if (H % 8 != 0) throw std::runtime_error("dropout_combine: H must be a multiple of 8");
  uint4 k = make_uint4(keys[0], G > 1 ? keys[1] : 0, G > 2 ? keys[2] : 0, G > 3 ? keys[3] : 0);
  const long long n_vec = (long long)M * H / 8;
  const int grid = (int)std::min<long long>((n_vec + 255) / 256, (long long)num_sms() * 8);
  dropout_combine_kernel<<<grid, 256, 0, s>>>((const bf16*)base, (const bf16*)parts, part_stride, ld_parts, (bf16*)out, n_vec, H, G, seed_ptr, k,
                                              thr16, inv_keep);
  RB_CHECK_LAUNCH("dropout_combine");
}

// ============================================================================================ rotary
// one thread per (row, head, pair i < rotary_dim/2): y1 = x1 c - x2 s ; y2 = x2 c + x1 s  (backward: s -> -s)
__global__ void __launch_bounds__(256) rope_kernel(bf16* __restrict__ buf, long long ld, long long total, int T, int n_heads, int hd,
                                                   int half, const bf16* __restrict__ cosp, const bf16* __restrict__ sinp, float sgn,
                                                   int pos0) {
  const int pairs2 = half / 2;  // process two adjacent pairs per thread (bf16x2 accesses)
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int pp = int(i % pairs2);
    const long long t = i / pairs2;
    const int h = int(t % n_heads);
    const long long row = t / n_heads;
    const int pos = int(row % T) + pos0;
    bf16* base = buf + row * ld + (long long)h * hd;
    const int j = pp * 2;
    __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(base + j);
    __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(base + j + half);
    const __nv_bfloat162 c = *reinterpret_cast<const __nv_bfloat162*>(cosp + (long long)pos * 2 * half + j);
    const __nv_bfloat162 sn = *reinterpret_cast<const __nv_bfloat162*>(sinp + (long long)pos * 2 * half + j);
    const float2 af = __bfloat1622float2(a), bfv = __bfloat1622float2(b), cf = __bfloat1622float2(c), sf = __bfloat1622float2(sn);
    const float s0 = sf.x * sgn, s1 = sf.y * sgn;
    *reinterpret_cast<__nv_bfloat162*>(base + j) = __floats2bfloat162_rn(af.x * cf.x - bfv.x * s0, af.y * cf.y - bfv.y * s1);
    *reinterpret_cast<__nv_bfloat162*>(base + j + half) = __floats2bfloat162_rn(bfv.x * cf.x + af.x * s0, bfv.y * cf.y + af.y * s1);
  }
}

void rope_inplace(void* buf, long long ld, int M, int T, int n_rot_heads, int hd, int rotary_dim, const void* cos, const void* sin,
                  bool backward, int pos0, cudaStream_t s) {
  if (rope_inplace_vec(buf, ld, M, T, n_rot_heads, hd, rotary_dim, cos, sin, backward, pos0, s)) return;
  const int half = rotary_dim / 2;
  if (rotary_dim % 4 != 0 || hd % 2 != 0) throw std::runtime_error("rope: rotary_dim must be a multiple of 4");
  const long long total = (long long)M * n_rot_heads * (half / 2);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 16);
  rope_kernel<<<grid, 256, 0, s>>>((bf16*)buf, ld, total, T, n_rot_heads, hd, half, (const bf16*)cos, (const bf16*)sin,
                                   backward ? -1.f : 1.f, pos0);
  RB_CHECK_LAUNCH("rope");
}

// ============================================================================================ SwiGLU
// h = silu(gate) * up ; optionally also hd = keep ⊙ h / (1-p) (the dropout-expanded copy the LoRA down-projection of
// down_proj consumes) so that h is not re-read by a separate dropout kernel.  Two vectors in flight per thread.
__global__ void __launch_bounds__(256) swiglu_fwd_kernel(const bf16* __restrict__ gu, long long ldgu, bf16* __restrict__ h, long long ldh,
                                                         int M, int F, bf16* __restrict__ hd, long long ldhd,
                                                         const uint32_t* __restrict__ seed_ptr, uint32_t key, uint32_t thr16, float inv_keep,
                                                         Fp8Out f8, MxOut mo) {
  pdl_wait();
  pdl_launch_dependents();
  const float q_inv = f8.q != nullptr ? *f8.inv_scale : 0.f;
  float q_max = 0.f;
  const int fv = F / 8;
  const long long total = (long long)M * fv;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const uint32_t seed = hd != nullptr ? mix_seed(seed_ptr ? *seed_ptr : 0u, key) : 0u;
  for (long long i0 = blockIdx.x * (long long)blockDim.x + threadIdx.x; i0 < total; i0 += 2 * stride) {
    const long long i1 = i0 + stride;
    const bool has1 = i1 < total;
    const long long r0 = i0 / fv, r1 = has1 ? i1 / fv : r0;
    const int c0 = int(i0 % fv) * 8, c1 = has1 ? int(i1 % fv) * 8 : c0;
    const bf16x8 g0 = *reinterpret_cast<const bf16x8*>(gu + r0 * ldgu + c0);
    const bf16x8 u0 = *reinterpret_cast<const bf16x8*>(gu + r0 * ldgu + F + c0);
    const bf16x8 g1 = *reinterpret_cast<const bf16x8*>(gu + r1 * ldgu + c1);
    const bf16x8 u1 = *reinterpret_cast<const bf16x8*>(gu + r1 * ldgu + F + c1);
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      if (t == 1 && !has1) break;
      const long long row = t ? r1 : r0;
      const int c = t ? c1 : c0;
      float g[8], u[8], o[8];
      unpack8(t ? g1 : g0, g);
      unpack8(t ? u1 : u0, u);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = __fdividef(g[j], 1.f + __expf(-g[j])) * u[j];  // MUFU.EX2 + MUFU.RCP, no IEEE division sequence
      const bf16x8 packed = pack8(o);
      *reinterpret_cast<bf16x8*>(h + row * ldh + c) = packed;
      if (mo.q != nullptr) {  // F % 128 == 0 and the stride is a multiple of 4: each 4-thread group holds one 32-column block
        float ob8[8];
        unpack8(packed, ob8);
        mx_emit8(mo, row, c, ob8, mx_group_mask());
      }
      if (f8.q != nullptr) {
        float ob8[8];
        unpack8(packed, ob8);
        *reinterpret_cast<uint2*>(f8.q + row * f8.ld + c) = pack8_e4m3(ob8, q_inv);
        q_max = fmaxf(q_max, absmax8(ob8));
      }
      if (hd != nullptr) {
        float ob[8], d[8];
        unpack8(packed, ob);  // the mask multiplies the rounded activation, exactly like dropout_expand(h)
#pragma unroll
        for (int j = 0; j < 8; ++j) d[j] = keep_drop(seed, (uint32_t)row, (uint32_t)(c + j), thr16) ? ob[j] * inv_keep : 0.f;
        *reinterpret_cast<bf16x8*>(hd + row * ldhd + c) = pack8(d);
      }
    }
  }
  if (f8.q != nullptr) amax_commit(q_max, f8.amax);
}
__global__ void __launch_bounds__(256) swiglu_bwd_kernel(const bf16* __restrict__ dh, long long lddh, const bf16* __restrict__ gu,
                                                         long long ldgu, bf16* __restrict__ dgu, long long lddgu, int M, int F) {
  pdl_wait();
  pdl_launch_dependents();
  const int fv = F / 8;
  const long long total = (long long)M * fv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / fv;
    const int c = int(i % fv) * 8;
    float g[8], u[8], d[8], dg[8], du[8];
    unpack8(*reinterpret_cast<const bf16x8*>(gu + row * ldgu + c), g);
    unpack8(*reinterpret_cast<const bf16x8*>(gu + row * ldgu + F + c), u);
    unpack8(*reinterpret_cast<const bf16x8*>(dh + row * lddh + c), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sg = __fdividef(1.f, 1.f + __expf(-g[j]));
      const float silu = g[j] * sg;
      du[j] = d[j] * silu;
      dg[j] = d[j] * u[j] * (sg + silu * (1.f - sg));
    }
    *reinterpret_cast<bf16x8*>(dgu + row * lddgu + c) = pack8(dg);
    *reinterpret_cast<bf16x8*>(dgu + row * lddgu + F + c) = pack8(du);
  }
}
void swiglu_fwd(const void* gu, long long ldgu, void* h, long long ldh, int M, int F, void* hd, long long ldhd,
                const uint32_t* seed_ptr, uint32_t key, uint32_t thr16, float inv_keep, Fp8Out f8, MxOut mo, cudaStream_t s) {
  if (F % 8) throw std::runtime_error("swiglu: F must be a multiple of 8");
  if (mo.q != nullptr && F % 128) throw std::runtime_error("swiglu: the MX output needs F to be a multiple of 128");
  const long long total = (long long)M * (F / 8);
  const int grid = (int)std::min<long long>((total + 511) / 512, (long long)num_sms() * 8);
  launch_k(swiglu_fwd_kernel, grid > 0 ? grid : 1, 256, 0, s, (const bf16*)gu, ldgu, (bf16*)h, ldh, M, F, (bf16*)hd, ldhd, seed_ptr, key, thr16, inv_keep, f8, mo);
  RB_CHECK_LAUNCH("swiglu_fwd");
}
void swiglu_bwd(const void* dh, long long lddh, const void* gu, long long ldgu, void* dgu, long long lddgu, int M, int F,
                cudaStream_t s) {
  if (F % 8) throw std::runtime_error("swiglu_bwd: F must be a multiple of 8");
  const long long total = (long long)M * (F / 8);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 8);
  launch_k(swiglu_bwd_kernel, grid, 256, 0, s, (const bf16*)dh, lddh, (const bf16*)gu, ldgu, (bf16*)dgu, lddgu, M, F);
  RB_CHECK_LAUNCH("swiglu_bwd");
}

// ============================================================================================ embedding
__global__ void __launch_bounds__(256) embedding_fwd_kernel(const int64_t* __restrict__ ids, const bf16* __restrict__ table,
                                                            bf16* __restrict__ out, long long total, int hv) {
  pdl_wait();
  pdl_launch_dependents();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / hv;
    const int c = int(i % hv);
    reinterpret_cast<bf16x8*>(out)[i] = reinterpret_cast<const bf16x8*>(table)[ids[row] * hv + c];
  }
}
__global__ void __launch_bounds__(256) embedding_bwd_kernel(const int64_t* __restrict__ ids, const bf16* __restrict__ dout,
                                                            float* __restrict__ dtable, long long total, int hv, long long padding_idx) {
  pdl_wait();
  pdl_launch_dependents();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / hv;
    const int c = int(i % hv);
    const long long id = ids[row];
    if (id == padding_idx) continue;
    float f[8];
    unpack8(reinterpret_cast<const bf16x8*>(dout)[i], f);
    float* dst = dtable + (id * hv + c) * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) atomicAdd(dst + j, f[j]);
  }
}
// Deterministic variant: `sorted_ids` / `perm` are the token ids in ascending order (stable) and the positions they came from.
// One block per sorted position; only the first position of every run of equal ids works: it adds the rows of that token's
// occurrences in position order (fixed summation order) and is the only writer of its table row -- no atomics, so the result
// is bit-identical from run to run and across ranks (SURVEY K9; torch's dense embedding backward is atomic, too).
__global__ void __launch_bounds__(128) embedding_bwd_sorted_kernel(const int64_t* __restrict__ sorted_ids, const int64_t* __restrict__ perm,
                                                                   const bf16* __restrict__ dout, float* __restrict__ dtable, int M, int hv,
                                                                   long long padding_idx) {
  pdl_wait();
  pdl_launch_dependents();
  const int i = blockIdx.x;
  const long long id = sorted_ids[i];
  if (id == padding_idx || (i > 0 && sorted_ids[i - 1] == id)) return;
  for (int c = threadIdx.x; c < hv; c += blockDim.x) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int k = i; k < M && sorted_ids[k] == id; ++k) {
      float f[8];
      unpack8(reinterpret_cast<const bf16x8*>(dout)[perm[k] * hv + c], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
    float4* dst = reinterpret_cast<float4*>(dtable + (id * hv + c) * 8);
    float4 a = dst[0], b = dst[1];
    a.x += acc[0]; a.y += acc[1]; a.z += acc[2]; a.w += acc[3];
    b.x += acc[4]; b.y += acc[5]; b.z += acc[6]; b.w += acc[7];
    dst[0] = a;
    dst[1] = b;
  }
}
void embedding_bwd_sorted(const int64_t* sorted_ids, const int64_t* perm, const void* dout, float* dtable, int M, int H,
                          long long padding_idx, cudaStream_t s) {
  if (H % 8) throw std::runtime_error("embedding: H must be a multiple of 8");
  if (M <= 0) return;
  launch_k(embedding_bwd_sorted_kernel, M, 128, 0, s, sorted_ids, perm, (const bf16*)dout, dtable, M, H / 8, padding_idx);
  RB_CHECK_LAUNCH("embedding_bwd_sorted");
}
void embedding_fwd(const int64_t* ids, const void* table, void* out, int M, int H, cudaStream_t s) {
  if (H % 8) throw std::runtime_error("embedding: H must be a multiple of 8");
  const long long total = (long long)M * (H / 8);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 8);
  launch_k(embedding_fwd_kernel, grid, 256, 0, s, ids, (const bf16*)table, (bf16*)out, total, H / 8);
  RB_CHECK_LAUNCH("embedding_fwd");
}
void embedding_bwd(const int64_t* ids, const void* dout, float* dtable, int M, int H, long long padding_idx, cudaStream_t s) {
  if (H % 8) throw std::runtime_error("embedding: H must be a multiple of 8");
  const long long total = (long long)M * (H / 8);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 8);
  launch_k(embedding_bwd_kernel, grid, 256, 0, s, ids, (const bf16*)dout, dtable, total, H / 8, padding_idx);
  RB_CHECK_LAUNCH("embedding_bwd");
}

// ============================================================================================ misc
__global__ void transpose_kernel(const bf16* __restrict__ in, long long ld_in, bf16* __restrict__ out, long long ld_out, int R, int C) {
  __shared__ bf16 tile[32][33];
  const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int r = by + j, c = bx + threadIdx.x;
    if (r < R && c < C) tile[j][threadIdx.x] = in[(long long)r * ld_in + c];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = bx + j, r = by + threadIdx.x;
    if (r < R && c < C) out[(long long)c * ld_out + r] = tile[threadIdx.x][j];
  }
}
void transpose_bf16(const void* in, long long ld_in, void* out, long long ld_out, int R, int C, cudaStream_t s) {
  dim3 grid(ceil_div(C, 32), ceil_div(R, 32)), block(32, 8);
  transpose_kernel<<<grid, block, 0, s>>>((const bf16*)in, ld_in, (bf16*)out, ld_out, R, C);
  RB_CHECK_LAUNCH("transpose");
}

__global__ void __launch_bounds__(256) add_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, bf16* __restrict__ out, long long nv) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nv; i += (long long)gridDim.x * blockDim.x) {
    float x[8], y[8];
    unpack8(reinterpret_cast<const bf16x8*>(a)[i], x);
    unpack8(reinterpret_cast<const bf16x8*>(b)[i], y);
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] += y[j];
    reinterpret_cast<bf16x8*>(out)[i] = pack8(x);
  }
}
void add_bf16(const void* a, const void* b, void* out, long long n, cudaStream_t s) {
  if (n % 8) throw std::runtime_error("add: n must be a multiple of 8");
  const long long nv = n / 8;
  const int grid = (int)std::min<long long>((nv + 255) / 256, (long long)num_sms() * 8);
  add_kernel<<<grid, 256, 0, s>>>((const bf16*)a, (const bf16*)b, (bf16*)out, nv);
  RB_CHECK_LAUNCH("add");
}

__global__ void __launch_bounds__(256) cast_kernel(const float* __restrict__ in, bf16* __restrict__ out, long long nv, float scale) {
  pdl_wait();
  pdl_launch_dependents();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nv; i += (long long)gridDim.x * blockDim.x) {
    const float4 a = reinterpret_cast<const float4*>(in)[2 * i], b = reinterpret_cast<const float4*>(in)[2 * i + 1];
    float f[8] = {a.x * scale, a.y * scale, a.z * scale, a.w * scale, b.x * scale, b.y * scale, b.z * scale, b.w * scale};
    reinterpret_cast<bf16x8*>(out)[i] = pack8(f);
  }
}
void cast_f32_to_bf16(const float* in, void* out, long long n, float scale, cudaStream_t s) {
  if (n % 8) throw std::runtime_error("cast: n must be a multiple of 8");
  const long long nv = n / 8;
  const int grid = (int)std::min<long long>((nv + 255) / 256, (long long)num_sms() * 8);
  launch_k(cast_kernel, grid, 256, 0, s, in, (bf16*)out, nv, scale);
  RB_CHECK_LAUNCH("cast");
}

__global__ void __launch_bounds__(256) fill_uniform_kernel(bf16* __restrict__ out, int R, int C, long long ld, uint32_t seed, float bound) {
  const long long total = (long long)R * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = int(i / C), c = int(i % C);
    const float u = (float)(hash_rc(seed, (uint32_t)r, (uint32_t)c) >> 8) * (1.0f / 16777216.0f);
    out[(long long)r * ld + c] = __float2bfloat16_rn((2.f * u - 1.f) * bound);
  }
}
void fill_uniform_hash(void* out, int R, int C, long long ld, uint32_t seed, float bound, cudaStream_t s) {
  const long long total = (long long)R * C;
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 8);
  fill_uniform_kernel<<<grid, 256, 0, s>>>((bf16*)out, R, C, ld, seed, bound);
  RB_CHECK_LAUNCH("fill_uniform");
}

__global__ void seed_advance_kernel(uint32_t* seed) {
  pdl_wait();
  pdl_launch_dependents(); *seed = lowbias32(*seed + 0x9E3779B9u); }
void seed_advance(uint32_t* seed, cudaStream_t s) {
  launch_k(seed_advance_kernel, 1, 1, 0, s, seed);
  RB_CHECK_LAUNCH("seed_advance");
}

}  // namespace rb
