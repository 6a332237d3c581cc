// Kernels of the GPT-NeoX / Pythia block that the Llama executor does not have (SURVEY K16):
//
//   layernorm_fwd / layernorm_bwd   nn.LayerNorm with affine weight + bias (reference modeling_pythia.py:413-414), warp per row,
//                                   fp32 statistics saved for the backward; dw / db accumulated through shared-memory block
//                                   partials and one 16-byte vector reduction per 4 columns per block
//   layernorm_fwd_dual / _bwd_dual  executor forms: two norms of one input, LoRA-dropout copies, dx += residual gradient, its column sum
//   gelu_fwd / gelu_bwd             exact (erf) and tanh GELU (modeling_pythia.py:395-406), 128-bit accesses; optional dropout copy
//                                   of the output, optional column sum of dz (bias gradient of dense_h_to_4h)
//   colsum                          Σ rows of a bf16 matrix into fp32 (bias gradients)
//   neox_rope                       partial rotary embedding on the fused query_key_value output [rows, nh, 3*hd]
//                                   (q | k | v per head, first `rot` dims of q and k rotated, fp32 tables; :172-197), in place,
//                                   forward and inverse (backward) direction
#include "common.cuh"
#include "kernels.h"

namespace rb {

namespace {
constexpr int kRowsPerBlock = 8;  // one warp per row

// One pass over x for up to two norms of the same row (GPT-NeoX parallel residual: LN1(x) and LN2(x) share mean / rstd), each
// optionally followed by its LoRA-dropout copy xd = keep ⊙ y / (1 - p) with the mask stream mix_seed(*seed, key) of csrc/common.cuh.
template <int VPL>
__global__ void __launch_bounds__(kRowsPerBlock * 32) layernorm_fwd_kernel(const bf16* __restrict__ x, const LnFwdOut n1, const LnFwdOut n2,
                                                                          float* __restrict__ mean_out, float* __restrict__ rstd_out, int M,
                                                                          int H, float eps, LnDrop drop) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int row = blockIdx.x * kRowsPerBlock + warp;
  if (row >= M) return;
  const int nvec = H / 8;
  const uint4* xr = reinterpret_cast<const uint4*>(x + (long long)row * H);
  uint4 xv[VPL];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c = lane + i * 32;
    if (c < nvec) {
      xv[i] = xr[c];
      float f[8];
      unpack8(xv[i], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += f[j];
    }
  }
  const float mean = warp_sum(s) / (float)H;
  float ss = 0.f;  // two-pass variance on the registers: no cancellation
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c = lane + i * 32;
    if (c < nvec) {
      float f[8];
      unpack8(xv[i], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) ss += (f[j] - mean) * (f[j] - mean);
    }
  }
  const float rstd = rsqrtf(warp_sum(ss) / (float)H + eps);
  if (lane == 0) {
    mean_out[row] = mean;
    rstd_out[row] = rstd;
  }
  const uint32_t base = drop.seed_ptr != nullptr ? *drop.seed_ptr : 0u;
#pragma unroll
  for (int n = 0; n < 2; ++n) {
    const LnFwdOut& o_ = n == 0 ? n1 : n2;
    if (o_.y == nullptr) break;
    const uint32_t sd = mix_seed(base, o_.key);
    uint4* yr = reinterpret_cast<uint4*>(static_cast<bf16*>(o_.y) + (long long)row * H);
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int c = lane + i * 32;
      if (c < nvec) {
        float f[8], wf[8], bf[8], o[8];
        unpack8(xv[i], f);
        unpack8(reinterpret_cast<const uint4*>(o_.w)[c], wf);
        if (o_.b != nullptr) unpack8(reinterpret_cast<const uint4*>(o_.b)[c], bf);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (f[j] - mean) * rstd * wf[j] + (o_.b != nullptr ? bf[j] : 0.f);
        const uint4 packed = pack8(o);
        yr[c] = packed;
        if (o_.xd != nullptr) {  // the mask multiplies the rounded output, exactly like dropout_expand(y)
          unpack8(packed, o);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = keep_drop(sd, (uint32_t)row, (uint32_t)(c * 8 + j), drop.thr16) ? o[j] * drop.inv_keep : 0.f;
          reinterpret_cast<uint4*>(static_cast<bf16*>(o_.xd) + (long long)row * H)[c] = pack8(o);
        }
      }
    }
  }
}

// dx = rstd * (g - mean(g) - xhat * mean(g * xhat)),  g = dy * w;   dw += sum_rows dy * xhat;   db += sum_rows dy
template <int VPL>
__global__ void __launch_bounds__(kRowsPerBlock * 32) layernorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                                                          const bf16* __restrict__ w, const float* __restrict__ mean,
                                                                          const float* __restrict__ rstd, bf16* __restrict__ dx,
                                                                          float* __restrict__ dw, float* __restrict__ db, int M, int H) {
  extern __shared__ float sacc[];  // [2][H] block partials of dw, db
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nvec = H / 8;
  for (int c = threadIdx.x; c < 2 * H; c += blockDim.x) sacc[c] = 0.f;
  __syncthreads();
  uint4 wv[VPL];
  float dwacc[VPL][8], dbacc[VPL][8];
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c = lane + i * 32;
    wv[i] = (c < nvec) ? reinterpret_cast<const uint4*>(w)[c] : make_uint4(0, 0, 0, 0);
#pragma unroll
    for (int j = 0; j < 8; ++j) dwacc[i][j] = dbacc[i][j] = 0.f;
  }
  for (int row = blockIdx.x * kRowsPerBlock + warp; row < M; row += gridDim.x * kRowsPerBlock) {
    const float mu = mean[row], rs = rstd[row];
    uint4 dyv[VPL], xv[VPL];
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int c = lane + i * 32;
      if (c < nvec) {
        dyv[i] = reinterpret_cast<const uint4*>(dy + (long long)row * H)[c];
        xv[i] = reinterpret_cast<const uint4*>(x + (long long)row * H)[c];
        float dyf[8], xf[8], wf[8];
        unpack8(dyv[i], dyf);
        unpack8(xv[i], xf);
        unpack8(wv[i], wf);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xh = (xf[j] - mu) * rs, g = dyf[j] * wf[j];
          sg += g;
          sgx += g * xh;
          dwacc[i][j] += dyf[j] * xh;
          dbacc[i][j] += dyf[j];
        }
      }
    }
    sg = warp_sum(sg) / (float)H;
    sgx = warp_sum(sgx) / (float)H;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int c = lane + i * 32;
      if (c < nvec) {
        float dyf[8], xf[8], wf[8], o[8];
        unpack8(dyv[i], dyf);
        unpack8(xv[i], xf);
        unpack8(wv[i], wf);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rs * (dyf[j] * wf[j] - sg - (xf[j] - mu) * rs * sgx);
        reinterpret_cast<uint4*>(dx + (long long)row * H)[c] = pack8(o);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c = lane + i * 32;
    if (c < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        atomicAdd(&sacc[c * 8 + j], dwacc[i][j]);
        atomicAdd(&sacc[H + c * 8 + j], dbacc[i][j]);
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x * 4; c < H; c += blockDim.x * 4) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dw + c), "f"(sacc[c]), "f"(sacc[c + 1]), "f"(sacc[c + 2]), "f"(sacc[c + 3])
                 : "memory");
    if (db != nullptr)
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(db + c), "f"(sacc[H + c]), "f"(sacc[H + c + 1]), "f"(sacc[H + c + 2]),
                   "f"(sacc[H + c + 3])
                   : "memory");
  }
}

// Executor form of the backward: dx = dres + LN1ᵀ(dy1) [+ LN2ᵀ(dy2)] for norms of the same x, the γ / β gradients of each norm and,
// optionally, Σ rows of dres (the bias gradient of the projections whose output gradient dres is).  Block partials go through
// shared memory, laid out [quantity][j][column vector] so that the lanes of a warp hit consecutive words.  With two Σ dres
// outputs the blocks add their partials into `dsum1` as a zeroed total, which ln_add_total then adds to both outputs.
template <int VPL>
__global__ void __launch_bounds__(kRowsPerBlock * 32) layernorm_bwd_dual_kernel(const bf16* __restrict__ x, const float* __restrict__ mean,
                                                                               const float* __restrict__ rstd, const LnBwdNorm n1,
                                                                               const LnBwdNorm n2, const bf16* __restrict__ dres,
                                                                               bf16* __restrict__ dx, float* __restrict__ dsum1,
                                                                               int M, int H) {
  extern __shared__ float sacc[];  // [5][H]: dw1, db1, dw2, db2, Σ dres
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nvec = H / 8;
  const int nq = 5;
  for (int c = threadIdx.x; c < nq * H; c += blockDim.x) sacc[c] = 0.f;
  __syncthreads();
  const bool two = n2.dy != nullptr, sum = dsum1 != nullptr;
  for (int row = blockIdx.x * kRowsPerBlock + warp; row < M; row += gridDim.x * kRowsPerBlock) {
    const float mu = mean[row], rs = rstd[row];
    float sg[2] = {0.f, 0.f}, sgx[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int c = lane + i * 32;
      if (c < nvec) {
        float xf[8];
        unpack8(reinterpret_cast<const uint4*>(x + (long long)row * H)[c], xf);
#pragma unroll
        for (int n = 0; n < 2; ++n) {
          const LnBwdNorm& nn = n == 0 ? n1 : n2;
          if (n == 1 && !two) break;
          float dyf[8], wf[8];
          unpack8(reinterpret_cast<const uint4*>(static_cast<const bf16*>(nn.dy) + (long long)row * H)[c], dyf);
          unpack8(reinterpret_cast<const uint4*>(nn.w)[c], wf);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float xh = (xf[j] - mu) * rs, g = dyf[j] * wf[j];
            sg[n] += g;
            sgx[n] += g * xh;
            atomicAdd(&sacc[(2 * n) * H + j * nvec + c], dyf[j] * xh);
            atomicAdd(&sacc[(2 * n + 1) * H + j * nvec + c], dyf[j]);
          }
        }
      }
    }
#pragma unroll
    for (int n = 0; n < 2; ++n) {
      sg[n] = warp_sum(sg[n]) / (float)H;
      sgx[n] = warp_sum(sgx[n]) / (float)H;
    }
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int c = lane + i * 32;
      if (c < nvec) {
        float xf[8], o[8];
        unpack8(reinterpret_cast<const uint4*>(x + (long long)row * H)[c], xf);
        if (dres != nullptr) {
          unpack8(reinterpret_cast<const uint4*>(dres + (long long)row * H)[c], o);
          if (sum) {
#pragma unroll
            for (int j = 0; j < 8; ++j) atomicAdd(&sacc[4 * H + j * nvec + c], o[j]);
          }
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = 0.f;
        }
#pragma unroll
        for (int n = 0; n < 2; ++n) {
          const LnBwdNorm& nn = n == 0 ? n1 : n2;
          if (n == 1 && !two) break;
          float dyf[8], wf[8];
          unpack8(reinterpret_cast<const uint4*>(static_cast<const bf16*>(nn.dy) + (long long)row * H)[c], dyf);
          unpack8(reinterpret_cast<const uint4*>(nn.w)[c], wf);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += rs * (dyf[j] * wf[j] - sg[n] - (xf[j] - mu) * rs * sgx[n]);
        }
        reinterpret_cast<uint4*>(dx + (long long)row * H)[c] = pack8(o);
      }
    }
  }
  __syncthreads();
  float* dst[5] = {n1.dw, n1.db, n2.dw, n2.db, dsum1};
#pragma unroll
  for (int q = 0; q < nq; ++q) {
    if (dst[q] == nullptr) continue;
    for (int col = threadIdx.x; col < H; col += blockDim.x) {
      atomicAdd(dst[q] + col, sacc[q * H + (col & 7) * nvec + (col >> 3)]);
    }
  }
}

// out1 += total; out2 += total: the two bias gradients that share Σ dres receive the same rounded sum, whatever order the
// blocks' atomics added it up in
__global__ void ln_add_total_kernel(const float* __restrict__ total, float* __restrict__ out1, float* __restrict__ out2, int H) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < H) {
    const float t = total[c];
    out1[c] += t;
    out2[c] += t;
  }
}

int pick_vpl(int nvec) {
  const int need = (nvec + 31) / 32;
  for (int v : {1, 2, 3, 4, 8, 16}) if (need <= v) return v;
  return 0;
}

__device__ __forceinline__ float gelu_erf(float z) { return 0.5f * z * (1.f + erff(z * 0.70710678118654752f)); }
__device__ __forceinline__ float dgelu_erf(float z) {
  return 0.5f * (1.f + erff(z * 0.70710678118654752f)) + z * 0.3989422804014327f * __expf(-0.5f * z * z);
}
__device__ __forceinline__ float gelu_tanh(float z) {
  const float u = 0.7978845608028654f * (z + 0.044715f * z * z * z);
  return 0.5f * z * (1.f + tanhf(u));
}
__device__ __forceinline__ float dgelu_tanh(float z) {
  const float u = 0.7978845608028654f * (z + 0.044715f * z * z * z), t = tanhf(u);
  return 0.5f * (1.f + t) + 0.5f * z * (1.f - t * t) * 0.7978845608028654f * (1.f + 3.f * 0.044715f * z * z);
}

// xd (optional): LoRA-dropout copy of the rounded output with the mask stream mix_seed(*seed, key); row width N for the mask positions
template <bool TANH>
__global__ void __launch_bounds__(256) gelu_fwd_kernel(const bf16* __restrict__ z, bf16* __restrict__ a, long long nvec, bf16* __restrict__ xd,
                                                       int N, uint32_t key, LnDrop drop) {
  const uint32_t sd = xd != nullptr ? mix_seed(drop.seed_ptr != nullptr ? *drop.seed_ptr : 0u, key) : 0u;
  const int nv_row = N / 8;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float f[8];
    unpack8(reinterpret_cast<const uint4*>(z)[i], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = TANH ? gelu_tanh(f[j]) : gelu_erf(f[j]);
    const uint4 packed = pack8(f);
    reinterpret_cast<uint4*>(a)[i] = packed;
    if (xd != nullptr) {
      const uint32_t row = (uint32_t)(i / nv_row), c8 = (uint32_t)(i % nv_row) * 8;
      unpack8(packed, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = keep_drop(sd, row, c8 + j, drop.thr16) ? f[j] * drop.inv_keep : 0.f;
      reinterpret_cast<uint4*>(xd)[i] = pack8(f);
    }
  }
}
template <bool TANH>
__global__ void __launch_bounds__(256) gelu_bwd_kernel(const bf16* __restrict__ da, const bf16* __restrict__ z, bf16* __restrict__ dz,
                                                       long long nvec) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float g[8], f[8];
    unpack8(reinterpret_cast<const uint4*>(da)[i], g);
    unpack8(reinterpret_cast<const uint4*>(z)[i], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] *= TANH ? dgelu_tanh(f[j]) : dgelu_erf(f[j]);
    reinterpret_cast<uint4*>(dz)[i] = pack8(g);
  }
}

// Column sums of a [M, N] bf16 matrix added into fp32 out[N] (a bias gradient).  MODE 0: of x itself; MODE 1 / 2: x is the GELU output
// gradient da, the kernel also writes dz = da · gelu'(z) (erf / tanh) and sums the rounded dz.  Thread = 8 columns x a strided set of
// rows; the 8 row lanes of a block are combined in shared memory before one vector reduction per 4 columns.
constexpr int kColRows = 8;
template <int MODE>
__global__ void __launch_bounds__(32 * kColRows) colsum_kernel(const bf16* __restrict__ x, const bf16* __restrict__ z, bf16* __restrict__ dz,
                                                              float* __restrict__ out, int M, int N) {
  __shared__ float part[kColRows][32 * 8];
  const int nvec = N / 8;
  const int c = blockIdx.x * 32 + threadIdx.x;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (c < nvec) {
    for (int row = blockIdx.y * kColRows + threadIdx.y; row < M; row += gridDim.y * kColRows) {
      const long long i = (long long)row * nvec + c;
      float g[8];
      unpack8(reinterpret_cast<const uint4*>(x)[i], g);
      if (MODE != 0) {
        float f[8];
        unpack8(reinterpret_cast<const uint4*>(z)[i], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] *= MODE == 2 ? dgelu_tanh(f[j]) : dgelu_erf(f[j]);
        const uint4 packed = pack8(g);
        reinterpret_cast<uint4*>(dz)[i] = packed;
        unpack8(packed, g);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += g[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) part[threadIdx.y][threadIdx.x * 8 + j] = acc[j];
  __syncthreads();
  const int t = threadIdx.y * 32 + threadIdx.x;  // 256 threads: 64 groups of 4 columns
  if (t < 64) {
    const int col = blockIdx.x * 256 + t * 4;
    if (col < N) {
      float v[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int r = 0; r < kColRows; ++r)
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] += part[r][t * 4 + k];
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(out + col), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]) : "memory");
    }
  }
}

void launch_colsum(int mode, const bf16* x, const bf16* z, bf16* dz, float* out, int M, int N, cudaStream_t s) {
  if (N % 8 != 0) throw std::runtime_error("colsum: N must be a multiple of 8");
  if (M <= 0) return;
  const int gx = ceil_div(N / 8, 32);
  const int gy = std::max(1, std::min(ceil_div(M, kColRows * 16), 4 * num_sms() / gx));
  const dim3 grid(gx, gy), block(32, kColRows);
  if (mode == 0) launch_k(colsum_kernel<0>, grid, block, 0, s, x, z, dz, out, M, N);
  else if (mode == 1) launch_k(colsum_kernel<1>, grid, block, 0, s, x, z, dz, out, M, N);
  else launch_k(colsum_kernel<2>, grid, block, 0, s, x, z, dz, out, M, N);
  RB_CHECK_LAUNCH("colsum");
}

// one thread per (row, head, q|k, pair index i < rot/2): (a, b) = (x[i], x[i + rot/2]) -> (a cos - b sin, b cos + a sin)
__global__ void __launch_bounds__(256) neox_rope_kernel(bf16* __restrict__ qkv, long long ld, long long rows, int T, int nh, int hd, int rot,
                                                        const float* __restrict__ cos, const float* __restrict__ sin, int pos0, bool inverse) {
  const int half = rot / 2;
  const long long total = rows * nh * 2 * half;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int p = int(i % half);
    long long r = i / half;
    const int which = int(r % 2);  // 0 = q, 1 = k
    r /= 2;
    const int h = int(r % nh);
    const long long row = r / nh;
    const int pos = int(row % T) + pos0;
    bf16* base = qkv + row * ld + (long long)h * 3 * hd + which * hd;
    const float c = cos[(long long)pos * rot + p], s = inverse ? -sin[(long long)pos * rot + p] : sin[(long long)pos * rot + p];
    const float a = __bfloat162float(base[p]), b = __bfloat162float(base[p + half]);
    base[p] = __float2bfloat16_rn(a * c - b * s);
    base[p + half] = __float2bfloat16_rn(b * c + a * s);
  }
}
}  // namespace

bool layernorm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, int M, int H, float eps, cudaStream_t s) {
  LnFwdOut n1{(const bf16*)w, (const bf16*)b, (bf16*)y, nullptr, 0}, n2{};
  return layernorm_fwd_dual(x, n1, n2, mean, rstd, M, H, eps, LnDrop{}, s);
}

bool layernorm_fwd_dual(const void* x, const LnFwdOut& n1, const LnFwdOut& n2, float* mean, float* rstd, int M, int H, float eps,
                        const LnDrop& drop, cudaStream_t s) {
  const int vpl = (H % 8 == 0) ? pick_vpl(H / 8) : 0;
  if (vpl == 0 || M <= 0) return false;
  const int grid = ceil_div(M, kRowsPerBlock);
  const bf16* xp = (const bf16*)x;
#define L(V) launch_k(layernorm_fwd_kernel<V>, grid, kRowsPerBlock * 32, 0, s, xp, n1, n2, mean, rstd, M, H, eps, drop)
  switch (vpl) {
    case 1: L(1); break;
    case 2: L(2); break;
    case 3: L(3); break;
    case 4: L(4); break;
    case 8: L(8); break;
    default: L(16); break;
  }
#undef L
  RB_CHECK_LAUNCH("layernorm_fwd");
  return true;
}

bool layernorm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, void* dx, float* dw, float* db, int M,
                   int H, cudaStream_t s) {
  const int vpl = (H % 8 == 0) ? pick_vpl(H / 8) : 0;
  if (vpl == 0 || vpl > 8 || M <= 0) return false;
  const size_t smem = 2 * (size_t)H * sizeof(float);
  const int grid = std::min(ceil_div(M, kRowsPerBlock), 2 * num_sms());
  const bf16 *a = (const bf16*)dy, *bx = (const bf16*)x, *c = (const bf16*)w;
#define L(V) launch_k(layernorm_bwd_kernel<V>, grid, kRowsPerBlock * 32, smem, s, a, bx, c, mean, rstd, (bf16*)dx, dw, db, M, H)
  switch (vpl) {
    case 1: L(1); break;
    case 2: L(2); break;
    case 3: L(3); break;
    case 4: L(4); break;
    default: L(8); break;
  }
#undef L
  RB_CHECK_LAUNCH("layernorm_bwd");
  return true;
}

bool layernorm_bwd_dual(const void* x, const float* mean, const float* rstd, const LnBwdNorm& n1, const LnBwdNorm& n2, const void* dres,
                        void* dx, float* dsum1, float* dsum2, float* dsum_tmp, int M, int H, cudaStream_t s) {
  const int vpl = (H % 8 == 0) ? pick_vpl(H / 8) : 0;
  if (vpl == 0 || vpl > 8 || M <= 0) return false;
  if (dsum2 != nullptr && (dsum1 == nullptr || dsum_tmp == nullptr)) throw std::runtime_error("layernorm_bwd: dsum2 needs dsum1 and dsum_tmp");
  const size_t smem = 5 * (size_t)H * sizeof(float);
  const int grid = std::min(ceil_div(M, kRowsPerBlock), 2 * num_sms());
  const bf16 *xp = (const bf16*)x, *rp = (const bf16*)dres;
  float* dsum = dsum1;
  if (dsum2 != nullptr) {
    check(cudaMemsetAsync(dsum_tmp, 0, (size_t)H * sizeof(float), s), "cudaMemsetAsync(layernorm_bwd total)");
    dsum = dsum_tmp;
  }
#define L(V) launch_k(layernorm_bwd_dual_kernel<V>, grid, kRowsPerBlock * 32, smem, s, xp, mean, rstd, n1, n2, rp, (bf16*)dx, dsum, M, H)
  switch (vpl) {
    case 1: L(1); break;
    case 2: L(2); break;
    case 3: L(3); break;
    case 4: L(4); break;
    default: L(8); break;
  }
#undef L
  RB_CHECK_LAUNCH("layernorm_bwd_dual");
  if (dsum2 != nullptr) {
    launch_k(ln_add_total_kernel, ceil_div(H, 256), 256, 0, s, (const float*)dsum_tmp, dsum1, dsum2, H);
    RB_CHECK_LAUNCH("ln_add_total");
  }
  return true;
}

void gelu_fwd(const void* z, void* a, long long n, bool tanh_approx, cudaStream_t s, void* xd, int N, uint32_t key, const LnDrop& drop) {
  if (n % 8) throw std::runtime_error("gelu: element count must be a multiple of 8");
  if (xd != nullptr && (N <= 0 || N % 8 || n % N)) throw std::runtime_error("gelu: dropout copy needs a row width that is a multiple of 8");
  const long long nvec = n / 8;
  const int grid = (int)std::min<long long>((nvec + 255) / 256, (long long)num_sms() * 8);
  if (grid <= 0) return;
  if (tanh_approx) launch_k(gelu_fwd_kernel<true>, grid, 256, 0, s, (const bf16*)z, (bf16*)a, nvec, (bf16*)xd, N, key, drop);
  else launch_k(gelu_fwd_kernel<false>, grid, 256, 0, s, (const bf16*)z, (bf16*)a, nvec, (bf16*)xd, N, key, drop);
  RB_CHECK_LAUNCH("gelu_fwd");
}
void gelu_bwd(const void* da, const void* z, void* dz, long long n, bool tanh_approx, cudaStream_t s) {
  if (n % 8) throw std::runtime_error("gelu: element count must be a multiple of 8");
  const long long nvec = n / 8;
  const int grid = (int)std::min<long long>((nvec + 255) / 256, (long long)num_sms() * 8);
  if (grid <= 0) return;
  if (tanh_approx) launch_k(gelu_bwd_kernel<true>, grid, 256, 0, s, (const bf16*)da, (const bf16*)z, (bf16*)dz, nvec);
  else launch_k(gelu_bwd_kernel<false>, grid, 256, 0, s, (const bf16*)da, (const bf16*)z, (bf16*)dz, nvec);
  RB_CHECK_LAUNCH("gelu_bwd");
}
void gelu_bwd_colsum(const void* da, const void* z, void* dz, float* dbias, int M, int N, bool tanh_approx, cudaStream_t s) {
  launch_colsum(tanh_approx ? 2 : 1, (const bf16*)da, (const bf16*)z, (bf16*)dz, dbias, M, N, s);
}
void colsum(const void* x, float* out, int M, int N, cudaStream_t s) { launch_colsum(0, (const bf16*)x, nullptr, nullptr, out, M, N, s); }

void neox_rope(void* qkv, long long ld, long long rows, int T, int nh, int hd, int rot, const float* cos, const float* sin, int pos0,
               bool inverse, cudaStream_t s) {
  if (rot <= 0) return;
  if (rot % 2 || rot > hd) throw std::runtime_error("neox_rope: rotary dims must be even and <= head_dim");
  const long long total = rows * nh * rot;  // 2 (q, k) * rot / 2 pairs
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 16);
  if (grid <= 0) return;
  launch_k(neox_rope_kernel, grid, 256, 0, s, (bf16*)qkv, ld, rows, T, nh, hd, rot, cos, sin, pos0, inverse);
  RB_CHECK_LAUNCH("neox_rope");
}

}  // namespace rb
