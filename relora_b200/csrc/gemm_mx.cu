// Block-scaled MXFP8 path for the frozen weights (SURVEY K15): e4m3 wgmma per 32-element scale block with the ue8m0 scale
// factors applied to the fp32 partial products in registers, plus the quantisation / requantisation kernels.
//
// Replaces the reference's bitsandbytes storage (peft_pretraining/relora.py:222-238 Params4bit / Int8Params, :314-317 matmul_4bit /
// bnb.matmul, :277-299 dequantise -> add -> requantise merge).  Formats (OCP MX): E4M3 elements, one UE8M0 (power of two) scale per
// 32 elements of the reduction dimension.
//
//   * activations / gradients  [M, K]: scales per (row, 32 columns)                              mx_quantize_rows
//   * frozen weights           [N, K]: ONE scale per 32 x 32 tile, so the same bytes serve        mx_quantize_weight_2d
//       - the forward GEMM  y = x · Wᵀ   (B operand K-major,  scale of (n, k/32) = tile scale)
//       - the backward GEMM dx = dy · W  (B operand MN-major, scale of (k, n/32) = the same tile scale)
//     -> 1 byte per parameter + two expanded scale arrays (1/32 byte each) instead of two fp8 copies.
//     wgmma reads 8-bit operands K-major only: an MN-major B tile is transposed in shared memory by the consumer warpgroups.
//
// Scale-factor layout in global memory: for a block of 128 rows x 4 scale columns (= 128 reduction elements) 512 contiguous bytes,
//     byte[(r % 32) * 16 + (r / 32) * 4 + j]  =  scale(row r, scale column j)
// blocks ordered [row block][k group].
#include <cuda.h>
#include <cuda_fp8.h>

#include <cstdlib>
#include <stdexcept>

#include "common.cuh"
#include "kernels.h"
#include "sm90.cuh"
#include "tensormap.h"

namespace rb {

using namespace sm90;

namespace {

constexpr int BM = 128, BN = 128;
constexpr int KB8 = 128;  // fp8 elements per k-block (128 bytes = one swizzle row)
constexpr int KB16 = 64;  // bf16 elements per k-block of the optional second (LoRA) segment
constexpr int kStages = 5;
constexpr int kTileBytes = BM * 128;           // 16 KB per operand tile
constexpr int kStageBytes = 2 * kTileBytes;    // A + B
constexpr int kSfBytes = 512;                  // one 128-row x 4-scale block
constexpr int kSmemTiles = kStages * kStageBytes;             // 160 KB
constexpr int kSmemSf = kStages * 2 * kSfBytes;               // 5 KB
constexpr int kSmemTotal = kSmemTiles + kTileBytes + kSmemSf + 1024 + 1024;  // + transposed B tile, barriers, alignment

__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ float ue8m0_value(uint8_t e) { return __uint_as_float(e == 0 ? 0x00400000u : uint32_t(e) << 23); }
__device__ __forceinline__ int sf_byte(int r, int j) { return (r & 31) * 16 + (r >> 5) * 4 + j; }

struct MxArgs {
  int M, N, K8, K2;                 // K8: fp8 reduction length (multiple of 128), K2: bf16 LoRA segment (multiple of 64, may be 0)
  const uint8_t* sfa;               // [m blocks][sfa_kg][512]
  const uint8_t* sfb;               // [n blocks][sfb_kg][512]
  int sfa_kg, sfb_kg;               // 128-element k groups per row block in the arrays
  int num_m_tiles, num_n_tiles;
  bf16* out;
  long long ldc;
  const bf16* residual;
  long long ldr;
};

// 256 consumer threads: MN-major [128 K rows][128 N bytes] (128-byte swizzle) -> K-major [128 N rows][128 K bytes] (same swizzle)
__device__ __forceinline__ void transpose_fp8_tile(const uint8_t* src, uint8_t* dst, int t) {
#pragma unroll 1
  for (int item = t; item < 128 * 8; item += 256) {
    const int n = item & 127, c = item >> 7;  // output row n, 16-byte chunk c (K = 16c .. 16c + 15)
    uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
    for (int e = 0; e < 16; ++e) {
      const int k = c * 16 + e;
      const uint32_t v = src[k * 128 + ((((n >> 4) ^ (k & 7))) << 4) + (n & 15)];
      w[e >> 2] |= v << ((e & 3) * 8);
    }
    *reinterpret_cast<uint4*>(dst + n * 128 + ((c ^ (n & 7)) << 4)) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

template <bool B_MN>
__global__ void __launch_bounds__(384, 1)
gemm_mx_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const __grid_constant__ CUtensorMap map_a2,
               const __grid_constant__ CUtensorMap map_b2, const MxArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* bt = smem + kSmemTiles;  // transposed B tile (MN-major B only)
  uint8_t* sf_base = bt + kTileBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sf_base + kSmemSf);
  uint64_t* empty_bar = full_bar + kStages;

  const uint32_t warp = warp_id();
  const int wg = threadIdx.x / 128;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    if (p.K2 > 0) {
      tma_prefetch_desc(&map_a2);
      tma_prefetch_desc(&map_b2);
    }
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 256);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int num_tiles = p.num_m_tiles * p.num_n_tiles;
  const int kb8 = p.K8 / KB8, kb16 = p.K2 / KB16;

  if (wg == 0) {
    // ===================================================================== TMA producer (whole warp walks the loop, one lane issues)
    setmaxnreg_dec<40>();
    if (warp != 0) return;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int tm = tile / p.num_n_tiles, tn = tile % p.num_n_tiles;
      const int m0 = tm * BM, n0 = tn * BN;
      for (int kb = 0; kb < kb8 + kb16; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem + stage * kStageBytes;
        uint8_t* sb = sa + kTileBytes;
        if (!elect_one()) {
        } else if (kb < kb8) {
          mbar_arrive_expect_tx(&full_bar[stage], kStageBytes + 2 * kSfBytes);
          tma_load_2d(&map_a, &full_bar[stage], sa, kb * KB8, m0, kEvictNormal);
          if constexpr (B_MN) tma_load_2d(&map_b, &full_bar[stage], sb, n0, kb * KB8, kEvictLast);  // box {128 (MN), 128 (K rows)}
          else tma_load_2d(&map_b, &full_bar[stage], sb, kb * KB8, n0, kEvictLast);
          bulk_copy_g2s(sf_base + stage * 2 * kSfBytes, p.sfa + ((long long)tm * p.sfa_kg + kb) * kSfBytes, kSfBytes, &full_bar[stage]);
          bulk_copy_g2s(sf_base + stage * 2 * kSfBytes + kSfBytes, p.sfb + ((long long)tn * p.sfb_kg + kb) * kSfBytes, kSfBytes,
                        &full_bar[stage]);
        } else {  // bf16 LoRA segment: [x | u]·[W | B]ᵀ shares the accumulator
          const int k = (kb - kb8) * KB16;
          mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
          tma_load_2d(&map_a2, &full_bar[stage], sa, k, m0, kEvictNormal);
          tma_load_2d(&map_b2, &full_bar[stage], sb, k, n0, kEvictLast);
        }
        __syncwarp();
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  // ======================================================================= consumers: 64 rows each
  setmaxnreg_inc<232>();
  const int cw = wg - 1;
  const int ct = threadIdx.x - 128;
  const uint32_t smem0 = smem_u32(smem);
  int stage = 0;
  uint32_t phase = 0;
  float acc[BN / 2], part[BN / 2];
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m0 = (tile / p.num_n_tiles) * BM, n0 = (tile % p.num_n_tiles) * BN;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < kb8 + kb16; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem0 + stage * kStageBytes + cw * 8192;
      uint32_t sb = smem0 + stage * kStageBytes + kTileBytes;
      if (kb < kb8) {
        if constexpr (B_MN) {
          named_bar_sync(1, 256);  // both warpgroups are done with the previous transposed tile
          transpose_fp8_tile(smem + stage * kStageBytes + kTileBytes, bt, ct);
          fence_proxy_async_smem();
          named_bar_sync(1, 256);
          sb = smem_u32(bt);
        }
        const uint8_t* sfa = sf_base + stage * 2 * kSfBytes;
        const uint8_t* sfb = sfa + kSfBytes;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {  // one K = 32 wgmma per scale column, scaled into the accumulator
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) part[i] = 0.f;
          wgmma_fence();
          wgmma_e4m3_ss_n128(part, desc_kmajor(sa + kk * 32), desc_kmajor(sb + kk * 32));
          wgmma_commit();
          wgmma_wait<0>();
          fence_regs(part);
          const float s_lo = ue8m0_value(sfa[sf_byte(cw * 64 + frag_row(0), kk)]);
          const float s_hi = ue8m0_value(sfa[sf_byte(cw * 64 + frag_row(2), kk)]);
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) {
            const float sbv = ue8m0_value(sfb[sf_byte(frag_col(i), kk)]);
            acc[i] = fmaf(part[i], (((i >> 1) & 1) ? s_hi : s_lo) * sbv, acc[i]);
          }
        }
      } else {
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < KB16 / 16; ++k) wgmma_bf16_ss_n128<0, 0>(acc, desc_kmajor(sa + k * 32), desc_kmajor(sb + k * 32));
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(acc);
      }
      mbar_arrive(&empty_bar[stage]);
      if (++stage == kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
      const int row = m0 + cw * 64 + frag_row(i), col = n0 + frag_col(i);
      if (row >= p.M || col >= p.N) continue;  // N is a multiple of 8: column pairs are whole
      float v0 = acc[i], v1 = acc[i + 1];
      if (p.residual != nullptr) {
        const float2 r = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.residual + (long long)row * p.ldr + col));
        v0 += r.x;
        v1 += r.y;
      }
      *reinterpret_cast<uint32_t*>(p.out + (long long)row * p.ldc + col) = pack_bf16x2(v0, v1);
    }
  }
}


// ---------------------------------------------------------------------------------------------- quantisation
__device__ __forceinline__ uint32_t sf_offset(long long row, int sfcol, int kg_per_block) {
  // byte offset of scale (row, scale column) in the [row block][k group][512] layout
  const long long rb = row >> 7;
  const int r = int(row & 127), kg = sfcol >> 2, j = sfcol & 3;
  return uint32_t(((rb * kg_per_block + kg) << 9) + ((r & 31) << 4) + ((r >> 5) << 2) + j);
}
// smallest power of two s = 2^e with amax / s <= 448 (E4M3 max); returns the biased UE8M0 byte and 1/s
__device__ __forceinline__ uint8_t ue8m0_for(float amax, float& inv_scale) {
  int e = -127;
  if (amax > 0.f) {
    e = (int)ceilf(log2f(amax * (1.f / 448.f)));
    e = max(-127, min(127, e));
  }
  inv_scale = exp2f((float)-e);
  return (uint8_t)(e + 127);
}

// rows: one warp per (row, 4 blocks of 32 columns): lane l holds 4 consecutive elements of column block l / 8
__global__ void __launch_bounds__(256) mx_quantize_rows_kernel(const bf16* __restrict__ x, long long ldx, uint8_t* __restrict__ q, long long ldq,
                                                               uint8_t* __restrict__ sf, int M, int K, int Kpad, int kg_per_block) {
  const int lane = threadIdx.x & 31;
  const long long warp_global = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int groups_per_row = Kpad / 128;
  const long long total = (long long)((M + 127) / 128 * 128) * groups_per_row;
  for (long long w = warp_global; w < total; w += ((long long)gridDim.x * blockDim.x) >> 5) {
    const long long row = w / groups_per_row;
    const int kg = int(w % groups_per_row);
    const int col = kg * 128 + lane * 4;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (row < M && col < K) {  // K is a multiple of 8: a 4-element group is entirely inside or outside
      const uint2 raw = *reinterpret_cast<const uint2*>(x + row * ldx + col);
      const float2 a = unpack_bf16x2(raw.x), b = unpack_bf16x2(raw.y);
      v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
    }
    float amax = fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3])));
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));  // 8 lanes = one 32-column block
    float inv;
    const uint8_t e = ue8m0_for(amax, inv);
    if ((lane & 7) == 0) sf[sf_offset(row, kg * 4 + (lane >> 3), kg_per_block)] = e;
    if (row < M && col < Kpad) {
      const __nv_fp8x2_storage_t lo = __nv_cvt_float2_to_fp8x2(make_float2(v[0] * inv, v[1] * inv), __NV_SATFINITE, __NV_E4M3);
      const __nv_fp8x2_storage_t hi = __nv_cvt_float2_to_fp8x2(make_float2(v[2] * inv, v[3] * inv), __NV_SATFINITE, __NV_E4M3);
      *reinterpret_cast<uint32_t*>(q + row * ldq + col) = (uint32_t)lo | ((uint32_t)hi << 16);
    }
  }
}

// weights: one warp per 32 x 32 tile (lane = row of the tile, 32 columns each); optional fp32 `delta` is added first (merge)
__global__ void __launch_bounds__(256) mx_quantize_weight_2d_kernel(const bf16* __restrict__ w, long long ldw, const uint8_t* __restrict__ q_old,
                                                                    const uint8_t* __restrict__ sf_old, const float* __restrict__ delta,
                                                                    long long ldd, uint8_t* __restrict__ q, long long ldq,
                                                                    uint8_t* __restrict__ sf_fwd, uint8_t* __restrict__ sf_bwd, int N, int K,
                                                                    int Npad, int Kpad, int kg_fwd, int kg_bwd) {
  const int lane = threadIdx.x & 31;
  const long long warp_global = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int tiles_k = Kpad / 32;
  const long long total = (long long)(Npad / 32) * tiles_k;
  for (long long t = warp_global; t < total; t += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int tn = int(t / tiles_k), tk = int(t % tiles_k);
    const long long n = (long long)tn * 32 + lane;
    float v[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = 0.f;
    if (n < N) {
      if (w != nullptr) {
#pragma unroll
        for (int j = 0; j < 32; j += 8) {
          const int k = tk * 32 + j;
          if (k < K) {
            float f[8];
            unpack8(*reinterpret_cast<const uint4*>(w + n * ldw + k), f);
#pragma unroll
            for (int i = 0; i < 8; ++i) v[j + i] = f[i];
          }
        }
      } else {  // requantisation: start from the packed weight and its (forward-layout) scale
        const float s_old = exp2f((float)sf_old[sf_offset(n, tk, kg_fwd)] - 127.f);
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          const int k = tk * 32 + j;
          if (k < Kpad) {
            const uint32_t raw = *reinterpret_cast<const uint32_t*>(q_old + n * ldq + k);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const __half_raw h = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)((raw >> (8 * i)) & 0xff), __NV_E4M3);
              v[j + i] = __half2float(*reinterpret_cast<const __half*>(&h)) * s_old;
            }
          }
        }
      }
      if (delta != nullptr) {
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int k = tk * 32 + j;
          if (k < K) v[j] += delta[n * ldd + k];
        }
      }
    }
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) amax = fmaxf(amax, fabsf(v[j]));
    amax = warp_max(amax);
    float inv;
    const uint8_t e = ue8m0_for(amax, inv);
    // forward layout: scale of (row n, k block tk); backward layout: scale of (row k, n block tn) for the 32 k of this tile
    if (n < Npad) sf_fwd[sf_offset(n, tk, kg_fwd)] = e;
    {
      const long long k = (long long)tk * 32 + lane;
      if (k < Kpad) sf_bwd[sf_offset(k, tn, kg_bwd)] = e;
    }
    if (n < Npad) {
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const int k = tk * 32 + j;
        if (k < Kpad) {
          const __nv_fp8x2_storage_t lo = __nv_cvt_float2_to_fp8x2(make_float2(v[j] * inv, v[j + 1] * inv), __NV_SATFINITE, __NV_E4M3);
          const __nv_fp8x2_storage_t hi = __nv_cvt_float2_to_fp8x2(make_float2(v[j + 2] * inv, v[j + 3] * inv), __NV_SATFINITE, __NV_E4M3);
          *reinterpret_cast<uint32_t*>(q + n * ldq + k) = (uint32_t)lo | ((uint32_t)hi << 16);
        }
      }
    }
  }
}

// dense bf16 copy of a packed weight (checkpoints, numerics oracle)
__global__ void __launch_bounds__(256) mx_dequantize_weight_kernel(const uint8_t* __restrict__ q, long long ldq, const uint8_t* __restrict__ sf,
                                                                   bf16* __restrict__ out, long long ldo, int N, int K, int kg) {
  const long long total = (long long)N * (K / 4);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / (K / 4);
    const int k = int(i % (K / 4)) * 4;
    const float s = exp2f((float)sf[sf_offset(n, k >> 5, kg)] - 127.f);
    const uint32_t raw = *reinterpret_cast<const uint32_t*>(q + n * ldq + k);
    float f[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __half_raw h = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)((raw >> (8 * j)) & 0xff), __NV_E4M3);
      f[j] = __half2float(*reinterpret_cast<const __half*>(&h)) * s;
    }
    uint2 o;
    o.x = pack_bf16x2(f[0], f[1]);
    o.y = pack_bf16x2(f[2], f[3]);
    *reinterpret_cast<uint2*>(out + n * ldo + k) = o;
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------- host
long long mx_sf_bytes(long long rows, long long k_elems) { return ((rows + 127) / 128) * ((k_elems + 127) / 128) * 512; }

void mx_quantize_rows(const void* x, long long ldx, void* q, long long ldq, void* sf, int M, int K, cudaStream_t s) {
  if (K % 8) throw std::runtime_error("mx_quantize_rows: K must be a multiple of 8");
  const int Kpad = (K + 127) / 128 * 128;
  if (ldq < Kpad) throw std::runtime_error("mx_quantize_rows: the fp8 buffer needs a row pitch >= K rounded up to 128");
  const long long warps = (long long)((M + 127) / 128 * 128) * (Kpad / 128);
  const int grid = (int)std::min<long long>((warps * 32 + 255) / 256, (long long)num_sms() * 16);
  if (grid <= 0) return;
  launch_k(mx_quantize_rows_kernel, grid, 256, 0, s, (const bf16*)x, ldx, (uint8_t*)q, ldq, (uint8_t*)sf, M, K, Kpad, Kpad / 128);
  RB_CHECK_LAUNCH("mx_quantize_rows");
}

void mx_quantize_weight_2d(const void* w, long long ldw, const void* q_old, const void* sf_old, const float* delta, long long ldd, void* q,
                           long long ldq, void* sf_fwd, void* sf_bwd, int N, int K, cudaStream_t s) {
  if (K % 8) throw std::runtime_error("mx_quantize_weight_2d: K must be a multiple of 8");
  const int Npad = (N + 127) / 128 * 128, Kpad = (K + 127) / 128 * 128;
  if (ldq < Kpad) throw std::runtime_error("mx_quantize_weight_2d: the fp8 buffer needs a row pitch >= K rounded up to 128");
  const long long warps = (long long)(Npad / 32) * (Kpad / 32);
  const int grid = (int)std::min<long long>((warps * 32 + 255) / 256, (long long)num_sms() * 16);
  launch_k(mx_quantize_weight_2d_kernel, grid, 256, 0, s, (const bf16*)w, ldw, (const uint8_t*)q_old, (const uint8_t*)sf_old, delta, ldd,
           (uint8_t*)q, ldq, (uint8_t*)sf_fwd, (uint8_t*)sf_bwd, N, K, Npad, Kpad, Kpad / 128, Npad / 128);
  RB_CHECK_LAUNCH("mx_quantize_weight_2d");
}

void mx_dequantize_weight(const void* q, long long ldq, const void* sf_fwd, void* out, long long ldo, int N, int K, cudaStream_t s) {
  if (K % 4) throw std::runtime_error("mx_dequantize_weight: K must be a multiple of 4");
  const int Kpad = (K + 127) / 128 * 128;
  const long long total = (long long)N * (K / 4);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 16);
  if (grid <= 0) return;
  launch_k(mx_dequantize_weight_kernel, grid, 256, 0, s, (const uint8_t*)q, ldq, (const uint8_t*)sf_fwd, (bf16*)out, ldo, N, K, Kpad / 128);
  RB_CHECK_LAUNCH("mx_dequantize_weight");
}

void gemm_mx(const MxGemmDesc& d, cudaStream_t stream) {
  if (d.M <= 0 || d.N <= 0) return;
  const int K8 = (d.K + 127) / 128 * 128;
  if (d.K2 % KB16) throw std::runtime_error("gemm_mx: the bf16 segment must be a multiple of 64");
  if (d.ldc % 8 || (reinterpret_cast<uintptr_t>(d.out) & 15)) throw std::runtime_error("gemm_mx: output must be 16-byte aligned");
  if (d.N % 8) throw std::runtime_error("gemm_mx: N must be a multiple of 8");
  MxArgs p;
  p.M = d.M; p.N = d.N; p.K8 = K8; p.K2 = d.K2;
  p.sfa = reinterpret_cast<const uint8_t*>(d.sfa); p.sfb = reinterpret_cast<const uint8_t*>(d.sfb);
  p.sfa_kg = K8 / 128; p.sfb_kg = K8 / 128;
  p.num_m_tiles = ceil_div(d.M, BM); p.num_n_tiles = ceil_div(d.N, BN);
  p.out = reinterpret_cast<bf16*>(d.out); p.ldc = d.ldc;
  p.residual = reinterpret_cast<const bf16*>(d.residual); p.ldr = d.ldr;
  // operands: fp8 bytes; A [M, K8] K-major (pitch lda); B K-major [N, K8] (pitch ldb) or MN-major [K8 rows, N] (pitch ldb)
  CUtensorMap ma = make_map_2d_sw128(d.a, K8, d.M, d.lda, KB8, BM, 1);
  CUtensorMap mb = d.b_mn_major ? make_map_2d_sw128(d.b, d.N, K8, d.ldb, 128, KB8, 1) : make_map_2d_sw128(d.b, K8, d.N, d.ldb, KB8, BN, 1);
  CUtensorMap ma2 = ma, mb2 = mb;
  if (d.K2 > 0) {
    ma2 = make_map_2d_sw128(d.a2, d.K2, d.M, d.lda2, KB16, BM, 2);
    mb2 = make_map_2d_sw128(d.b2, d.K2, d.N, d.ldb2, KB16, BN, 2);
  }
  if (d.residual != nullptr) {
    if (d.ldr % 8 || (reinterpret_cast<uintptr_t>(d.residual) & 15)) throw std::runtime_error("gemm_mx: residual must be 16-byte aligned");
  }
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  if (d.b_mn_major) {
    static bool cfg = false;
    if (!cfg) { check(cudaFuncSetAttribute(gemm_mx_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotal), "attr(gemm_mx)"); cfg = true; }
    launch_k(gemm_mx_kernel<true>, grid, 384, kSmemTotal, stream, ma, mb, ma2, mb2, p);
  } else {
    static bool cfg = false;
    if (!cfg) { check(cudaFuncSetAttribute(gemm_mx_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotal), "attr(gemm_mx)"); cfg = true; }
    launch_k(gemm_mx_kernel<false>, grid, 384, kSmemTotal, stream, ma, mb, ma2, mb2, p);
  }
  RB_CHECK_LAUNCH("gemm_mx");
}

}  // namespace rb
