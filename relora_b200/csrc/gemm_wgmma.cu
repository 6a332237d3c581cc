// Persistent warp-specialised bf16 / fp8 GEMM for sm_90a: TMA -> shared memory (128B swizzle) -> wgmma with fp32
// accumulators in registers -> epilogue straight from registers.
//
//   D[M,N] = alpha * ( A1[M,K1]·B1[N,K1]ᵀ + A2[M,K2]·B2[N,K2]ᵀ ) (+ bias) (+ residual) (+ D)
//
// The second product is the fused LoRA up-projection: it simply extends the K loop ("concat-K"), so the frozen
// weight GEMM and the low-rank branch share one accumulator, one read of x and one write of y.
// Reference behaviour being replaced: relora.py:319-322 (F.linear + dropout + two small GEMMs + mul + add).
//
// Roles (384 threads, 1 CTA / SM, persistent over output tiles):
//   warpgroup 0   TMA producer (warp 0, one elected lane issues)        smem ring: full[s] / empty[s]
//   warpgroups 1-2 consumers: each issues the wgmma of its 64 rows of the 128-row tile and writes them out
#include <cuda.h>

#include <cstdlib>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "gemm.h"
#include "tensormap.h"
#include "sm90.cuh"

namespace rb {

long long g_launch_count = 0;

using namespace sm90;

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 bytes = one swizzle row (fp8: 128 elements)
constexpr int kNumThreads = 384;

struct KernelArgs {
  int M, N, K1, K2;
  int n_per_group, a1_group_kofs, a2_group_kofs;
  int b1_group_kofs, b1_local_n;        // B1: K-window offset per N-group; MN coordinate relative to the group
  int m_per_group, b1_mn_ofs_per_mgroup; // B1: extra MN offset selected by the M-tile's group (weight gradients)
  void* out;
  long long ldc;
  const bf16* residual;
  long long ldr;
  const bf16* bias;  // [N], added in fp32 (Pythia projections carry biases)
  float alpha;
  const float* alpha_dev;  // optional device scalar multiplied into alpha (fp8 dequantisation scales live on the device)
  int fp8;                 // segment 1 (A1, B1) holds fp8 bytes: k-blocks of 128 elements, e4m3 wgmma (2: A1 is E5M2)
  int out_f32, accumulate;
  int num_m_tiles, num_n_tiles;
  int tiles_per_group;  // N-tiles per output-column group (the last one of a group may be ragged)
  int split_k;  // >1: each output tile is computed by split_k CTAs over disjoint K ranges, combined with fp32 atomics
};

template <int BLOCK_N>
struct SmemLayout {
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;  // 16 KB
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (192 * 1024) / kStageBytes;  // 6 stages of 128-wide tiles, 4 of 256-wide tiles
  static constexpr int kTileBytes = kStages * kStageBytes;
  static constexpr int kTotal = kTileBytes + 1024 + 1024;  // barriers, manual 1024-byte alignment
};
static_assert(SmemLayout<256>::kTotal <= 232448 && SmemLayout<128>::kTotal <= 232448, "shared memory budget");

// Issue the TMA loads of one operand tile (BLOCK_MN x BLOCK_K) into `dst`.
template <int BLOCK_MN, bool MN_MAJOR>
__device__ __forceinline__ void load_operand(const CUtensorMap* map, uint64_t* bar, uint8_t* dst, int mn0, int k0, uint64_t hint) {
  if constexpr (!MN_MAJOR) {
    tma_load_2d(map, bar, dst, k0, mn0, hint);  // box {64 (K), BLOCK_MN}
  } else {
#pragma unroll
    for (int j = 0; j < BLOCK_MN / 64; ++j) tma_load_2d(map, bar, dst + j * 8192, mn0 + j * 64, k0, hint);  // box {64 (MN), 64 (K)}
  }
}

// One k-block of MMAs of a consumer warpgroup: A = its 64 rows of the stage's A tile, B = the whole B tile.
template <int BLOCK_N, bool A_MN, bool B_MN>
__device__ __forceinline__ void mma_bf16_kblock(float (&acc)[BLOCK_N / 2], uint32_t sa, uint32_t sb) {
  const uint64_t da = A_MN ? desc_mnmajor(sa) : desc_kmajor(sa);
  const uint64_t db = B_MN ? desc_mnmajor(sb) : desc_kmajor(sb);
  constexpr uint64_t kStepA = A_MN ? 128 : 2, kStepB = B_MN ? 128 : 2;  // (byte offset >> 4) per K = 16
#pragma unroll
  for (int k = 0; k < BLOCK_K / 16; ++k) {
    if constexpr (BLOCK_N == 256) wgmma_bf16_ss_n256<A_MN, B_MN>(acc, da + kStepA * k, db + kStepB * k);
    else if constexpr (BLOCK_N == 128) wgmma_bf16_ss_n128<A_MN, B_MN>(acc, da + kStepA * k, db + kStepB * k);
    else wgmma_bf16_ss_n64<A_MN, B_MN>(acc, da + kStepA * k, db + kStepB * k);
  }
}
template <int BLOCK_N>
__device__ __forceinline__ void mma_fp8_kblock(float (&acc)[BLOCK_N / 2], uint32_t sa, uint32_t sb, bool a_e5m2) {
  const uint64_t da = desc_kmajor(sa), db = desc_kmajor(sb);
#pragma unroll
  for (int k = 0; k < 4; ++k) {  // rows of 128 bytes: four K = 32 steps
    if constexpr (BLOCK_N == 256) {
      if (a_e5m2) wgmma_e5m2_ss_n256(acc, da + 2 * k, db + 2 * k);
      else wgmma_e4m3_ss_n256(acc, da + 2 * k, db + 2 * k);
    } else {
      if (a_e5m2) wgmma_e5m2_ss_n128(acc, da + 2 * k, db + 2 * k);
      else wgmma_e4m3_ss_n128(acc, da + 2 * k, db + 2 * k);
    }
  }
}

template <int BLOCK_N, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap map_a1, const __grid_constant__ CUtensorMap map_b1,
            const __grid_constant__ CUtensorMap map_a2, const __grid_constant__ CUtensorMap map_b2, const KernelArgs p) {
  using L = SmemLayout<BLOCK_N>;
  constexpr int kStages = L::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kTileBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const uint32_t warp = warp_id();
  const int wg = threadIdx.x / 128;
  if (threadIdx.x == 0) {
    pdl_launch_dependents();
    tma_prefetch_desc(&map_a1);
    tma_prefetch_desc(&map_b1);
    if (p.K2 > 0) {
      tma_prefetch_desc(&map_a2);
      tma_prefetch_desc(&map_b2);
    }
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 256);  // every consumer thread releases the slot
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();  // everything above is CTA-local: it overlaps the tail of the previous kernel in the stream (PDL)

  const int num_tiles = p.num_m_tiles * p.num_n_tiles;
  const int num_work = num_tiles * p.split_k;
  const int kstep1 = p.fp8 ? 2 * BLOCK_K : BLOCK_K;  // elements per k-block of segment 1 (always 128 bytes per row)
  const int kb1 = (p.K1 + kstep1 - 1) / kstep1;
  const int kb2 = (p.K2 + BLOCK_K - 1) / BLOCK_K;
  const int num_kb = kb1 + kb2;
  const int kb_per_split = (num_kb + p.split_k - 1) / p.split_k;

  if (wg == 0) {
    // ===================================================================== TMA producer (whole warp walks the loop)
    setmaxnreg_dec<40>();
    if (warp != 0) return;
    int stage = 0;
    uint32_t phase = 0;
    for (int work = blockIdx.x; work < num_work; work += gridDim.x) {
      const int tile = work / p.split_k, split = work % p.split_k;
      const int m0 = (tile / p.num_n_tiles) * BLOCK_M;
      const int tn = tile % p.num_n_tiles;
      const int g = tn / p.tiles_per_group;
      const int nl = (tn % p.tiles_per_group) * BLOCK_N;  // column offset inside the group
      const int n0 = g * p.n_per_group + nl;
      const int a1_k = g * p.a1_group_kofs;
      const int a2_k = g * p.a2_group_kofs;
      const int b1_k = g * p.b1_group_kofs;
      const int b1_n = (p.b1_local_n ? nl : n0) + (m0 / p.m_per_group) * p.b1_mn_ofs_per_mgroup;
      const int kb_begin = split * kb_per_split, kb_end = min(num_kb, kb_begin + kb_per_split);
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (elect_one()) {
          uint8_t* sa = smem + stage * L::kStageBytes;
          uint8_t* sb = sa + L::kABytes;
          mbar_arrive_expect_tx(&full_bar[stage], L::kStageBytes);
          if (kb < kb1) {
            load_operand<BLOCK_M, A_MN>(&map_a1, &full_bar[stage], sa, m0, a1_k + kb * kstep1, kEvictNormal);
            load_operand<BLOCK_N, B_MN>(&map_b1, &full_bar[stage], sb, b1_n, b1_k + kb * kstep1, kEvictLast);
          } else {
            const int k = (kb - kb1) * BLOCK_K;
            load_operand<BLOCK_M, false>(&map_a2, &full_bar[stage], sa, m0, a2_k + k, kEvictNormal);
            load_operand<BLOCK_N, false>(&map_b2, &full_bar[stage], sb, n0, k, kEvictLast);
          }
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
  const uint32_t smem0 = smem_u32(smem);
  const float alpha_eff = p.alpha * (p.alpha_dev != nullptr ? *p.alpha_dev : 1.0f);
  const bool out_vec = (p.ldc % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.out) & 7) == 0);
  const bool res_vec = p.residual != nullptr && (p.ldr % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.residual) & 3) == 0);
  int stage = 0;
  uint32_t phase = 0;
  float acc[BLOCK_N / 2];
  for (int work = blockIdx.x; work < num_work; work += gridDim.x) {
    const int tile = work / p.split_k, split = work % p.split_k;
    const int m0 = (tile / p.num_n_tiles) * BLOCK_M;
    const int tn = tile % p.num_n_tiles;
    const int nl = (tn % p.tiles_per_group) * BLOCK_N;
    const int n0 = (tn / p.tiles_per_group) * p.n_per_group + nl;
    const int n_lim = min(p.N, n0 + min(BLOCK_N, p.n_per_group - nl));  // a group's last tile may be ragged
    const int kb_begin = split * kb_per_split, kb_end = min(num_kb, kb_begin + kb_per_split);
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
    for (int kb = kb_begin; kb < kb_end; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem0 + stage * L::kStageBytes + cw * 8192;  // this warpgroup's 64 rows (either major)
      const uint32_t sb = smem0 + stage * L::kStageBytes + L::kABytes;
      wgmma_fence();
      if (kb < kb1 && p.fp8) mma_fp8_kblock<BLOCK_N>(acc, sa, sb, p.fp8 == 2);
      else if (kb < kb1) mma_bf16_kblock<BLOCK_N, A_MN, B_MN>(acc, sa, sb);
      else mma_bf16_kblock<BLOCK_N, false, false>(acc, sa, sb);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(acc);
      mbar_arrive(&empty_bar[stage]);
      if (++stage == kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    if (kb_begin >= kb_end) continue;  // nothing was accumulated for this work item
    // ---- epilogue: each thread owns column pairs of two rows (accumulator fragment order)
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; i += 2) {
      const int row = m0 + cw * 64 + frag_row(i);
      const int col = n0 + frag_col(i);
      if (row >= p.M || col >= n_lim) continue;
      const bool pair_ok = col + 1 < n_lim;
      float v0 = acc[i] * alpha_eff, v1 = acc[i + 1] * alpha_eff;
      if (p.split_k > 1) {
        float* op = reinterpret_cast<float*>(p.out) + (long long)row * p.ldc + col;
        atomicAdd(op, v0);
        if (pair_ok) atomicAdd(op + 1, v1);
      } else if (p.out_f32) {
        float* op = reinterpret_cast<float*>(p.out) + (long long)row * p.ldc + col;
        if (pair_ok && out_vec) {
          float2 o = make_float2(v0, v1);
          if (p.accumulate) {
            const float2 old = *reinterpret_cast<const float2*>(op);
            o.x += old.x;
            o.y += old.y;
          }
          *reinterpret_cast<float2*>(op) = o;
        } else {
          op[0] = p.accumulate ? op[0] + v0 : v0;
          if (pair_ok) op[1] = p.accumulate ? op[1] + v1 : v1;
        }
      } else {
        bf16* op = reinterpret_cast<bf16*>(p.out) + (long long)row * p.ldc + col;
        if (p.bias != nullptr) {
          v0 += __bfloat162float(p.bias[col]);
          if (pair_ok) v1 += __bfloat162float(p.bias[col + 1]);
        }
        if (p.residual != nullptr) {
          const bf16* rp = p.residual + (long long)row * p.ldr + col;
          if (pair_ok && res_vec) {
            const float2 r = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(rp));
            v0 += r.x;
            v1 += r.y;
          } else {
            v0 += __bfloat162float(rp[0]);
            if (pair_ok) v1 += __bfloat162float(rp[1]);
          }
        }
        if (pair_ok && out_vec) {
          uint32_t* o32 = reinterpret_cast<uint32_t*>(op);
          if (p.accumulate) {
            const float2 old = unpack_bf16x2(*o32);
            v0 += old.x;
            v1 += old.y;
          }
          *o32 = pack_bf16x2(v0, v1);
        } else {
          op[0] = __float2bfloat16_rn(p.accumulate ? __bfloat162float(op[0]) + v0 : v0);
          if (pair_ok) op[1] = __float2bfloat16_rn(p.accumulate ? __bfloat162float(op[1]) + v1 : v1);
        }
      }
    }
  }
}

// =============================================================================================
// Fused backward of a stacked LoRA group (input gradient):
//
//   dx[M,N] = dy[M,Kb] · W[Kb,N]  +  inv_keep · Σ_g keep_g(row, col) ⊙ ( du_g[M,r] · A_g[r,N] )
//
// (Kb = G·Ng: the group's stacked output width; N: the group's input width.)  The dropout mask sits on the LoRA
// *input*, i.e. on the output of this backward product, so the low-rank terms cannot share the accumulator of the
// frozen path.  Each consumer warpgroup runs the G short LoRA products first into one register accumulator, folds each
// one, masked, into a second, and then lets the long frozen-path reduction accumulate on top of the combined term: one
// write of dx instead of base-GEMM + parts-GEMM + dropout_combine.  With Kb == 0 the frozen-path product `base` was
// computed by a separate GEMM and is added from global memory.
// Reference math: backward of relora.py:319-322 with nn.Dropout on the LoRA input.
struct LoraDxArgs {
  int M, N, Kb, r, G;
  bf16* out;
  long long ldc;
  const bf16* base;
  long long ld_base;
  int num_m_tiles, num_n_tiles;
  uint32_t thr16;
  float inv_keep;
  const uint32_t* seed_ptr;
  uint32_t keys[3];
};

__global__ void __launch_bounds__(kNumThreads, 1)
lora_dx_kernel(const __grid_constant__ CUtensorMap map_dy, const __grid_constant__ CUtensorMap map_w,
               const __grid_constant__ CUtensorMap map_du, const __grid_constant__ CUtensorMap map_a, const LoraDxArgs p) {
  constexpr int BLOCK_N = 128;
  using L = SmemLayout<BLOCK_N>;
  constexpr int kStages = L::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kTileBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const uint32_t warp = warp_id();
  const int wg = threadIdx.x / 128;
  if (threadIdx.x == 0) {
    pdl_launch_dependents();
    tma_prefetch_desc(&map_du);
    tma_prefetch_desc(&map_a);
    if (p.Kb > 0) {
      tma_prefetch_desc(&map_dy);
      tma_prefetch_desc(&map_w);
    }
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 256);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  const int num_tiles = p.num_m_tiles * p.num_n_tiles;
  const int kb_lora = p.r / BLOCK_K;  // r is a multiple of 64
  const int kb_base = (p.Kb + BLOCK_K - 1) / BLOCK_K;

  if (wg == 0) {
    // ===================================================================== TMA producer
    setmaxnreg_dec<40>();
    if (warp != 0) return;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m0 = (tile / p.num_n_tiles) * BLOCK_M;
      const int n0 = (tile % p.num_n_tiles) * BLOCK_N;
      for (int kb = 0; kb < p.G * kb_lora + kb_base; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (elect_one()) {
          uint8_t* sa = smem + stage * L::kStageBytes;
          mbar_arrive_expect_tx(&full_bar[stage], L::kStageBytes);
          if (kb < p.G * kb_lora) {  // du [M, G·r] K-major ; A [G·r, N] MN-major
            load_operand<BLOCK_M, false>(&map_du, &full_bar[stage], sa, m0, kb * BLOCK_K, kEvictNormal);
            load_operand<BLOCK_N, true>(&map_a, &full_bar[stage], sa + L::kABytes, n0, kb * BLOCK_K, kEvictLast);
          } else {                   // dy [M, Kb] K-major ; W [Kb, N] MN-major
            const int k = (kb - p.G * kb_lora) * BLOCK_K;
            load_operand<BLOCK_M, false>(&map_dy, &full_bar[stage], sa, m0, k, kEvictNormal);
            load_operand<BLOCK_N, true>(&map_w, &full_bar[stage], sa + L::kABytes, n0, k, kEvictLast);
          }
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

  setmaxnreg_inc<232>();
  const int cw = wg - 1;
  const uint32_t smem0 = smem_u32(smem);
  const uint32_t seed0 = p.seed_ptr ? *p.seed_ptr : 0u;
  uint32_t seeds[3];
#pragma unroll
  for (int g = 0; g < 3; ++g) seeds[g] = mix_seed(seed0, p.keys[g]);
  int stage = 0;
  uint32_t phase = 0;
  auto mma_blocks = [&](float (&acc)[BLOCK_N / 2], int n) {
    for (int kb = 0; kb < n; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem0 + stage * L::kStageBytes + cw * 8192;
      wgmma_fence();
      mma_bf16_kblock<BLOCK_N, false, true>(acc, sa, smem0 + stage * L::kStageBytes + L::kABytes);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(acc);
      mbar_arrive(&empty_bar[stage]);
      if (++stage == kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
  };
  float acc[BLOCK_N / 2], cmb[BLOCK_N / 2];
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m0 = (tile / p.num_n_tiles) * BLOCK_M + cw * 64;
    const int n0 = (tile % p.num_n_tiles) * BLOCK_N;
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) cmb[i] = 0.f;
    for (int g = 0; g < p.G; ++g) {
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
      mma_blocks(acc, kb_lora);
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; i += 2) {  // one hash per column pair (common.cuh:keep_drop)
        const uint32_t row = m0 + frag_row(i), col = n0 + frag_col(i);
        const uint32_t hsh = lowbias32((row * 0x9E3779B1u) ^ seeds[g] ^ ((col >> 1) * 0x85EBCA77u));
        if ((hsh & 0xFFFFu) >= p.thr16) cmb[i] += acc[i];
        if ((hsh >> 16) >= p.thr16) cmb[i + 1] += acc[i + 1];
      }
    }
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = cmb[i] * p.inv_keep;
    if (kb_base > 0) mma_blocks(acc, kb_base);  // the frozen-path product accumulates on top of the combined LoRA term
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; i += 2) {
      const int row = m0 + frag_row(i), col = n0 + frag_col(i);
      if (row >= p.M || col >= p.N) continue;  // N is a multiple of 8: column pairs are whole
      float v0 = acc[i], v1 = acc[i + 1];
      if (kb_base == 0) {
        const float2 b = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.base + (long long)row * p.ld_base + col));
        v0 += b.x;
        v1 += b.y;
      }
      *reinterpret_cast<uint32_t*>(p.out + (long long)row * p.ldc + col) = pack_bf16x2(v0, v1);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host: tensor-map construction (driver entry point resolved at run time; no link against libcuda)
// ---------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    check(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q), "cudaGetDriverEntryPoint");
    if (q != cudaDriverEntryPointSuccess || p == nullptr) throw std::runtime_error("cuTensorMapEncodeTiled not available");
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

struct MapKey {
  const void* ptr;
  long long inner, outer, ld;
  int box_inner, box_outer, esize;
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && inner == o.inner && outer == o.outer && ld == o.ld && box_inner == o.box_inner && box_outer == o.box_outer && esize == o.esize;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.ptr);
    auto mix = [&](long long v) { h ^= std::hash<long long>()(v) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
    mix(k.inner); mix(k.outer); mix(k.ld); mix(k.box_inner); mix(k.box_outer); mix(k.esize);
    return h;
  }
};
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;
static std::mutex g_maps_mu;

void gemm_clear_descriptor_cache() {
  std::lock_guard<std::mutex> lk(g_maps_mu);
  g_maps.clear();
}

// 2-D bf16 tensor, `inner` contiguous elements per row, `outer` rows `ld` elements apart, 128B swizzle.
static CUtensorMap make_map_2d(const void* ptr, long long inner, long long outer, long long ld, int box_inner, int box_outer,
                               int esize = 2) {
  MapKey key{ptr, inner, outer, ld, box_inner, box_outer, esize};
  {
    std::lock_guard<std::mutex> lk(g_maps_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) return it->second;
  }
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0) throw std::runtime_error("gemm operand pointer must be 16-byte aligned");
  if ((ld * esize) % 16 != 0) throw std::runtime_error("gemm operand leading dimension must be a multiple of 16 bytes");
  CUtensorMap m;
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)ld * esize};
  cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer};
  const CUtensorMapDataType dt = esize == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode()(&m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_ERROR_INVALID_CONTEXT) {
    // the driver call needs the primary context current on THIS thread; autograd worker threads only bind it lazily.
    // cudaSetDevice binds it and, unlike cudaFree(0), is legal while a stream is being captured.
    int dev = 0;
    check(cudaGetDevice(&dev), "cudaGetDevice");
    check(cudaSetDevice(dev), "cudaSetDevice");
    r = get_encode()(&m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
  std::lock_guard<std::mutex> lk(g_maps_mu);
  if (g_maps.size() > 8192) g_maps.clear();  // eager runs see fresh activation pointers every step: bound the cache
  g_maps.emplace(key, m);
  return m;
}

// 3-D bf16 tensor map (128B swizzle, zero fill outside the tensor): dims d0 (contiguous) x d1 x d2 with strides s1 / s2 elements.
// Attention views the packed [rows, 3*hidden] qkv buffer as [head_dim, heads, rows]; a 64-wide box over a 48-wide head is
// zero padded by the TMA unit.
CUtensorMap make_map_3d_bf16(const void* ptr, long long d0, long long d1, long long d2, long long s1, long long s2, int b0, int b1,
                             int b2) {
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (s1 * 2) % 16 != 0 || (s2 * 2) % 16 != 0)
    throw std::runtime_error("tensor map: base and strides must be 16-byte aligned");
  CUtensorMap m;
  cuuint64_t dims[3] = {(cuuint64_t)d0, (cuuint64_t)d1, (cuuint64_t)d2};
  cuuint64_t strides[2] = {(cuuint64_t)s1 * 2, (cuuint64_t)s2 * 2};
  cuuint32_t box[3] = {(cuuint32_t)b0, (cuuint32_t)b1, (cuuint32_t)b2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = CUDA_SUCCESS;
  for (int attempt = 0; attempt < 2; ++attempt) {
    r = get_encode()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_ERROR_INVALID_CONTEXT) break;
    int dev = 0;  // bind the primary context on this thread (legal during stream capture), then retry
    check(cudaGetDevice(&dev), "cudaGetDevice");
    check(cudaSetDevice(dev), "cudaSetDevice");
  }
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled(3d) failed with code " + std::to_string((int)r));
  return m;
}

// exported for the other translation units (gemm_mx.cu): same cache, same checks
CUtensorMap make_map_2d_sw128(const void* ptr, long long inner, long long outer, long long ld, int box_inner, int box_outer, int esize) {
  return make_map_2d(ptr, inner, outer, ld, box_inner, box_outer, esize);
}


// Operand covering `mn` rows/cols of the output dimension and `k` of the reduction dimension.
static CUtensorMap operand_map(const Operand& o, long long mn, long long k, int block_mn, bool fp8 = false) {
  if (fp8) return make_map_2d(o.ptr, k, mn, o.ld, 2 * BLOCK_K, block_mn, 1);  // E4M3 bytes, K-major only
  if (!o.mn_major) return make_map_2d(o.ptr, k, mn, o.ld, BLOCK_K, block_mn);
  return make_map_2d(o.ptr, mn, k, o.ld, 64, BLOCK_K);
}

template <int BLOCK_N, bool A_MN, bool B_MN>
static void launch(const GemmDesc& d, cudaStream_t stream) {
  using L = SmemLayout<BLOCK_N>;
  KernelArgs p;
  p.M = d.M; p.N = d.N; p.K1 = d.K1; p.K2 = d.K2;
  p.n_per_group = d.n_per_group > 0 ? d.n_per_group : (d.N > 0 ? d.N : 1);
  p.a1_group_kofs = d.a1_group_kofs; p.a2_group_kofs = d.a2_group_kofs;
  p.b1_group_kofs = d.b1_group_kofs; p.b1_local_n = d.b1_local_n ? 1 : 0;
  p.m_per_group = d.m_per_group > 0 ? d.m_per_group : (1 << 30); p.b1_mn_ofs_per_mgroup = d.b1_mn_ofs_per_mgroup;
  p.out = d.out; p.ldc = d.ldc; p.residual = reinterpret_cast<const bf16*>(d.residual); p.ldr = d.ldr;
  p.bias = reinterpret_cast<const bf16*>(d.bias);
  if (d.bias != nullptr && d.out_f32) throw std::runtime_error("gemm: bias is only fused for bf16 outputs");
  p.alpha = d.alpha; p.alpha_dev = d.alpha_dev; p.fp8 = d.fp8 ? (d.fp8_a_e5m2 ? 2 : 1) : 0; p.out_f32 = d.out_f32 ? 1 : 0; p.accumulate = d.accumulate ? 1 : 0;
  p.num_m_tiles = ceil_div(d.M, BLOCK_M);
  const int groups = ceil_div(d.N, p.n_per_group);
  // tiles never straddle a group: the last tile of a group may be ragged (its tail columns are computed but not stored)
  if (groups > 1 && (p.n_per_group % 64) != 0) throw std::runtime_error("gemm: n_per_group must be a multiple of 64");
  p.tiles_per_group = ceil_div(p.n_per_group, BLOCK_N);
  p.num_n_tiles = groups * p.tiles_per_group;

  // K extents of the global tensors include the per-group windows
  const long long a1_k_total = (long long)d.K1 + (long long)(groups - 1) * d.a1_group_kofs;
  if (d.fp8 && (A_MN || B_MN)) throw std::runtime_error("gemm: fp8 operands must be K-major");
  CUtensorMap ma1 = operand_map(d.a1, d.M, a1_k_total, BLOCK_M, d.fp8);
  const int mgroups = d.m_per_group > 0 ? ceil_div(d.M, d.m_per_group) : 1;
  const long long b1_mn_total = (d.b1_local_n ? (long long)p.n_per_group : (long long)d.N) + (long long)(mgroups - 1) * d.b1_mn_ofs_per_mgroup;
  const long long b1_k_total = (long long)d.K1 + (long long)(groups - 1) * d.b1_group_kofs;
  if (d.m_per_group > 0 && (d.m_per_group % BLOCK_M) != 0) throw std::runtime_error("gemm: m_per_group must be a multiple of the M tile");
  CUtensorMap mb1 = operand_map(d.b1, b1_mn_total, b1_k_total, BLOCK_N, d.fp8);
  CUtensorMap ma2 = ma1, mb2 = mb1;
  if (d.K2 > 0) {
    if (d.a2.mn_major || d.b2.mn_major) throw std::runtime_error("gemm: the LoRA (A2/B2) operands must be K-major");
    const long long a2_k_total = (long long)d.K2 + (long long)(groups - 1) * d.a2_group_kofs;
    ma2 = operand_map(d.a2, d.M, a2_k_total, BLOCK_M);
    mb2 = operand_map(d.b2, d.N, d.K2, BLOCK_N);
  }
  auto kern = gemm_kernel<BLOCK_N, A_MN, B_MN>;
  static bool configured = false;
  if (!configured) {
    check(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal), "cudaFuncSetAttribute(gemm)");
    configured = true;
  }
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  const int num_kb = ceil_div(d.K1, d.fp8 ? 2 * BLOCK_K : BLOCK_K) + ceil_div(d.K2, BLOCK_K);
  int split = d.split_k;
  if (split == 0) {  // auto: fill the machine when there are few output tiles and a long reduction
    split = 1;
    if (d.out_f32 && d.accumulate && d.residual == nullptr && tiles * 2 <= num_sms() && num_kb >= 16)
      split = std::min(std::min(num_sms() / tiles, num_kb / 4), 64);
  }
  if (split > 1 && !(d.out_f32 && d.accumulate && d.residual == nullptr))
    throw std::runtime_error("gemm: split_k needs an fp32 accumulate output without residual");
  if (split < 1) split = 1;
  p.split_k = split;
  const int work = tiles * split;
  const int grid = work < num_sms() ? work : num_sms();
  if (grid <= 0) return;
  launch_k(kern, grid, kNumThreads, L::kTotal, stream, ma1, mb1, ma2, mb2, p);
  RB_CHECK_LAUNCH("gemm_kernel");
}

template <int BLOCK_N>
static void dispatch_major(const GemmDesc& d, cudaStream_t s) {
  if (d.a1.mn_major) {
    if (d.b1.mn_major) launch<BLOCK_N, true, true>(d, s);
    else launch<BLOCK_N, true, false>(d, s);
  } else {
    if (d.b1.mn_major) launch<BLOCK_N, false, true>(d, s);
    else launch<BLOCK_N, false, false>(d, s);
  }
}

void gemm_bf16(const GemmDesc& d, cudaStream_t stream) {
  if (d.n_lora_acc != 0) throw std::runtime_error("gemm: dropout-combine epilogue not built into this kernel variant");
  if (d.M <= 0 || d.N <= 0) return;
  int bn = d.block_n;
  if (bn == 0) {
    // wide tiles halve the shared-memory traffic per MMA; keep 128 when the group size demands it or there are too few tiles
    const int npg = d.n_per_group > 0 ? d.n_per_group : d.N;
    const bool groups_ok = (npg % 256 == 0) || (npg >= d.N) || (npg % 64 == 0 && npg >= 2048);  // ragged last tile: <= 6 % waste
    bn = (d.N >= 512 && groups_ok && ceil_div(d.M, BLOCK_M) * ceil_div(d.N, 256) >= num_sms() / 2) ? 256 : 128;
  }
  if (bn == 256) dispatch_major<256>(d, stream);
  else dispatch_major<128>(d, stream);
}

void lora_dx(const LoraDxDesc& d, cudaStream_t stream) {
  if (d.M <= 0 || d.N <= 0) return;
  if (d.groups < 1 || d.groups > 3) throw std::runtime_error("lora_dx: 1..3 stacked LoRA groups");
  if (d.r <= 0 || d.r % BLOCK_K != 0) throw std::runtime_error("lora_dx: the LoRA rank must be a multiple of 64");
  if (d.Kb == 0 && (d.base == nullptr || d.ld_base % 8 != 0 || (reinterpret_cast<uintptr_t>(d.base) & 15) != 0))
    throw std::runtime_error("lora_dx: Kb == 0 needs a 16-byte aligned base product");
  if (d.ldc % 8 != 0 || (reinterpret_cast<uintptr_t>(d.out) & 15) != 0) throw std::runtime_error("lora_dx: output must be 16-byte aligned");
  if (d.N % 2 != 0) throw std::runtime_error("lora_dx: N must be even");
  using L = SmemLayout<128>;
  LoraDxArgs p;
  p.M = d.M; p.N = d.N; p.Kb = d.Kb; p.r = d.r; p.G = d.groups;
  p.out = reinterpret_cast<bf16*>(d.out); p.ldc = d.ldc;
  p.base = reinterpret_cast<const bf16*>(d.base); p.ld_base = d.ld_base;
  p.num_m_tiles = ceil_div(d.M, BLOCK_M);
  p.num_n_tiles = ceil_div(d.N, 128);
  p.thr16 = d.drop_threshold16; p.inv_keep = d.inv_keep; p.seed_ptr = d.seed_ptr;
  for (int g = 0; g < 3; ++g) p.keys[g] = d.seed_key[g];
  CUtensorMap m_du = make_map_2d(d.du, (long long)d.groups * d.r, d.M, d.ld_du, BLOCK_K, BLOCK_M);
  CUtensorMap m_a = make_map_2d(d.a, d.N, (long long)d.groups * d.r, d.ld_a, 64, BLOCK_K);
  CUtensorMap m_dy = m_du, m_w = m_a;  // unused when the frozen-path product is supplied (Kb == 0)
  if (d.Kb > 0) {
    m_dy = make_map_2d(d.dy, d.Kb, d.M, d.ld_dy, BLOCK_K, BLOCK_M);
    m_w = make_map_2d(d.w, d.N, d.Kb, d.ld_w, 64, BLOCK_K);
  }
  static bool configured = false;
  if (!configured) {
    check(cudaFuncSetAttribute(lora_dx_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal), "cudaFuncSetAttribute(lora_dx)");
    configured = true;
  }
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  launch_k(lora_dx_kernel, grid, kNumThreads, L::kTotal, stream, m_dy, m_w, m_du, m_a, p);
  RB_CHECK_LAUNCH("lora_dx_kernel");
}

}  // namespace rb
