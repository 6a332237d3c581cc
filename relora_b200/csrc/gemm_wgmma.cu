// Persistent warp-specialised bf16 / fp8 GEMM for sm_90a: TMA -> shared memory (128B swizzle) -> wgmma with fp32
// accumulators in registers -> epilogue.  bf16 outputs of the 128- and 192-wide tiles leave through a shared-memory staging
// buffer and TMA stores that drain while the next tile's k-loop runs; fp32, split-K and unaligned outputs are stored from
// registers.
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
// Long reductions into wide outputs run as clusters of two CTAs that share each B tile (CtaPair, gemm_pairs).
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
  int tma_store;  // bf16 output through shared memory and TMA stores (map_out); else stored from registers
  int paired;     // clusters of 2 CTAs own M-tiles (2i, 2i + 1) of one N tile and multicast the B tile (CtaPair)
  int block_n;    // tile width: 128 or 192 in gemm_kernel<128, ...>, 256 in gemm_kernel<256, ...>
};

template <int BLOCK_N>
struct SmemLayout {
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;  // 16 KB
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (192 * 1024) / kStageBytes;  // 6 stages of 128-wide tiles, 4 of 192- and 256-wide tiles
  static constexpr int kTileBytes = kStages * kStageBytes;
  static constexpr int kRingTotal = kTileBytes + 1024 + 1024;  // ring, barriers, manual 1024-byte alignment (lora_dx)
  // + the store staging of the bf16 epilogue, one 64 x 64 sub-tile (8 KB, 128B-swizzled) per 64 columns of each consumer
  // warpgroup's rows.  Not for 256-wide tiles: with their 128 accumulator registers the staging code spills.
  static constexpr int kSubTiles = BLOCK_N == 256 ? 0 : BLOCK_N / 64;
  static constexpr int kStoreBytes = 2 * kSubTiles * 64 * 64 * 2;
  static constexpr int kTotal = kRingTotal + kStoreBytes;
};
static_assert(SmemLayout<128>::kTotal <= 232448 && SmemLayout<192>::kTotal <= 232448 && SmemLayout<256>::kTotal <= 232448,
              "shared memory budget");

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

// CTA pairs: a cluster of 2 CTAs computes M tiles 2u and 2u + 1 of one N tile over the same k range.  Each CTA loads its own
// A tile and half of the B tile, which the TMA unit multicasts into the same stage of both CTAs, so each B tile crosses from
// L2 once per pair instead of once per CTA.  A stage's full barrier still expects the whole stage; its empty barrier also
// counts one arrival from each consumer warp of the peer, whose multicast writes into this CTA's stage.  When the last pair
// has a second tile past M, that CTA still loads its half of B, computes on zero-filled A and stores nothing.  Unpaired, each
// CTA is a work unit of its own and nothing below changes the single-CTA schedule.
struct CtaPair {
  int on;
  uint32_t rank;  // in the cluster; 0 unpaired
  __device__ __forceinline__ explicit CtaPair(int paired) : on(paired), rank(paired ? cluster_ctarank() : 0) {}
  __device__ __forceinline__ int m_units(int num_m_tiles) const { return on ? (num_m_tiles + 1) / 2 : num_m_tiles; }
  __device__ __forceinline__ int first_unit() const { return blockIdx.x >> on; }
  __device__ __forceinline__ int unit_stride() const { return gridDim.x >> on; }
  __device__ __forceinline__ int m_tile(int m_unit) const { return (m_unit << on) + rank; }
  __device__ __forceinline__ uint32_t empty_arrivals() const { return on ? 256 + 8 : 256; }
  // consumer release of a stage: every consumer thread arrives here; paired, lane 0 of each warp also arrives at the peer
  __device__ __forceinline__ void release(uint64_t* bar) const {
    mbar_arrive(bar);
    if (on && lane_id() == 0) mbar_arrive_cluster(bar, rank ^ 1);
  }
  // after barrier init: the peer may multicast into this CTA or arrive on its barriers only once they are initialised
  __device__ __forceinline__ void start() const {
    if (on) cluster_sync();
    else __syncthreads();
  }
  // before exit: no CTA leaves while its peer may still arrive on its barriers
  __device__ __forceinline__ void finish() const {
    if (on) cluster_sync();
  }
};

// Loads of the B tile, which both CTAs of a pair share: unpaired the whole tile, paired this CTA's half (64-row or 64-wide MN
// chunk; K-major maps of a pair have a box of BLOCK_MN / 2 rows), multicast to both CTAs.
template <int BLOCK_MN, bool MN_MAJOR>
__device__ __forceinline__ void load_shared_operand(const CtaPair& pair, const CUtensorMap* map, uint64_t* bar, uint8_t* dst, int mn0,
                                                    int k0, uint64_t hint) {
  if (!pair.on) {
    load_operand<BLOCK_MN, MN_MAJOR>(map, bar, dst, mn0, k0, hint);
    return;
  }
  const int ofs = pair.rank * (BLOCK_MN / 2);  // rows of 128 bytes either way
  if constexpr (!MN_MAJOR) {
    tma_load_2d_multicast(map, bar, dst + ofs * 128, k0, mn0 + ofs, 0x3, hint);
  } else {
#pragma unroll
    for (int j = 0; j < BLOCK_MN / 128; ++j) tma_load_2d_multicast(map, bar, dst + ofs * 128 + j * 8192, mn0 + ofs + j * 64, k0, 0x3, hint);
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
    else if constexpr (BLOCK_N == 192) wgmma_bf16_ss_n192<A_MN, B_MN>(acc, da + kStepA * k, db + kStepB * k);
    else if constexpr (BLOCK_N == 128) wgmma_bf16_ss_n128<A_MN, B_MN>(acc, da + kStepA * k, db + kStepB * k);
    else wgmma_bf16_ss_n64<A_MN, B_MN>(acc, da + kStepA * k, db + kStepB * k);
  }
}
template <int BLOCK_N, bool A_E5M2>
__device__ __forceinline__ void mma_fp8_kblock(float (&acc)[BLOCK_N / 2], uint32_t sa, uint32_t sb) {
  const uint64_t da = desc_kmajor(sa), db = desc_kmajor(sb);
#pragma unroll
  for (int k = 0; k < 4; ++k) {  // rows of 128 bytes: four K = 32 steps
    if constexpr (BLOCK_N == 256) {
      if constexpr (A_E5M2) wgmma_e5m2_ss_n256(acc, da + 2 * k, db + 2 * k);
      else wgmma_e4m3_ss_n256(acc, da + 2 * k, db + 2 * k);
    } else {
      if constexpr (A_E5M2) wgmma_e5m2_ss_n128(acc, da + 2 * k, db + 2 * k);
      else wgmma_e4m3_ss_n128(acc, da + 2 * k, db + 2 * k);
    }
  }
}

// Consumer side of the shared-memory ring with one k-block of wgmma in flight: after issuing k-block kb as one batch the
// warpgroup waits only for k-block kb - 1, then hands that k-block's stage back to the producer.  `held` is the stage the
// batch still in flight reads (-1: none); drain() retires it.  Accumulator registers are only touched by the wgmma
// instructions between drains, so no operand fences sit between in-flight batches.
template <int kStages, int kStageBytes>
struct MmaRing {
  const uint32_t smem0;
  uint64_t* const full_bar;
  uint64_t* const empty_bar;
  const CtaPair pair;
  int stage = 0;
  uint32_t phase = 0;
  int held = -1;

  // n k-blocks through mma(stage smem address)
  template <typename Mma>
  __device__ __forceinline__ void run(int n, Mma mma) {
    for (int i = 0; i < n; ++i) {
      mbar_wait(&full_bar[stage], phase);
      wgmma_fence();
      mma(smem0 + stage * kStageBytes);
      wgmma_commit();
      wgmma_wait<1>();
      if (held >= 0) pair.release(&empty_bar[held]);
      held = stage;
      if (++stage == kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
  }
  // wait for every issued batch, then release the last stage; the caller fences the accumulator before reading it
  __device__ __forceinline__ void drain() {
    wgmma_wait<0>();
    if (held >= 0) pair.release(&empty_bar[held]);
    held = -1;
  }
};

// The whole persistent schedule of one tile width (the body of gemm_kernel).
template <int BLOCK_N, bool A_MN, bool B_MN>
__device__ __forceinline__ void gemm_tiles(const CUtensorMap& map_a1, const CUtensorMap& map_b1, const CUtensorMap& map_a2,
                                           const CUtensorMap& map_b2, const CUtensorMap& map_out, const KernelArgs& p) {
  using L = SmemLayout<BLOCK_N>;
  constexpr int kStages = L::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kTileBytes + L::kStoreBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const uint32_t warp = warp_id();
  const int wg = threadIdx.x / 128;
  const CtaPair pair(p.paired);
  if (threadIdx.x == 0) {
    pdl_launch_dependents();
    tma_prefetch_desc(&map_a1);
    tma_prefetch_desc(&map_b1);
    if (p.K2 > 0) {
      tma_prefetch_desc(&map_a2);
      tma_prefetch_desc(&map_b2);
    }
    if (p.tma_store) tma_prefetch_desc(&map_out);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], pair.empty_arrivals());  // every consumer thread releases the slot (+ the peer's warps)
    }
    fence_barrier_init();
  }
  pair.start();
  pdl_wait();  // everything above is CTA-local: it overlaps the tail of the previous kernel in the stream (PDL)

  // work unit: (M unit, N tile, split); an M unit is one M tile, or a pair's two
  const int num_work = pair.m_units(p.num_m_tiles) * p.num_n_tiles * p.split_k;
  const int kstep1 = p.fp8 ? 2 * BLOCK_K : BLOCK_K;  // elements per k-block of segment 1 (always 128 bytes per row)
  const int kb1 = (p.K1 + kstep1 - 1) / kstep1;
  const int kb2 = (p.K2 + BLOCK_K - 1) / BLOCK_K;
  const int num_kb = kb1 + kb2;
  const int kb_per_split = (num_kb + p.split_k - 1) / p.split_k;

  if (wg == 0) {
    // ===================================================================== TMA producer (whole warp walks the loop)
    setmaxnreg_dec<40>();
    int stage = 0;
    uint32_t phase = 0;
    for (int work = pair.first_unit(); warp == 0 && work < num_work; work += pair.unit_stride()) {
      const int tile = work / p.split_k, split = work % p.split_k;
      const int mu = tile / p.num_n_tiles;
      const int m0 = pair.m_tile(mu) * BLOCK_M;
      const int tn = tile % p.num_n_tiles;
      const int g = tn / p.tiles_per_group;
      const int nl = (tn % p.tiles_per_group) * BLOCK_N;  // column offset inside the group
      const int n0 = g * p.n_per_group + nl;
      const int a1_k = g * p.a1_group_kofs;
      const int a2_k = g * p.a2_group_kofs;
      const int b1_k = g * p.b1_group_kofs;
      // the M group of the unit's first tile: a pair never straddles M groups (m_per_group is a multiple of 2 tiles)
      const int b1_n = (p.b1_local_n ? nl : n0) + (pair.m_tile(mu) - pair.rank) * BLOCK_M / p.m_per_group * p.b1_mn_ofs_per_mgroup;
      const int kb_begin = split * kb_per_split, kb_end = min(num_kb, kb_begin + kb_per_split);
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (elect_one()) {
          uint8_t* sa = smem + stage * L::kStageBytes;
          uint8_t* sb = sa + L::kABytes;
          mbar_arrive_expect_tx(&full_bar[stage], L::kStageBytes);
          if (kb < kb1) {
            load_operand<BLOCK_M, A_MN>(&map_a1, &full_bar[stage], sa, m0, a1_k + kb * kstep1, kEvictNormal);
            load_shared_operand<BLOCK_N, B_MN>(pair, &map_b1, &full_bar[stage], sb, b1_n, b1_k + kb * kstep1, kEvictLast);
          } else {
            const int k = (kb - kb1) * BLOCK_K;
            load_operand<BLOCK_M, false>(&map_a2, &full_bar[stage], sa, m0, a2_k + k, kEvictNormal);
            load_shared_operand<BLOCK_N, false>(pair, &map_b2, &full_bar[stage], sb, n0, k, kEvictLast);
          }
        }
        __syncwarp();
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    pair.finish();
    return;
  }

  // ======================================================================= consumers: 64 rows each
  setmaxnreg_inc<232>();
  const int cw = wg - 1;
  const uint32_t smem0 = smem_u32(smem);
  const float alpha_eff = p.alpha * (p.alpha_dev != nullptr ? *p.alpha_dev : 1.0f);
  const bool out_vec = (p.ldc % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.out) & 7) == 0);
  const bool res_vec = p.residual != nullptr && (p.ldr % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.residual) & 3) == 0);
  MmaRing<kStages, L::kStageBytes> ring{smem0, full_bar, empty_bar, pair};
  const uint32_t a_ofs = cw * 8192;  // this warpgroup's 64 rows of the A tile (either major)
  const bool store_lead = (threadIdx.x & 127) == 0;  // issues and waits for this warpgroup's TMA stores
  const uint32_t stage_u32 = smem0 + L::kTileBytes;  // store staging, 1024-byte aligned (128B swizzle)
  const bool plain = p.bias == nullptr && p.residual == nullptr && !p.accumulate;
  const bool res_only = p.bias == nullptr && res_vec && !p.accumulate;  // residual, read as aligned column pairs
  float acc[BLOCK_N / 2];
  for (int work = pair.first_unit(); work < num_work; work += pair.unit_stride()) {
    const int tile = work / p.split_k, split = work % p.split_k;
    const int m0 = pair.m_tile(tile / p.num_n_tiles) * BLOCK_M;
    const int tn = tile % p.num_n_tiles;
    const int nl = (tn % p.tiles_per_group) * BLOCK_N;
    const int n0 = (tn / p.tiles_per_group) * p.n_per_group + nl;
    const int n_lim = min(p.N, n0 + min(BLOCK_N, p.n_per_group - nl));  // a group's last tile may be ragged
    const int kb_begin = split * kb_per_split, kb_end = min(num_kb, kb_begin + kb_per_split);
    if (kb_begin >= kb_end) continue;  // nothing to accumulate for this work item
    const int kb_mid = max(kb_begin, min(kb1, kb_end));  // segment 1: [kb_begin, kb_mid), segment 2: [kb_mid, kb_end)
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
    fence_regs(acc);
    // The operand type is chosen once per segment, so each loop body is one straight batch of wgmma.
    if constexpr (BLOCK_N == 192) {  // bf16 operands only (the host refuses fp8 at this width)
      ring.run(kb_mid - kb_begin, [&](uint32_t s) { mma_bf16_kblock<BLOCK_N, A_MN, B_MN>(acc, s + a_ofs, s + L::kABytes); });
    } else if (p.fp8 == 2) {
      ring.run(kb_mid - kb_begin, [&](uint32_t s) { mma_fp8_kblock<BLOCK_N, true>(acc, s + a_ofs, s + L::kABytes); });
    } else if (p.fp8) {
      ring.run(kb_mid - kb_begin, [&](uint32_t s) { mma_fp8_kblock<BLOCK_N, false>(acc, s + a_ofs, s + L::kABytes); });
    } else {
      ring.run(kb_mid - kb_begin, [&](uint32_t s) { mma_bf16_kblock<BLOCK_N, A_MN, B_MN>(acc, s + a_ofs, s + L::kABytes); });
    }
    ring.run(kb_end - kb_mid, [&](uint32_t s) { mma_bf16_kblock<BLOCK_N, false, false>(acc, s + a_ofs, s + L::kABytes); });
    ring.drain();
    fence_regs(acc);
    if (m0 >= p.M) continue;  // a pair's second tile past M
    if (L::kSubTiles > 0 && p.tma_store) {
      // ---- bf16 epilogue through shared memory: every 64-column sub-tile of the warpgroup's 64 rows is written to a staging
      // buffer in the TMA box layout, then one proxy fence and one barrier, and one thread stores them; the stores drain
      // while the next tile's k-loop runs.  Same fp32 operations in the same order as the register path below, one
      // rounding.  A group's ragged last tile stores only the sub-tiles inside the group (group widths are multiples of 64);
      // the TMA unit clips rows and columns past the tensor, so without bias, residual or accumulation (`plain`) no element
      // needs a bounds check: that path is a multiply, a pack and a shared store per column pair, where the general one
      // spends tens of instructions on uniform tests and bounds (about 3 us per tile at N 5120, K 768).  A residual alone
      // over a sub-tile wholly inside M and the group adds one 4-byte load per column pair to that path.
      if (store_lead) bulk_wait_read<0>();  // the previous tile's stores, issued a whole k-loop ago, have read the staging
      named_bar_sync(1 + cw, 128);
#pragma unroll
      for (int j = 0; j < L::kSubTiles; ++j) {
        if (n0 + j * 64 >= n_lim) break;
        const uint32_t buf = stage_u32 + (cw * L::kSubTiles + j) * 8192;
        if (res_only && m0 + cw * 64 + 64 <= p.M && n0 + j * 64 + 64 <= n_lim) {
          // the thread's two rows (frag_row: r and r + 8), column pair (threadIdx.x & 3) of each 8-column chunk
          const uint32_t* res = reinterpret_cast<const uint32_t*>(p.residual + (long long)(m0 + cw * 64 + frag_row(0)) * p.ldr + n0 +
                                                                  j * 64 + (threadIdx.x & 3) * 2);
          const long long res8 = 4 * p.ldr;  // 8 rows, in 4-byte pairs
#pragma unroll
          for (int q = 0; q < 32; q += 2) {
            const int i = j * 32 + q;
            const int r = frag_row(i);
            const float2 rv = unpack_bf16x2(res[((q >> 1) & 1) * res8 + (q >> 2) * 4]);
            // __fadd_rn: a product and a sum, never contracted into one fma, as in the general path
            st_shared_u32(buf + r * 128 + (((q >> 2) ^ (r & 7)) << 4) + (threadIdx.x & 3) * 4,
                          pack_bf16x2(__fadd_rn(acc[i] * alpha_eff, rv.x), __fadd_rn(acc[i + 1] * alpha_eff, rv.y)));
          }
          continue;
        }
        if (plain) {
#pragma unroll
          for (int q = 0; q < 32; q += 2) {
            const int i = j * 32 + q;
            const int r = frag_row(i);
            st_shared_u32(buf + r * 128 + (((q >> 2) ^ (r & 7)) << 4) + (threadIdx.x & 3) * 4,
                          pack_bf16x2(acc[i] * alpha_eff, acc[i + 1] * alpha_eff));
          }
          continue;
        }
#pragma unroll
        for (int q = 0; q < 32; q += 2) {
          const int i = j * 32 + q;
          const int r = frag_row(i);
          const int row = m0 + cw * 64 + r, col = n0 + frag_col(i);
          float v0 = acc[i] * alpha_eff, v1 = acc[i + 1] * alpha_eff;
          if (row < p.M && col < n_lim) {
            const bool pair_ok = col + 1 < n_lim;
            if (p.bias != nullptr) {
              v0 += __bfloat162float(p.bias[col]);
              if (pair_ok) v1 += __bfloat162float(p.bias[col + 1]);
            }
            if (p.residual != nullptr) {
              const bf16* rp = p.residual + (long long)row * p.ldr + col;
              if (pair_ok && res_vec) {
                const float2 rv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(rp));
                v0 += rv.x;
                v1 += rv.y;
              } else {
                v0 += __bfloat162float(rp[0]);
                if (pair_ok) v1 += __bfloat162float(rp[1]);
              }
            }
            if (p.accumulate) {
              const bf16* op = reinterpret_cast<const bf16*>(p.out) + (long long)row * p.ldc + col;
              v0 += __bfloat162float(op[0]);
              if (pair_ok) v1 += __bfloat162float(op[1]);
            }
          }
          // 16-byte chunk (q / 4) of row r, XOR-swizzled by r % 8: conflict-free, and the layout the TMA unit reads
          st_shared_u32(buf + r * 128 + (((q >> 2) ^ (r & 7)) << 4) + (threadIdx.x & 3) * 4, pack_bf16x2(v0, v1));
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(1 + cw, 128);
      if (store_lead) {
#pragma unroll
        for (int j = 0; j < L::kSubTiles; ++j) {
          if (n0 + j * 64 >= n_lim) break;
          tma_store_2d(&map_out, stage_u32 + (cw * L::kSubTiles + j) * 8192, n0 + j * 64, m0 + cw * 64);
        }
        bulk_commit();
      }
      continue;
    }
    // ---- epilogue from registers: each thread owns column pairs of two rows (accumulator fragment order)
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
  if (store_lead && p.tma_store) bulk_wait_all();  // the staging buffers must outlive the stores that read them
  pair.finish();
}

// One kernel per operand-major combination and tile family: the 128-wide instantiation also runs 192-wide tiles (p.block_n),
// whose shared-memory layout fits in the 128-wide one's opt-in; the 256-wide tile has its own.
template <int BLOCK_N, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap map_a1, const __grid_constant__ CUtensorMap map_b1,
            const __grid_constant__ CUtensorMap map_a2, const __grid_constant__ CUtensorMap map_b2,
            const __grid_constant__ CUtensorMap map_out, const KernelArgs p) {
  if constexpr (BLOCK_N == 128) {
    if (p.block_n == 192) {
      gemm_tiles<192, A_MN, B_MN>(map_a1, map_b1, map_a2, map_b2, map_out, p);
      return;
    }
  }
  gemm_tiles<BLOCK_N, A_MN, B_MN>(map_a1, map_b1, map_a2, map_b2, map_out, p);
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
// computed by a separate GEMM and is added from global memory.  With one group (kOneGroup) the mask is applied to the LoRA
// product in place, so a 192-wide tile needs only its 96 accumulator registers.  Two or three groups keep the 128-wide
// tile: a 192-wide one would hold two 96-register accumulators, and ptxas spills it (288 bytes) within the kernel's 168
// registers per thread.
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
  int paired;     // CTA pairs share the MN-major A / W tile (CtaPair)
  int tma_store;  // output through shared memory and TMA stores (map_out); else stored from registers
  int block_n;    // 128, or 192 (one group only)
};

// The whole persistent schedule of one tile width (the body of lora_dx_kernel).
template <int BLOCK_N, bool kOneGroup>
__device__ __forceinline__ void lora_dx_tiles(const CUtensorMap& map_dy, const CUtensorMap& map_w, const CUtensorMap& map_du,
                                              const CUtensorMap& map_a, const CUtensorMap& map_out, const LoraDxArgs& p) {
  static_assert(BLOCK_N == 128 || kOneGroup, "two or more groups run on the 128-wide tile");
  using L = SmemLayout<BLOCK_N>;
  constexpr int kStages = L::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kTileBytes + L::kStoreBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const uint32_t warp = warp_id();
  const int wg = threadIdx.x / 128;
  const CtaPair pair(p.paired);
  if (threadIdx.x == 0) {
    pdl_launch_dependents();
    tma_prefetch_desc(&map_du);
    tma_prefetch_desc(&map_a);
    if (p.Kb > 0) {
      tma_prefetch_desc(&map_dy);
      tma_prefetch_desc(&map_w);
    }
    if (p.tma_store) tma_prefetch_desc(&map_out);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], pair.empty_arrivals());
    }
    fence_barrier_init();
  }
  pair.start();
  pdl_wait();

  const int num_work = pair.m_units(p.num_m_tiles) * p.num_n_tiles;
  const int kb_lora = p.r / BLOCK_K;  // r is a multiple of 64
  const int kb_base = (p.Kb + BLOCK_K - 1) / BLOCK_K;

  if (wg == 0) {
    // ===================================================================== TMA producer
    setmaxnreg_dec<40>();
    int stage = 0;
    uint32_t phase = 0;
    for (int work = pair.first_unit(); warp == 0 && work < num_work; work += pair.unit_stride()) {
      const int m0 = pair.m_tile(work / p.num_n_tiles) * BLOCK_M;
      const int n0 = (work % p.num_n_tiles) * BLOCK_N;
      for (int kb = 0; kb < p.G * kb_lora + kb_base; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (elect_one()) {
          uint8_t* sa = smem + stage * L::kStageBytes;
          mbar_arrive_expect_tx(&full_bar[stage], L::kStageBytes);
          if (kb < p.G * kb_lora) {  // du [M, G·r] K-major ; A [G·r, N] MN-major
            load_operand<BLOCK_M, false>(&map_du, &full_bar[stage], sa, m0, kb * BLOCK_K, kEvictNormal);
            load_shared_operand<BLOCK_N, true>(pair, &map_a, &full_bar[stage], sa + L::kABytes, n0, kb * BLOCK_K, kEvictLast);
          } else {                   // dy [M, Kb] K-major ; W [Kb, N] MN-major
            const int k = (kb - p.G * kb_lora) * BLOCK_K;
            load_operand<BLOCK_M, false>(&map_dy, &full_bar[stage], sa, m0, k, kEvictNormal);
            load_shared_operand<BLOCK_N, true>(pair, &map_w, &full_bar[stage], sa + L::kABytes, n0, k, kEvictLast);
          }
        }
        __syncwarp();
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    pair.finish();
    return;
  }

  setmaxnreg_inc<232>();
  const int cw = wg - 1;
  const uint32_t smem0 = smem_u32(smem);
  const uint32_t seed0 = p.seed_ptr ? *p.seed_ptr : 0u;
  MmaRing<kStages, L::kStageBytes> ring{smem0, full_bar, empty_bar, pair};
  const bool store_lead = (threadIdx.x & 127) == 0;  // issues and waits for this warpgroup's TMA stores
  const uint32_t stage_u32 = smem0 + L::kTileBytes;  // store staging, 1024-byte aligned (128B swizzle)
  // n k-blocks into acc with one batch in flight, drained before the caller reads acc
  auto mma_blocks = [&](float (&acc)[BLOCK_N / 2], int n) {
    fence_regs(acc);
    ring.run(n, [&](uint32_t s) { mma_bf16_kblock<BLOCK_N, false, true>(acc, s + cw * 8192, s + L::kABytes); });
    ring.drain();
    fence_regs(acc);
  };
  float acc[BLOCK_N / 2], cmb[kOneGroup ? 1 : BLOCK_N / 2];
  for (int work = pair.first_unit(); work < num_work; work += pair.unit_stride()) {
    const int m0 = pair.m_tile(work / p.num_n_tiles) * BLOCK_M + cw * 64;
    const int n0 = (work % p.num_n_tiles) * BLOCK_N;
    if constexpr (kOneGroup) {
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
      mma_blocks(acc, kb_lora);
      const uint32_t seed = mix_seed(seed0, p.keys[0]);
      // (0 + acc) * inv_keep where kept, else 0: the values of the G >= 2 form below, the sign of a zero included
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; i += 2) {
        const uint32_t row = m0 + frag_row(i), col = n0 + frag_col(i);
        const uint32_t hsh = lowbias32((row * 0x9E3779B1u) ^ seed ^ ((col >> 1) * 0x85EBCA77u));
        acc[i] = (hsh & 0xFFFFu) >= p.thr16 ? __fmul_rn(__fadd_rn(0.f, acc[i]), p.inv_keep) : 0.f;
        acc[i + 1] = (hsh >> 16) >= p.thr16 ? __fmul_rn(__fadd_rn(0.f, acc[i + 1]), p.inv_keep) : 0.f;
      }
    } else {
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) cmb[i] = 0.f;
      for (int g = 0; g < p.G; ++g) {
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
        mma_blocks(acc, kb_lora);
        const uint32_t seed = mix_seed(seed0, g == 0 ? p.keys[0] : g == 1 ? p.keys[1] : p.keys[2]);
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; i += 2) {  // one hash per column pair (common.cuh:keep_drop)
          const uint32_t row = m0 + frag_row(i), col = n0 + frag_col(i);
          const uint32_t hsh = lowbias32((row * 0x9E3779B1u) ^ seed ^ ((col >> 1) * 0x85EBCA77u));
          if ((hsh & 0xFFFFu) >= p.thr16) cmb[i] += acc[i];
          if ((hsh >> 16) >= p.thr16) cmb[i + 1] += acc[i + 1];
        }
      }
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = cmb[i] * p.inv_keep;
    }
    if (kb_base > 0) mma_blocks(acc, kb_base);  // the frozen-path product accumulates on top of the combined LoRA term
    if (m0 >= p.M) continue;  // rows past M: a ragged last tile's second warpgroup, or a pair's second tile past M
    if (p.tma_store) {
      // ---- through shared memory, as gemm_kernel's bf16 epilogue: each 64-column sub-tile of the warpgroup's 64 rows is
      // written to a staging buffer in the TMA box layout and stored by one thread, draining while the next tile's k-loop
      // runs.  The TMA unit clips rows past M and columns past N.
#pragma unroll
      for (int j = 0; j < BLOCK_N / 64; ++j) {
        if (n0 + j * 64 >= p.N) break;
        if (store_lead) {
          if (j == 0) bulk_wait_read<0>();
          else bulk_wait_read<1>();
        }
        named_bar_sync(1 + cw, 128);
        const uint32_t buf = stage_u32 + (cw * L::kSubTiles + j) * 8192;
#pragma unroll
        for (int q = 0; q < 32; q += 2) {
          const int i = j * 32 + q;
          const int r = frag_row(i);
          const int row = m0 + r, col = n0 + frag_col(i);
          float v0 = acc[i], v1 = acc[i + 1];
          if (kb_base == 0 && row < p.M && col < p.N) {
            const float2 b = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.base + (long long)row * p.ld_base + col));
            v0 += b.x;
            v1 += b.y;
          }
          st_shared_u32(buf + r * 128 + (((q >> 2) ^ (r & 7)) << 4) + (threadIdx.x & 3) * 4, pack_bf16x2(v0, v1));
        }
        fence_proxy_async_smem();
        named_bar_sync(1 + cw, 128);
        if (store_lead) {
          tma_store_2d(&map_out, buf, n0 + j * 64, m0);
          bulk_commit();
        }
      }
      continue;
    }
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; i += 2) {
      const int row = m0 + frag_row(i), col = n0 + frag_col(i);
      if (row >= p.M || col >= p.N) continue;  // N is a multiple of 2: column pairs are whole
      float v0 = acc[i], v1 = acc[i + 1];
      if (kb_base == 0) {
        const float2 b = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.base + (long long)row * p.ld_base + col));
        v0 += b.x;
        v1 += b.y;
      }
      *reinterpret_cast<uint32_t*>(p.out + (long long)row * p.ldc + col) = pack_bf16x2(v0, v1);
    }
  }
  if (store_lead && p.tma_store) bulk_wait_all();  // the staging buffers must outlive the stores that read them
  pair.finish();
}

__global__ void __launch_bounds__(kNumThreads, 1)
lora_dx_kernel(const __grid_constant__ CUtensorMap map_dy, const __grid_constant__ CUtensorMap map_w,
               const __grid_constant__ CUtensorMap map_du, const __grid_constant__ CUtensorMap map_a,
               const __grid_constant__ CUtensorMap map_out, const LoraDxArgs p) {
  if (p.block_n == 192) lora_dx_tiles<192, true>(map_dy, map_w, map_du, map_a, map_out, p);
  else lora_dx_tiles<128, false>(map_dy, map_w, map_du, map_a, map_out, p);
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


// Map of an operand over its stored extent e (gemm_operand_extents); boxes of block_mn rows/cols of the output dimension.
static CUtensorMap operand_map(const Operand& o, const GemmExtent& e, int block_mn, bool fp8 = false) {
  if (fp8) return make_map_2d(o.ptr, e.cols, e.rows, o.ld, 2 * BLOCK_K, block_mn, 1);  // E4M3 bytes, K-major only
  if (!o.mn_major) return make_map_2d(o.ptr, e.cols, e.rows, o.ld, BLOCK_K, block_mn);
  return make_map_2d(o.ptr, e.cols, e.rows, o.ld, 64, BLOCK_K);
}

static int gemm_n_per_group(const GemmDesc& d) { return d.n_per_group > 0 ? d.n_per_group : (d.N > 0 ? d.N : 1); }

GemmExtents gemm_operand_extents(const GemmDesc& d) {
  // K extents include the per-group windows, B1's MN extent the per-M-group offsets
  const int groups = ceil_div(d.N, gemm_n_per_group(d));
  const int mgroups = d.m_per_group > 0 ? ceil_div(d.M, d.m_per_group) : 1;
  const auto stored = [](const Operand& o, long long mn, long long k) { return o.mn_major ? GemmExtent{k, mn} : GemmExtent{mn, k}; };
  GemmExtents e;
  e.a1 = stored(d.a1, d.M, (long long)d.K1 + (long long)(groups - 1) * d.a1_group_kofs);
  e.b1 = stored(d.b1, (d.b1_local_n ? (long long)gemm_n_per_group(d) : (long long)d.N) + (long long)(mgroups - 1) * d.b1_mn_ofs_per_mgroup,
                (long long)d.K1 + (long long)(groups - 1) * d.b1_group_kofs);
  if (d.K2 > 0) {
    e.a2 = stored(d.a2, d.M, (long long)d.K2 + (long long)(groups - 1) * d.a2_group_kofs);
    e.b2 = stored(d.b2, d.N, d.K2);
  }
  return e;
}

// The TMA store needs a 16-byte aligned base and row pitch, and a row length of whole 16-byte chunks: past a ragged last
// chunk it writes beyond column N.  fp32 outputs (weight gradients, accumulated or split-K with atomics) and 256-wide tiles
// keep the register epilogue.
bool gemm_uses_tma_store(const GemmDesc& d, int block_n, int split_k) {
  return block_n != 256 && !d.out_f32 && split_k == 1 && (reinterpret_cast<uintptr_t>(d.out) & 15) == 0 && d.ldc % 8 == 0 &&
         d.N % 8 == 0;
}

template <int BLOCK_N, bool A_MN, bool B_MN>
static void launch(const GemmDesc& d, cudaStream_t stream) {
  using L = SmemLayout<BLOCK_N>;
  KernelArgs p;
  p.M = d.M; p.N = d.N; p.K1 = d.K1; p.K2 = d.K2;
  p.n_per_group = gemm_n_per_group(d);
  p.a1_group_kofs = d.a1_group_kofs; p.a2_group_kofs = d.a2_group_kofs;
  p.b1_group_kofs = d.b1_group_kofs; p.b1_local_n = d.b1_local_n ? 1 : 0;
  p.m_per_group = d.m_per_group > 0 ? d.m_per_group : (1 << 30); p.b1_mn_ofs_per_mgroup = d.b1_mn_ofs_per_mgroup;
  p.out = d.out; p.ldc = d.ldc; p.residual = reinterpret_cast<const bf16*>(d.residual); p.ldr = d.ldr;
  p.bias = reinterpret_cast<const bf16*>(d.bias);
  if (d.bias != nullptr && d.out_f32) throw std::runtime_error("gemm: bias is only fused for bf16 outputs");
  if (d.residual != nullptr && d.out_f32) throw std::runtime_error("gemm: residual is only fused for bf16 outputs");
  p.alpha = d.alpha; p.alpha_dev = d.alpha_dev; p.fp8 = d.fp8 ? (d.fp8_a_e5m2 ? 2 : 1) : 0; p.out_f32 = d.out_f32 ? 1 : 0; p.accumulate = d.accumulate ? 1 : 0;
  p.num_m_tiles = ceil_div(d.M, BLOCK_M);
  const int groups = ceil_div(d.N, p.n_per_group);
  // tiles never straddle a group: the last tile of a group may be ragged (its tail columns are computed but not stored)
  if (groups > 1 && (p.n_per_group % 64) != 0) throw std::runtime_error("gemm: n_per_group must be a multiple of 64");
  p.tiles_per_group = ceil_div(p.n_per_group, BLOCK_N);
  p.num_n_tiles = groups * p.tiles_per_group;
  // The last k-block of a K window narrower than a whole number of k-blocks runs into the next group's window, which lies
  // inside the tensor map, so TMA does not zero-fill it.  With only one of A1 / B1 windowed the other one's map ends at K1 and
  // the overhang multiplies zeros; with both windowed it would add the next group's terms.
  if (groups > 1 && d.a1_group_kofs != 0 && d.b1_group_kofs != 0 && d.K1 % (d.fp8 ? 2 * BLOCK_K : BLOCK_K) != 0)
    throw std::runtime_error("gemm: with per-group K windows on both A1 and B1, K1 must be a multiple of the k-block (64, fp8: 128)");

  const GemmExtents e = gemm_operand_extents(d);
  if (d.fp8 && (A_MN || B_MN)) throw std::runtime_error("gemm: fp8 operands must be K-major");
  CUtensorMap ma1 = operand_map(d.a1, e.a1, BLOCK_M, d.fp8);
  if (d.m_per_group > 0 && (d.m_per_group % BLOCK_M) != 0) throw std::runtime_error("gemm: m_per_group must be a multiple of the M tile");
  if (BLOCK_N == 192 && d.fp8) throw std::runtime_error("gemm: fp8 operands run on the 128- or 256-wide tile");
  const bool paired = gemm_pairs(d, BLOCK_N);
  p.paired = paired ? 1 : 0;
  const int b_box = paired ? BLOCK_N / 2 : BLOCK_N;  // each CTA of a pair loads half of the B tile
  CUtensorMap mb1 = operand_map(d.b1, e.b1, b_box, d.fp8);
  CUtensorMap ma2 = ma1, mb2 = mb1;
  if (d.K2 > 0) {
    if (d.a2.mn_major || d.b2.mn_major) throw std::runtime_error("gemm: the LoRA (A2/B2) operands must be K-major");
    ma2 = operand_map(d.a2, e.a2, BLOCK_M);
    mb2 = operand_map(d.b2, e.b2, b_box);
  }
  // 192-wide tiles run in the 128-wide kernel, whose opt-in covers both layouts
  constexpr int kKernelN = BLOCK_N == 192 ? 128 : BLOCK_N;
  constexpr int kOptIn = SmemLayout<kKernelN>::kTotal;
  static_assert(L::kTotal <= kOptIn, "a tile's layout must fit in its kernel's opt-in");
  auto kern = gemm_kernel<kKernelN, A_MN, B_MN>;
  p.block_n = BLOCK_N;
  static int max_pairs = 0;  // clusters of 2 resident at once
  if (max_pairs == 0) {
    check(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kOptIn), "cudaFuncSetAttribute(gemm)");
    max_pairs = max_active_clusters(kern, 2, kNumThreads, kOptIn);
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
  p.tma_store = gemm_uses_tma_store(d, BLOCK_N, split) ? 1 : 0;
  const CUtensorMap mout = p.tma_store ? make_map_2d(d.out, d.N, d.M, d.ldc, 64, 64) : ma1;
  const int cta_per_unit = paired ? 2 : 1;
  const int work = ceil_div(p.num_m_tiles, cta_per_unit) * p.num_n_tiles * split;
  const int grid = std::min(work, paired ? max_pairs : num_sms()) * cta_per_unit;
  if (grid <= 0) return;
  launch_k_cluster(cta_per_unit, kern, grid, kNumThreads, L::kTotal, stream, ma1, mb1, ma2, mb2, mout, p);
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

// Width of the output tiles by wave count: the grid is one CTA per SM and tiles go round-robin, so a width costs
// ceil(tiles / SMs) tile-times, each tile-time scaled by the width's per-tile cost; a ragged tile counts whole.  The
// 192-wide tile costs kCost192 of a 128-wide one.  It is taken only when strictly cheaper, so ties go to 128.  kCost192 = 1.5
// is the ratio of the widths, not a measured per-tile cost (bench/gemm_ksweep.py's bn192 column measures it); at 1.5 the
// llama_250m N 768 outputs and the qkv projection take 192 and N 5120 ties.  On an H100 80GB HBM3 at 700 W this rule took
// bench.py's llama_250m from 213,744 - 214,913 tokens/s to 227,530 - 227,713 (3 runs each, alternating).
int tile_width_by_waves(int m, int n, int n_per_group, int sms) {
  constexpr double kCost192 = 1.5;
  if (sms <= 0 || m <= 0 || n <= 0 || n_per_group <= 0) return 128;
  const long long m_tiles = ceil_div(m, BLOCK_M), groups = ceil_div(n, n_per_group);
  const auto waves = [&](int bn) { return ceil_div(m_tiles * groups * ceil_div(n_per_group, bn), sms); };
  return kCost192 * waves(192) < waves(128) ? 192 : 128;
}

// Tile width (block_n 0 = auto; 128, 192 or 256 on request).  Auto runs bf16 outputs of bf16 operands at 192 where the
// wave count says so (tile_width_by_waves), and at 128 otherwise: fp32, accumulated and split-K outputs, fp8 operands, and
// calls that pair at 128 (gemm_pairs), whose shared B tile is worth more than a wave.  On an H100 80GB HBM3 at 700 W
// (bench/gemm_bench.py, M 12288, plain bf16 GEMM with the register epilogue) the 256-wide tile ran at 192 - 387 TFLOP/s
// on the llama_1b shapes and 410 at 8192^3, the 128-wide one at 466 - 548 and 440; with the fused LoRA branch the
// 256-wide tile took 2.0 - 2.5x as long on every llama_250m / llama_1b projection.  The K sweep (bench/gemm_ksweep.py)
// puts the difference in the per-tile fixed cost: 528 vs 260 us at K = 128, N = 5120.  The 256-wide tile has no
// TMA-store epilogue (it would spill), so auto never picks it.
int gemm_block_n(const GemmDesc& d, int sms) {
  if (d.block_n != 0) return d.block_n == 256 || d.block_n == 192 ? d.block_n : 128;
  if (d.out_f32 || d.accumulate || d.split_k > 1 || d.fp8 || gemm_pairs(d, 128)) return 128;
  return tile_width_by_waves(d.M, d.N, gemm_n_per_group(d), sms > 0 ? sms : num_sms());
}

int gemm_smem_bytes(int block_n) {
  return block_n == 256 ? SmemLayout<256>::kTotal : block_n == 192 ? SmemLayout<192>::kTotal : SmemLayout<128>::kTotal;
}

// CTA pairs (CtaPair): the 128-wide tile only, M of at least two tiles, and M groups (weight gradients) that hold whole
// pairs, since a pair shares one B tile.  Auto (pair = -1) pairs long reductions into wide outputs: N >= 2048 and at least
// 32 k-blocks.  Measured on an H100 80GB HBM3 at 700 W (bench/gemm_bench.py, bench/gemm_ksweep.py, M 12288): pairs cut the
// per-k-block slope at N 5120 from 14.7 to 11.9 us (cuBLAS 10.1) and ran 2 - 6 % faster on every llama_1b projection
// (K 2048 - 11008) and 14 % faster at 8192^3; at K 768 (N 2304, 5120) they tied, and at N 768 they ran 7 - 14 % slower
// (o / down of llama_250m and its N 768, K 5120 input gradient), where B is small enough to stay in L2.
bool gemm_pairs(const GemmDesc& d, int block_n) {
  if (d.pair == 0 || block_n != 128 || ceil_div(d.M, BLOCK_M) < 2) return false;
  if (d.m_per_group > 0 && d.m_per_group % (2 * BLOCK_M) != 0) return false;
  const int num_kb = ceil_div(d.K1, d.fp8 ? 2 * BLOCK_K : BLOCK_K) + ceil_div(d.K2, BLOCK_K);
  return d.pair == 1 || (d.N >= 2048 && num_kb >= 32);
}

void gemm_bf16(const GemmDesc& d, cudaStream_t stream) {
  if (d.n_lora_acc != 0) throw std::runtime_error("gemm: dropout-combine epilogue not built into this kernel variant");
  if (d.M <= 0 || d.N <= 0) return;
  const int bn = gemm_block_n(d);
  if (bn == 256) dispatch_major<256>(d, stream);
  else if (bn == 192) dispatch_major<192>(d, stream);
  else dispatch_major<128>(d, stream);
}

// Pairs share the A / W tile (MN-major, 64-wide chunks); every call form of the 128-wide tile can pair.  Auto: the GEMM's rule
// (bench/lora_dx_bench.py, same card: pairs 15 % faster on llama_1b down (N 5504) and 3 % on o (N 2048), 7 - 13 % slower
// at N 768).
static bool lora_dx_pairs_at_128(const LoraDxDesc& d) {
  if (d.pair == 0 || ceil_div(d.M, BLOCK_M) < 2) return false;
  const int num_kb = d.groups * d.r / BLOCK_K + ceil_div(d.Kb, BLOCK_K);
  return d.pair == 1 || (d.N >= 2048 && num_kb >= 32);
}
// Tile width: 128 for two or three groups (lora_dx_kernel); with one group, 192 on request, and on auto the GEMM's wave
// rule over N unless the call pairs at 128.
int lora_dx_block_n(const LoraDxDesc& d) {
  if (d.groups > 1 || d.block_n == 128) return 128;
  if (d.block_n == 192) return 192;
  return lora_dx_pairs_at_128(d) ? 128 : tile_width_by_waves(d.M, d.N, d.N, num_sms());
}
bool lora_dx_pairs(const LoraDxDesc& d) { return lora_dx_block_n(d) == 128 && lora_dx_pairs_at_128(d); }
// the base, pitch and alignment rules below hold for every call; only a ragged last 16-byte chunk of a row keeps the
// register epilogue (a TMA store would write past column N)
bool lora_dx_uses_tma_store(const LoraDxDesc& d) { return d.N % 8 == 0; }


template <int BLOCK_N>
static void lora_dx_launch(const LoraDxDesc& d, cudaStream_t stream) {
  using L = SmemLayout<BLOCK_N>;
  constexpr int kOptIn = SmemLayout<128>::kTotal;  // the larger layout: one opt-in for both widths
  static_assert(L::kTotal <= kOptIn, "a tile's layout must fit in the kernel's opt-in");
  auto kern = lora_dx_kernel;
  LoraDxArgs p;
  p.block_n = BLOCK_N;
  p.M = d.M; p.N = d.N; p.Kb = d.Kb; p.r = d.r; p.G = d.groups;
  p.out = reinterpret_cast<bf16*>(d.out); p.ldc = d.ldc;
  p.base = reinterpret_cast<const bf16*>(d.base); p.ld_base = d.ld_base;
  p.num_m_tiles = ceil_div(d.M, BLOCK_M);
  p.num_n_tiles = ceil_div(d.N, BLOCK_N);
  p.thr16 = d.drop_threshold16; p.inv_keep = d.inv_keep; p.seed_ptr = d.seed_ptr;
  for (int g = 0; g < 3; ++g) p.keys[g] = d.seed_key[g];
  CUtensorMap m_du = make_map_2d(d.du, (long long)d.groups * d.r, d.M, d.ld_du, BLOCK_K, BLOCK_M);
  CUtensorMap m_a = make_map_2d(d.a, d.N, (long long)d.groups * d.r, d.ld_a, 64, BLOCK_K);
  CUtensorMap m_dy = m_du, m_w = m_a;  // unused when the frozen-path product is supplied (Kb == 0)
  if (d.Kb > 0) {
    m_dy = make_map_2d(d.dy, d.Kb, d.M, d.ld_dy, BLOCK_K, BLOCK_M);
    m_w = make_map_2d(d.w, d.N, d.Kb, d.ld_w, 64, BLOCK_K);
  }
  p.paired = lora_dx_pairs(d) ? 1 : 0;
  p.tma_store = lora_dx_uses_tma_store(d) ? 1 : 0;
  const CUtensorMap m_out = p.tma_store ? make_map_2d(d.out, d.N, d.M, d.ldc, 64, 64) : m_du;
  static int max_pairs = 0;  // clusters of 2 resident at once
  if (max_pairs == 0) {
    check(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kOptIn), "cudaFuncSetAttribute(lora_dx)");
    max_pairs = max_active_clusters(kern, 2, kNumThreads, kOptIn);
  }
  const int cta_per_unit = p.paired ? 2 : 1;
  const int work = ceil_div(p.num_m_tiles, cta_per_unit) * p.num_n_tiles;
  const int grid = std::min(work, p.paired ? max_pairs : num_sms()) * cta_per_unit;
  launch_k_cluster(cta_per_unit, kern, grid, kNumThreads, L::kTotal, stream, m_dy, m_w, m_du, m_a, m_out, p);
  RB_CHECK_LAUNCH("lora_dx_kernel");
}

void lora_dx(const LoraDxDesc& d, cudaStream_t stream) {
  if (d.M <= 0 || d.N <= 0) return;
  if (d.r <= 0 || d.r % BLOCK_K != 0) throw std::runtime_error("lora_dx: the LoRA rank must be a multiple of 64");
  if (d.Kb == 0 && d.base == nullptr) throw std::runtime_error("lora_dx: Kb == 0 needs the base product");
  if (d.N % 2 != 0) throw std::runtime_error("lora_dx: N must be even");
  if (lora_dx_block_n(d) == 192) lora_dx_launch<192>(d, stream);  // one group (lora_dx_block_n)
  else lora_dx_launch<128>(d, stream);
}

}  // namespace rb
