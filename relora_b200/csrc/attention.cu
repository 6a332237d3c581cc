// Causal flash attention for sm_90a: wgmma with the scores, probabilities and outputs in registers, TMA loads straight out
// of the packed qkv projection buffer.
//
// Replaces the reference's F.scaled_dot_product_attention call (peft_pretraining/modeling_llama.py:241-247 and
// modeling_pythia.py attention) for head_dim <= 256 (a multiple of 8).  Three kernels, one warpgroup (128 threads, 64 rows)
// per CTA:
//
//   attn_fwd_kernel      CTA = (64 queries, head, batch); per 64 keys:  S = Q·Kᵀ -> online softmax -> O += P·V
//   attn_bwd_dq_kernel   CTA = (64 queries, head, batch); per 64 keys:  S, dP = dO·Vᵀ -> dS -> dQ += dS·K
//   attn_bwd_dkv_kernel  CTA = (64 keys, KV head, batch); per 64 queries of each query head of the group:  Sᵀ = K·Qᵀ, dPᵀ = V·dOᵀ -> Pᵀ, dSᵀ -> dV += Pᵀ·dO, dK += dSᵀ·Q
//
// Each kernel is instantiated for NP = ceil(head_dim / 64) in {1, 2, 3, 4}.  An operand tile is NP shared-memory panels of
// [64 rows x 64 columns] bf16 (128 bytes per row, 128-byte swizzle), loaded by NP TMA boxes at column offsets 64·p; columns
// past head_dim are zero filled.  The same panel serves as a K-major operand (reduction over head_dim) and as an MN-major
// operand (reduction over its rows) by descriptor alone.  Products that reduce over head_dim issue only the ceil(hd / 16)
// K = 16 steps that hold data when the head spans several panels; products that produce head_dim columns run one
// register-A wgmma chain per panel, and the padded columns of the last panel are computed but never stored.  The
// probabilities / score gradients never leave registers: the accumulator fragment of one wgmma is, packed to bf16, the register A operand of the next.  The streamed
// operand pair is double buffered.  Each product (or the pair of independent products S, dP) is issued as one wgmma batch,
// and the warpgroup waits for it only where softmax or the next product reads the result.
//
// Register budget.  The output accumulators take 32 fp32 registers per panel per thread, on top of the two 32-register
// score fragments of the backward kernels.  Where the whole head does not fit one warpgroup without spilling (dQ at NP = 4,
// dK/dV at NP >= 3), the backward kernels split the output columns across CTAs: each CTA owns at most two panels
// (128 columns) of dQ, or of both dK and dV, and recomputes S / dP (Sᵀ / dPᵀ) over the full head for them.  Splitting by
// columns rather than computing dK and dV in separate CTAs keeps one kernel body for every head size.
#include <cuda.h>

#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>

#include "attention.h"
#include "common.cuh"
#include "sm90.cuh"
#include "tensormap.h"

namespace rb {

using namespace sm90;

namespace {

constexpr int BQ = 64;                // rows per CTA (queries in fwd / dq, keys in dkv)
constexpr int kPanel = 64 * 128;      // bytes of a [64 x 64] bf16 panel
constexpr int kThreads = 128;
constexpr int kMaxHeadDim = 256;
constexpr float kNegInf = -1e30f;

// dynamic shared memory: NRES resident tiles, two double-buffered streamed tiles, barriers + row statistics, alignment
constexpr int smem_bytes(int nres, int np) { return (nres + 4) * np * kPanel + 1024 + 1024; }
// output panels per CTA of the backward kernels (see "Register budget" above)
constexpr int dq_out_panels(int np) { return np <= 3 ? np : 2; }
constexpr int dkv_out_panels(int np) { return np <= 2 ? np : 2; }
constexpr int splits(int np, int no) { return (np + no - 1) / no; }

__device__ __forceinline__ float fast_exp2(float x) {  // one MUFU.EX2 (inputs are <= ~8; -1e30 -> 0)
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// acc(64 rows, cols 16kk..16kk+15) as the register A operand of a K = 16 wgmma
__device__ __forceinline__ void frag_to_a(const float (&d)[32], int kk, uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(d[8 * kk + 0], d[8 * kk + 1]);
  a[1] = pack_bf16x2(d[8 * kk + 2], d[8 * kk + 3]);
  a[2] = pack_bf16x2(d[8 * kk + 4], d[8 * kk + 5]);
  a[3] = pack_bf16x2(d[8 * kk + 6], d[8 * kk + 7]);
}
template <int NSTEPS>
__device__ __forceinline__ void mma_steps_kk(float (&d)[32], uint32_t a, uint32_t b) {
#pragma unroll
  for (int ks = 0; ks < NSTEPS; ++ks) {
    const uint32_t ofs = (ks >> 2) * kPanel + (ks & 3) * 32;
    wgmma_bf16_ss_n64<0, 0>(d, desc_kmajor(a + ofs), desc_kmajor(b + ofs));
  }
}
// d += A · Bᵀ with A, B both [64 x 64·NP] K-major tiles (reduction over head_dim); only the first nks K = 16 steps hold data.
// A single-panel head issues all four steps unconditionally (zero-filled columns add nothing).  Wider heads pick the step
// count with one uniform branch into straight-line runs: a wgmma under a condition of its own makes ptxas serialise every
// wgmma of the batch.
template <int NP>
__device__ __forceinline__ void mma_tiles_kk(float (&d)[32], uint32_t a, uint32_t b, int nks) {
  if constexpr (NP == 1) {
    mma_steps_kk<4>(d, a, b);
  } else {
    switch (nks - 4 * (NP - 1)) {
      case 1: mma_steps_kk<4 * NP - 3>(d, a, b); break;
      case 2: mma_steps_kk<4 * NP - 2>(d, a, b); break;
      case 3: mma_steps_kk<4 * NP - 1>(d, a, b); break;
      default: mma_steps_kk<4 * NP>(d, a, b); break;
    }
  }
}
// P (rows x 64, an accumulator fragment) as the register A operands of the four K = 16 steps of mma_regs_tile.  Call it
// before wgmma_fence(): packing between the wgmma of one batch would make ptxas serialise them.
__device__ __forceinline__ void pack_a(const float (&p)[32], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    frag_to_a(p, kk, a[kk]);
    fence_regs(a[kk]);
  }
}
// d[j] += P · T_j for the first nout of NO consecutive panels T_j starting at t, read MN-major (reduction over their rows);
// P packed by pack_a.  N counts the panels of the straight-line run; a smaller nout is peeled off by uniform branches
// (as in mma_tiles_kk).
template <int NO, int N = NO>
__device__ __forceinline__ void mma_regs_tile(float (&d)[NO][32], const uint32_t (&a)[4][4], uint32_t t, int nout) {
  if constexpr (N > 1) {
    if (nout < N) return mma_regs_tile<NO, N - 1>(d, a, t, nout);
  }
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
    for (int j = 0; j < N; ++j) wgmma_bf16_rs_n64<1>(d[j], a[kk], desc_mnmajor(t + j * kPanel + kk * 2048));
  }
}
__device__ __forceinline__ void zero32(float (&d)[32]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) d[i] = 0.f;
}

struct Smem {
  uint8_t* res[2];     // resident tiles
  uint8_t* str[2][2];  // streamed tiles [buffer][operand]
  uint64_t* res_bar;
  uint64_t* str_bar;   // [2]
  float* col_lse;      // [64]: per-column row statistics of the streamed block (dK/dV kernel)
  float* col_delta;    // [64]
};
template <int NRES, int NP>
__device__ __forceinline__ Smem smem_layout() {
  constexpr int kTile = NP * kPanel;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* s = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  Smem m;
  m.res[0] = s;
  m.res[1] = s + (NRES - 1) * kTile;
  for (int b = 0; b < 2; ++b)
    for (int o = 0; o < 2; ++o) m.str[b][o] = s + (NRES + 2 * b + o) * kTile;
  m.res_bar = reinterpret_cast<uint64_t*>(s + (NRES + 4) * kTile);
  m.str_bar = m.res_bar + 1;
  m.col_lse = reinterpret_cast<float*>(s + (NRES + 4) * kTile + 64);
  m.col_delta = m.col_lse + 64;
  return m;
}
// Barriers (thread 0), then the resident tiles and the first two streamed pairs (one elected lane of warp 0 issues every TMA load:
// the whole warp takes the branch, so ptxas needs no uniformisation loop around the loads).
struct TileSrc {
  const CUtensorMap* map;
  int head;
};
template <int NP>
__device__ __forceinline__ void load_tile(TileSrc s, uint64_t* bar, uint8_t* dst, int row) {
#pragma unroll
  for (int pn = 0; pn < NP; ++pn) tma_load_3d(s.map, bar, dst + pn * kPanel, 64 * pn, s.head, row);
}
template <int NP>
__device__ __forceinline__ void issue_pair(const Smem& m, int buf, TileSrc s0, TileSrc s1, int row) {
  mbar_arrive_expect_tx(&m.str_bar[buf], 2 * NP * kPanel);
  load_tile<NP>(s0, &m.str_bar[buf], m.str[buf][0], row);
  load_tile<NP>(s1, &m.str_bar[buf], m.str[buf][1], row);
}
template <int NRES, int NP>
__device__ __forceinline__ void prologue(const Smem& m, TileSrc r0, TileSrc r1, int res_row, TileSrc s0, TileSrc s1, int row0, int nblk) {
  if (threadIdx.x == 0) {
    mbar_init(m.res_bar, 1);
    mbar_init(&m.str_bar[0], 1);
    mbar_init(&m.str_bar[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  if (warp_id() == 0) {
    if (elect_one()) {
      mbar_arrive_expect_tx(m.res_bar, NRES * NP * kPanel);
      load_tile<NP>(r0, m.res_bar, m.res[0], res_row);
      if (NRES == 2) load_tile<NP>(r1, m.res_bar, m.res[1], res_row);
      for (int j = 0; j < 2 && j < nblk; ++j) issue_pair<NP>(m, j, s0, s1, row0 + j * BQ);
    }
    __syncwarp();
  }
  mbar_wait(m.res_bar, 0);
}

// Head map of the packed qkv buffer, in head-columns of hd: query head h sits at h·hs; it reads KV head kv = h / group, whose
// k and v sit at kv·hs + wk and kv·hs + wv.  Default layout [q: nh | k: nkv | v: nkv] x hd: hs = 1, wk = nh, wv = nh + nkv,
// group = nh / nkv (grouped-query attention; 1 for multi-head).  Interleaved (GPT-NeoX query_key_value) [nh, (q|k|v), hd]:
// hs = 3, wk = 1, wv = 2, group = 1.
struct HeadMap {
  int hs, wk, wv, group;
  __device__ __forceinline__ int q(int h) const { return h * hs; }
  __device__ __forceinline__ int k(int kv) const { return kv * hs + wk; }
  __device__ __forceinline__ int v(int kv) const { return kv * hs + wv; }
};
struct FwdArgs {
  bf16* out;
  long long ld_out;
  float* lse;
  int B, T, nh, hd;
  float scale_log2;
  HeadMap hm;
};

// =============================================================================================== forward
template <int NP>
__global__ void __launch_bounds__(kThreads) attn_fwd_kernel(const __grid_constant__ CUtensorMap map_qkv, const FwdArgs p) {
  if (threadIdx.x == 0) pdl_launch_dependents();
  const int nqb = (p.T + BQ - 1) / BQ;
  const int qb = nqb - 1 - blockIdx.x;  // longest rows first
  const int h = blockIdx.y, b = blockIdx.z;
  const int q0 = qb * BQ, rowbase = b * p.T;
  const int nkb = qb + 1;
  const int nks = (p.hd + 15) / 16;
  const Smem m = smem_layout<1, NP>();
  // resident: Q; streamed: K, V
  const int kv = h / p.hm.group;
  const int hq = p.hm.q(h), hk = p.hm.k(kv), hv = p.hm.v(kv);
  prologue<1, NP>(m, {&map_qkv, hq}, {&map_qkv, hq}, rowbase + q0, {&map_qkv, hk}, {&map_qkv, hv}, rowbase, nkb);
  const uint32_t sq = smem_u32(m.res[0]);
  float o[NP][32], mrow[2] = {kNegInf, kNegInf}, lrow[2] = {0.f, 0.f};
#pragma unroll
  for (int pn = 0; pn < NP; ++pn) zero32(o[pn]);
  const int r_lo = q0 + frag_row(0);  // this thread's two query rows: r_lo and r_lo + 8
  for (int j = 0; j < nkb; ++j) {
    const int buf = j & 1;
    mbar_wait(&m.str_bar[buf], (j >> 1) & 1);
    float s[32];
    zero32(s);
    wgmma_fence();
    mma_tiles_kk<NP>(s, sq, smem_u32(m.str[buf][0]), nks);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    float mx[2] = {mrow[0], mrow[1]};
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int hr = (i >> 1) & 1;
      float v = s[i] * p.scale_log2;
      if (j == qb && j * BQ + frag_col(i) > r_lo + 8 * hr) v = kNegInf;  // causal mask on the diagonal block
      s[i] = v;
      mx[hr] = fmaxf(mx[hr], v);
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 1));
      mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 2));
    }
    const float corr[2] = {fast_exp2(mrow[0] - mx[0]), fast_exp2(mrow[1] - mx[1])};
    float ls[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int hr = (i >> 1) & 1;
      s[i] = fast_exp2(s[i] - mx[hr]);
      ls[hr] += s[i];
#pragma unroll
      for (int pn = 0; pn < NP; ++pn) o[pn][i] *= corr[hr];
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      lrow[hr] = lrow[hr] * corr[hr] + ls[hr];
      mrow[hr] = mx[hr];
    }
    uint32_t pa[4][4];
    pack_a(s, pa);
#pragma unroll
    for (int pn = 0; pn < NP; ++pn) fence_regs(o[pn]);  // the rescaled accumulator is written before the batch
    wgmma_fence();
    mma_regs_tile<NP>(o, pa, smem_u32(m.str[buf][1]), NP);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int pn = 0; pn < NP; ++pn) fence_regs(o[pn]);
    __syncthreads();  // every warp is done with this buffer
    if (warp_id() == 0 && j + 2 < nkb) {
      if (elect_one()) issue_pair<NP>(m, buf, {&map_qkv, hk}, {&map_qkv, hv}, rowbase + (j + 2) * BQ);
      __syncwarp();
    }
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    lrow[hr] += __shfl_xor_sync(0xffffffffu, lrow[hr], 1);
    lrow[hr] += __shfl_xor_sync(0xffffffffu, lrow[hr], 2);
  }
#pragma unroll
  for (int pn = 0; pn < NP; ++pn) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int hr = (i >> 1) & 1;
      const int q = r_lo + 8 * hr, c = 64 * pn + frag_col(i);
      if (q >= p.T || c >= p.hd) continue;
      const float inv = 1.f / lrow[hr];
      *reinterpret_cast<uint32_t*>(p.out + (long long)(rowbase + q) * p.ld_out + h * p.hd + c) =
          pack_bf16x2(o[pn][i] * inv, o[pn][i + 1] * inv);
    }
  }
  if ((threadIdx.x & 3) == 0) {
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int q = r_lo + 8 * hr;
      if (q < p.T) p.lse[((long long)b * p.nh + h) * p.T + q] = mrow[hr] + __log2f(lrow[hr]);
    }
  }
}

// =============================================================================================== backward: delta
// delta[b, h, t] = sum_d dO[b, t, h, d] * O[b, t, h, d]
__global__ void __launch_bounds__(256) attn_delta_kernel(const bf16* __restrict__ o, long long ld_o, const bf16* __restrict__ dout,
                                                         long long ld_do, float* __restrict__ delta, int B, int T, int nh, int hd) {
  pdl_wait();
  pdl_launch_dependents();
  const long long total = (long long)B * T * nh;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int h = int(i % nh);
    const long long row = i / nh;
    const bf16* a = o + row * ld_o + h * hd;
    const bf16* g = dout + row * ld_do + h * hd;
    float acc = 0.f;
    for (int q = 0; q < hd; q += 8) {
      float x[8], y[8];
      unpack8(*reinterpret_cast<const uint4*>(a + q), x);
      unpack8(*reinterpret_cast<const uint4*>(g + q), y);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc += x[j] * y[j];
    }
    const long long bb = row / T, t = row % T;
    delta[(bb * nh + h) * T + t] = acc;
  }
}

struct BwdArgs {
  const float* lse;
  const float* delta;
  bf16* dqkv;
  long long ld_dqkv;
  int B, T, nh, hd;
  float scale, scale_log2;
  HeadMap hm;  // of qkv / dqkv (see FwdArgs)
};

__device__ __forceinline__ void store_rows(bf16* base, long long ld, int row0, int rows_valid, int col_ofs, int hd, const float (&d)[32], float sc) {
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int r = frag_row(i), c = frag_col(i);
    if (row0 + r >= rows_valid || c >= hd) continue;
    *reinterpret_cast<uint32_t*>(base + (long long)row0 * ld + (long long)r * ld + col_ofs + c) = pack_bf16x2(d[i] * sc, d[i + 1] * sc);
  }
}
// output panels j < nout of a CTA that owns head columns 64·pn0 ..: panel j lands at column 64·(pn0 + j) of the head at col_ofs
template <int NO>
__device__ __forceinline__ void store_panels(bf16* base, long long ld, int row0, int rows_valid, int col_ofs, int hd, int pn0, int nout,
                                             const float (&d)[NO][32], float sc) {
#pragma unroll
  for (int j = 0; j < NO; ++j)
    if (j < nout) store_rows(base, ld, row0, rows_valid, col_ofs + 64 * (pn0 + j), hd - 64 * (pn0 + j), d[j], sc);
}

// =============================================================================================== backward: dQ
template <int NP>
__global__ void __launch_bounds__(kThreads) attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap map_qkv,
                                                               const __grid_constant__ CUtensorMap map_do, const BwdArgs p) {
  constexpr int NO = dq_out_panels(NP), NSPLIT = splits(NP, dq_out_panels(NP));
  if (threadIdx.x == 0) pdl_launch_dependents();
  const int nqb = (p.T + BQ - 1) / BQ;
  const int qb = nqb - 1 - blockIdx.x / NSPLIT;
  const int pn0 = (blockIdx.x % NSPLIT) * NO;  // first output panel of this CTA
  const int nout = NP % NO == 0 ? NO : min(NO, NP - pn0);
  const int h = blockIdx.y, b = blockIdx.z;
  const int q0 = qb * BQ, rowbase = b * p.T;
  const int nkb = qb + 1;
  const int nks = (p.hd + 15) / 16;
  const Smem m = smem_layout<2, NP>();
  const int kv = h / p.hm.group;
  const int hq = p.hm.q(h), hk = p.hm.k(kv), hv = p.hm.v(kv);
  prologue<2, NP>(m, {&map_qkv, hq}, {&map_do, h}, rowbase + q0, {&map_qkv, hk}, {&map_qkv, hv}, rowbase, nkb);
  const long long bh = (long long)b * p.nh + h;
  const int r_lo = q0 + frag_row(0);
  float lse[2], dlt[2];
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int q = min(r_lo + 8 * hr, p.T - 1);
    lse[hr] = p.lse[bh * p.T + q];
    dlt[hr] = p.delta[bh * p.T + q];
  }
  float dq[NO][32];
#pragma unroll
  for (int j = 0; j < NO; ++j) zero32(dq[j]);
  for (int j = 0; j < nkb; ++j) {
    const int buf = j & 1;
    mbar_wait(&m.str_bar[buf], (j >> 1) & 1);
    float s[32], dp[32];
    zero32(s);
    zero32(dp);
    wgmma_fence();
    mma_tiles_kk<NP>(s, smem_u32(m.res[0]), smem_u32(m.str[buf][0]), nks);   // S = Q·Kᵀ
    mma_tiles_kk<NP>(dp, smem_u32(m.res[1]), smem_u32(m.str[buf][1]), nks);  // dP = dO·Vᵀ
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    fence_regs(dp);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int hr = (i >> 1) & 1;
      const bool ok = !(j == qb && j * BQ + frag_col(i) > r_lo + 8 * hr);
      const float pr = ok ? fast_exp2(s[i] * p.scale_log2 - lse[hr]) : 0.f;
      s[i] = pr * (dp[i] - dlt[hr]);  // dS (w.r.t. the scaled scores)
    }
    uint32_t pa[4][4];
    pack_a(s, pa);
    wgmma_fence();
    mma_regs_tile<NO>(dq, pa, smem_u32(m.str[buf][0]) + pn0 * kPanel, nout);  // dQ += dS·K
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int jo = 0; jo < NO; ++jo) fence_regs(dq[jo]);
    __syncthreads();
    if (warp_id() == 0 && j + 2 < nkb) {
      if (elect_one()) issue_pair<NP>(m, buf, {&map_qkv, hk}, {&map_qkv, hv}, rowbase + (j + 2) * BQ);
      __syncwarp();
    }
  }
  store_panels<NO>(p.dqkv + (long long)rowbase * p.ld_dqkv, p.ld_dqkv, q0, p.T, hq * p.hd, p.hd, pn0, nout, dq, p.scale);
}

// =============================================================================================== backward: dK, dV
// CTA = (64 keys, KV head, batch).  Under grouped-query attention (GQA) the CTA streams the (Q, dO) blocks of each query head of its
// group in turn and accumulates dK / dV over the whole group in registers: one writer per output element and a fixed summation
// order, so no atomics and bit-reproducible results.  Stream item jj is query block kb + jb of query head h0 + g, with
// jj = g·nblk + jb; the query head and first row are stepped as counters rather than divided out (the kernel runs at the edge of the
// register file).
template <int NP>
__global__ void __launch_bounds__(kThreads) attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap map_qkv,
                                                                const __grid_constant__ CUtensorMap map_do, const BwdArgs p) {
  constexpr int NO = dkv_out_panels(NP), NSPLIT = splits(NP, dkv_out_panels(NP));
  if (threadIdx.x == 0) pdl_launch_dependents();
  const int nkb = (p.T + BQ - 1) / BQ;
  const int kb = blockIdx.x / NSPLIT;  // key block; query blocks kb .. nkb-1
  const int pn0 = (blockIdx.x % NSPLIT) * NO;
  const int nout = NP % NO == 0 ? NO : min(NO, NP - pn0);
  const int kv = blockIdx.y, b = blockIdx.z;
  const int k0 = kb * BQ, rowbase = b * p.T;
  const int nblk = nkb - kb;
  const int nks = (p.hd + 15) / 16;
  const Smem m = smem_layout<2, NP>();
  const int h0 = kv * p.hm.group;  // first query head of the group
  prologue<2, NP>(m, {&map_qkv, p.hm.k(kv)}, {&map_qkv, p.hm.v(kv)}, rowbase + k0, {&map_qkv, p.hm.q(h0)}, {&map_do, h0}, rowbase + k0, nblk);
  if (nblk == 1 && p.hm.group > 1 && warp_id() == 0) {  // the prologue streamed only the first head's single block
    if (elect_one()) issue_pair<NP>(m, 1, {&map_qkv, p.hm.q(h0 + 1)}, {&map_do, h0 + 1}, rowbase + k0);
    __syncwarp();
  }
  const int key_lo = k0 + frag_row(0);
  float dk[NO][32], dv[NO][32];
#pragma unroll
  for (int j = 0; j < NO; ++j) {
    zero32(dk[j]);
    zero32(dv[j]);
  }
  int hg = h0, qs = k0;  // query head and first query row of stream item jj
  // the bound is re-derived from blockIdx and the kernel parameters, so it occupies no register across the loop
  for (int jj = 0; hg < ((int)blockIdx.y + 1) * p.hm.group; ++jj) {
    const int buf = jj & 1;
    const long long bh = (long long)b * p.nh + hg;
    if (threadIdx.x < BQ) {  // row statistics of this block's 64 queries, read by every thread below
      const int qc = min(qs + (int)threadIdx.x, p.T - 1);
      m.col_lse[threadIdx.x] = p.lse[bh * p.T + qc];
      m.col_delta[threadIdx.x] = p.delta[bh * p.T + qc];
    }
    __syncthreads();
    mbar_wait(&m.str_bar[buf], (jj >> 1) & 1);
    float st[32], dpt[32];
    zero32(st);
    zero32(dpt);
    wgmma_fence();
    mma_tiles_kk<NP>(st, smem_u32(m.res[0]), smem_u32(m.str[buf][0]), nks);   // Sᵀ = K·Qᵀ
    mma_tiles_kk<NP>(dpt, smem_u32(m.res[1]), smem_u32(m.str[buf][1]), nks);  // dPᵀ = V·dOᵀ
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(st);
    fence_regs(dpt);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int q = qs + frag_col(i), key = key_lo + 8 * ((i >> 1) & 1);
      const bool ok = q < p.T && key <= q;
      const float pr = ok ? fast_exp2(st[i] * p.scale_log2 - m.col_lse[frag_col(i)]) : 0.f;
      dpt[i] = pr * (dpt[i] - m.col_delta[frag_col(i)]);  // dSᵀ
      st[i] = pr;                                       // Pᵀ
    }
    uint32_t pa[4][4], dsa[4][4];
    pack_a(st, pa);
    pack_a(dpt, dsa);
    wgmma_fence();
    mma_regs_tile<NO>(dv, pa, smem_u32(m.str[buf][1]) + pn0 * kPanel, nout);   // dV += Pᵀ·dO
    mma_regs_tile<NO>(dk, dsa, smem_u32(m.str[buf][0]) + pn0 * kPanel, nout);  // dK += dSᵀ·Q
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < NO; ++j) {
      fence_regs(dv[j]);
      fence_regs(dk[j]);
    }
    __syncthreads();
    if (warp_id() == 0) {
      int h2 = hg, q2 = qs + 2 * BQ;  // item jj + 2
      while (q2 >= p.T) {
        q2 -= nkb * BQ - k0;
        ++h2;
      }
      if (h2 < ((int)blockIdx.y + 1) * p.hm.group) {
        if (elect_one()) issue_pair<NP>(m, buf, {&map_qkv, p.hm.q(h2)}, {&map_do, h2}, rowbase + q2);
        __syncwarp();
      }
    }
    qs += BQ;
    if (qs >= p.T) {
      qs = k0;
      ++hg;
    }
  }
  bf16* base = p.dqkv + (long long)rowbase * p.ld_dqkv;
  store_panels<NO>(base, p.ld_dqkv, k0, p.T, p.hm.k(blockIdx.y) * p.hd, p.hd, pn0, nout, dk, p.scale);
  store_panels<NO>(base, p.ld_dqkv, k0, p.T, p.hm.v(blockIdx.y) * p.hd, p.hd, pn0, nout, dv, 1.0f);
}

// ---------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------
struct HeadMapKey {
  const void* ptr;
  long long ld, rows;
  int hd, heads;
  bool operator==(const HeadMapKey& o) const { return ptr == o.ptr && ld == o.ld && rows == o.rows && hd == o.hd && heads == o.heads; }
};
struct HeadMapHash {
  size_t operator()(const HeadMapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.ptr);
    h ^= std::hash<long long>()(k.ld * 1315423911ll + k.rows) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
    h ^= std::hash<long long>()(((long long)k.hd << 32) | (unsigned)k.heads) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
    return h;
  }
};
std::unordered_map<HeadMapKey, CUtensorMap, HeadMapHash> g_head_maps;
std::mutex g_head_maps_mu;

// [rows, heads*hd] bf16 (row stride ld) viewed as [hd, heads, rows]; box = 64 x 1 x 64 rows
CUtensorMap head_map(const void* ptr, long long ld, long long rows, int hd, int heads) {
  HeadMapKey key{ptr, ld, rows, hd, heads};
  {
    std::lock_guard<std::mutex> lk(g_head_maps_mu);
    auto it = g_head_maps.find(key);
    if (it != g_head_maps.end()) return it->second;
  }
  CUtensorMap m = make_map_3d_bf16(ptr, hd, heads, rows, hd, ld, 64, 1, 64);
  std::lock_guard<std::mutex> lk(g_head_maps_mu);
  if (g_head_maps.size() > 4096) g_head_maps.clear();
  g_head_maps.emplace(key, m);
  return m;
}

void check_shape(int B, int T, int nh, int nkv, int hd, bool interleaved) {
  if (B <= 0 || T <= 0 || nh <= 0) throw std::runtime_error("attention: empty problem");
  if (hd <= 0 || hd % 8 != 0 || hd > kMaxHeadDim)
    throw std::runtime_error("attention: head_dim must be a multiple of 8 and <= 256, got " + std::to_string(hd));
  if (nkv <= 0 || nh % nkv != 0)
    throw std::runtime_error("attention: nh (" + std::to_string(nh) + ") must be a multiple of nkv (" + std::to_string(nkv) + ")");
  if (interleaved && nkv != nh) throw std::runtime_error("attention: the interleaved qkv layout has no grouped-query form (nkv must equal nh)");
}

HeadMap head_map_of(int nh, int nkv, bool interleaved) {
  return interleaved ? HeadMap{3, 1, 2, 1} : HeadMap{1, nh, nh + nkv, nh / nkv};
}

template <int NP>
void fwd_np(const AttnDesc& d, const CUtensorMap& map, cudaStream_t stream) {
  constexpr int smem = smem_bytes(1, NP);
  static const bool configured =
      (check(cudaFuncSetAttribute(attn_fwd_kernel<NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem), "cudaFuncSetAttribute(attn_fwd)"), true);
  (void)configured;
  FwdArgs p;
  p.out = reinterpret_cast<bf16*>(d.out); p.ld_out = d.ld_out; p.lse = d.lse;
  p.B = d.B; p.T = d.T; p.nh = d.nh; p.hd = d.hd;
  p.scale_log2 = d.scale * 1.4426950408889634f;
  p.hm = head_map_of(d.nh, d.nkv, d.interleaved);
  const dim3 grid((unsigned)((d.T + BQ - 1) / BQ), (unsigned)d.nh, (unsigned)d.B);
  launch_k(attn_fwd_kernel<NP>, grid, kThreads, smem, stream, map, p);
  RB_CHECK_LAUNCH("attn_fwd_kernel");
}

template <int NP>
void bwd_np(const AttnBwdDesc& d, const CUtensorMap& map_qkv, const CUtensorMap& map_do, cudaStream_t stream) {
  constexpr int smem = smem_bytes(2, NP);
  static const bool configured =
      (check(cudaFuncSetAttribute(attn_bwd_dq_kernel<NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem), "cudaFuncSetAttribute(attn_dq)"),
       check(cudaFuncSetAttribute(attn_bwd_dkv_kernel<NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem), "cudaFuncSetAttribute(attn_dkv)"),
       true);
  (void)configured;
  BwdArgs p;
  p.lse = d.lse; p.delta = d.delta; p.dqkv = reinterpret_cast<bf16*>(d.dqkv); p.ld_dqkv = d.ld_dqkv;
  p.B = d.B; p.T = d.T; p.nh = d.nh; p.hd = d.hd;
  p.scale = d.scale; p.scale_log2 = d.scale * 1.4426950408889634f;
  p.hm = head_map_of(d.nh, d.nkv, d.interleaved);
  const unsigned nblk = (unsigned)((d.T + BQ - 1) / BQ);
  const dim3 grid_dkv(nblk * splits(NP, dkv_out_panels(NP)), (unsigned)d.nkv, (unsigned)d.B);
  launch_k(attn_bwd_dkv_kernel<NP>, grid_dkv, kThreads, smem, stream, map_qkv, map_do, p);
  RB_CHECK_LAUNCH("attn_bwd_dkv_kernel");
  const dim3 grid_dq(nblk * splits(NP, dq_out_panels(NP)), (unsigned)d.nh, (unsigned)d.B);
  launch_k(attn_bwd_dq_kernel<NP>, grid_dq, kThreads, smem, stream, map_qkv, map_do, p);
  RB_CHECK_LAUNCH("attn_bwd_dq_kernel");
}

int panels(int hd) { return (hd + 63) / 64; }

}  // namespace

void attention_fwd(const AttnDesc& d, cudaStream_t stream) {
  check_shape(d.B, d.T, d.nh, d.nkv, d.hd, d.interleaved);
  const long long rows = (long long)d.B * d.T;
  CUtensorMap map = head_map(d.qkv, d.ld_qkv, rows, d.hd, d.nh + 2 * d.nkv);
  switch (panels(d.hd)) {
    case 1: fwd_np<1>(d, map, stream); break;
    case 2: fwd_np<2>(d, map, stream); break;
    case 3: fwd_np<3>(d, map, stream); break;
    default: fwd_np<4>(d, map, stream); break;
  }
}

void attention_bwd(const AttnBwdDesc& d, cudaStream_t stream) {
  check_shape(d.B, d.T, d.nh, d.nkv, d.hd, d.interleaved);
  const long long rows = (long long)d.B * d.T;
  CUtensorMap map_qkv = head_map(d.qkv, d.ld_qkv, rows, d.hd, d.nh + 2 * d.nkv);
  CUtensorMap map_do = head_map(d.dout, d.ld_dout, rows, d.hd, d.nh);
  {
    const long long total = rows * d.nh;
    const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 8);
    launch_k(attn_delta_kernel, grid, 256, 0, stream, reinterpret_cast<const bf16*>(d.out), d.ld_out, reinterpret_cast<const bf16*>(d.dout),
             d.ld_dout, d.delta, d.B, d.T, d.nh, d.hd);
    RB_CHECK_LAUNCH("attn_delta_kernel");
  }
  switch (panels(d.hd)) {
    case 1: bwd_np<1>(d, map_qkv, map_do, stream); break;
    case 2: bwd_np<2>(d, map_qkv, map_do, stream); break;
    case 3: bwd_np<3>(d, map_qkv, map_do, stream); break;
    default: bwd_np<4>(d, map_qkv, map_do, stream); break;
  }
}

int attention_smem_bytes(int hd) { return smem_bytes(2, panels(hd)); }

long long attention_ds_pitch(int T) { return ((long long)T + 63) / 64 * 64; }
long long attention_ds_workspace_elems(int B, int T, int nh) {
  const long long Tp = attention_ds_pitch(T);
  return (long long)B * nh * Tp * Tp;
}

}  // namespace rb
