// Causal flash attention for sm_90a: wgmma with the scores, probabilities and outputs in registers, TMA loads straight out
// of the packed qkv projection buffer.
//
// Replaces the reference's F.scaled_dot_product_attention call (peft_pretraining/modeling_llama.py:241-247 and
// modeling_pythia.py attention) for head_dim <= 64.  Three kernels, one warpgroup (128 threads, 64 rows) per CTA:
//
//   attn_fwd_kernel      CTA = (64 queries, head, batch); per 64 keys:  S = Q·Kᵀ -> online softmax -> O += P·V
//   attn_bwd_dq_kernel   CTA = (64 queries, head, batch); per 64 keys:  S, dP = dO·Vᵀ -> dS -> dQ += dS·K
//   attn_bwd_dkv_kernel  CTA = (64 keys, head, batch); per 64 queries:  Sᵀ = K·Qᵀ, dPᵀ = V·dOᵀ -> Pᵀ, dSᵀ -> dV += Pᵀ·dO, dK += dSᵀ·Q
//
// Shared-memory tiles are [64 rows x 64 columns] bf16 (128 bytes per row, 128-byte swizzle), so the same tile serves as a
// K-major operand (reduction over head_dim) and as an MN-major operand (reduction over its rows) by descriptor alone.  The
// probabilities / score gradients never leave registers: the accumulator fragment of one wgmma is, packed to bf16, the
// register A operand of the next.  The streamed operand pair is double buffered.  Each consumer issues one k-block of wgmma
// and waits for it before the dependent math; the overlap this forgoes has not been measured on the H100.
#include <cuda.h>

#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <stdexcept>
#include <unordered_map>

#include "attention.h"
#include "common.cuh"
#include "sm90.cuh"
#include "tensormap.h"

namespace rb {

using namespace sm90;

namespace {

constexpr int BQ = 64;                // rows per CTA (queries in fwd / dq, keys in dkv)
constexpr int kTile = 64 * 128;       // bytes of a [64 x 64] bf16 tile
constexpr int kThreads = 128;
constexpr int kSmem = 6 * kTile + 1024 + 1024;  // two resident tiles, two double-buffered streamed tiles, barriers, alignment
constexpr float kNegInf = -1e30f;

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
// d += A · Bᵀ with A, B both [64 x 64] K-major tiles (reduction over head_dim)
__device__ __forceinline__ void mma_tiles_kk(float (&d)[32], uint32_t a, uint32_t b) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) wgmma_bf16_ss_n64<0, 0>(d, desc_kmajor(a + kk * 32), desc_kmajor(b + kk * 32));
}
// d += P · T with P in registers (rows x 64) and T a [64 x 64] tile read MN-major (reduction over its rows)
__device__ __forceinline__ void mma_regs_tile(float (&d)[32], const float (&p)[32], uint32_t t) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    uint32_t a[4];
    frag_to_a(p, kk, a);
    wgmma_bf16_rs_n64<1>(d, a, desc_mnmajor(t + kk * 2048));
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
__device__ __forceinline__ Smem smem_layout() {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* s = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  Smem m;
  m.res[0] = s;
  m.res[1] = s + kTile;
  for (int b = 0; b < 2; ++b)
    for (int o = 0; o < 2; ++o) m.str[b][o] = s + (2 + 2 * b + o) * kTile;
  m.res_bar = reinterpret_cast<uint64_t*>(s + 6 * kTile);
  m.str_bar = m.res_bar + 1;
  m.col_lse = reinterpret_cast<float*>(s + 6 * kTile + 64);
  m.col_delta = m.col_lse + 64;
  return m;
}
// Barriers (thread 0), then the resident tiles and the first two streamed pairs (one elected lane of warp 0 issues every TMA load:
// the whole warp takes the branch, so ptxas needs no uniformisation loop around the loads).
struct TileSrc {
  const CUtensorMap* map;
  int head;
};
__device__ __forceinline__ void issue_pair(const Smem& m, int buf, TileSrc s0, TileSrc s1, int row) {
  mbar_arrive_expect_tx(&m.str_bar[buf], 2 * kTile);
  tma_load_3d(s0.map, &m.str_bar[buf], m.str[buf][0], 0, s0.head, row);
  tma_load_3d(s1.map, &m.str_bar[buf], m.str[buf][1], 0, s1.head, row);
}
template <int NRES>
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
      mbar_arrive_expect_tx(m.res_bar, NRES * kTile);
      tma_load_3d(r0.map, m.res_bar, m.res[0], 0, r0.head, res_row);
      if (NRES == 2) tma_load_3d(r1.map, m.res_bar, m.res[1], 0, r1.head, res_row);
      for (int j = 0; j < 2 && j < nblk; ++j) issue_pair(m, j, s0, s1, row0 + j * BQ);
    }
    __syncwarp();
  }
  mbar_wait(m.res_bar, 0);
}

struct FwdArgs {
  bf16* out;
  long long ld_out;
  float* lse;
  int B, T, nh, hd;
  float scale_log2;
};

// =============================================================================================== forward
__global__ void __launch_bounds__(kThreads) attn_fwd_kernel(const __grid_constant__ CUtensorMap map_qkv, const FwdArgs p) {
  if (threadIdx.x == 0) pdl_launch_dependents();
  const int nqb = (p.T + BQ - 1) / BQ;
  const int qb = nqb - 1 - blockIdx.x;  // longest rows first
  const int h = blockIdx.y, b = blockIdx.z;
  const int q0 = qb * BQ, rowbase = b * p.T;
  const int nkb = qb + 1;
  const Smem m = smem_layout();
  // resident: Q; streamed: K, V
  prologue<1>(m, {&map_qkv, h}, {&map_qkv, h}, rowbase + q0, {&map_qkv, p.nh + h}, {&map_qkv, 2 * p.nh + h}, rowbase, nkb);
  const uint32_t sq = smem_u32(m.res[0]);
  float o[32], mrow[2] = {kNegInf, kNegInf}, lrow[2] = {0.f, 0.f};
  zero32(o);
  const int r_lo = q0 + frag_row(0);  // this thread's two query rows: r_lo and r_lo + 8
  for (int j = 0; j < nkb; ++j) {
    const int buf = j & 1;
    mbar_wait(&m.str_bar[buf], (j >> 1) & 1);
    float s[32];
    zero32(s);
    wgmma_fence();
    mma_tiles_kk(s, sq, smem_u32(m.str[buf][0]));
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
      o[i] *= corr[hr];
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      lrow[hr] = lrow[hr] * corr[hr] + ls[hr];
      mrow[hr] = mx[hr];
    }
    wgmma_fence();
    mma_regs_tile(o, s, smem_u32(m.str[buf][1]));
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    __syncthreads();  // every warp is done with this buffer
    if (warp_id() == 0 && j + 2 < nkb) {
      if (elect_one()) issue_pair(m, buf, {&map_qkv, p.nh + h}, {&map_qkv, 2 * p.nh + h}, rowbase + (j + 2) * BQ);
      __syncwarp();
    }
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    lrow[hr] += __shfl_xor_sync(0xffffffffu, lrow[hr], 1);
    lrow[hr] += __shfl_xor_sync(0xffffffffu, lrow[hr], 2);
  }
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int hr = (i >> 1) & 1;
    const int q = r_lo + 8 * hr, c = frag_col(i);
    if (q >= p.T || c >= p.hd) continue;
    const float inv = 1.f / lrow[hr];
    *reinterpret_cast<uint32_t*>(p.out + (long long)(rowbase + q) * p.ld_out + h * p.hd + c) = pack_bf16x2(o[i] * inv, o[i + 1] * inv);
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
};

__device__ __forceinline__ void store_rows(bf16* base, long long ld, int row0, int rows_valid, int col_ofs, int hd, const float (&d)[32], float sc) {
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int r = frag_row(i), c = frag_col(i);
    if (row0 + r >= rows_valid || c >= hd) continue;
    *reinterpret_cast<uint32_t*>(base + (long long)row0 * ld + (long long)r * ld + col_ofs + c) = pack_bf16x2(d[i] * sc, d[i + 1] * sc);
  }
}

// =============================================================================================== backward: dQ
__global__ void __launch_bounds__(kThreads) attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap map_qkv,
                                                               const __grid_constant__ CUtensorMap map_do, const BwdArgs p) {
  if (threadIdx.x == 0) pdl_launch_dependents();
  const int nqb = (p.T + BQ - 1) / BQ;
  const int qb = nqb - 1 - blockIdx.x;
  const int h = blockIdx.y, b = blockIdx.z;
  const int q0 = qb * BQ, rowbase = b * p.T;
  const int nkb = qb + 1;
  const Smem m = smem_layout();
  prologue<2>(m, {&map_qkv, h}, {&map_do, h}, rowbase + q0, {&map_qkv, p.nh + h}, {&map_qkv, 2 * p.nh + h}, rowbase, nkb);
  const long long bh = (long long)b * p.nh + h;
  const int r_lo = q0 + frag_row(0);
  float lse[2], dlt[2];
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int q = min(r_lo + 8 * hr, p.T - 1);
    lse[hr] = p.lse[bh * p.T + q];
    dlt[hr] = p.delta[bh * p.T + q];
  }
  float dq[32];
  zero32(dq);
  for (int j = 0; j < nkb; ++j) {
    const int buf = j & 1;
    mbar_wait(&m.str_bar[buf], (j >> 1) & 1);
    float s[32], dp[32];
    zero32(s);
    zero32(dp);
    wgmma_fence();
    mma_tiles_kk(s, smem_u32(m.res[0]), smem_u32(m.str[buf][0]));   // S = Q·Kᵀ
    mma_tiles_kk(dp, smem_u32(m.res[1]), smem_u32(m.str[buf][1]));  // dP = dO·Vᵀ
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
    wgmma_fence();
    mma_regs_tile(dq, s, smem_u32(m.str[buf][0]));  // dQ += dS·K
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(dq);
    __syncthreads();
    if (warp_id() == 0 && j + 2 < nkb) {
      if (elect_one()) issue_pair(m, buf, {&map_qkv, p.nh + h}, {&map_qkv, 2 * p.nh + h}, rowbase + (j + 2) * BQ);
      __syncwarp();
    }
  }
  store_rows(p.dqkv + (long long)rowbase * p.ld_dqkv, p.ld_dqkv, q0, p.T, h * p.hd, p.hd, dq, p.scale);
}

// =============================================================================================== backward: dK, dV
__global__ void __launch_bounds__(kThreads) attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap map_qkv,
                                                                const __grid_constant__ CUtensorMap map_do, const BwdArgs p) {
  if (threadIdx.x == 0) pdl_launch_dependents();
  const int nkb = (p.T + BQ - 1) / BQ;
  const int kb = blockIdx.x;  // key block; query blocks kb .. nkb-1
  const int h = blockIdx.y, b = blockIdx.z;
  const int k0 = kb * BQ, rowbase = b * p.T;
  const int nblk = nkb - kb;
  const Smem m = smem_layout();
  prologue<2>(m, {&map_qkv, p.nh + h}, {&map_qkv, 2 * p.nh + h}, rowbase + k0, {&map_qkv, h}, {&map_do, h}, rowbase + k0, nblk);
  const long long bh = (long long)b * p.nh + h;
  const int key_lo = k0 + frag_row(0);
  float dk[32], dv[32];
  zero32(dk);
  zero32(dv);
  for (int jj = 0; jj < nblk; ++jj) {
    const int buf = jj & 1;
    const int qs = (kb + jj) * BQ;
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
    mma_tiles_kk(st, smem_u32(m.res[0]), smem_u32(m.str[buf][0]));   // Sᵀ = K·Qᵀ
    mma_tiles_kk(dpt, smem_u32(m.res[1]), smem_u32(m.str[buf][1]));  // dPᵀ = V·dOᵀ
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
    wgmma_fence();
    mma_regs_tile(dv, st, smem_u32(m.str[buf][1]));   // dV += Pᵀ·dO
    mma_regs_tile(dk, dpt, smem_u32(m.str[buf][0]));  // dK += dSᵀ·Q
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(dv);
    fence_regs(dk);
    __syncthreads();
    if (warp_id() == 0 && jj + 2 < nblk) {
      if (elect_one()) issue_pair(m, buf, {&map_qkv, h}, {&map_do, h}, rowbase + qs + 2 * BQ);
      __syncwarp();
    }
  }
  bf16* base = p.dqkv + (long long)rowbase * p.ld_dqkv;
  store_rows(base, p.ld_dqkv, k0, p.T, (p.nh + h) * p.hd, p.hd, dk, p.scale);
  store_rows(base, p.ld_dqkv, k0, p.T, (2 * p.nh + h) * p.hd, p.hd, dv, 1.0f);
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

void check_shape(int B, int T, int nh, int hd) {
  if (B <= 0 || T <= 0 || nh <= 0) throw std::runtime_error("attention: empty problem");
  if (hd % 8 != 0 || hd > 64) throw std::runtime_error("attention: head_dim must be a multiple of 8 and <= 64");
}

}  // namespace

void attention_fwd(const AttnDesc& d, cudaStream_t stream) {
  check_shape(d.B, d.T, d.nh, d.hd);
  const long long rows = (long long)d.B * d.T;
  CUtensorMap map = head_map(d.qkv, d.ld_qkv, rows, d.hd, 3 * d.nh);
  static bool configured = false;
  if (!configured) {
    check(cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem), "cudaFuncSetAttribute(attn_fwd)");
    configured = true;
  }
  FwdArgs p;
  p.out = reinterpret_cast<bf16*>(d.out); p.ld_out = d.ld_out; p.lse = d.lse;
  p.B = d.B; p.T = d.T; p.nh = d.nh; p.hd = d.hd;
  p.scale_log2 = d.scale * 1.4426950408889634f;
  const dim3 grid((unsigned)((d.T + BQ - 1) / BQ), (unsigned)d.nh, (unsigned)d.B);
  launch_k(attn_fwd_kernel, grid, kThreads, kSmem, stream, map, p);
  RB_CHECK_LAUNCH("attn_fwd_kernel");
}

void attention_bwd(const AttnBwdDesc& d, cudaStream_t stream) {
  check_shape(d.B, d.T, d.nh, d.hd);
  const long long rows = (long long)d.B * d.T;
  CUtensorMap map_qkv = head_map(d.qkv, d.ld_qkv, rows, d.hd, 3 * d.nh);
  CUtensorMap map_do = head_map(d.dout, d.ld_dout, rows, d.hd, d.nh);
  static bool configured = false;
  if (!configured) {
    check(cudaFuncSetAttribute(attn_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem), "cudaFuncSetAttribute(attn_dq)");
    check(cudaFuncSetAttribute(attn_bwd_dkv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem), "cudaFuncSetAttribute(attn_dkv)");
    configured = true;
  }
  {
    const long long total = rows * d.nh;
    const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 8);
    launch_k(attn_delta_kernel, grid, 256, 0, stream, reinterpret_cast<const bf16*>(d.out), d.ld_out, reinterpret_cast<const bf16*>(d.dout),
             d.ld_dout, d.delta, d.B, d.T, d.nh, d.hd);
    RB_CHECK_LAUNCH("attn_delta_kernel");
  }
  BwdArgs p;
  p.lse = d.lse; p.delta = d.delta; p.dqkv = reinterpret_cast<bf16*>(d.dqkv); p.ld_dqkv = d.ld_dqkv;
  p.B = d.B; p.T = d.T; p.nh = d.nh; p.hd = d.hd;
  p.scale = d.scale; p.scale_log2 = d.scale * 1.4426950408889634f;
  const dim3 grid((unsigned)((d.T + BQ - 1) / BQ), (unsigned)d.nh, (unsigned)d.B);
  launch_k(attn_bwd_dkv_kernel, grid, kThreads, kSmem, stream, map_qkv, map_do, p);
  RB_CHECK_LAUNCH("attn_bwd_dkv_kernel");
  launch_k(attn_bwd_dq_kernel, grid, kThreads, kSmem, stream, map_qkv, map_do, p);
  RB_CHECK_LAUNCH("attn_bwd_dq_kernel");
}

long long attention_ds_pitch(int T) { return ((long long)T + 63) / 64 * 64; }
long long attention_ds_workspace_elems(int B, int T, int nh) {
  const long long Tp = attention_ds_pitch(T);
  return (long long)B * nh * Tp * Tp;
}

}  // namespace rb
