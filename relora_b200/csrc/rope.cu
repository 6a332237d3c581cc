// Rotary position embedding kernels with 128-bit accesses.
//   rope_inplace_vec : in-place rotation of q,k heads inside the packed [tokens, 3h] QKV buffer (forward / backward)
//   rope_pack_bwd    : attention-backward epilogue: gathers dq [B, nh, T, hd], dk, dv [B, nkv, T, hd] (arbitrary batch/head/token
//                      strides) into the packed dQKV buffer [q: nh | k: nkv | v: nkv] and applies the inverse rotation to dq, dk on the way
//                      (replaces three strided copies + an in-place rotation pass).
// Half-rotation layout (reference modeling_llama.py:126-141): y1 = x1 c - x2 s, y2 = x2 c + x1 s; backward uses -s.
#include "common.cuh"
#include "kernels.h"

namespace rb {

__device__ __forceinline__ void rotate8(const uint4& a, const uint4& b, const uint4& c, const uint4& s, float sgn, uint4& oa, uint4& ob) {
  float x1[8], x2[8], cf[8], sf[8], y1[8], y2[8];
  unpack8(a, x1);
  unpack8(b, x2);
  unpack8(c, cf);
  unpack8(s, sf);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float sn = sf[i] * sgn;
    y1[i] = x1[i] * cf[i] - x2[i] * sn;
    y2[i] = x2[i] * cf[i] + x1[i] * sn;
  }
  oa = pack8(y1);
  ob = pack8(y2);
}

__global__ void __launch_bounds__(256) rope_vec_kernel(bf16* __restrict__ buf, long long ld, long long total, int T, int n_heads, int hd,
                                                       int half, const bf16* __restrict__ cosp, const bf16* __restrict__ sinp, float sgn,
                                                       int pos0) {
  pdl_wait();
  pdl_launch_dependents();
  const int nr = half / 8;  // vectors per half
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int j = int(i % nr);
    const long long t = i / nr;
    const int h = int(t % n_heads);
    const long long row = t / n_heads;
    const int pos = int(row % T) + pos0;
    bf16* base = buf + row * ld + (long long)h * hd + j * 8;
    const uint4 c = *reinterpret_cast<const uint4*>(cosp + (long long)pos * 2 * half + j * 8);
    const uint4 s = *reinterpret_cast<const uint4*>(sinp + (long long)pos * 2 * half + j * 8);
    uint4 oa, ob;
    rotate8(*reinterpret_cast<const uint4*>(base), *reinterpret_cast<const uint4*>(base + half), c, s, sgn, oa, ob);
    *reinterpret_cast<uint4*>(base) = oa;
    *reinterpret_cast<uint4*>(base + half) = ob;
  }
}

bool rope_inplace_vec(void* buf, long long ld, int M, int T, int n_rot_heads, int hd, int rotary_dim, const void* cos, const void* sin,
                      bool backward, int pos0, cudaStream_t s) {
  const int half = rotary_dim / 2;
  if (half % 8 != 0 || hd % 8 != 0 || ld % 8 != 0 || ((reinterpret_cast<uintptr_t>(buf) | reinterpret_cast<uintptr_t>(cos) |
                                                         reinterpret_cast<uintptr_t>(sin)) & 15) != 0)
    return false;
  const long long total = (long long)M * n_rot_heads * (half / 8);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 16);
  launch_k(rope_vec_kernel, grid, 256, 0, s, (bf16*)buf, ld, total, T, n_rot_heads, hd, half, (const bf16*)cos, (const bf16*)sin,
                                       backward ? -1.f : 1.f, pos0);
  RB_CHECK_LAUNCH("rope_vec");
  return true;
}

// one thread per 8 columns of a query head; the threads of heads h < nkv also carry KV head h
__global__ void __launch_bounds__(256) rope_pack_bwd_kernel(const bf16* __restrict__ dq, const bf16* __restrict__ dk, const bf16* __restrict__ dv,
                                                            long long sB, long long sH, long long sT, long long kB, long long kH, long long kT,
                                                            bf16* __restrict__ out, long long ldo, long long total, int T, int nh, int nkv, int hd,
                                                            int half, const bf16* __restrict__ cosp, const bf16* __restrict__ sinp, int pos0) {
  pdl_wait();
  pdl_launch_dependents();
  const int nv = hd / 8, nr = half / 8;
  const long long qsz = (long long)nh * hd, ksz = (long long)nkv * hd;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int j = int(i % nv);
    const long long t = i / nv;
    const int h = int(t % nh);
    const long long row = t / nh;
    const long long b = row / T, tt = row % T;
    const long long src = b * sB + h * sH + tt * sT + j * 8;
    const long long ksrc = b * kB + h * kH + tt * kT + j * 8;
    const bool kv = h < nkv;
    bf16* o = out + row * ldo + (long long)h * hd + j * 8;
    // v: plain gather
    if (kv) *reinterpret_cast<uint4*>(o + qsz + ksz) = *reinterpret_cast<const uint4*>(dv + ksrc);
    if (j < nr) {
      const int pos = int(tt) + pos0;
      const uint4 c = *reinterpret_cast<const uint4*>(cosp + (long long)pos * 2 * half + j * 8);
      const uint4 s = *reinterpret_cast<const uint4*>(sinp + (long long)pos * 2 * half + j * 8);
      uint4 oa, ob;
      rotate8(*reinterpret_cast<const uint4*>(dq + src), *reinterpret_cast<const uint4*>(dq + src + half), c, s, -1.f, oa, ob);
      *reinterpret_cast<uint4*>(o) = oa;
      *reinterpret_cast<uint4*>(o + half) = ob;
      if (kv) {
        rotate8(*reinterpret_cast<const uint4*>(dk + ksrc), *reinterpret_cast<const uint4*>(dk + ksrc + half), c, s, -1.f, oa, ob);
        *reinterpret_cast<uint4*>(o + qsz) = oa;
        *reinterpret_cast<uint4*>(o + qsz + half) = ob;
      }
    } else if (j >= 2 * nr) {  // dims beyond the rotary part pass through
      *reinterpret_cast<uint4*>(o) = *reinterpret_cast<const uint4*>(dq + src);
      if (kv) *reinterpret_cast<uint4*>(o + qsz) = *reinterpret_cast<const uint4*>(dk + ksrc);
    }
  }
}

void rope_pack_bwd(const void* dq, const void* dk, const void* dv, long long sB, long long sH, long long sT, long long kB, long long kH,
                   long long kT, void* out, long long ldo, int B, int T, int nh, int nkv, int hd, int rotary_dim, const void* cos,
                   const void* sin, int pos0, cudaStream_t s) {
  const int half = rotary_dim / 2;
  if (half % 8 != 0 || hd % 8 != 0) throw std::runtime_error("rope_pack_bwd: head_dim and rotary_dim must allow 128-bit accesses");
  if (nkv <= 0 || nkv > nh || nh % nkv != 0) throw std::runtime_error("rope_pack_bwd: nh must be a multiple of nkv");
  const long long total = (long long)B * T * nh * (hd / 8);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 16);
  launch_k(rope_pack_bwd_kernel, grid, 256, 0, s, (const bf16*)dq, (const bf16*)dk, (const bf16*)dv, sB, sH, sT, kB, kH, kT, (bf16*)out, ldo,
                                            total, T, nh, nkv, hd, half, (const bf16*)cos, (const bf16*)sin, pos0);
  RB_CHECK_LAUNCH("rope_pack_bwd");
}

}  // namespace rb
