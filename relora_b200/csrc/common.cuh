// Shared device helpers: counter-based RNG (dropout masks / re-init), reductions, vector access,
// plus the host-side launch counter and error macro used by every launcher.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp8.h>

#include "fp8out.h"
#include <cuda_runtime.h>

#include <cstdlib>
#include <utility>
#include <stdint.h>
#include <stdio.h>

#include <stdexcept>
#include <string>

typedef __nv_bfloat16 bf16;

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
namespace rb {

// number of kernels launched by this extension since the last reset (bench.py: "gpu_launches")
extern long long g_launch_count;
inline void count_launch(int n = 1) { g_launch_count += n; }

inline void check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string("CUDA error in ") + what + ": " + cudaGetErrorString(e));
}
#define RB_CHECK_LAUNCH(name)                \
  do {                                       \
    rb::count_launch();                      \
    rb::check(cudaGetLastError(), name);     \
  } while (0)

// ---- programmatic dependent launch (PDL): a kernel launched with the attribute may start (and run its prologue) while its
// predecessor in the stream is still draining; it must call pdl_wait() before touching global memory.  Predecessors call
// pdl_launch_dependents() early so the next grid's CTAs are scheduled as soon as SM resources free up.  Inside captured CUDA graphs
// these become programmatic dependency edges.  Enabled with RB_PDL=1.
inline bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("RB_PDL");  // opt-in
    v = (e != nullptr && atoi(e) != 0) ? 1 : 0;
  }
  return v != 0;
}
template <typename... KArgs, typename... Args>
inline void launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  check(cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...), "cudaLaunchKernelEx");
}
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#endif

inline int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}
inline int ceil_div(long long a, long long b) { return int((a + b - 1) / b); }

}  // namespace rb

// ---------------------------------------------------------------------------------------------
// device side
// ---------------------------------------------------------------------------------------------
// keep(row, col) = (lowbias32(row*C1 ^ col*C2 ^ seed) >> 8) >= threshold24     (ops/reference.py)
__host__ __device__ __forceinline__ uint32_t lowbias32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7FEB352Du;
  x ^= x >> 15;
  x *= 0x846CA68Bu;
  x ^= x >> 16;
  return x;
}
__host__ __device__ __forceinline__ uint32_t hash_rc(uint32_t seed, uint32_t row, uint32_t col) {
  return lowbias32((row * 0x9E3779B1u) ^ (col * 0x85EBCA77u) ^ seed);
}
__host__ __device__ __forceinline__ bool keep_bit(uint32_t seed, uint32_t row, uint32_t col, uint32_t threshold24) {
  return (hash_rc(seed, row, col) >> 8) >= threshold24;
}
// Dropout keep mask: one hash per column PAIR, 16-bit threshold (halves the integer work of every dropout consumer;
// it was the bound of the fused LoRA-backward epilogue and of the RMSNorm forward with three expanded copies):
//   h = lowbias32(row*C1 ^ (col>>1)*C2 ^ seed);  keep(row, col) = ((col & 1) ? h >> 16 : h & 0xFFFF) >= round(p * 2^16)
// Same definition in ops/reference.py:dropout_keep_mask.
__host__ __device__ __forceinline__ uint32_t drop_hash2(uint32_t seed, uint32_t row, uint32_t col) {
  return lowbias32((row * 0x9E3779B1u) ^ ((col >> 1) * 0x85EBCA77u) ^ seed);
}
__host__ __device__ __forceinline__ bool keep_drop(uint32_t seed, uint32_t row, uint32_t col, uint32_t thr16) {
  const uint32_t h = drop_hash2(seed, row, col);
  return ((col & 1u) ? (h >> 16) : (h & 0xFFFFu)) >= thr16;
}
__host__ __device__ __forceinline__ uint32_t mix_seed(uint32_t base, uint32_t key) {
  uint32_t x = base ^ key;
  x = (x ^ (x >> 16)) * 0x7FEB352Du;
  x = (x ^ (x >> 15)) * 0x846CA68Bu;
  return x ^ (x >> 16);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- optional E4M3 side output of a producer kernel (fp8 frozen-weight path, see fp8.cu): q = sat_e4m3(value * *inv_scale),
// amax(|value|) recorded for the next micro-step's delayed scale
__device__ __forceinline__ uint2 pack8_e4m3(const float (&f)[8], float inv) {
  uint32_t w[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const __nv_fp8x2_storage_t lo = __nv_cvt_float2_to_fp8x2(make_float2(f[h * 4] * inv, f[h * 4 + 1] * inv), __NV_SATFINITE, __NV_E4M3);
    const __nv_fp8x2_storage_t hi = __nv_cvt_float2_to_fp8x2(make_float2(f[h * 4 + 2] * inv, f[h * 4 + 3] * inv), __NV_SATFINITE, __NV_E4M3);
    w[h] = (uint32_t)lo | ((uint32_t)hi << 16);
  }
  return make_uint2(w[0], w[1]);
}
__device__ __forceinline__ float absmax8(const float (&f)[8]) {
  float m = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) m = fmaxf(m, fabsf(f[j]));
  return m;
}
// warp-level: one atomic only when this warp raises the running maximum (almost never after the first few warps)
__device__ __forceinline__ void amax_commit(float lane_max, float* amax) {
  const float m = warp_max(lane_max);
  if ((threadIdx.x & 31) == 0 && m > *reinterpret_cast<volatile float*>(amax))
    atomicMax(reinterpret_cast<unsigned int*>(amax), __float_as_uint(m));
}
// block-wide sum; `scratch` must hold >= 32 floats; result broadcast to every thread
__device__ __forceinline__ float block_sum(float v, float* scratch) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) scratch[w] = v;
  __syncthreads();
  float t = (lane < nw) ? scratch[lane] : 0.f;
  return warp_sum(t);
}
__device__ __forceinline__ float block_max(float v, float* scratch) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) scratch[w] = v;
  __syncthreads();
  float t = (lane < nw) ? scratch[lane] : -INFINITY;
  return warp_max(t);
}

// 8 packed bf16 moved as one 128-bit access.  (A struct of four bfloat162 is copied member-wise by nvcc, which
// turns every load/store into four 32-bit transactions; the builtin vector type keeps LDG/STG.128.)
typedef uint4 bf16x8;
__device__ __forceinline__ void unpack8(const bf16x8& p, float (&f)[8]) {
  const uint32_t w[4] = {p.x, p.y, p.z, p.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(&w[i]);
    float2 t = __bfloat1622float2(b);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ bf16x8 pack8(const float (&f)[8]) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat162 b = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    w[i] = *reinterpret_cast<uint32_t*>(&b);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
