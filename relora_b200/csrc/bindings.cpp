// Python bindings (pybind11 over torch::Tensor) for the sm_90a kernels.  Every function launches on the
// current PyTorch CUDA stream, so the ops compose with torch streams and CUDA-graph capture.
//
// This is where Python tensors become raw pointers, so every tensor argument goes through arg() once, before anything
// launches: a call that got past the host with a wrong operand would fault on the device instead of raising.  The launchers
// keep only the limits of what their kernels support (row widths, head dims, tile multiples).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "comm.h"
#include "attention.h"
#include "gemm.h"
#include "kernels.h"

namespace rb {
extern long long g_launch_count;
}

namespace {

using torch::Tensor;
using OptTensor = c10::optional<Tensor>;
constexpr auto BF = at::kBFloat16;
constexpr auto F32 = at::kFloat;

cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

// The binding being called and the device all of its tensors must be on.
struct Call {
  const char* fn;
  c10::Device dev;
};

// Numbers are formatted with std::to_string: streaming an integer into a TORCH_CHECK message from this extension is not
// safe against every libstdc++ the torch wheels are built with.
std::string dims(c10::IntArrayRef v) {
  std::string s = "[";
  for (size_t i = 0; i < v.size(); ++i) s += (i ? ", " : "") + std::to_string(v[i]);
  return s + "]";
}

// Checks one tensor argument of binding c.fn and returns its data pointer.  The tensor must be a CUDA tensor on c.dev of
// dtype `dt` (at::kByte: any one-byte type) that covers `shape`, the extent the kernel touches:
//   - one entry: at least shape[0] elements of a contiguous tensor of any rank;
//   - more: that rank, a unit inner stride and at least shape[d] entries in dimension d; `strides`, if given, pins the
//     stride of every outer dimension (a kernel that derives the pitch itself).
// `align` (bytes) is what the kernel's vector or TMA accesses need of the base and of every outer stride.  As for
// is_contiguous(), the stride of a dimension of size 1 is never used and not checked.
template <class T = void>
T* arg(const Call& c, const Tensor& t, const char* name, at::ScalarType dt, c10::IntArrayRef shape, int64_t align = 1,
       c10::IntArrayRef strides = {}) {
  TORCH_CHECK(t.is_cuda() && t.device() == c.dev, c.fn, ": ", name, " must be a CUDA tensor on ", c.dev.str(), ", got ", t.device().str());
  TORCH_CHECK(dt == at::kByte ? t.element_size() == 1 : t.scalar_type() == dt, c.fn, ": ", name, " must be ",
              dt == at::kByte ? "a one-byte type" : c10::toString(dt), ", got ", c10::toString(t.scalar_type()));
  const int64_t r = (int64_t)shape.size();
  if (r == 1) {
    TORCH_CHECK(t.is_contiguous(), c.fn, ": ", name, " must be contiguous");
    TORCH_CHECK(t.numel() >= shape[0], c.fn, ": ", name, " has ", std::to_string(t.numel()), " elements, smaller than the ",
                std::to_string(shape[0]), " expected");
  } else {
    TORCH_CHECK(t.dim() == r && t.stride(r - 1) == 1, c.fn, ": ", name, " must be ", std::to_string(r), "-D with unit inner stride, got sizes ",
                dims(t.sizes()), " and strides ", dims(t.strides()));
    for (int64_t d = 0; d < r; ++d)
      TORCH_CHECK(t.size(d) >= shape[d], c.fn, ": ", name, " ", dims(t.sizes()), " is smaller than the ", dims(shape), " expected");
    for (int64_t d = 0; d + 1 < r && !strides.empty(); ++d)
      TORCH_CHECK(t.size(d) <= 1 || t.stride(d) == strides[d], c.fn, ": ", name, " must have strides ", dims(strides), " in its outer dimensions, got ",
                  dims(t.strides()));
  }
  bool aligned = reinterpret_cast<uintptr_t>(t.data_ptr()) % align == 0;
  for (int64_t d = 0; d + 1 < r; ++d) aligned = aligned && (t.size(d) <= 1 || t.stride(d) * t.element_size() % align == 0);
  TORCH_CHECK(aligned, c.fn, ": ", name, " needs a ", std::to_string(align), "-byte-aligned base and row pitch, got strides ",
              dims(t.strides()));
  return static_cast<T*>(t.data_ptr());
}
// optional tensors: nullptr when absent
template <class T = void>
T* arg(const Call& c, const OptTensor& t, const char* name, at::ScalarType dt, c10::IntArrayRef shape, int64_t align = 1,
       c10::IntArrayRef strides = {}) {
  return t.has_value() ? arg<T>(c, *t, name, dt, shape, align, strides) : nullptr;
}

// The LoRA-dropout arguments of one call: the device seed (absent: seed 0), min_keys .. max_keys mask keys (one per group)
// and p in [0, 1).
struct Dropout {
  const uint32_t* seed = nullptr;
  uint32_t keys[4] = {0, 0, 0, 0};
  int groups = 0;
  uint32_t thr16 = 0;  // round(p * 65536)
  float inv_keep = 1.f;
  rb::LnDrop ln() const { return {seed, thr16, inv_keep}; }
};
Dropout dropout(const Call& c, const OptTensor& seed, const std::vector<int64_t>& keys, double p, int min_keys, int max_keys) {
  const int n = (int)keys.size();
  TORCH_CHECK(n >= min_keys && n <= max_keys, c.fn, ": ", std::to_string(n), " dropout keys, expected ", std::to_string(min_keys), " to ",
              std::to_string(max_keys));
  TORCH_CHECK(p >= 0.0 && p < 1.0, c.fn, ": dropout p must be in [0, 1), got ", std::to_string(p));
  Dropout d;
  d.seed = arg<const uint32_t>(c, seed, "seed", at::kInt, {1});
  d.groups = n;
  for (int i = 0; i < n; ++i) d.keys[i] = (uint32_t)keys[i];
  d.thr16 = (uint32_t)llround(p * 65536.0);
  d.inv_keep = (float)(1.0 / (1.0 - p));
  return d;
}

rb::Fp8Out fp8_out(const Call& c, const OptTensor& q8, const OptTensor& inv_scale, const OptTensor& amax, int64_t rows, int64_t cols) {
  rb::Fp8Out f;
  if (!q8.has_value()) return f;
  TORCH_CHECK(inv_scale.has_value() && amax.has_value(), c.fn, ": the fp8 output q8 needs q_inv_scale and q_amax");
  f.q = arg<uint8_t>(c, q8, "q8", at::kByte, {rows, cols}, 8);  // 8-byte stores
  f.ld = q8->stride(0);
  f.inv_scale = arg<const float>(c, inv_scale, "q_inv_scale", F32, {1});
  f.amax = arg<float>(c, amax, "q_amax", F32, {1});
  return f;
}

// out[M,N] = alpha*(a1·b1ᵀ + a2·b2ᵀ) (+ residual) (+ out)
void gemm(const Tensor& a1, const Tensor& b1, Tensor& out, int64_t M, int64_t N, int64_t K1, const OptTensor& a2, const OptTensor& b2,
          int64_t K2, bool a1_mn, bool b1_mn, int64_t n_per_group, int64_t a1_group_kofs, int64_t a2_group_kofs,
          const OptTensor& residual, double alpha, bool accumulate, int64_t block_n, int64_t split_k, int64_t b1_group_kofs,
          bool b1_local_n, int64_t m_per_group, int64_t b1_mn_ofs_per_mgroup, const OptTensor& bias, int64_t pair, int64_t fp8,
          const OptTensor& alpha_dev) {
  const Call c{"gemm", out.device()};
  rb::GemmDesc d;
  d.M = (int)M; d.N = (int)N; d.K1 = (int)K1; d.K2 = (int)K2;
  d.a1.mn_major = a1_mn; d.b1.mn_major = b1_mn;
  d.fp8 = fp8 != 0; d.fp8_a_e5m2 = fp8 == 2;  // E4M3 / E5M2 bytes (torch.uint8 / float8 storage), leading dimensions in bytes
  d.n_per_group = (int)n_per_group; d.a1_group_kofs = (int)a1_group_kofs; d.a2_group_kofs = (int)a2_group_kofs;
  d.b1_group_kofs = (int)b1_group_kofs; d.b1_local_n = b1_local_n; d.m_per_group = (int)m_per_group;
  d.b1_mn_ofs_per_mgroup = (int)b1_mn_ofs_per_mgroup;
  d.accumulate = accumulate; d.alpha = (float)alpha; d.block_n = (int)block_n; d.split_k = (int)split_k; d.pair = (int)pair;
  TORCH_CHECK(K2 <= 0 || (a2.has_value() && b2.has_value()), "gemm: a2 and b2 are required when K2 > 0");
  // the tensor maps span these extents, so each operand must cover them
  const rb::GemmExtents e = rb::gemm_operand_extents(d);
  const auto in = d.fp8 ? at::kByte : BF;
  d.a1.ptr = arg(c, a1, "a1", in, {e.a1.rows, e.a1.cols}, 16); d.a1.ld = a1.stride(0);
  d.b1.ptr = arg(c, b1, "b1", in, {e.b1.rows, e.b1.cols}, 16); d.b1.ld = b1.stride(0);
  if (K2 > 0) {
    d.a2.ptr = arg(c, a2, "a2", BF, {e.a2.rows, e.a2.cols}, 16); d.a2.ld = a2->stride(0);
    d.b2.ptr = arg(c, b2, "b2", BF, {e.b2.rows, e.b2.cols}, 16); d.b2.ld = b2->stride(0);
  }
  d.out_f32 = out.scalar_type() == F32;
  d.out = arg(c, out, "out", d.out_f32 ? F32 : BF, {M, N}); d.ldc = out.stride(0);
  d.residual = arg(c, residual, "residual", BF, {M, N}); d.ldr = residual.has_value() ? residual->stride(0) : 0;
  d.bias = arg(c, bias, "bias", BF, {N});
  d.alpha_dev = arg<const float>(c, alpha_dev, "alpha_dev", F32, {1});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::gemm_bf16(d, cur_stream());
}

void rmsnorm_fwd(const Tensor& x, const Tensor& w, Tensor& y, Tensor& rstd, double eps, const OptTensor& xd, const OptTensor& seed,
                 std::vector<int64_t> keys, double p, const OptTensor& q8, const OptTensor& q_inv_scale, const OptTensor& q_amax) {
  const Call c{"rmsnorm_fwd", x.device()};
  const void* xp = arg(c, x, "x", BF, {0}, 16);
  const int64_t H = x.size(-1), M = x.numel() / H;
  const Dropout dr = dropout(c, seed, keys, p, xd.has_value() ? 1 : 0, 4);
  const int G = xd.has_value() ? dr.groups : 0;
  void* xdp = arg(c, xd, "xd", BF, {M * G * H}, 16);
  const void* wp = arg(c, w, "w", BF, {H}, 16);
  void* yp = arg(c, y, "y", BF, {M * H}, 16);
  float* rp = arg<float>(c, rstd, "rstd", F32, {M});
  const rb::Fp8Out f8 = fp8_out(c, q8, q_inv_scale, q_amax, M, H);
  c10::cuda::CUDAGuard guard(c.dev);
  rb::rmsnorm_fwd(xp, wp, yp, rp, (int)M, (int)H, (float)eps, xdp, G, dr.seed, dr.keys, dr.thr16, dr.inv_keep, f8, cur_stream());
}

void rmsnorm_bwd(const Tensor& dy, const Tensor& x, const Tensor& w, const Tensor& rstd, const OptTensor& dx_add, Tensor& dx, Tensor& dw,
                 const OptTensor& ws, const OptTensor& ticket) {
  const Call c{"rmsnorm_bwd", x.device()};
  const void* xp = arg(c, x, "x", BF, {0}, 16);
  const int64_t H = x.size(-1), M = x.numel() / H;
  const void* dyp = arg(c, dy, "dy", BF, {M * H}, 16);
  const void* wp = arg(c, w, "w", BF, {H}, 16);
  const float* rp = arg<const float>(c, rstd, "rstd", F32, {M});
  const void* add = arg(c, dx_add, "dx_add", BF, {M * H}, 16);
  void* dxp = arg(c, dx, "dx", BF, {M * H}, 16);
  float* dwp = arg<float>(c, dw, "dw", F32, {H});
  // the warp-per-row kernel runs only with both its workspace and ticket
  const bool warp = ws.has_value() && ticket.has_value();
  float* wsp = warp ? arg<float>(c, ws, "ws", F32, {rb::rmsnorm_bwd_ws_blocks() * H}) : nullptr;
  auto* tk = warp ? arg<unsigned int>(c, ticket, "ticket", at::kInt, {1}) : nullptr;
  c10::cuda::CUDAGuard guard(c.dev);
  rb::rmsnorm_bwd(dyp, xp, wp, rp, add, dxp, dwp, (int)M, (int)H, wsp, tk, cur_stream());
}

void dropout_expand(const Tensor& x, Tensor& xd, const OptTensor& seed, std::vector<int64_t> keys, double p, const OptTensor& q8,
                    const OptTensor& q_inv_scale, const OptTensor& q_amax) {
  const Call c{"dropout_expand", x.device()};
  const void* xp = arg(c, x, "x", BF, {0}, 16);
  const int64_t H = x.size(-1), M = x.numel() / H;
  const Dropout dr = dropout(c, seed, keys, p, 1, 4);
  void* xdp = arg(c, xd, "xd", BF, {M * dr.groups * H}, 16);
  const rb::Fp8Out f8 = fp8_out(c, q8, q_inv_scale, q_amax, M, H);
  c10::cuda::CUDAGuard guard(c.dev);
  rb::dropout_expand(xp, xdp, (int)M, (int)H, dr.groups, dr.seed, dr.keys, dr.thr16, dr.inv_keep, f8, cur_stream());
}

void dropout_combine(const OptTensor& base, const Tensor& parts, Tensor& out, const OptTensor& seed, std::vector<int64_t> keys, double p) {
  const Call c{"dropout_combine", out.device()};
  void* op = arg(c, out, "out", BF, {0, 0}, 16, {out.size(-1)});
  const int64_t M = out.size(0), H = out.size(1);
  const Dropout dr = dropout(c, seed, keys, p, 1, 4);
  const int64_t G = dr.groups;
  // parts: [G, M, H] contiguous, or [M, G*H] row-major with group g at column offset g*H
  const bool stacked = parts.dim() == 3;
  const void* pp = stacked ? arg(c, parts, "parts", BF, {G, M, H}, 16, {M * H, H}) : arg(c, parts, "parts", BF, {M, G * H}, 16);
  const void* bp = arg(c, base, "base", BF, {M * H}, 16);
  c10::cuda::CUDAGuard guard(c.dev);
  rb::dropout_combine(bp, pp, stacked ? M * H : H, stacked ? H : parts.stride(0), op, (int)M, (int)H, (int)G, dr.seed, dr.keys,
                      dr.thr16, dr.inv_keep, cur_stream());
}

void fp8_quantize_weight(const Tensor& w, Tensor& w8, Tensor& scratch, Tensor& scale, Tensor& inv_scale, const OptTensor& w8t) {
  const Call c{"fp8_quantize_weight", w.device()};
  const void* wp = arg(c, w, "w", BF, {0, 0}, 16);
  const int64_t R = w.size(0), C = w.size(1);
  void* w8p = arg(c, w8, "w8", at::kByte, {R, C}, 16);
  void* tp = arg(c, w8t, "w8t", at::kByte, {C, R});
  float* sp = arg<float>(c, scratch, "scratch", F32, {1});
  float* scp = arg<float>(c, scale, "scale", F32, {1});
  float* isp = arg<float>(c, inv_scale, "inv_scale", F32, {1});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::fp8_quantize_weight(wp, w.stride(0), w8p, w8.stride(0), tp, w8t.has_value() ? w8t->stride(0) : 0, (int)R, (int)C, sp, scp, isp,
                          cur_stream());
}
void fp8_quantize_act(const Tensor& x, Tensor& x8, const Tensor& inv_scale, const OptTensor& amax_cur, bool e5m2) {
  const Call c{"fp8_quantize_act", x.device()};
  const void* xp = arg(c, x, "x", BF, {0, 0}, 16);
  const int64_t R = x.size(0), C = x.size(1);
  void* x8p = arg(c, x8, "x8", at::kByte, {R, C}, 16);
  const float* isp = arg<const float>(c, inv_scale, "inv_scale", F32, {1});
  float* ap = arg<float>(c, amax_cur, "amax_cur", F32, {1});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::fp8_quantize_act(xp, x.stride(0), x8p, x8.stride(0), (int)R, (int)C, isp, ap, e5m2, cur_stream());
}
void fp8_prep(Tensor& state, const Tensor& w_scale, Tensor& inv_sx, Tensor& alpha_main, Tensor& alpha_inv, double margin, int64_t n_e4m3) {
  const Call c{"fp8_prep", w_scale.device()};
  const float* wsp = arg<const float>(c, w_scale, "w_scale", F32, {0});
  const int64_t n = w_scale.numel();
  float* sp = arg<float>(c, state, "state", F32, {2 * n});
  float* ip = arg<float>(c, inv_sx, "inv_sx", F32, {n});
  float* mp = arg<float>(c, alpha_main, "alpha_main", F32, {n});
  float* ap = arg<float>(c, alpha_inv, "alpha_inv", F32, {n});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::fp8_prep(sp, wsp, ip, mp, ap, (int)n, (float)margin, n_e4m3 < 0 ? (int)n : (int)n_e4m3, cur_stream());
}

// out[M,N] = dy[M,Kb]·W[Kb,N] + Σ_g keep_g ⊙ (du_g·A_g)/(1-p)     (fused input gradient of a stacked LoRA group)
void lora_dx(const OptTensor& dy, const OptTensor& w, const Tensor& du, const Tensor& a, Tensor& out, const OptTensor& seed,
             std::vector<int64_t> keys, double p, const OptTensor& base, int64_t pair, int64_t block_n) {
  const Call c{"lora_dx", out.device()};
  const Dropout dr = dropout(c, seed, keys, p, 1, 3);
  rb::LoraDxDesc d;
  d.groups = dr.groups;
  d.du = arg(c, du, "du", BF, {0, 0}, 16); d.ld_du = du.stride(0);
  const int64_t du_cols = du.size(1);  // du = [du_0 | du_1 | ...], [M, G*r]
  TORCH_CHECK(du_cols % d.groups == 0, "lora_dx: du must be [M, G*r] for the G = ", std::to_string(d.groups), " dropout keys");
  d.M = (int)du.size(0); d.r = (int)(du_cols / d.groups);
  d.a = arg(c, a, "a", BF, {(int64_t)d.groups * d.r, 0}, 16); d.ld_a = a.stride(0);
  d.N = (int)a.size(1);
  d.out = arg(c, out, "out", BF, {d.M, d.N}, 16); d.ldc = out.stride(0);
  if (base.has_value()) {
    // two-kernel form: base = dy·W from the plain GEMM, this launch adds the masked low-rank terms
    d.base = arg(c, base, "base", BF, {d.M, d.N}, 16); d.ld_base = base->stride(0); d.Kb = 0;
  } else {
    TORCH_CHECK(dy.has_value() && w.has_value(), "lora_dx: pass (dy, w) or base");
    d.dy = arg(c, dy, "dy", BF, {d.M, 0}, 16); d.ld_dy = dy->stride(0);
    d.Kb = (int)dy->size(1);
    d.w = arg(c, w, "w", BF, {d.Kb, d.N}, 16); d.ld_w = w->stride(0);
  }
  d.drop_threshold16 = dr.thr16; d.inv_keep = dr.inv_keep; d.seed_ptr = dr.seed;
  for (int i = 0; i < 3; ++i) d.seed_key[i] = dr.keys[i];
  d.pair = (int)pair;
  TORCH_CHECK(block_n == 0 || block_n == 128 || block_n == 192, "lora_dx: block_n must be 0 (auto), 128 or 192");
  d.block_n = (int)block_n;
  c10::cuda::CUDAGuard guard(c.dev);
  rb::lora_dx(d, cur_stream());
}

// causal flash attention over the packed (post-RoPE) qkv buffer [B*T, (nh + 2*nkv)*hd]; nkv < 0 means nkv = nh.  The kernels
// read out rows with 16-byte loads and store 4-byte pairs into out / dqkv, so those tensors obey the rule the TMA maps enforce
// for qkv / dout: a 16-byte-aligned base and row pitch.
void attention_fwd(const Tensor& qkv, Tensor& out, Tensor& lse, int64_t B, int64_t T, int64_t nh, int64_t hd, double scale, bool interleaved,
                   int64_t nkv) {
  if (nkv < 0) nkv = nh;
  const Call c{"attention_fwd", qkv.device()};
  rb::AttnDesc d;
  d.qkv = arg(c, qkv, "qkv", BF, {B * T, (nh + 2 * nkv) * hd}, 16); d.ld_qkv = qkv.stride(0);
  d.out = arg(c, out, "out", BF, {B * T, nh * hd}, 16); d.ld_out = out.stride(0);
  d.lse = arg<float>(c, lse, "lse", F32, {B * nh * T});
  d.B = (int)B; d.T = (int)T; d.nh = (int)nh; d.nkv = (int)nkv; d.hd = (int)hd; d.scale = (float)scale; d.interleaved = interleaved;
  c10::cuda::CUDAGuard guard(c.dev);
  rb::attention_fwd(d, cur_stream());
}
void attention_bwd(const Tensor& qkv, const Tensor& out, const Tensor& dout, const Tensor& lse, Tensor& delta, Tensor& dqkv, int64_t B,
                   int64_t T, int64_t nh, int64_t hd, double scale, const OptTensor& ds_workspace, bool interleaved, int64_t nkv) {
  if (nkv < 0) nkv = nh;
  const Call c{"attention_bwd", qkv.device()};
  rb::AttnBwdDesc d;
  d.qkv = arg(c, qkv, "qkv", BF, {B * T, (nh + 2 * nkv) * hd}, 16); d.ld_qkv = qkv.stride(0);
  d.out = arg(c, out, "out", BF, {B * T, nh * hd}, 16); d.ld_out = out.stride(0);
  d.dout = arg(c, dout, "dout", BF, {B * T, nh * hd}, 16); d.ld_dout = dout.stride(0);
  d.lse = arg<float>(c, lse, "lse", F32, {B * nh * T});
  d.delta = arg<float>(c, delta, "delta", F32, {B * nh * T});
  d.dqkv = arg(c, dqkv, "dqkv", BF, {B * T, (nh + 2 * nkv) * hd}, 16); d.ld_dqkv = dqkv.stride(0);
  d.ds_workspace = arg(c, ds_workspace, "ds_workspace", BF, {rb::attention_ds_workspace_elems((int)B, (int)T, (int)nh)});
  d.B = (int)B; d.T = (int)T; d.nh = (int)nh; d.nkv = (int)nkv; d.hd = (int)hd; d.scale = (float)scale; d.interleaved = interleaved;
  c10::cuda::CUDAGuard guard(c.dev);
  rb::attention_bwd(d, cur_stream());
}

// operand name of the bf16 rotary tables: rows are positions, pitch rotary_dim
constexpr const char* kCos = "cos (rotary table [pos, rotary_dim])";
constexpr const char* kSin = "sin (rotary table [pos, rotary_dim])";

void rope_inplace(Tensor& buf, int64_t T, int64_t n_rot_heads, int64_t hd, int64_t rotary_dim, const Tensor& cos, const Tensor& sin,
                  bool backward, int64_t pos0) {
  TORCH_CHECK(rotary_dim > 0 && rotary_dim <= hd, "rope_inplace: rotary_dim must be in (0, hd]");
  const Call c{"rope_inplace", buf.device()};
  // the scalar kernel (taken when the 16-byte one cannot run) moves element pairs with 4-byte accesses
  void* bp = arg(c, buf, "buf", BF, {0, n_rot_heads * hd}, 4);
  const void* cp = arg(c, cos, kCos, BF, {T + pos0, rotary_dim}, 4, {rotary_dim});
  const void* sp = arg(c, sin, kSin, BF, {T + pos0, rotary_dim}, 4, {rotary_dim});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::rope_inplace(bp, buf.stride(0), (int)buf.size(0), (int)T, (int)n_rot_heads, (int)hd, (int)rotary_dim, cp, sp, backward, (int)pos0,
                   cur_stream());
}

// dq [B, nh, T, hd]; dk, dv [B, nkv, T, hd] (nkv < 0 means nh), nh % nkv == 0 -> out [B*T, (nh + 2*nkv)*hd]
void rope_pack_bwd(const Tensor& dq, const Tensor& dk, const Tensor& dv, Tensor& out, int64_t rotary_dim, const Tensor& cos,
                   const Tensor& sin, int64_t pos0, int64_t nkv) {
  const Call c{"rope_pack_bwd", out.device()};
  const void* dqp = arg(c, dq, "dq", BF, {0, 0, 0, 0}, 16);
  const int64_t B = dq.size(0), nh = dq.size(1), T = dq.size(2), hd = dq.size(3);
  if (nkv < 0) nkv = nh;
  TORCH_CHECK(rotary_dim > 0 && rotary_dim <= hd, "rope_pack_bwd: rotary_dim must be in (0, hd]");
  const void* dkp = arg(c, dk, "dk", BF, {B, nkv, T, hd}, 16);
  const void* dvp = arg(c, dv, "dv", BF, {B, nkv, T, hd}, 16, dk.strides());  // dk and dv share the strides kB, kH, kT
  void* op = arg(c, out, "out", BF, {B * T, (nh + 2 * nkv) * hd}, 16);
  const void* cp = arg(c, cos, kCos, BF, {T + pos0, rotary_dim}, 16, {rotary_dim});
  const void* sp = arg(c, sin, kSin, BF, {T + pos0, rotary_dim}, 16, {rotary_dim});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::rope_pack_bwd(dqp, dkp, dvp, dq.stride(0), dq.stride(1), dq.stride(2), dk.stride(0), dk.stride(1), dk.stride(2), op, out.stride(0),
                    (int)B, (int)T, (int)nh, (int)nkv, (int)hd, (int)rotary_dim, cp, sp, (int)pos0, cur_stream());
}

void swiglu_fwd(const Tensor& gu, Tensor& h, const OptTensor& hd, const OptTensor& seed, int64_t key, double p, const OptTensor& q8,
                const OptTensor& q_inv_scale, const OptTensor& q_amax) {
  const Call c{"swiglu_fwd", h.device()};
  void* hp = arg(c, h, "h", BF, {0, 0}, 16);
  const int64_t M = h.size(0), F = h.size(1);
  const void* gp = arg(c, gu, "gu", BF, {M, 2 * F}, 16);
  void* hdp = arg(c, hd, "hd", BF, {M, F}, 16);
  const Dropout dr = dropout(c, seed, {key}, p, 1, 1);
  const rb::Fp8Out f8 = fp8_out(c, q8, q_inv_scale, q_amax, M, F);
  c10::cuda::CUDAGuard guard(c.dev);
  rb::swiglu_fwd(gp, gu.stride(0), hp, h.stride(0), (int)M, (int)F, hdp, hd.has_value() ? hd->stride(0) : 0, dr.seed, dr.keys[0],
                 dr.thr16, dr.inv_keep, f8, cur_stream());
}
void swiglu_bwd(const Tensor& dh, const Tensor& gu, Tensor& dgu) {
  const Call c{"swiglu_bwd", dh.device()};
  const void* dhp = arg(c, dh, "dh", BF, {0, 0}, 16);
  const int64_t M = dh.size(0), F = dh.size(1);
  const void* gp = arg(c, gu, "gu", BF, {M, 2 * F}, 16);
  void* dgp = arg(c, dgu, "dgu", BF, {M, 2 * F}, 16);
  c10::cuda::CUDAGuard guard(c.dev);
  rb::swiglu_bwd(dhp, dh.stride(0), gp, gu.stride(0), dgp, dgu.stride(0), (int)M, (int)F, cur_stream());
}

// ---------------------------------------------------------------------------------------------- block-scaled MXFP8
int64_t mx_sf_bytes(int64_t rows, int64_t k) { return rb::mx_sf_bytes(rows, k); }
int64_t pad128(int64_t n) { return (n + 127) / 128 * 128; }
// the quantisers load 4 bf16 (8 bytes) or, for the weight, 8 bf16 (16 bytes) and store 4 bytes of q per access
void mx_quantize_rows(const Tensor& x, Tensor& q, Tensor& sf) {
  const Call c{"mx_quantize_rows", x.device()};
  const void* xp = arg(c, x, "x", BF, {0, 0}, 8);
  const int64_t M = x.size(0), K = x.size(1);
  void* qp = arg(c, q, "q", at::kByte, {M, pad128(K)}, 4);
  void* sp = arg(c, sf, "sf", at::kByte, {rb::mx_sf_bytes(M, K)});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::mx_quantize_rows(xp, x.stride(0), qp, q.stride(0), sp, (int)M, (int)K, cur_stream());
}
void mx_quantize_weight_2d(const OptTensor& w, const OptTensor& delta, Tensor& q, Tensor& sf_fwd, Tensor& sf_bwd, int64_t N, int64_t K) {
  const Call c{"mx_quantize_weight_2d", q.device()};
  void* qp = arg(c, q, "q", at::kByte, {pad128(N), pad128(K)}, 4);
  void* fp = arg(c, sf_fwd, "sf_fwd", at::kByte, {rb::mx_sf_bytes(N, K)});
  void* bp = arg(c, sf_bwd, "sf_bwd", at::kByte, {rb::mx_sf_bytes(K, N)});
  const void* wp = arg(c, w, "w", BF, {N, K}, 16);
  const float* dp = arg<const float>(c, delta, "delta", F32, {N, K});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::mx_quantize_weight_2d(wp, w.has_value() ? w->stride(0) : 0, qp, fp, dp, delta.has_value() ? delta->stride(0) : 0, qp, q.stride(0), fp,
                            bp, (int)N, (int)K, cur_stream());
}
void mx_dequantize_weight(const Tensor& q, const Tensor& sf_fwd, Tensor& out) {
  const Call c{"mx_dequantize_weight", out.device()};
  void* op = arg(c, out, "out", BF, {0, 0}, 8);
  const int64_t N = out.size(0), K = out.size(1);
  const void* qp = arg(c, q, "q", at::kByte, {N, K}, 4);
  const void* fp = arg(c, sf_fwd, "sf_fwd", at::kByte, {rb::mx_sf_bytes(N, K)});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::mx_dequantize_weight(qp, q.stride(0), fp, op, out.stride(0), (int)N, (int)K, cur_stream());
}
void gemm_mx(const Tensor& a, const Tensor& sfa, const Tensor& b, const Tensor& sfb, Tensor& out, int64_t M, int64_t N, int64_t K, bool b_mn_major,
             const OptTensor& a2, const OptTensor& b2, const OptTensor& residual) {
  TORCH_CHECK(!a2.has_value() || b2.has_value(), "gemm_mx: a2 needs b2");
  const Call c{"gemm_mx", out.device()};
  rb::MxGemmDesc d;
  const int64_t Kpad = pad128(K);
  d.a = arg(c, a, "a", at::kByte, {M, Kpad}, 16); d.lda = a.stride(0);
  d.b = b_mn_major ? arg(c, b, "b", at::kByte, {Kpad, N}, 16) : arg(c, b, "b", at::kByte, {N, Kpad}, 16); d.ldb = b.stride(0);
  d.sfa = arg(c, sfa, "sfa", at::kByte, {rb::mx_sf_bytes(M, K)});
  d.sfb = arg(c, sfb, "sfb", at::kByte, {rb::mx_sf_bytes(N, K)});
  d.out = arg(c, out, "out", BF, {M, N}, 16); d.ldc = out.stride(0);
  d.b_mn_major = b_mn_major; d.M = (int)M; d.N = (int)N; d.K = (int)K;
  if (a2.has_value()) {
    d.a2 = arg(c, a2, "a2", BF, {M, 0}, 16); d.lda2 = a2->stride(0); d.K2 = (int)a2->size(1);
    d.b2 = arg(c, b2, "b2", BF, {N, d.K2}, 16); d.ldb2 = b2->stride(0);
  }
  d.residual = arg(c, residual, "residual", BF, {M, N}, 16); d.ldr = residual.has_value() ? residual->stride(0) : 0;
  c10::cuda::CUDAGuard guard(c.dev);
  rb::gemm_mx(d, cur_stream());
}

// ---------------------------------------------------------------------------------------------- GPT-NeoX / Pythia block
// y = LN(x; w, b).  Executor options: y2 = LN(x; w2, b2) from the same statistics, and dropout copies xd (of y, mask key `keys[0]`) /
// xd2 (of y2, `keys[1]`) with probability p from the device seed.
void layernorm_fwd(const Tensor& x, const Tensor& w, const OptTensor& b, Tensor& y, Tensor& mean, Tensor& rstd, double eps, const OptTensor& w2,
                   const OptTensor& b2, const OptTensor& y2, const OptTensor& xd, const OptTensor& xd2, const OptTensor& seed,
                   std::vector<int64_t> keys, double p) {
  TORCH_CHECK(y2.has_value() == w2.has_value(), "layernorm_fwd: y2 and w2 go together");
  TORCH_CHECK(!xd2.has_value() || y2.has_value(), "layernorm_fwd: xd2 needs y2");
  const bool copies = xd.has_value() || xd2.has_value();
  TORCH_CHECK(!copies || seed.has_value(), "layernorm_fwd: dropout copies need the seed");
  const Call c{"layernorm_fwd", x.device()};
  const void* xp = arg(c, x, "x", BF, {0, 0}, 16, {x.size(-1)});
  const int64_t M = x.size(0), H = x.size(1);
  const Dropout dr = dropout(c, seed, keys, p, copies ? 2 : 0, 2);
  rb::LnFwdOut n1, n2;
  n1.w = arg(c, w, "w", BF, {H}, 16); n1.b = arg(c, b, "b", BF, {H}, 16); n1.y = arg(c, y, "y", BF, {M * H}, 16);
  n1.xd = arg(c, xd, "xd", BF, {M * H}, 16);
  n2.w = arg(c, w2, "w2", BF, {H}, 16); n2.b = arg(c, b2, "b2", BF, {H}, 16); n2.y = arg(c, y2, "y2", BF, {M * H}, 16);
  n2.xd = arg(c, xd2, "xd2", BF, {M * H}, 16);
  n1.key = dr.keys[0]; n2.key = dr.keys[1];
  float* mp = arg<float>(c, mean, "mean", F32, {M});
  float* rp = arg<float>(c, rstd, "rstd", F32, {M});
  c10::cuda::CUDAGuard guard(c.dev);
  const bool ok = rb::layernorm_fwd_dual(xp, n1, n2, mp, rp, (int)M, (int)H, (float)eps, copies ? dr.ln() : rb::LnDrop{}, cur_stream());
  TORCH_CHECK(ok, "layernorm_fwd: hidden size must be a multiple of 8 and <= 4096");
}

// Module form: dx = LNᵀ(dy).  Executor form (any of dres / dy2 / dres_sum given): dx = dres + LNᵀ(dy) [+ LN2ᵀ(dy2)], γ / β gradients of
// both norms, dres_sum (and dres_sum2) += Σ rows of dres.  All fp32 gradients accumulate.
void layernorm_bwd(const Tensor& dy, const Tensor& x, const Tensor& w, const Tensor& mean, const Tensor& rstd, Tensor& dx, Tensor& dw,
                   const OptTensor& db, const OptTensor& dres, const OptTensor& dy2, const OptTensor& w2, const OptTensor& dw2,
                   const OptTensor& db2, const OptTensor& dres_sum, const OptTensor& dres_sum2) {
  TORCH_CHECK(dy2.has_value() == w2.has_value() && dy2.has_value() == dw2.has_value(), "layernorm_bwd: dy2, w2 and dw2 go together");
  TORCH_CHECK(!dres_sum.has_value() || dres.has_value(), "layernorm_bwd: dres_sum needs dres");
  TORCH_CHECK(!dres_sum2.has_value() || dres_sum.has_value(), "layernorm_bwd: dres_sum2 needs dres_sum");
  const Call c{"layernorm_bwd", x.device()};
  const void* xp = arg(c, x, "x", BF, {0, 0}, 16, {x.size(-1)});
  const int64_t M = x.size(0), H = x.size(1);
  const bool dual = dres.has_value() || dy2.has_value() || dres_sum.has_value();
  // the module form adds dw / db with 16-byte reductions, the executor form with scalar atomics
  const int64_t wgrad_align = dual ? 4 : 16;
  rb::LnBwdNorm n1, n2;
  n1.dy = arg(c, dy, "dy", BF, {M * H}, 16); n1.w = arg(c, w, "w", BF, {H}, 16);
  n1.dw = arg<float>(c, dw, "dw", F32, {H}, wgrad_align); n1.db = arg<float>(c, db, "db", F32, {H}, wgrad_align);
  n2.dy = arg(c, dy2, "dy2", BF, {M * H}, 16); n2.w = arg(c, w2, "w2", BF, {H}, 16);
  n2.dw = arg<float>(c, dw2, "dw2", F32, {H}); n2.db = arg<float>(c, db2, "db2", F32, {H});
  const float* mp = arg<const float>(c, mean, "mean", F32, {M});
  const float* rp = arg<const float>(c, rstd, "rstd", F32, {M});
  void* dxp = arg(c, dx, "dx", BF, {M * H}, 16);
  const void* drp = arg(c, dres, "dres", BF, {M * H}, 16);
  float* s1 = arg<float>(c, dres_sum, "dres_sum", F32, {H});
  float* s2 = arg<float>(c, dres_sum2, "dres_sum2", F32, {H});
  c10::cuda::CUDAGuard guard(c.dev);
  bool ok;
  if (!dual) {
    ok = rb::layernorm_bwd(n1.dy, xp, n1.w, mp, rp, dxp, n1.dw, n1.db, (int)M, (int)H, cur_stream());
  } else {
    Tensor total;  // Σ rows of dres, formed once when it goes to two outputs
    if (s2 != nullptr) total = at::empty({H}, x.options().dtype(F32));
    ok = rb::layernorm_bwd_dual(xp, mp, rp, n1, n2, drp, dxp, s1, s2, s2 != nullptr ? total.data_ptr<float>() : nullptr, (int)M, (int)H,
                                cur_stream());
  }
  TORCH_CHECK(ok, "layernorm_bwd: hidden size must be a multiple of 8 and <= 2048");
}
// a = GELU(z); xd (optional): dropout copy of a with mask key `key` (rows of z.size(-1) elements)
void gelu_fwd(const Tensor& z, Tensor& a, bool tanh_approx, const OptTensor& xd, const OptTensor& seed, int64_t key, double p) {
  TORCH_CHECK(!xd.has_value() || seed.has_value(), "gelu_fwd: the dropout copy needs the seed");
  const Call c{"gelu_fwd", z.device()};
  const void* zp = arg(c, z, "z", BF, {0}, 16);
  const int64_t n = z.numel();
  void* ap = arg(c, a, "a", BF, {n}, 16);
  void* xdp = arg(c, xd, "xd", BF, {n}, 16);
  const Dropout dr = dropout(c, seed, {key}, p, 1, 1);
  c10::cuda::CUDAGuard guard(c.dev);
  rb::gelu_fwd(zp, ap, n, tanh_approx, cur_stream(), xdp, (int)z.size(-1), dr.keys[0], xdp != nullptr ? dr.ln() : rb::LnDrop{});
}
// dz = da · GELU'(z); dbias (optional, fp32 [N]) += Σ rows of dz
void gelu_bwd(const Tensor& da, const Tensor& z, Tensor& dz, bool tanh_approx, const OptTensor& dbias) {
  const Call c{"gelu_bwd", z.device()};
  const void* zp = arg(c, z, "z", BF, {0}, 16);
  const int64_t n = z.numel(), N = z.size(-1);
  const void* dap = arg(c, da, "da", BF, {n}, 16);
  void* dzp = arg(c, dz, "dz", BF, {n}, 16);
  float* bp = arg<float>(c, dbias, "dbias", F32, {N}, 16);
  c10::cuda::CUDAGuard guard(c.dev);
  if (bp != nullptr) rb::gelu_bwd_colsum(dap, zp, dzp, bp, (int)(n / N), (int)N, tanh_approx, cur_stream());
  else rb::gelu_bwd(dap, zp, dzp, n, tanh_approx, cur_stream());
}
// out (fp32 [N]) += Σ rows of x [M, N]
void colsum(const Tensor& x, Tensor& out) {
  const Call c{"colsum", x.device()};
  const void* xp = arg(c, x, "x", BF, {0, 0}, 16, {x.size(-1)});
  float* op = arg<float>(c, out, "out", F32, {x.size(1)}, 16);
  c10::cuda::CUDAGuard guard(c.dev);
  rb::colsum(xp, op, (int)x.size(0), (int)x.size(1), cur_stream());
}
void neox_rope(Tensor& qkv, int64_t T, int64_t nh, int64_t hd, int64_t rot, const Tensor& cos, const Tensor& sin, int64_t pos0, bool inverse) {
  const Call c{"neox_rope", qkv.device()};
  void* qp = arg(c, qkv, "qkv", BF, {0, nh * 3 * hd});
  const float* cp = arg<const float>(c, cos, "cos (rotary table [pos, rot])", F32, {T + pos0, rot}, 1, {rot});
  const float* sp = arg<const float>(c, sin, "sin (rotary table [pos, rot])", F32, {T + pos0, rot}, 1, {rot});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::neox_rope(qp, qkv.stride(0), qkv.size(0), (int)T, (int)nh, (int)hd, (int)rot, cp, sp, (int)pos0, inverse, cur_stream());
}

void embedding_fwd(const Tensor& ids, const Tensor& table, Tensor& out) {
  const Call c{"embedding_fwd", out.device()};
  const int64_t* ip = arg<const int64_t>(c, ids, "ids", at::kLong, {0});
  const void* tp = arg(c, table, "table", BF, {0, 0}, 16, {table.size(-1)});
  const int64_t M = ids.numel(), H = table.size(1);
  void* op = arg(c, out, "out", BF, {M * H}, 16);
  c10::cuda::CUDAGuard guard(c.dev);
  rb::embedding_fwd(ip, tp, op, (int)M, (int)H, cur_stream());
}
void embedding_bwd(const Tensor& ids, const Tensor& dout, Tensor& dtable, int64_t padding_idx) {
  const Call c{"embedding_bwd", dout.device()};
  const int64_t* ip = arg<const int64_t>(c, ids, "ids", at::kLong, {0});
  float* tp = arg<float>(c, dtable, "dtable", F32, {0, 0}, 1, {dtable.size(-1)});
  const int64_t M = ids.numel(), H = dtable.size(1);
  const void* dp = arg(c, dout, "dout", BF, {M * H}, 16);
  c10::cuda::CUDAGuard guard(c.dev);
  rb::embedding_bwd(ip, dp, tp, (int)M, (int)H, padding_idx, cur_stream());
}
void embedding_bwd_sorted(const Tensor& sorted_ids, const Tensor& perm, const Tensor& dout, Tensor& dtable, int64_t padding_idx) {
  const Call c{"embedding_bwd_sorted", dout.device()};
  const int64_t* ip = arg<const int64_t>(c, sorted_ids, "sorted_ids", at::kLong, {0});
  const int64_t M = sorted_ids.numel();
  const int64_t* pp = arg<const int64_t>(c, perm, "perm", at::kLong, {M});
  float* tp = arg<float>(c, dtable, "dtable", F32, {0, 0}, 16, {dtable.size(-1)});  // 16-byte read-modify-writes
  const int64_t H = dtable.size(1);
  const void* dp = arg(c, dout, "dout", BF, {M * H}, 16);
  c10::cuda::CUDAGuard guard(c.dev);
  rb::embedding_bwd_sorted(ip, pp, dp, tp, (int)M, (int)H, padding_idx, cur_stream());
}

void cross_entropy_fwd_bwd(Tensor& logits, const Tensor& labels, int64_t V, double grad_scale, int64_t ignore_index, Tensor& loss_sum,
                           Tensor& count) {
  const Call c{"cross_entropy_fwd_bwd", logits.device()};
  void* lp = arg(c, logits, "logits", BF, {0, V}, 16);
  const int64_t M = logits.size(0);
  const int64_t* yp = arg<const int64_t>(c, labels, "labels", at::kLong, {M});
  float* sp = arg<float>(c, loss_sum, "loss_sum", F32, {1});
  float* np = arg<float>(c, count, "count", F32, {1});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::cross_entropy_fwd_bwd(lp, logits.stride(0), yp, (int)M, (int)V, (float)grad_scale, ignore_index, sp, np, cur_stream());
}

void transpose(const Tensor& in, Tensor& out) {
  const Call c{"transpose", in.device()};
  const void* ip = arg(c, in, "in", BF, {0, 0});
  const int64_t R = in.size(0), C = in.size(1);
  void* op = arg(c, out, "out", BF, {C, R});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::transpose_bf16(ip, in.stride(0), op, out.stride(0), (int)R, (int)C, cur_stream());
}
void add(const Tensor& a, const Tensor& b, Tensor& out) {
  const Call c{"add", a.device()};
  const void* ap = arg(c, a, "a", BF, {0}, 16);
  const int64_t n = a.numel();
  const void* bp = arg(c, b, "b", BF, {n}, 16);
  void* op = arg(c, out, "out", BF, {n}, 16);
  c10::cuda::CUDAGuard guard(c.dev);
  rb::add_bf16(ap, bp, op, n, cur_stream());
}
void cast_f32_to_bf16(const Tensor& in, Tensor& out, double scale) {
  const Call c{"cast_f32_to_bf16", in.device()};
  const float* ip = arg<const float>(c, in, "in", F32, {0}, 16);
  void* op = arg(c, out, "out", BF, {in.numel()}, 16);
  c10::cuda::CUDAGuard guard(c.dev);
  rb::cast_f32_to_bf16(ip, op, in.numel(), (float)scale, cur_stream());
}
void fill_uniform_hash(Tensor& out, int64_t seed, double bound) {
  const Call c{"fill_uniform_hash", out.device()};
  void* op = arg(c, out, "out", BF, {0, 0});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::fill_uniform_hash(op, (int)out.size(0), (int)out.size(1), out.stride(0), (uint32_t)seed, (float)bound, cur_stream());
}
void seed_advance(Tensor& seed) {
  const Call c{"seed_advance", seed.device()};
  uint32_t* sp = arg<uint32_t>(c, seed, "seed", at::kInt, {1});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::seed_advance(sp, cur_stream());
}

// bf16 or fp32 flat buffers: the dtype is the tensor's own, and must be one of the two
at::ScalarType bf16_or_f32(const Tensor& t) { return t.scalar_type() == F32 ? F32 : BF; }

void adamw_flat(Tensor& p, const Tensor& g, Tensor& m, Tensor& v, double lr, double b1, double b2, double eps, double wd, int64_t step,
                const OptTensor& grad_scale, double grad_scale_host, const OptTensor& skip, const OptTensor& step_dev) {
  const Call c{"adamw_flat", p.device()};
  void* pp = arg(c, p, "param", BF, {0}, 16);
  const int64_t n = p.numel();
  const auto gt = bf16_or_f32(g), st = bf16_or_f32(m);
  const void* gp = arg(c, g, "grad", gt, {n});
  void* mp = arg(c, m, "exp_avg", st, {n});
  void* vp = arg(c, v, "exp_avg_sq", st, {n});
  const float* gsp = arg<const float>(c, grad_scale, "grad_scale", F32, {1});
  const float* skp = arg<const float>(c, skip, "skip", F32, {1});
  const float* sdp = arg<const float>(c, step_dev, "step_dev", F32, {1});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::adamw_flat(pp, gp, gt == F32, mp, vp, st == F32, n, (float)lr, (float)b1, (float)b2, (float)eps, (float)wd, (int)step, gsp,
                 (float)grad_scale_host, skp, sdp, cur_stream());
}
void sumsq(const Tensor& x, Tensor& out) {
  const Call c{"sumsq", x.device()};
  const auto xt = bf16_or_f32(x);
  const void* xp = arg(c, x, "x", xt, {0});
  float* op = arg<float>(c, out, "out", F32, {1});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::sumsq(xp, xt == F32, x.numel(), op, cur_stream());
}
void random_prune(Tensor& x, double ratio, int64_t seed, int64_t col_offset) {
  const Call c{"random_prune", x.device()};
  const auto xt = bf16_or_f32(x);
  void* xp = arg(c, x, "x", xt, {0});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::random_prune(xp, xt == F32, x.numel(), (float)ratio, (uint32_t)seed, col_offset, cur_stream());
}
void magnitude_prune(Tensor& x, double ratio, Tensor& workspace, Tensor& thr) {
  const Call c{"magnitude_prune", x.device()};
  const auto xt = bf16_or_f32(x);
  void* xp = arg(c, x, "x", xt, {0});
  void* wp = arg(c, workspace, "workspace", at::kByte, {(int64_t)rb::magnitude_quantile_workspace_bytes()});
  float* tp = arg<float>(c, thr, "thr", F32, {1});
  c10::cuda::CUDAGuard guard(c.dev);
  rb::magnitude_quantile(xp, xt == F32, x.numel(), (float)ratio, tp, wp, cur_stream());
  rb::threshold_prune(xp, xt == F32, x.numel(), tp, cur_stream());
}

// ---------------------------------------------------------------------------------------------- NVLink collectives
// The peer and multicast addresses are raw integers from the symmetric-memory allocator and cannot be checked here; the
// tensor arguments are.
rb::PeerPtrs peer_ptrs(const std::vector<int64_t>& v) {
  TORCH_CHECK((int)v.size() <= rb::kMaxPeers, "at most 8 peers");
  rb::PeerPtrs p;
  for (int i = 0; i < rb::kMaxPeers; ++i) p.ptr[i] = i < (int)v.size() ? reinterpret_cast<void*>(v[i]) : nullptr;
  return p;
}
rb::CommCtx comm_ctx(const Call& c, const std::vector<int64_t>& flag_ptrs, int64_t rank, int64_t world, Tensor& local_go) {
  rb::CommCtx x;
  x.rank = (int)rank; x.world = (int)world; x.flags = peer_ptrs(flag_ptrs);
  x.local_go = arg<uint32_t>(c, local_go, "local_go", at::kInt, {2});
  return x;
}
void comm_barrier(std::vector<int64_t> flag_ptrs, int64_t rank, int64_t world, Tensor& local_go, int64_t set, int64_t epoch) {
  const Call c{"comm_barrier", local_go.device()};
  const rb::CommCtx x = comm_ctx(c, flag_ptrs, rank, world, local_go);
  c10::cuda::CUDAGuard guard(c.dev);
  rb::xgpu_barrier(x, (int)set, (uint32_t)epoch, cur_stream());
}
void comm_allreduce_bf16(std::vector<int64_t> flag_ptrs, int64_t rank, int64_t world, Tensor& local_go, std::vector<int64_t> buf_ptrs,
                         int64_t mc_ptr, int64_t off_elems, int64_t n, int64_t epoch, int64_t max_blocks) {
  const Call c{"comm_allreduce_bf16", local_go.device()};
  const rb::CommCtx x = comm_ctx(c, flag_ptrs, rank, world, local_go);
  c10::cuda::CUDAGuard guard(c.dev);
  rb::allreduce_bf16(x, peer_ptrs(buf_ptrs), reinterpret_cast<void*>(mc_ptr), off_elems, n, (uint32_t)epoch, (int)max_blocks, cur_stream());
}
void comm_fused_update(std::vector<int64_t> flag_ptrs, int64_t rank, int64_t world, Tensor& local_go, const OptTensor& grads_f32,
                       std::vector<int64_t> grad_ptrs, int64_t grad_mc, Tensor& gred, std::vector<int64_t> param_ptrs, int64_t param_mc,
                       Tensor& exp_avg, Tensor& exp_avg_sq, int64_t n, double lr, double b1, double b2, double eps, double wd, int64_t step,
                       double max_norm, const OptTensor& skip, Tensor& norm_out, Tensor& scratch, int64_t epoch, int64_t max_blocks,
                       const OptTensor& step_dev, const OptTensor& loss_in, const OptTensor& loss_out) {
  TORCH_CHECK(world >= 1, "comm_fused_update: world must be positive");
  const Call c{"comm_fused_update", local_go.device()};
  const rb::CommCtx x = comm_ctx(c, flag_ptrs, rank, world, local_go);
  const int64_t shard = (n + world - 1) / world;  // this rank's slice of the reduced gradient and of the moments
  rb::FusedUpdateArgs a;
  a.grads_f32 = arg<float>(c, grads_f32, "grads_f32", F32, {n});
  a.grad_bufs = peer_ptrs(grad_ptrs); a.grad_mc = reinterpret_cast<void*>(grad_mc);
  a.gred = arg<float>(c, gred, "gred", F32, {shard});
  a.param_bufs = peer_ptrs(param_ptrs); a.param_mc = reinterpret_cast<void*>(param_mc);
  a.exp_avg = arg(c, exp_avg, "exp_avg", BF, {shard});
  a.exp_avg_sq = arg(c, exp_avg_sq, "exp_avg_sq", BF, {shard});
  a.n = n; a.lr = (float)lr; a.beta1 = (float)b1; a.beta2 = (float)b2; a.eps = (float)eps; a.weight_decay = (float)wd;
  a.step = (int)step; a.step_dev = arg<const float>(c, step_dev, "step_dev", F32, {1}); a.max_norm = (float)max_norm;
  a.inv_world = 1.0f / (float)world;
  a.loss_in = arg<const float>(c, loss_in, "loss_in", F32, {1}); a.loss_out = arg<float>(c, loss_out, "loss_out", F32, {1});
  a.skip = arg<const float>(c, skip, "skip", F32, {1});
  a.norm_out = arg<float>(c, norm_out, "norm_out", F32, {1});
  a.sq_accum = arg<float>(c, scratch, "scratch", F32, {3});
  a.max_blocks = (int)max_blocks;
  c10::cuda::CUDAGuard guard(c.dev);
  rb::fused_update(x, a, (uint32_t)epoch, cur_stream());
}

long long launch_count() { return rb::g_launch_count; }
void reset_launch_count() { rb::g_launch_count = 0; }

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "relora_b200 sm_90a kernels";
  m.def("gemm", &gemm, "wgmma GEMM with fused LoRA K-extension");
  m.def("gemm_clear_descriptor_cache", &rb::gemm_clear_descriptor_cache);
  // host-side schedule of one gemm call (no launch): (block_n, tma_store, dynamic shared memory bytes, CTA pairs); sms: the
  // SM count of the tile-width rule (0: this device's)
  m.def("gemm_plan", [](int64_t block_n, bool out_f32, int64_t out_addr, int64_t ldc, int64_t n, int64_t split_k, int64_t m,
                        int64_t m_per_group, int64_t pair, int64_t k, int64_t n_per_group, bool accumulate, int64_t sms) {
    rb::GemmDesc d;
    d.block_n = (int)block_n; d.out_f32 = out_f32; d.out = reinterpret_cast<void*>(out_addr); d.ldc = ldc; d.N = (int)n;
    d.M = (int)m; d.m_per_group = (int)m_per_group; d.pair = (int)pair; d.K1 = (int)k;
    d.n_per_group = (int)n_per_group; d.accumulate = accumulate; d.split_k = (int)split_k;
    const int bn = rb::gemm_block_n(d, (int)sms);
    return py::make_tuple(bn, rb::gemm_uses_tma_store(d, bn, (int)split_k), rb::gemm_smem_bytes(bn), rb::gemm_pairs(d, bn));
  }, py::arg("block_n"), py::arg("out_f32"), py::arg("out_addr"), py::arg("ldc"), py::arg("n"), py::arg("split_k"),
     py::arg("m") = 0, py::arg("m_per_group") = 0, py::arg("pair") = -1, py::arg("k") = 0, py::arg("n_per_group") = 0,
     py::arg("accumulate") = false, py::arg("sms") = 0);
  // (CTA pairs, TMA-store epilogue) of one lora_dx call with G = 1 and rank r
  m.def("lora_dx_plan", [](int64_t m, int64_t n, int64_t pair, int64_t kb, int64_t r) {
    rb::LoraDxDesc d;
    d.M = (int)m; d.N = (int)n; d.pair = (int)pair; d.Kb = (int)kb; d.r = (int)r;
    return py::make_tuple(rb::lora_dx_pairs(d), rb::lora_dx_uses_tma_store(d));
  }, py::arg("m"), py::arg("n"), py::arg("pair") = -1, py::arg("kb") = 0, py::arg("r") = 128);
  m.def("rmsnorm_fwd", &rmsnorm_fwd, py::arg("x"), py::arg("w"), py::arg("y"), py::arg("rstd"), py::arg("eps"), py::arg("xd"), py::arg("seed"),
        py::arg("keys"), py::arg("p"), py::arg("q8") = py::none(), py::arg("q_inv_scale") = py::none(), py::arg("q_amax") = py::none());
  m.def("rmsnorm_bwd", &rmsnorm_bwd);
  m.def("rmsnorm_bwd_ws_blocks", &rb::rmsnorm_bwd_ws_blocks);
  m.def("dropout_expand", &dropout_expand, py::arg("x"), py::arg("xd"), py::arg("seed"), py::arg("keys"), py::arg("p"), py::arg("q8") = py::none(),
        py::arg("q_inv_scale") = py::none(), py::arg("q_amax") = py::none());
  m.def("dropout_combine", &dropout_combine);
  m.def("fp8_quantize_weight", &fp8_quantize_weight, py::arg("w"), py::arg("w8"), py::arg("scratch"), py::arg("scale"), py::arg("inv_scale"),
        py::arg("w8t") = py::none());
  m.def("fp8_quantize_act", &fp8_quantize_act, py::arg("x"), py::arg("x8"), py::arg("inv_scale"), py::arg("amax_cur") = py::none(), py::arg("e5m2") = false);
  m.def("fp8_prep", &fp8_prep, py::arg("state"), py::arg("w_scale"), py::arg("inv_sx"), py::arg("alpha_main"), py::arg("alpha_inv"), py::arg("margin"),
        py::arg("n_e4m3") = -1);
  m.def("attention_smem_bytes", [](int64_t hd) { return rb::attention_smem_bytes((int)hd); });
  m.def("attention_fwd", &attention_fwd, py::arg("qkv"), py::arg("out"), py::arg("lse"), py::arg("B"), py::arg("T"), py::arg("nh"), py::arg("hd"),
        py::arg("scale"), py::arg("interleaved") = false, py::arg("nkv") = -1);
  m.def("attention_bwd", &attention_bwd, py::arg("qkv"), py::arg("out"), py::arg("dout"), py::arg("lse"), py::arg("delta"), py::arg("dqkv"),
        py::arg("B"), py::arg("T"), py::arg("nh"), py::arg("hd"), py::arg("scale"), py::arg("ds_workspace") = py::none(),
        py::arg("interleaved") = false, py::arg("nkv") = -1);
  m.def("attention_ds_workspace_elems", &rb::attention_ds_workspace_elems);
  m.def("lora_dx", &lora_dx, py::arg("dy"), py::arg("w"), py::arg("du"), py::arg("a"), py::arg("out"), py::arg("seed"), py::arg("keys"),
        py::arg("p"), py::arg("base") = py::none(), py::arg("pair") = -1, py::arg("block_n") = 0);
  m.def("rope_inplace", &rope_inplace);
  m.def("rope_pack_bwd", &rope_pack_bwd, py::arg("dq"), py::arg("dk"), py::arg("dv"), py::arg("out"), py::arg("rotary_dim"), py::arg("cos"),
        py::arg("sin"), py::arg("pos0"), py::arg("nkv") = -1);
  m.def("swiglu_fwd", &swiglu_fwd, py::arg("gu"), py::arg("h"), py::arg("hd") = py::none(), py::arg("seed") = py::none(),
        py::arg("key") = 0, py::arg("p") = 0.0, py::arg("q8") = py::none(), py::arg("q_inv_scale") = py::none(), py::arg("q_amax") = py::none());
  m.def("swiglu_bwd", &swiglu_bwd);
  m.def("mx_sf_bytes", &mx_sf_bytes);
  m.def("mx_quantize_rows", &mx_quantize_rows);
  m.def("mx_quantize_weight_2d", &mx_quantize_weight_2d);
  m.def("mx_dequantize_weight", &mx_dequantize_weight);
  m.def("gemm_mx", &gemm_mx, py::arg("a"), py::arg("sfa"), py::arg("b"), py::arg("sfb"), py::arg("out"), py::arg("M"), py::arg("N"), py::arg("K"),
        py::arg("b_mn_major") = false, py::arg("a2") = py::none(), py::arg("b2") = py::none(), py::arg("residual") = py::none());
  m.def("layernorm_fwd", &layernorm_fwd, py::arg("x"), py::arg("w"), py::arg("b"), py::arg("y"), py::arg("mean"), py::arg("rstd"), py::arg("eps"),
        py::arg("w2") = py::none(), py::arg("b2") = py::none(), py::arg("y2") = py::none(), py::arg("xd") = py::none(), py::arg("xd2") = py::none(),
        py::arg("seed") = py::none(), py::arg("keys") = std::vector<int64_t>{}, py::arg("p") = 0.0);
  m.def("layernorm_bwd", &layernorm_bwd, py::arg("dy"), py::arg("x"), py::arg("w"), py::arg("mean"), py::arg("rstd"), py::arg("dx"), py::arg("dw"),
        py::arg("db"), py::arg("dres") = py::none(), py::arg("dy2") = py::none(), py::arg("w2") = py::none(), py::arg("dw2") = py::none(),
        py::arg("db2") = py::none(), py::arg("dres_sum") = py::none(), py::arg("dres_sum2") = py::none());
  m.def("gelu_fwd", &gelu_fwd, py::arg("z"), py::arg("a"), py::arg("tanh_approx"), py::arg("xd") = py::none(), py::arg("seed") = py::none(),
        py::arg("key") = 0, py::arg("p") = 0.0);
  m.def("gelu_bwd", &gelu_bwd, py::arg("da"), py::arg("z"), py::arg("dz"), py::arg("tanh_approx"), py::arg("dbias") = py::none());
  m.def("colsum", &colsum);
  m.def("neox_rope", &neox_rope);
  m.def("embedding_fwd", &embedding_fwd);
  m.def("embedding_bwd", &embedding_bwd);
  m.def("embedding_bwd_sorted", &embedding_bwd_sorted);
  m.def("cross_entropy_fwd_bwd", &cross_entropy_fwd_bwd);
  m.def("transpose", &transpose);
  m.def("add", &add);
  m.def("cast_f32_to_bf16", &cast_f32_to_bf16);
  m.def("fill_uniform_hash", &fill_uniform_hash);
  m.def("seed_advance", &seed_advance);
  m.def("adamw_flat", &adamw_flat);
  m.def("sumsq", &sumsq);
  m.def("random_prune", &random_prune);
  m.def("magnitude_prune", &magnitude_prune);
  m.def("quantile_workspace_bytes", &rb::magnitude_quantile_workspace_bytes);
  m.def("comm_barrier", &comm_barrier);
  m.def("comm_allreduce_bf16", &comm_allreduce_bf16);
  m.def("comm_fused_update", &comm_fused_update);
  m.def("launch_count", &launch_count);
  m.def("reset_launch_count", &reset_launch_count);
}
