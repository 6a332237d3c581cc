"""Every binding refuses, on the host and before any launch, a tensor operand that does not cover the extent its kernel takes
from the other arguments, or that has the wrong dtype; then the valid call runs.

Each case is one valid call on small shapes.  Every tensor sits at the start of a larger allocation, so the short views
(one row short, one column short) and the wider-dtype copies stay inside live, aligned device memory even if a check were
missing.  A refusal must name the binding and the operand, launch nothing and leave every allocation bit-for-bit unchanged."""
import pytest
import torch

BF, F32, F64, I32, I64, U8 = torch.bfloat16, torch.float32, torch.float64, torch.int32, torch.int64, torch.uint8
WIDER = {BF: F32, F32: F64, I32: I64, I64: F64, U8: torch.int16}

# bindings that take no tensor, or only raw peer addresses next to their tensors (comm_*: exercised by the multi-GPU tests)
EXEMPT = {
    "gemm_clear_descriptor_cache": "drops cached tensor maps, takes no tensor",
    "gemm_plan": "host-side schedule query",
    "lora_dx_plan": "host-side schedule query",
    "rmsnorm_bwd_ws_blocks": "size query",
    "attention_smem_bytes": "size query",
    "attention_ds_workspace_elems": "size query",
    "mx_sf_bytes": "size query",
    "quantile_workspace_bytes": "size query",
    "launch_count": "launch counter",
    "reset_launch_count": "launch counter",
    "comm_barrier": "peer flags are raw addresses; needs peers",
    "comm_allreduce_bf16": "peer buffers are raw addresses; needs peers",
    "comm_fused_update": "peer buffers are raw addresses; needs peers",
}


class Op:
    """A tensor operand: `name` as the binding reports it, its shape and dtype, row-major with a padded row pitch
    (`pitched`) or contiguous, and the refusals to probe: r(ow short), c(olumn short), d(type)."""

    def __init__(self, name, shape, dtype=BF, pitched=False, probe="rcd", init=None, wrong=None):
        self.name, self.shape, self.dtype, self.pitched, self.init = name, tuple(shape), dtype, pitched, init
        self.probe = probe if len(self.shape) > 1 else probe.replace("c", "")
        self.wrong = wrong or WIDER[dtype]


def _rows(n):
    return lambda s, d: torch.randint(0, n, s, device="cuda").to(d)


def _const(v):
    return lambda s, d: torch.full(s, v, device="cuda").to(d)


def _sorted(n):
    return lambda s, d: torch.randint(0, n, s, device="cuda").sort().values.to(d)


M, H, N, K, V = 128, 256, 256, 128, 512
SEED = Op("seed", (1,), I32, init=_const(7))


def _gemm(a1, b1, out, M, N, K1, *, a2=None, b2=None, K2=0, a1_mn=False, b1_mn=False, n_per_group=0, a1_group_kofs=0, residual=None,
          accumulate=False, m_per_group=0, b1_mn_ofs_per_mgroup=0, bias=None, fp8=0, alpha_dev=None):
    """A gemm call in the binding's positional order (it declares no keywords)."""
    return ["gemm", a1, b1, out, M, N, K1, a2, b2, K2, a1_mn, b1_mn, n_per_group, a1_group_kofs, 0, residual, 1.0, accumulate, 0, 1, 0, False,
            m_per_group, b1_mn_ofs_per_mgroup, bias, -1, fp8, alpha_dev]


def _gemm_forms():
    """The footprint forms of gemm_operand_extents: K-major bf16 with the LoRA operands, MN-major B1, per-group K windows of
    A1, per-M-group offsets of B1 (stacked weight gradients), and fp8 bytes."""
    out = lambda *shape, **kw: Op("out", shape, pitched=True, probe="", **kw)  # noqa: E731
    Ng, r = 128, 64
    return {
        "gemm": _gemm(Op("a1", (M, K), pitched=True), Op("b1", (N, K), pitched=True), Op("out", (M, N), pitched=True, wrong=F64), M, N, K,
                      a2=Op("a2", (M, 64), pitched=True), b2=Op("b2", (N, 64), pitched=True), K2=64,
                      residual=Op("residual", (M, N), pitched=True), bias=Op("bias", (N,)), alpha_dev=Op("alpha_dev", (1,), F32, init=_const(1.0))),
        "gemm-mn_major": _gemm(Op("a1", (M, K), pitched=True, probe=""), Op("b1", (K, N), pitched=True, probe="rc"), out(M, N), M, N, K,
                               b1_mn=True),
        "gemm-k_windows": _gemm(Op("a1", (M, 2 * K), pitched=True, probe="rc"), Op("b1", (N, K), pitched=True, probe=""), out(M, N), M, N, K,
                                n_per_group=N // 2, a1_group_kofs=K),
        "gemm-m_groups": _gemm(Op("a1", (K, 2 * Ng), pitched=True, probe=""), Op("b1", (K, 2 * r), pitched=True, probe="rc"),
                               out(2 * Ng, r, dtype=F32), 2 * Ng, r, K, a1_mn=True, b1_mn=True, accumulate=True, m_per_group=Ng,
                               b1_mn_ofs_per_mgroup=r),
        "gemm-fp8": _gemm(Op("a1", (M, K), U8, pitched=True, init=_const(0)), Op("b1", (N, K), U8, pitched=True, probe="", init=_const(0)),
                          out(M, N), M, N, K, fp8=1),
    }


def _lora_dx():
    return ["lora_dx", Op("dy", (M, 128), pitched=True, probe="rd"), Op("w", (128, N), pitched=True), Op("du", (M, 64), pitched=True, probe="d"),
            Op("a", (64, N), pitched=True, probe="rd"), Op("out", (M, N), pitched=True), SEED, [3], 0.1, None, -1]


def _attention_bwd(C):
    B, T, nh, hd = 1, 128, 2, 64
    ws = C.attention_ds_workspace_elems(B, T, nh)
    return ["attention_bwd", Op("qkv", (B * T, 3 * nh * hd), pitched=True), Op("out", (B * T, nh * hd), pitched=True),
            Op("dout", (B * T, nh * hd), pitched=True), Op("lse", (B * nh * T,), F32), Op("delta", (B * nh * T,), F32),
            Op("dqkv", (B * T, 3 * nh * hd), pitched=True), B, T, nh, hd, 0.125, Op("ds_workspace", (ws,)), False, -1]


def _mx(C):
    sf = C.mx_sf_bytes
    return {
        "mx_quantize_rows": ["mx_quantize_rows", Op("x", (M, K), pitched=True, probe="d"), Op("q", (M, K), U8, pitched=True),
                             Op("sf", (sf(M, K),), U8)],
        "mx_quantize_weight_2d": ["mx_quantize_weight_2d", Op("w", (N, K), pitched=True), None, Op("q", (N, K), U8, pitched=True),
                                  Op("sf_fwd", (sf(N, K),), U8), Op("sf_bwd", (sf(K, N),), U8), N, K],
        "mx_dequantize_weight": ["mx_dequantize_weight", Op("q", (N, K), U8, pitched=True, init=_const(0)), Op("sf_fwd", (sf(N, K),), U8, init=_const(127)),
                                 Op("out", (N, K), pitched=True, probe="d")],
        "gemm_mx": ["gemm_mx", Op("a", (M, K), U8, pitched=True, init=_const(0)), Op("sfa", (sf(M, K),), U8, init=_const(127)),
                    Op("b", (N, K), U8, pitched=True, init=_const(0)), Op("sfb", (sf(N, K),), U8, init=_const(127)),
                    Op("out", (M, N), pitched=True), M, N, K, False, Op("a2", (M, 64), pitched=True, probe="rd"),
                    Op("b2", (N, 64), pitched=True), Op("residual", (M, N), pitched=True)],
    }


def _cases(C):
    n, T, nh, hd = 4096, 64, 2, 64
    cos = lambda rot, dt=BF: Op("cos", (T, rot), dt)  # noqa: E731
    sin = lambda rot, dt=BF: Op("sin", (T, rot), dt)  # noqa: E731
    return {
        **_gemm_forms(),
        "rmsnorm_fwd": ["rmsnorm_fwd", Op("x", (M, H), probe="d"), Op("w", (H,)), Op("y", (M, H)), Op("rstd", (M,), F32), 1e-6,
                        Op("xd", (M, 2 * H)), SEED, [1, 2], 0.1],
        "rmsnorm_bwd": ["rmsnorm_bwd", Op("dy", (M, H)), Op("x", (M, H), probe="d"), Op("w", (H,)), Op("rstd", (M,), F32, init=_const(1.0)),
                        None, Op("dx", (M, H)), Op("dw", (H,), F32), None, None],
        "dropout_expand": ["dropout_expand", Op("x", (M, H), probe="d"), Op("xd", (M, 2 * H)), SEED, [1, 2], 0.1],
        "dropout_combine": ["dropout_combine", Op("base", (M, H)), Op("parts", (M, 2 * H), pitched=True), Op("out", (M, H), probe="d"), SEED,
                            [1, 2], 0.1],
        "fp8_quantize_weight": ["fp8_quantize_weight", Op("w", (N, K), pitched=True, probe="d"), Op("w8", (N, K), U8, pitched=True),
                                Op("scratch", (1,), F32), Op("scale", (1,), F32), Op("inv_scale", (1,), F32),
                                Op("w8t", (K, N), U8, pitched=True)],
        "fp8_quantize_act": ["fp8_quantize_act", Op("x", (M, K), pitched=True, probe="d"), Op("x8", (M, K), U8, pitched=True),
                             Op("inv_scale", (1,), F32, init=_const(1.0)), Op("amax_cur", (1,), F32), False],
        "fp8_prep": ["fp8_prep", Op("state", (8,), F32, init=_const(1.0)), Op("w_scale", (4,), F32, probe="d", init=_const(1.0)),
                     Op("inv_sx", (4,), F32), Op("alpha_main", (4,), F32), Op("alpha_inv", (4,), F32), 0.0, -1],
        "lora_dx": _lora_dx(),
        "attention_fwd": ["attention_fwd", Op("qkv", (T, 3 * nh * hd), pitched=True), Op("out", (T, nh * hd), pitched=True),
                          Op("lse", (nh * T,), F32), 1, T, nh, hd, 0.125, False, -1],
        "attention_bwd": _attention_bwd(C),
        "rope_inplace": ["rope_inplace", Op("buf", (T, 2 * nh * hd), pitched=True, probe="cd"), T, 2 * nh, hd, hd, cos(hd), sin(hd), False, 0],
        "rope_pack_bwd": ["rope_pack_bwd", Op("dq", (2, nh, T, hd), probe="d"), Op("dk", (2, nh, T, hd)), Op("dv", (2, nh, T, hd)),
                          Op("out", (2 * T, 3 * nh * hd), pitched=True), hd, cos(hd), sin(hd), 0, -1],
        "swiglu_fwd": ["swiglu_fwd", Op("gu", (M, 2 * H), pitched=True), Op("h", (M, H), pitched=True, probe="d"),
                       Op("hd", (M, H), pitched=True), SEED, 1, 0.1],
        "swiglu_bwd": ["swiglu_bwd", Op("dh", (M, H), pitched=True, probe="d"), Op("gu", (M, 2 * H), pitched=True),
                       Op("dgu", (M, 2 * H), pitched=True)],
        **_mx(C),
        "layernorm_fwd": ["layernorm_fwd", Op("x", (M, H), probe="d"), Op("w", (H,)), Op("b", (H,)), Op("y", (M, H)), Op("mean", (M,), F32),
                          Op("rstd", (M,), F32), 1e-5, None, None, None, Op("xd", (M, H)), None, SEED, [1, 2], 0.1],
        "layernorm_bwd": ["layernorm_bwd", Op("dy", (M, H)), Op("x", (M, H), probe="d"), Op("w", (H,)), Op("mean", (M,), F32),
                          Op("rstd", (M,), F32, init=_const(1.0)), Op("dx", (M, H)), Op("dw", (H,), F32), Op("db", (H,), F32)],
        "gelu_fwd": ["gelu_fwd", Op("z", (M, H), probe="d"), Op("a", (M, H)), False, Op("xd", (M, H)), SEED, 1, 0.1],
        "gelu_bwd": ["gelu_bwd", Op("da", (M, H)), Op("z", (M, H), probe="d"), Op("dz", (M, H)), False, Op("dbias", (H,), F32)],
        "colsum": ["colsum", Op("x", (M, H), probe="d"), Op("out", (H,), F32)],
        "neox_rope": ["neox_rope", Op("qkv", (T, 3 * nh * hd), pitched=True, probe="cd"), T, nh, hd, 16, cos(16, F32), sin(16, F32), 0, False],
        "embedding_fwd": ["embedding_fwd", Op("ids", (M,), I64, probe="d", init=_rows(V)), Op("table", (V, H), probe="cd"), Op("out", (M, H))],
        "embedding_bwd": ["embedding_bwd", Op("ids", (M,), I64, probe="d", init=_rows(V)), Op("dout", (M, H)),
                          Op("dtable", (V, H), F32, probe="cd"), -1],
        "embedding_bwd_sorted": ["embedding_bwd_sorted", Op("sorted_ids", (M,), I64, probe="d", init=_sorted(V)),
                                 Op("perm", (M,), I64, init=lambda s, d: torch.randperm(s[0], device="cuda").to(d)), Op("dout", (M, H)),
                                 Op("dtable", (V, H), F32, probe="cd"), -1],
        "cross_entropy_fwd_bwd": ["cross_entropy_fwd_bwd", Op("logits", (M, V), pitched=True, probe="cd"), Op("labels", (M,), I64, init=_rows(V)),
                                  V, 1.0, -100, Op("loss_sum", (1,), F32), Op("count", (1,), F32)],
        "transpose": ["transpose", Op("in", (M, N), pitched=True, probe="d"), Op("out", (N, M), pitched=True)],
        "add": ["add", Op("a", (n,), probe="d"), Op("b", (n,)), Op("out", (n,))],
        "cast_f32_to_bf16": ["cast_f32_to_bf16", Op("in", (n,), F32, probe="d"), Op("out", (n,)), 1.0],
        "fill_uniform_hash": ["fill_uniform_hash", Op("out", (M, N), pitched=True, probe="d"), 1, 0.1],
        "seed_advance": ["seed_advance", Op("seed", (1,), I32)],
        "adamw_flat": ["adamw_flat", Op("param", (n,), probe="d"), Op("grad", (n,), F32), Op("exp_avg", (n,), F32),
                       Op("exp_avg_sq", (n,), F32, init=_const(1.0)), 1e-3, 0.9, 0.999, 1e-8, 0.0, 1,
                       Op("grad_scale", (1,), F32, init=_const(1.0)), 1.0, Op("skip", (1,), F32, init=_const(0.0)),
                       Op("step_dev", (1,), F32, init=_const(1.0))],
        "sumsq": ["sumsq", Op("x", (n,), F32, probe="d"), Op("out", (1,), F32)],
        "random_prune": ["random_prune", Op("x", (n,), F32, probe="d"), 0.1, 1, 0],
        "magnitude_prune": ["magnitude_prune", Op("x", (n,), F32, probe="d"), 0.1, Op("workspace", (C.quantile_workspace_bytes(),), U8),
                            Op("thr", (1,), F32)],
    }


CASES = ("gemm gemm-mn_major gemm-k_windows gemm-m_groups gemm-fp8 rmsnorm_fwd rmsnorm_bwd dropout_expand dropout_combine fp8_quantize_weight fp8_quantize_act fp8_prep lora_dx attention_fwd "
         "attention_bwd rope_inplace rope_pack_bwd swiglu_fwd swiglu_bwd mx_quantize_rows mx_quantize_weight_2d mx_dequantize_weight gemm_mx "
         "layernorm_fwd layernorm_bwd gelu_fwd gelu_bwd colsum neox_rope embedding_fwd embedding_bwd embedding_bwd_sorted "
         "cross_entropy_fwd_bwd transpose add cast_f32_to_bf16 fill_uniform_hash seed_advance adamw_flat sumsq random_prune "
         "magnitude_prune").split()


class _Live:
    """Materialises the operands of one call, each at the start of an allocation one row (and, pitched, 16 columns) larger
    than its valid extent, with random bits in the slack; remembers every allocation to show that nothing was written."""

    def __init__(self):
        self.bufs = []

    def make(self, op: Op, mode=""):
        dtype = op.wrong if mode == "d" else op.dtype
        shape = list(op.shape)
        inner = 1
        for s in shape[1:]:
            inner *= s
        pitch = shape[-1] + 16 if op.pitched else shape[-1]
        total = (shape[0] + 1) * (inner // shape[-1] * pitch if len(shape) > 1 else 1) + 64
        buf = torch.randint(0, 256, (total * torch.tensor([], dtype=dtype).element_size(),), dtype=U8, device="cuda").view(dtype)
        full = buf[: shape[0] * (inner // shape[-1] * pitch if len(shape) > 1 else 1)].view(*shape[:-1], pitch)[..., : shape[-1]]
        g = torch.Generator(device="cuda").manual_seed(len(self.bufs))
        full.copy_(op.init(tuple(shape), dtype) if op.init else (torch.randn(shape, generator=g, device="cuda") * 0.1).to(dtype))
        self.bufs.append((buf, buf.clone()))
        if mode == "r":
            return full[: shape[0] - 1]
        if mode == "c":
            return full[..., : shape[-1] - 1]
        return full

    def unchanged(self):
        return all(torch.equal(b.view(U8), s.view(U8)) for b, s in self.bufs)


def _materialise(live, spec, target=None, mode=""):
    return [live.make(a, mode if a is target else "") if isinstance(a, Op) else a for a in spec[1:]]


@pytest.fixture(scope="module")
def C():
    from relora_b200.ops import native

    return native.require()


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_binding_refuses_short_or_mistyped_operands(C, case):
    spec = _cases(C)[case]
    name = spec[0]
    assert case.split("-")[0] == name
    fn = getattr(C, name)
    ops = [a for a in spec[1:] if isinstance(a, Op)]
    probed = 0
    for op in ops:
        for mode in op.probe:
            live = _Live()
            args = _materialise(live, spec, op, mode)
            torch.cuda.synchronize()
            before = C.launch_count()
            with pytest.raises(RuntimeError) as e:
                fn(*args)
            msg = str(e.value)
            assert f"{name}: {op.name}" in msg, f"{name} / {op.name} ({mode}): {msg}"
            assert C.launch_count() == before, f"{name} / {op.name} ({mode}) launched"
            torch.cuda.synchronize()
            assert live.unchanged(), f"{name} / {op.name} ({mode}) wrote to its operands"
            probed += 1
    assert probed > 0
    live = _Live()
    before = C.launch_count()
    fn(*_materialise(live, spec))
    torch.cuda.synchronize()
    assert C.launch_count() > before
