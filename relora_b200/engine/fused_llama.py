"""Whole-model fused executor for Llama + ReLoRA on H100.

The reference executes one ``ReLoRaLinear`` as ~8 eager kernels (``relora.py:319-322``) and a decoder
layer as ~100 (``modeling_llama.py:243-308``), re-reading every activation several times, and is
launch/CPU-bound at the 250M scale.  This executor instead

* keeps the frozen weights of a layer *stacked* (``Wqkv [3h,h]``, ``Wgu [2f,h]``) and the LoRA factors
  stacked alongside (``A_qkv [3r,h]``, ``B_qkv [3h,r]`` …) — the ``nn.Module`` parameters are views into these
  buffers, so checkpoints keep the reference layout;
* runs every projection as ONE wgmma GEMM launch with the low-rank up-projection folded into the K loop
  (``y = [x | u]·[W | B]ᵀ``, residual add in the epilogue), the three / two down-projections of a stacked group
  as one grouped launch, and all backward GEMMs (``dx``, ``du``, stacked ``dA`` / ``dB`` with split-K) on the same
  kernel reading operands MN-major in place — no transposed copies, no autograd graph;
* fuses RMSNorm with the LoRA-dropout expansion, computes LM-head + cross-entropy chunk-wise without ever
  materialising ``[tokens, V]`` logits, accumulates all gradients in one flat fp32 buffer;
* captures forward+backward of a micro-batch in a CUDA graph (dropout seeds live on the device and advance
  inside the graph), so a micro-step costs one graph launch on the host.

Math per layer (training, dropout p, scale s): see ``ops/reference.py`` — numerics tests compare this executor
with the module-by-module PyTorch path on identical weights and masks.
"""
from __future__ import annotations

import math
import os
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn.functional as F_

from ..models.llama import LlamaForCausalLM
from ..ops import fused, native
from ..parallel.dist import DistInfo
from ..parallel.flat import FlatAdamW, FlatParamStore
from ..parallel.grad_sync import GradSync, broadcast_params
from ..relora import ReLoRaLinear, ReLoRaModel
from .stepper import UpdateInfo

BF = torch.bfloat16


def supports(model, args=None) -> Tuple[bool, str]:
    if not isinstance(model, ReLoRaModel):
        return False, "full-rank training uses the module path"
    inner = model.wrapped_model
    if not isinstance(inner, LlamaForCausalLM):
        return False, "only Llama is fused"
    if model.lora_only or model.trainable_scaling or model._config.quantize is not None:
        return False, "lora_only / trainable scaling / quantized frozen weights use the module path"
    cfg = inner.config
    h, f, nh = cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads
    r = model.r
    hd = h // nh
    if h % 128 or r % 128:
        # the intermediate size may be anything (llama_1b: 5461): its buffers are zero-padded to a multiple of 128
        return False, f"hidden ({h}) and rank ({r}) must be multiples of 128 for stacked groups"
    if hd % 8 or hd % 4:
        return False, "head_dim must be a multiple of 8"
    p = next(inner.parameters())
    if not p.is_cuda or p.dtype != BF:
        return False, "needs CUDA + bfloat16"
    for m in inner.modules():
        if isinstance(m, ReLoRaLinear) and m.bias is not None:
            return False, "biased projections use the module path"
    return True, "ok"


class _Layer:
    """Stacked views of one decoder layer's parameters and gradients."""

    __slots__ = ("Wqkv", "Wo", "Wgu", "Wd", "A_qkv", "B_qkv", "A_o", "B_o", "A_gu", "B_gu", "A_d", "B_d", "w1", "w2",
                 "gA_qkv", "gB_qkv", "gA_o", "gB_o", "gA_gu", "gB_gu", "gA_d", "gB_d", "gw1", "gw2", "keys_qkv", "key_o",
                 "keys_gu", "key_d", "mods", "merge")


class FusedLlamaStepper:
    def __init__(self, model: ReLoRaModel, info: DistInfo, *, lr: float, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, clip_grad_norm: float = 1.0, grad_accumulation: int = 1, zero: bool = False,
                 transport: str = "nccl", native=None, symm_factory=None, cuda_graphs: bool = True, ce_chunk: int = 4096,
                 overlap_wgrad: bool = True, attention: str = "auto", fp8: bool = False, fp8_backward: bool = False,
                 deterministic: bool = False):
        ok, why = supports(model)
        if not ok:
            raise RuntimeError(why)
        self.model, self.info = model, info
        self.inner: LlamaForCausalLM = model.wrapped_model
        self.C = fused._C()
        self.ga = grad_accumulation
        self.clip = clip_grad_norm
        self.use_graphs = cuda_graphs
        self.ce_chunk = ce_chunk
        cfg = self.inner.config
        self.h, self.f, self.nh, self.V = cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads, cfg.vocab_size
        self.hd = self.h // self.nh
        self.fp = (self.f + 127) // 128 * 128  # padded intermediate size (zero rows / columns keep every GEMM extent a multiple of the 128-wide tile)
        self.r = model.r
        self.L = cfg.num_hidden_layers
        self.eps = cfg.rms_norm_eps
        self.p = float(model.lora_dropout)
        self.scale = float(model.lora_alpha) / model.r
        self.device = info.device
        broadcast_params(model)

        # ---------------------------------------------------------------- stacked frozen weights
        dev = self.device
        h, f, fp, r, L = self.h, self.f, self.fp, self.r, self.L
        self.Wqkv = torch.empty(L, 3 * h, h, dtype=BF, device=dev)
        self.Wo = torch.empty(L, h, h, dtype=BF, device=dev)
        self.Wgu = torch.zeros(L, 2 * fp, h, dtype=BF, device=dev)
        self.Wd = torch.zeros(L, h, fp, dtype=BF, device=dev)
        layers = self.inner.model.layers
        with torch.no_grad():
            for l, layer in enumerate(layers):
                at, mlp = layer.self_attn, layer.mlp
                for j, m in enumerate((at.q_proj, at.k_proj, at.v_proj)):
                    self._rehome(m.weight, self.Wqkv[l, j * h:(j + 1) * h])
                self._rehome(at.o_proj.weight, self.Wo[l])
                self._rehome(mlp.gate_proj.weight, self.Wgu[l, :f])
                self._rehome(mlp.up_proj.weight, self.Wgu[l, fp:fp + f])
                self._rehome(mlp.down_proj.weight, self.Wd[l][:, :f])

        # ---------------------------------------------------------------- flat trainable store (stack-friendly order)
        named: List[Tuple[str, torch.nn.Parameter]] = []
        name_of = {id(p): n for n, p in model.named_parameters()}

        def add(p):
            named.append((name_of[id(p)], p))

        for layer in layers:
            at, mlp = layer.self_attn, layer.mlp
            for m in (at.q_proj, at.k_proj, at.v_proj):
                add(m.lora_A.weight)
            for m in (at.q_proj, at.k_proj, at.v_proj):
                add(m.lora_B.weight)
            add(at.o_proj.lora_A.weight); add(at.o_proj.lora_B.weight)
            add(mlp.gate_proj.lora_A.weight); add(mlp.up_proj.lora_A.weight)
            add(mlp.gate_proj.lora_B.weight); add(mlp.up_proj.lora_B.weight)
            add(mlp.down_proj.lora_A.weight); add(mlp.down_proj.lora_B.weight)
            add(layer.input_layernorm.weight); add(layer.post_attention_layernorm.weight)
        add(self.inner.model.embed_tokens.weight)
        add(self.inner.model.norm.weight)
        add(self.inner.lm_head.weight)
        seen = {id(p) for _, p in named}
        extra = [(n, p) for n, p in model.named_parameters() if p.requires_grad and id(p) not in seen]
        if extra:
            raise RuntimeError(f"unexpected trainable parameters for the fused executor: {[n for n, _ in extra]}")
        # ---- transport: NVLink peer-memory kernels when symmetric memory is available, NCCL otherwise
        self.comm = None
        if info.world_size > 1 and transport in ("p2p", "auto"):
            from ..parallel.symm import SymmComm, symmetric_memory_available

            if symmetric_memory_available():
                try:
                    self.comm = SymmComm()
                except Exception as e:  # no P2P access, allocation failure, ...
                    if transport == "p2p":
                        raise
                    from ..obs import logger

                    logger.warning(f"peer-memory collectives unavailable ({type(e).__name__}: {e}); using NCCL")
            elif transport == "p2p":
                raise RuntimeError("--comm p2p needs torch symmetric memory over an NCCL process group")
        padded: Dict[int, Tuple[int, int]] = {}
        if fp != f:
            for layer in layers:
                mlp = layer.mlp
                padded[id(mlp.gate_proj.lora_B.weight)] = (fp, r)
                padded[id(mlp.up_proj.lora_B.weight)] = (fp, r)
                padded[id(mlp.down_proj.lora_A.weight)] = (r, fp)
        self.store = FlatParamStore(named, world_size=info.world_size, grad_dtype=torch.float32, bind_grads=False,
                                    allocator=self.comm.allocator() if self.comm is not None else None,
                                    storage_shapes=padded)
        self.trainable_params = [p for _, p in named]
        self.trainable_names = [n for n, _ in named]
        self.lora_params = [p for n, p in named if "lora_" in n]

        def pv(p, rows_mult=1):  # stacked view over `rows_mult` adjacent parameters (params and grads)
            o, n = self.store.segment(p)
            ps = self.store.storage.get(id(p), tuple(p.shape))  # padded block shape where one exists
            shape = (ps[0] * rows_mult, ps[1]) if p.dim() == 2 else (ps[0] * rows_mult,)
            tot = n * rows_mult
            return self.store.params[o:o + tot].view(shape), self.store.grads[o:o + tot].view(shape)

        self.layers: List[_Layer] = []
        for layer in layers:
            at, mlp = layer.self_attn, layer.mlp
            S = _Layer()
            l = len(self.layers)
            S.Wqkv, S.Wo, S.Wgu, S.Wd = self.Wqkv[l], self.Wo[l], self.Wgu[l], self.Wd[l]
            S.A_qkv, S.gA_qkv = pv(at.q_proj.lora_A.weight, 3)
            S.B_qkv, S.gB_qkv = pv(at.q_proj.lora_B.weight, 3)
            S.A_o, S.gA_o = pv(at.o_proj.lora_A.weight)
            S.B_o, S.gB_o = pv(at.o_proj.lora_B.weight)
            S.A_gu, S.gA_gu = pv(mlp.gate_proj.lora_A.weight, 2)
            S.B_gu, S.gB_gu = pv(mlp.gate_proj.lora_B.weight, 2)
            S.A_d, S.gA_d = pv(mlp.down_proj.lora_A.weight)
            S.B_d, S.gB_d = pv(mlp.down_proj.lora_B.weight)
            S.w1, S.gw1 = pv(layer.input_layernorm.weight)
            S.w2, S.gw2 = pv(layer.post_attention_layernorm.weight)
            S.keys_qkv = [m.module_index + 1 for m in (at.q_proj, at.k_proj, at.v_proj)]
            S.key_o = at.o_proj.module_index + 1
            S.keys_gu = [mlp.gate_proj.module_index + 1, mlp.up_proj.module_index + 1]
            S.key_d = mlp.down_proj.module_index + 1
            S.mods = (at.q_proj, at.k_proj, at.v_proj, at.o_proj, mlp.gate_proj, mlp.up_proj, mlp.down_proj)
            # sanity: the stacked views must alias the module parameters
            assert S.A_qkv[r:2 * r].data_ptr() == at.k_proj.lora_A.weight.data_ptr()
            assert S.B_gu[fp:].data_ptr() == mlp.up_proj.lora_B.weight.data_ptr()
            assert S.A_d.data_ptr() == mlp.down_proj.lora_A.weight.data_ptr() and S.A_d.shape == (r, fp)
            # (B, A, W) blocks of the merge GEMM  W += s·B·A  (padded blocks where the module views are strided)
            S.merge = [(m.lora_B.weight.data, m.lora_A.weight.data, m.weight.data) for m in S.mods[:4]]
            S.merge += [(S.B_gu[:fp], S.A_gu[:r], S.Wgu[:fp]), (S.B_gu[fp:], S.A_gu[r:], S.Wgu[fp:]), (S.B_d, S.A_d, S.Wd)]
            self.layers.append(S)
        emb = self.inner.model.embed_tokens
        self.W_emb, self.gW_emb = pv(emb.weight)
        self.pad_idx = emb.padding_idx if emb.padding_idx is not None else -1
        self.w_norm, self.gw_norm = pv(self.inner.model.norm.weight)
        self.W_head, self.gW_head = pv(self.inner.lm_head.weight)

        rot = layers[0].self_attn.rotary_emb
        self.cos = rot.cos_cached[0, 0].to(BF).contiguous()
        self.sin = rot.sin_cached[0, 0].to(BF).contiguous()

        # ---------------------------------------------------------------- optimizer / comm
        self.sync = GradSync(self.store, info, transport="nccl", zero=zero and self.comm is None)
        shard = self.sync.shard if (zero and self.comm is None) else None
        self._stage = None
        if self.comm is not None:
            # fused update: gradients travel as bf16 through a symmetric buffer, each rank owns 1/world of the
            # optimizer state (ZeRO-1 dataflow) and writes its updated parameters into every replica
            self.sync.transport = "p2p"
            self.param_buf = self.comm.buffer_of(self.store.params)
            self.grad_buf = self.comm.alloc(self.store.numel, BF)
            self.gred = torch.empty(self.store.numel // info.world_size, dtype=torch.float32, device=dev)
            shard = self.store.shard_bounds(info.rank, info.world_size)
        self.optimizer = FlatAdamW(self.store, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, shard=shard,
                                   native=native or fused.NativeOptim())
        self.seed = fused.seed_state.get(dev)
        self._shape = None
        self._graph = None
        self._replays = 0
        self._launches_per_micro = 0
        self._attn_saved: List = []
        # ---- fp8 frozen-weight path: E4M3 copies of the stacked weights + per-site activation scales (csrc/fp8.cu)
        self.fp8 = bool(fp8) or os.environ.get("RELORA_B200_FP8", "0") == "1"
        if self.fp8:
            u8 = lambda *sh: torch.zeros(*sh, dtype=torch.uint8, device=dev)  # noqa: E731
            self.W8 = [u8(L, 3 * h, h), u8(L, h, h), u8(L, 2 * fp, h), u8(L, h, fp)]  # sites: qkv, o, gate/up, down
            f32 = lambda *sh: torch.zeros(*sh, dtype=torch.float32, device=dev)  # noqa: E731
            # scale bookkeeping, index [direction, layer, site]: direction 0 = forward activations (E4M3), 1 = output gradients
            # (E5M2) of the same four projection groups
            self._w_scale2, self._act_state2 = f32(2, L, 4), f32(2, L, 4, 2)
            self._inv_sx2, self._alpha_main2, self._alpha_inv2 = f32(2, L, 4), f32(2, L, 4), f32(2, L, 4)
            self.w_scale, self.act_state = self._w_scale2[0], self._act_state2[0]
            self.inv_sx, self.alpha_main, self.alpha_inv = self._inv_sx2[0], self._alpha_main2[0], self._alpha_inv2[0]
            self.w_inv_scale, self._amax_scratch = f32(L, 4), f32(1)
            self.fp8_bwd = bool(fp8_backward) or os.environ.get("RELORA_B200_FP8_BWD", "0") == "1"
            self._fp8_bwd_calibrated = False
            # E4M3 copies of the transposed weights: K-major operands of the input-gradient GEMMs dy·W
            self.W8T = [u8(L, h, 3 * h), u8(L, h, h), u8(L, h, 2 * fp), u8(L, fp, h)] if self.fp8_bwd else None
            self.fp8_margin = float(os.environ.get("RELORA_B200_FP8_MARGIN", "1.5"))
            self._fp8_calibrated = False
            self._quantize_weights()
        self._fp8_calibrating = False
        if not self.fp8:
            self.fp8_bwd = False
        attention = os.environ.get("RELORA_B200_ATTENTION", attention)
        native_ok = self.hd % 8 == 0 and self.hd <= 64
        if attention == "native" and not native_ok:
            raise RuntimeError(f"--attention native supports head_dim <= 64 (multiple of 8), got {self.hd}")
        # auto: this repo's wgmma kernels (csrc/attention.cu) wherever they apply -- the hot path then contains no library
        # attention call; `--attention sdpa` selects torch SDPA (cuDNN; bench/attn_bench.py times both) and is what larger head
        # dims fall back to
        self.native_attn = attention == "native" or (attention == "auto" and native_ok)
        self.side = torch.cuda.Stream(device=dev) if overlap_wgrad else None
        self.fused_dx = os.environ.get("RELORA_B200_FUSED_DX", "1") != "0"
        # stacked output width from which dx uses two kernels (frozen-path GEMM on 256-wide tiles + a mask-and-add pass) instead of
        # the one-kernel form; the thresholds (4096 bf16, 2048 with fp8 input-gradient GEMMs) have not been re-tuned on the H100.
        self.dx_split_k = int(os.environ.get("RELORA_B200_DX_SPLIT_K", "0")) or (2048 if self.fp8_bwd else 4096)
        self._wg_done: Dict[str, torch.cuda.Event] = {}
        # --deterministic: the stacked dA / dB weight-gradient GEMMs run without split-K (one CTA owns an output tile for the whole token
        # reduction: fixed summation order instead of fp32 atomics from several CTAs).  Remaining order-dependent reductions are the
        # [h]-sized norm-weight gradients (block partials combined with vector atomics).
        self.wgrad_split_k = 1 if (deterministic or os.environ.get("RELORA_B200_DETERMINISTIC", "0") == "1") else 0
        # embedding backward without atomics (default); RELORA_B200_ATOMIC_EMBEDDING=1 selects the atomicAdd scatter
        self.deterministic_embedding = os.environ.get("RELORA_B200_ATOMIC_EMBEDDING", "0") != "1"

    # ------------------------------------------------------------------ plumbing
    @staticmethod
    def _rehome(param: torch.nn.Parameter, dst: torch.Tensor):
        dst.copy_(param.data)
        param.data = dst

    @torch.no_grad()
    def _quantize_weights(self):
        """(Re)build the E4M3 copies of the frozen weights and their per-tensor scales (at start-up and after every merge)."""
        stacks = (self.Wqkv, self.Wo, self.Wgu, self.Wd)
        for l in range(self.L):
            for s_i in range(4):
                self.C.fp8_quantize_weight(stacks[s_i][l], self.W8[s_i][l], self._amax_scratch, self.w_scale[l, s_i:s_i + 1],
                                           self.w_inv_scale[l, s_i:s_i + 1], self.W8T[s_i][l] if self.fp8_bwd else None)
        self._w_scale2[1].copy_(self._w_scale2[0])

    def _alloc(self, B: int, T: int):
        dev, h, f, r, L = self.device, self.h, self.fp, self.r, self.L  # f: padded intermediate size
        M = B * T
        e = lambda *s: torch.empty(*s, dtype=BF, device=dev)  # noqa: E731
        self.B_, self.T_, self.M_ = B, T, M
        self.ids = torch.zeros(B, T, dtype=torch.long, device=dev)
        self.labels = torch.zeros(M, dtype=torch.long, device=dev)
        self.x_in = e(L + 1, M, h)
        self.x1 = e(L, M, h)
        self.rstd1 = torch.empty(L, M, dtype=torch.float32, device=dev)
        self.rstd2 = torch.empty(L, M, dtype=torch.float32, device=dev)
        self.rstd_f = torch.empty(M, dtype=torch.float32, device=dev)
        G3, G2 = (3, 2) if self.p > 0 else (1, 1)
        self.xd_qkv = e(L, M, G3 * h)
        self.xd_o = e(L, M, h)
        self.xd_gu = e(L, M, G2 * h)
        self.xd_d = e(L, M, f)
        self.u_qkv = e(L, M, 3 * r)
        self.u_o = e(L, M, r)
        self.u_gu = e(L, M, 2 * r)
        self.u_d = e(L, M, r)
        self.qkv = e(L, M, 3 * h)
        self.gu = e(L, M, 2 * f)
        # transients
        self.xn = e(M, h)
        self.hmid = e(M, f)
        self.xf = e(M, h)
        self.dxf = e(M, h)
        self.dx_a, self.dx_b, self.dxn, self.dxn2 = e(M, h), e(M, h), e(M, h), e(M, h)
        self.dattn = e(M, h)
        self.dqkv = e(M, 3 * h)
        self.dgu = e(M, 2 * f)
        self.dhmid, self.dhmid2 = e(M, f), e(M, f)
        self.du_bufs = {"d": e(M, r), "gu": e(M, 2 * r), "o": e(M, r), "qkv": e(M, 3 * r)}
        if self.fp8:
            self.x8_h = torch.empty(M, h, dtype=torch.uint8, device=dev)
            self.x8_f = torch.empty(M, f, dtype=torch.uint8, device=dev)
            if self.fp8_bwd:
                self.dy8 = {w: torch.empty(M, w, dtype=torch.uint8, device=dev) for w in {h, 3 * h, 2 * f}}
        if self.native_attn:
            self.attn_o = e(L, M, h)
            self.lse = torch.empty(L, B, self.nh, T, dtype=torch.float32, device=dev)
            self.delta = torch.empty(B, self.nh, T, dtype=torch.float32, device=dev)
        self.parts = e(M, max(3 * h, f))
        ldv = (self.V + 7) // 8 * 8
        self.logits = torch.zeros(min(self.ce_chunk, M), ldv, dtype=BF, device=dev)
        self.loss_sum = torch.zeros(1, dtype=torch.float32, device=dev)
        self.count = torch.zeros(1, dtype=torch.float32, device=dev)
        self.loss_out = torch.zeros((), dtype=torch.float32, device=dev)
        self._shape = (B, T)

    # ------------------------------------------------------------------ forward + backward of one micro-batch
    def _attention(self, qkv: torch.Tensor, train: bool, sl: int = 0):
        B, T, nh, hd = self.B_, self.T_, self.nh, self.hd
        if self.native_attn:
            # wgmma flash attention straight out of the packed projection buffer (csrc/attention.cu); the output and the
            # log-sum-exp of the layer are what the backward kernels need
            out = self.attn_o[sl]
            self.C.attention_fwd(qkv, out, self.lse[sl], B, T, nh, hd, 1.0 / math.sqrt(hd))
            return out
        v5 = qkv.view(B, T, 3, nh, hd)
        q, k, v = (v5[:, :, i].transpose(1, 2) for i in range(3))
        if train:
            q, k, v = (t.detach().requires_grad_() for t in (q, k, v))
            with torch.enable_grad():
                o = F_.scaled_dot_product_attention(q, k, v, dropout_p=0.0, is_causal=True)
            self._attn_saved.append((o, q, k, v))
        else:
            o = F_.scaled_dot_product_attention(q, k, v, dropout_p=0.0, is_causal=True)
        return o.detach().transpose(1, 2).reshape(self.M_, self.h)

    def _q8(self, l, s_i, K):
        """(q8, inv_scale, amax_cur) arguments that make a producer kernel also emit the E4M3 copy of its output."""
        if not self.fp8:
            return (None, None, None)
        return (self.x8_h if K == self.h else self.x8_f, self.inv_sx[l, s_i:s_i + 1], self.act_state[l, s_i, 1:2])

    def _lora_group_fwd(self, xn, xd, A, B, W, u, out, *, G, K, Ng, residual=None, site=None, prequant=False):
        """u = s·xd_g·A_gᵀ (grouped) ; out = [xn | u]·[W | B]ᵀ (+ residual).

        fp8 path (``site = (layer, index)``): xn is quantised to E4M3 with the site's delayed scale and multiplied with the E4M3
        copy of W on the kind::f8f6f4 tensor-core path; the bf16 LoRA term shares the accumulator, so u is produced pre-divided
        by the product scale s_x·s_w, which the epilogue multiplies back."""
        g, r, M = fused.gemm, self.r, self.M_
        drop = self.p > 0 and xd.shape[1] == G * K
        if self.fp8 and site is not None:
            l, s_i = site
            x8 = self.x8_h if K == self.h else self.x8_f
            if not prequant:  # the producer of xn did not emit the E4M3 copy itself
                self.C.fp8_quantize_act(xn, x8, self.inv_sx[l, s_i:s_i + 1], self.act_state[l, s_i, 1:2])
        if self.fp8 and site is not None and not self._fp8_calibrating:
            g(xd, A, u, M=M, N=G * r, K1=K, n_per_group=r, a1_group_kofs=K if drop else 0, alpha=self.scale,
              alpha_dev=self.alpha_inv[l, s_i:s_i + 1])
            g(x8, self.W8[s_i][l], out, M=M, N=G * Ng, K1=K, a2=u, b2=B, K2=r, n_per_group=Ng, a2_group_kofs=r, residual=residual,
              fp8=True, alpha_dev=self.alpha_main[l, s_i:s_i + 1])
            return
        g(xd, A, u, M=M, N=G * r, K1=K, n_per_group=r, a1_group_kofs=K if drop else 0, alpha=self.scale)
        g(xn, W, out, M=M, N=G * Ng, K1=K, a2=u, b2=B, K2=r, n_per_group=Ng, a2_group_kofs=r, residual=residual)

    def _forward(self, train: bool):
        C, g, M, h, f, r = self.C, fused.gemm, self.M_, self.h, self.fp, self.r
        p = self.p if train else 0.0
        seed = self.seed
        C.embedding_fwd(self.ids.view(-1), self.W_emb, self.x_in[0])
        self._attn_saved.clear()
        for l, S in enumerate(self.layers):
            sl = l if train else 0
            x = self.x_in[l] if train else self.x_in[l % 2]
            x_next = self.x_in[l + 1] if train else self.x_in[(l + 1) % 2]
            x1 = self.x1[sl]
            qkv, gu = self.qkv[sl], self.gu[sl]
            # ---- attention block
            if p > 0:
                xd = self.xd_qkv[sl]
                C.rmsnorm_fwd(x, S.w1, self.xn, self.rstd1[sl], self.eps, xd, seed, S.keys_qkv, p, *self._q8(l, 0, h))
                xn = self.xn
            else:
                xn = self.xd_qkv[sl][:, :h] if self.p == 0 else self.xn  # p==0: the normed input is what dA needs
                xn = xn if xn.is_contiguous() else self.xn
                C.rmsnorm_fwd(x, S.w1, xn, self.rstd1[sl], self.eps, None, None, [], 0.0)
                xd = xn
            self._lora_group_fwd(xn, xd, S.A_qkv, S.B_qkv, S.Wqkv, self.u_qkv[sl], qkv, G=3, K=h, Ng=h, site=(l, 0), prequant=p > 0)
            C.rope_inplace(qkv, self.T_, 2 * self.nh, self.hd, self.hd, self.cos, self.sin, False, 0)
            attn = self._attention(qkv, train, sl)
            if p > 0:
                xd_o = self.xd_o[sl]
                C.dropout_expand(attn, xd_o, seed, [S.key_o], p, *self._q8(l, 1, h))
            else:
                xd_o = attn
                if train:
                    self.xd_o[sl].copy_(attn)
            self._lora_group_fwd(attn, xd_o, S.A_o, S.B_o, S.Wo, self.u_o[sl], x1, G=1, K=h, Ng=h, residual=x, site=(l, 1), prequant=p > 0)
            # ---- MLP block
            if p > 0:
                xd = self.xd_gu[sl]
                C.rmsnorm_fwd(x1, S.w2, self.xn, self.rstd2[sl], self.eps, xd, seed, S.keys_gu, p, *self._q8(l, 2, h))
                xn = self.xn
            else:
                xn = self.xd_gu[sl] if self.p == 0 else self.xn
                C.rmsnorm_fwd(x1, S.w2, xn, self.rstd2[sl], self.eps, None, None, [], 0.0)
                xd = xn
            self._lora_group_fwd(xn, xd, S.A_gu, S.B_gu, S.Wgu, self.u_gu[sl], gu, G=2, K=h, Ng=f, site=(l, 2), prequant=p > 0)
            if p > 0:
                xd_d = self.xd_d[sl]
                C.swiglu_fwd(gu, self.hmid, xd_d, seed, S.key_d, p, *self._q8(l, 3, f))  # activation, dropout copy (and E4M3 copy)
            else:
                C.swiglu_fwd(gu, self.hmid, None, None, 0, 0.0, *self._q8(l, 3, f))
                xd_d = self.hmid
                if train:
                    self.xd_d[sl].copy_(self.hmid)
            self._lora_group_fwd(self.hmid, xd_d, S.A_d, S.B_d, S.Wd, self.u_d[sl], x_next, G=1, K=f, Ng=h, residual=x1, site=(l, 3), prequant=True)
        x_last = self.x_in[self.L] if train else self.x_in[self.L % 2]
        C.rmsnorm_fwd(x_last, self.w_norm, self.xf, self.rstd_f, self.eps, None, None, [], 0.0)
        return x_last

    def _loss_and_head_backward(self, train: bool):
        """Chunked LM head + CE.  In training also dxf and dW_head (so logits never persist)."""
        C, g, M, h, V = self.C, fused.gemm, self.M_, self.h, self.V
        n_valid = self.B_ * (self.T_ - 1)
        self.loss_sum.zero_()
        self.count.zero_()
        grad_scale = 1.0 / (n_valid * self.ga)
        for s in range(0, M, self.ce_chunk):
            m = min(self.ce_chunk, M - s)
            hc = self.xf[s:s + m]
            lg = self.logits[:m]
            g(hc, self.W_head, lg, M=m, N=V, K1=h)
            C.cross_entropy_fwd_bwd(lg, self.labels[s:s + m], V, grad_scale, -100, self.loss_sum, self.count)
            if train:
                g(lg, self.W_head, self.dxf[s:s + m], M=m, N=h, K1=V, b1_mn=True)
                g(lg, hc, self.gW_head, M=V, N=h, K1=m, a1_mn=True, b1_mn=True, accumulate=True)
        torch.div(self.loss_sum[0], float(n_valid), out=self.loss_out)

    def _lora_group_bwd(self, dy, S_B, S_W, S_A, gA, gB, xd, u, keys, *, G, K, Ng, base_out, out, tag, site=None):
        """Backward of one stacked LoRA group.  dy [M, G·Ng] -> out [M, K] (grad of the group's input).

        The two weight-gradient GEMMs only read (dy, du, xd, u), so they are forked onto a side stream and fill the
        SMs that the skinny du / parts GEMMs and kernel tails of the main chain leave idle; ``self._wg_done[tag]``
        is the event the main stream waits on before it overwrites one of their inputs (see ``_backward``)."""
        C, g, M, r, s = self.C, fused.gemm, self.M_, self.r, self.scale
        du = self.du_bufs[tag]
        # du_g = s · dy_g · B_g          (B stacked [G·Ng, r], read MN-major; K window g·Ng)
        g(dy, S_B, du, M=M, N=G * r, K1=Ng, b1_mn=True, n_per_group=r, a1_group_kofs=Ng if G > 1 else 0,
          b1_group_kofs=Ng if G > 1 else 0, b1_local_n=True, alpha=s)
        drop = self.p > 0
        shared_x = (not drop) or xd.shape[1] != G * K

        def wgrads():  # fp32, accumulated across micro-batches, split-K over tokens
            g(du, xd, gA, M=G * r, N=K, K1=M, a1_mn=True, b1_mn=True, accumulate=True, split_k=self.wgrad_split_k,
              m_per_group=r if G > 1 else 0, b1_mn_ofs_per_mgroup=0 if shared_x else K)
            # fp8 path: the saved u is u / (s_x·s_w); the product scale is multiplied back here
            g(dy, u, gB, M=G * Ng, N=r, K1=M, a1_mn=True, b1_mn=True, accumulate=True, split_k=self.wgrad_split_k,
              m_per_group=Ng if G > 1 else 0, b1_mn_ofs_per_mgroup=r if G > 1 else 0,
              alpha_dev=self.alpha_main[site[0], site[1]:site[1] + 1] if (self.fp8 and site is not None) else None)

        if self.side is not None:
            fork = torch.cuda.Event()
            fork.record()
            self.side.wait_event(fork)
            with torch.cuda.stream(self.side):
                wgrads()
                done = torch.cuda.Event()
                done.record()
            self._wg_done[tag] = done
        if self.fused_dx:
            sd, ks, pp = (self.seed, list(keys), self.p) if drop else (None, [0] * G, 0.0)
            if G * Ng >= self.dx_split_k:
                # long reductions: the frozen-path product runs on the 256-wide / CTA-pair GEMM (1.3-1.5x the per-FLOP rate of
                # the 128-wide multi-accumulator tiles), then one light pass adds the masked low-rank terms
                if self.fp8_bwd and site is not None:
                    # E5M2 copy of the output gradient (delayed scale) x E4M3 copy of Wᵀ on the kind::f8f6f4 path
                    l_, s_i = site
                    dy8 = self.dy8[G * Ng]
                    C.fp8_quantize_act(dy, dy8, self._inv_sx2[1, l_, s_i:s_i + 1], self._act_state2[1, l_, s_i, 1:2], True)
                if self.fp8_bwd and site is not None and self._fp8_bwd_calibrated:
                    g(dy8, self.W8T[s_i][l_], base_out, M=M, N=K, K1=G * Ng, fp8=2, alpha_dev=self._alpha_main2[1, l_, s_i:s_i + 1])
                else:
                    g(dy, S_W, base_out, M=M, N=K, K1=G * Ng, b1_mn=True)
                C.lora_dx(None, None, du, S_A, out, sd, ks, pp, base_out)
            else:
                # one kernel: out = dy·W + Σ_g keep_g ⊙ (du_g·A_g)/(1-p)  (masked LoRA terms folded into the register accumulator)
                C.lora_dx(dy, S_W, du, S_A, out, sd, ks, pp)
        else:
            # frozen path: base = dy · W     (W stacked [G·Ng, K], read MN-major)
            g(dy, S_W, base_out, M=M, N=K, K1=G * Ng, b1_mn=True)
            # low-rank path per group: part_g = du_g · A_g
            parts = self.parts.view(-1)[: M * G * K].view(M, G * K)
            g(du, S_A, parts, M=M, N=G * K, K1=r, b1_mn=True, n_per_group=K, a1_group_kofs=r if G > 1 else 0,
              b1_group_kofs=r if G > 1 else 0, b1_local_n=True)
            if drop:
                C.dropout_combine(base_out, parts, out, self.seed, keys, self.p)
            else:
                torch.add(base_out, parts.view(M, G, K).sum(1) if G > 1 else parts, out=out)
        if self.side is None:
            wgrads()

    def _join(self, tag):
        """Main stream waits for the side-stream weight gradients tagged ``tag`` (no-op if none are pending)."""
        ev = self._wg_done.pop(tag, None)
        if ev is not None:
            torch.cuda.current_stream().wait_event(ev)

    def _backward(self):
        C, g, M, h, f, r = self.C, fused.gemm, self.M_, self.h, self.fp, self.r
        B, T, nh, hd = self.B_, self.T_, self.nh, self.hd
        dx, dx_other = self.dx_a, self.dx_b
        ws, tk = fused.norm_workspace(self.device, h)
        C.rmsnorm_bwd(self.dxf, self.x_in[self.L], self.w_norm, self.rstd_f, None, dx, self.gw_norm, ws, tk)
        for l in range(self.L - 1, -1, -1):
            S = self.layers[l]
            # ---- MLP: x_next = hmid·Wdᵀ + u_d·B_dᵀ + x1
            self._lora_group_bwd(dx, S.B_d, S.Wd, S.A_d, S.gA_d, S.gB_d, self.xd_d[l], self.u_d[l], [S.key_d],
                                 G=1, K=f, Ng=h, base_out=self.dhmid, out=self.dhmid2, tag="d", site=(l, 3))
            self._join("gu")  # the previous layer's gate/up weight gradients read dgu / du_gu
            C.swiglu_bwd(self.dhmid2, self.gu[l], self.dgu)
            self._lora_group_bwd(self.dgu, S.B_gu, S.Wgu, S.A_gu, S.gA_gu, S.gB_gu, self.xd_gu[l], self.u_gu[l], S.keys_gu,
                                 G=2, K=h, Ng=f, base_out=self.dxn, out=self.dxn2, tag="gu", site=(l, 2))
            self._join("o")  # ... and its o_proj weight gradients read the buffer this norm backward writes
            C.rmsnorm_bwd(self.dxn2, self.x1[l], S.w2, self.rstd2[l], dx, dx_other, S.gw2, ws, tk)
            dx, dx_other = dx_other, dx  # dx = grad wrt x1
            # ---- attention: x1 = attn·Woᵀ + u_o·B_oᵀ + x
            self._lora_group_bwd(dx, S.B_o, S.Wo, S.A_o, S.gA_o, S.gB_o, self.xd_o[l], self.u_o[l], [S.key_o],
                                 G=1, K=h, Ng=h, base_out=self.dxn, out=self.dattn, tag="o", site=(l, 1))
            if self.native_attn:
                self._join("qkv")  # the previous layer's qkv weight gradients read dqkv / du_qkv
                C.attention_bwd(self.qkv[l], self.attn_o[l], self.dattn, self.lse[l], self.delta, self.dqkv, B, T, nh, hd,
                                1.0 / math.sqrt(hd))
                C.rope_inplace(self.dqkv, T, 2 * nh, hd, hd, self.cos, self.sin, True, 0)  # back through the rotation of q, k
                dq = None
            else:
                o, q, k, v = self._attn_saved[l]
                dq, dk, dv = torch.autograd.grad(o, (q, k, v), self.dattn.view(B, T, nh, hd).transpose(1, 2))
                self._join("qkv")  # the previous layer's qkv weight gradients read dqkv / du_qkv
            if dq is None:
                pass
            elif dq.stride() == dk.stride() == dv.stride() and dq.stride(3) == 1:
                C.rope_pack_bwd(dq, dk, dv, self.dqkv, hd, self.cos, self.sin, 0)  # gather + inverse rotation in one pass
            else:
                d5 = self.dqkv.view(B, T, 3, nh, hd)
                d5[:, :, 0].copy_(dq.transpose(1, 2)); d5[:, :, 1].copy_(dk.transpose(1, 2)); d5[:, :, 2].copy_(dv.transpose(1, 2))
                C.rope_inplace(self.dqkv, T, 2 * nh, hd, hd, self.cos, self.sin, True, 0)
            self._lora_group_bwd(self.dqkv, S.B_qkv, S.Wqkv, S.A_qkv, S.gA_qkv, S.gB_qkv, self.xd_qkv[l], self.u_qkv[l],
                                 S.keys_qkv, G=3, K=h, Ng=h, base_out=self.dxn, out=self.dxn2, tag="qkv", site=(l, 0))
            self._join("d")  # this layer's down_proj weight gradients read the buffer written next
            C.rmsnorm_bwd(self.dxn2, self.x_in[l], S.w1, self.rstd1[l], dx, dx_other, S.gw1, ws, tk)
            dx, dx_other = dx_other, dx
        if self.deterministic_embedding:
            # stable sort of the token ids (12 K keys) -> one writer per table row, fixed summation order: bit-reproducible
            sorted_ids, perm = torch.sort(self.ids.view(-1), stable=True)
            C.embedding_bwd_sorted(sorted_ids, perm, dx, self.gW_emb, self.pad_idx)
        else:
            C.embedding_bwd(self.ids.view(-1), dx, self.gW_emb, self.pad_idx)
        for tag in ("d", "gu", "o", "qkv"):
            self._join(tag)
        self._attn_saved.clear()

    def _fp8_calibrate(self):
        """Bootstrap of the delayed activation scales: one bf16 forward that only *records* every site's amax.  (Starting the
        fp8 path cold would saturate the first sites, shrink everything downstream and need one pass per site to recover.)"""
        self._fp8_calibrating = True
        try:
            self.labels.view(self.B_, self.T_)[:, :-1].copy_(self.ids[:, 1:])
            self._forward(True)
        finally:
            self._fp8_calibrating = False
        self._fp8_calibrated = True

    def _micro_body(self):
        self.labels.view(self.B_, self.T_)[:, :-1].copy_(self.ids[:, 1:])
        self.labels.view(self.B_, self.T_)[:, -1].fill_(-100)
        if self.fp8:  # rotate the activation amax state, derive this micro-step's scales
            self.C.fp8_prep(self._act_state2, self._w_scale2, self._inv_sx2, self._alpha_main2, self._alpha_inv2, self.fp8_margin,
                            4 * self.L)
        self._forward(True)
        self._loss_and_head_backward(True)
        self._backward()
        if self.fp8_bwd:
            self._fp8_bwd_calibrated = True  # the first backward ran in bf16 and recorded the gradient amax of every site
        self.C.seed_advance(self.seed)

    # ------------------------------------------------------------------ public stepper interface
    @torch.no_grad()
    def micro_step(self, input_ids: torch.Tensor) -> torch.Tensor:
        B, T = input_ids.shape
        if self._shape != (B, T):
            self._alloc(B, T)
            self._graph = None
        self.ids.copy_(input_ids, non_blocking=True)
        if self.fp8 and not self._fp8_calibrated:
            self._fp8_calibrate()
        if not self.use_graphs:
            self._micro_body()
            return self.loss_out.clone()
        if self._graph is None:
            self._capture()
        else:
            self._graph.replay()
            self._replays += 1
        return self.loss_out.clone()

    def _capture(self):
        # warm-up (allocator, cuBLAS/flash workspaces, tensor-map cache) on a side stream, then capture
        grads_backup = self.store.grads.clone()
        seed_backup = self.seed.clone()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            self._micro_body()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.store.grads.copy_(grads_backup)
        self.seed.copy_(seed_backup)
        n0 = self.C.launch_count()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._micro_body()
        self._launches_per_micro = self.C.launch_count() - n0
        # capture does not execute: run the captured work once for this micro-batch
        self.store.grads.copy_(grads_backup)
        self.seed.copy_(seed_backup)
        del grads_backup
        graph.replay()
        self._replays += 1
        self._graph = graph

    @torch.no_grad()
    def eval_loss(self, input_ids: torch.Tensor) -> torch.Tensor:
        B, T = input_ids.shape
        if self._shape != (B, T):
            self._alloc(B, T)
            self._graph = None
        self.ids.copy_(input_ids)
        self.labels.view(B, T)[:, :-1].copy_(self.ids[:, 1:])
        self.labels.view(B, T)[:, -1].fill_(-100)
        if self.fp8 and not self._fp8_calibrated:
            # evaluation before the first training step: bootstrap the activation scales exactly like micro_step does
            self._fp8_calibrate()
            self.C.fp8_prep(self._act_state2, self._w_scale2, self._inv_sx2, self._alpha_main2, self._alpha_inv2, self.fp8_margin,
                            4 * self.L)
        self._forward(False)
        self._loss_and_head_backward(False)
        return self.loss_out.clone()

    @property
    def folds_loss_reduce(self) -> bool:
        """True when ``update(local_loss=...)`` combines loss / skip over ranks inside the NVLink kernel chain (no NCCL call)."""
        return self.comm is not None

    @torch.no_grad()
    def update(self, skip: Optional[torch.Tensor] = None, error_if_nonfinite: bool = False,
               local_loss: Optional[torch.Tensor] = None) -> UpdateInfo:
        opt = self.optimizer
        world = self.info.world_size
        if self.comm is not None:
            from .stepper import peer_memory_update

            return peer_memory_update(self, grads_f32=self.store.grads, skip=skip, error_if_nonfinite=error_if_nonfinite,
                                      local_loss=local_loss)
        grads = None
        if world > 1 and not self.sync.zero:
            # NCCL baseline: gradients cross the wire as bf16 (like the reference's bf16 DDP buckets), once per update
            if self._stage is None:
                self._stage = torch.empty(self.store.numel, dtype=BF, device=self.device)
            self.C.cast_f32_to_bf16(self.store.grads, self._stage, 1.0)
            dist.all_reduce(self._stage, op=dist.ReduceOp.SUM)
            grads = self._stage
            sq = torch.zeros(1, dtype=torch.float32, device=self.device)
            self.C.sumsq(grads, sq)
            total = sq[0].sqrt() / world
            coef = torch.clamp(self.clip / (total + 1e-6), max=1.0) if self.clip and self.clip > 0 else torch.ones_like(total)
            coef = torch.where(torch.isfinite(total), coef, torch.full_like(coef, float("nan")))  # non-finite norm: skip the update
            scale = coef / world
        else:
            self.sync.reduce()
            total, scale = self.sync.grad_norm_and_scale(self.clip)
        if error_if_nonfinite and not bool(torch.isfinite(total)):
            raise RuntimeError(f"The total norm of order 2.0 for gradients is non-finite ({float(total)}), so it cannot be clipped.")
        opt.step(grad_scale=scale, skip=skip, grads=grads)
        self.sync.gather_params()
        opt.zero_grad()
        return UpdateInfo(total, False)

    @torch.no_grad()
    def merge_and_reinit(self):
        """W += s·B@A on the stacked buffers (wgmma GEMM accumulating into W in fp32), then hash re-init."""
        from ..ops import reference as ref

        g, r = fused.gemm, self.r
        for S in self.layers:
            for m, (Bm, Am, Wm) in zip(S.mods, S.merge):
                g(Bm, Am, Wm, M=Wm.shape[0], N=Wm.shape[1], K1=r, b1_mn=True, alpha=self.scale, accumulate=True)
                sd = ref.mix_seed(self.model.seed, self.model.n_restarts, m.module_index)
                self.C.fill_uniform_hash(m.lora_A.weight.data, sd, 1.0 / math.sqrt(m.in_features))
                m.lora_B.weight.data.zero_()
        self.model.n_restarts += 1
        if self.fp8:
            self._quantize_weights()

    def launches_in_window(self, n_steps: int) -> int:
        """Kernel launches of this extension since ``reset_launch_count`` (graph replays included)."""
        return int(self.C.launch_count() + self._replays_since_reset() * self._launches_per_micro)

    def _replays_since_reset(self) -> int:
        return self._replays - getattr(self, "_replay_mark", 0)

    def mark_launch_window(self):
        self._replay_mark = self._replays
        self.C.reset_launch_count()

    def set_lr(self, lr: float) -> None:
        for grp in self.optimizer.param_groups:
            grp["lr"] = lr
