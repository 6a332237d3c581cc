"""Block-scaled low-precision storage for the frozen weight ``W`` (PyTorch reference implementation).

The reference offers ``--quantize 4bit|8bit`` through bitsandbytes NF4 / int8
(``peft_pretraining/relora.py:222-238, 277-299, 314-317``).  Blackwell tensor cores have native
block-scaled formats instead, so this engine stores the frozen weight as

* ``mxfp8``  — OCP MXFP8: e4m3 elements, one ue8m0 (power-of-two) scale per 32 elements of K;
* ``nvfp4``  — NVFP4: e2m1 elements, one e4m3 scale per 16 elements of K and one fp32 tensor scale.

``4bit`` and ``8bit`` are accepted as aliases (``4bit -> nvfp4``, ``8bit -> mxfp8``).  Layout: data
is row-major ``[N, K]`` (K contiguous, the K-major operand layout fp8 ``wgmma`` wants), scales are
``[N, K/block]``.  The functions here are the numerics oracle for the CUDA kernels and the CPU path.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch

from .reference import mx_encode_blocks

__all__ = ["QuantizedWeight", "quantize", "dequantize", "canonical_format", "FORMATS"]

FORMATS = ("mxfp8", "nvfp4")
_ALIASES = {"8bit": "mxfp8", "fp8": "mxfp8", "mxfp8": "mxfp8", "4bit": "nvfp4", "fp4": "nvfp4", "nvfp4": "nvfp4"}

_E4M3_MAX = 448.0
_E2M1_MAX = 6.0
# positive e2m1 code points, index = 3-bit magnitude code
_E2M1_VALUES = torch.tensor([0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0])


def canonical_format(name: Optional[str]) -> Optional[str]:
    if name is None or name is False:
        return None
    try:
        return _ALIASES[str(name).lower()]
    except KeyError:
        raise ValueError(f"Unknown quantize type: {name}") from None


@dataclass
class QuantizedWeight:
    """Packed frozen weight.  ``data``: uint8 (fp8 bytes, or two fp4 codes per byte, low nibble first)."""

    fmt: str
    shape: torch.Size
    data: torch.Tensor  # uint8
    scales: torch.Tensor  # uint8: ue8m0 exponents (mxfp8) or e4m3 bytes (nvfp4)
    tensor_scale: Optional[torch.Tensor] = None  # fp32 scalar (nvfp4)

    def to(self, device):
        return QuantizedWeight(
            self.fmt,
            self.shape,
            self.data.to(device),
            self.scales.to(device),
            None if self.tensor_scale is None else self.tensor_scale.to(device),
        )

    @property
    def nbytes(self) -> int:
        return self.data.numel() + self.scales.numel() + (4 if self.tensor_scale is not None else 0)


def _pad_k(w: torch.Tensor, block: int) -> torch.Tensor:
    k = w.shape[-1]
    pad = (-k) % block
    if pad:
        w = torch.nn.functional.pad(w, (0, pad))
    return w


def _quantize_mxfp8(w: torch.Tensor) -> QuantizedWeight:
    shape = w.shape
    wf = _pad_k(w.detach().to(torch.float32), 32)
    n, kp = wf.shape
    # the exponent rule and encoding of the CUDA quantisers (ops/reference.py: smallest power of two s with amax / s <= 448)
    q, scales = mx_encode_blocks(wf.view(n, kp // 32, 32))
    return QuantizedWeight("mxfp8", shape, q.reshape(n, kp), scales)


def _dequantize_mxfp8(qw: QuantizedWeight, dtype) -> torch.Tensor:
    n, kp = qw.data.shape
    vals = qw.data.view(torch.float8_e4m3fn).to(torch.float32).view(n, kp // 32, 32)
    scale = torch.exp2(qw.scales.to(torch.float32) - 127.0)
    out = (vals * scale.unsqueeze(-1)).view(n, kp)[:, : qw.shape[-1]]
    return out.to(dtype).contiguous()


def _quantize_nvfp4(w: torch.Tensor) -> QuantizedWeight:
    shape = w.shape
    wf = _pad_k(w.detach().to(torch.float32), 16)
    n, kp = wf.shape
    blocks = wf.view(n, kp // 16, 16)
    amax = blocks.abs().amax(dim=-1)
    gmax = amax.max().clamp(min=1e-30)
    # tensor scale chosen so that the largest block scale lands on e4m3 max
    tscale = gmax / (_E2M1_MAX * _E4M3_MAX)
    bscale = (amax / _E2M1_MAX / tscale).clamp(max=_E4M3_MAX).to(torch.float8_e4m3fn)
    bscale_f = bscale.to(torch.float32)
    denom = (bscale_f * tscale).clamp(min=1e-30).unsqueeze(-1)
    x = (blocks / denom).clamp(-_E2M1_MAX, _E2M1_MAX)
    table = _E2M1_VALUES.to(x.device)
    code = (x.abs().unsqueeze(-1) - table).abs().argmin(dim=-1).to(torch.uint8)
    code = code | ((x < 0).to(torch.uint8) << 3)
    code = code.view(n, kp)
    packed = code[:, 0::2] | (code[:, 1::2] << 4)
    return QuantizedWeight("nvfp4", shape, packed.contiguous(), bscale.view(torch.uint8), tscale.reshape(()).to(torch.float32))


def _dequantize_nvfp4(qw: QuantizedWeight, dtype) -> torch.Tensor:
    n, half = qw.data.shape
    kp = half * 2
    code = torch.empty(n, kp, dtype=torch.uint8, device=qw.data.device)
    code[:, 0::2] = qw.data & 0xF
    code[:, 1::2] = qw.data >> 4
    table = _E2M1_VALUES.to(qw.data.device)
    mag = table[(code & 0x7).long()]
    vals = torch.where((code & 0x8) != 0, -mag, mag).view(n, kp // 16, 16)
    bscale = qw.scales.view(torch.float8_e4m3fn).to(torch.float32)
    out = (vals * (bscale * qw.tensor_scale).unsqueeze(-1)).view(n, kp)[:, : qw.shape[-1]]
    return out.to(dtype).contiguous()


def quantize(w: torch.Tensor, fmt: str) -> QuantizedWeight:
    fmt = canonical_format(fmt)
    if w.dim() != 2:
        raise ValueError("expected a 2-D weight [N, K]")
    if fmt == "mxfp8":
        return _quantize_mxfp8(w)
    return _quantize_nvfp4(w)


def dequantize(qw: QuantizedWeight, dtype=torch.bfloat16) -> torch.Tensor:
    if qw.fmt == "mxfp8":
        return _dequantize_mxfp8(qw, dtype)
    return _dequantize_nvfp4(qw, dtype)
