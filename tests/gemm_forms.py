"""The GEMM call forms of one stacked LoRA group (``FusedStepperBase._lora_group_fwd`` / ``_lora_group_bwd``, bf16 path), shared
by the reference tests (test_gemm_reference.py) and the kernel sweep (test_gemm_modes_gpu.py).  Not a test module."""
import torch

BF = torch.bfloat16
FORMS = ("u", "y", "du", "parts", "dA", "dB")


def lora_group_shapes(*, G, K, Ng, M, r, drop):
    """Operand shapes (and dtypes) of one group: xn [M, K]; xd [M, G·K] with dropout windows, else [M, K]; A [G·r, K];
    W, B [G·Ng, K | r]; u [M, G·r]; y / dy / residual [M, G·Ng]; bias [G·Ng]; du [M, G·r]; parts [M, G·K]; fp32 gA, gB."""
    f32 = torch.float32
    return {
        "xn": ((M, K), BF), "xd": ((M, G * K if drop else K), BF), "A": ((G * r, K), BF), "W": ((G * Ng, K), BF),
        "B": ((G * Ng, r), BF), "u": ((M, G * r), BF), "y": ((M, G * Ng), BF), "res": ((M, G * Ng), BF), "bias": ((G * Ng,), BF),
        "dy": ((M, G * Ng), BF), "du": ((M, G * r), BF), "parts": ((M, G * K), BF), "gA": ((G * r, K), f32), "gB": ((G * Ng, r), f32),
    }


def lora_group_call(form, T, *, G, K, Ng, M, r, s, drop, split_k=0, bias=True, residual=True):
    """``(a1, b1, out, kwargs)`` of ``fused.gemm`` for one form, with the arguments the executors pass (``T``: tensors by the
    names of :func:`lora_group_shapes`).  ``drop``: per-group dropout copies of the input (xd holds G windows)."""
    shared_x = not drop
    if form == "u":    # u_g = s·xd_g·A_gᵀ
        return T["xd"], T["A"], T["u"], dict(M=M, N=G * r, K1=K, n_per_group=r, a1_group_kofs=K if drop else 0, alpha=s)
    if form == "y":    # y_g = xn·W_gᵀ + u_g·B_gᵀ (+ bias) (+ residual)
        return T["xn"], T["W"], T["y"], dict(M=M, N=G * Ng, K1=K, a2=T["u"], b2=T["B"], K2=r, n_per_group=Ng, a2_group_kofs=r,
                                             residual=T["res"] if residual else None, bias=T["bias"] if bias else None)
    if form == "du":   # du_g = s·dy_g·B_g
        return T["dy"], T["B"], T["du"], dict(M=M, N=G * r, K1=Ng, b1_mn=True, n_per_group=r, a1_group_kofs=Ng if G > 1 else 0,
                                              b1_group_kofs=Ng if G > 1 else 0, b1_local_n=True, alpha=s)
    if form == "parts":  # part_g = du_g·A_g
        return T["du"], T["A"], T["parts"], dict(M=M, N=G * K, K1=r, b1_mn=True, n_per_group=K, a1_group_kofs=r if G > 1 else 0,
                                                 b1_group_kofs=r if G > 1 else 0, b1_local_n=True)
    if form == "dA":   # gA_g += du_gᵀ·xd_g
        return T["du"], T["xd"], T["gA"], dict(M=G * r, N=K, K1=M, a1_mn=True, b1_mn=True, accumulate=True, split_k=split_k,
                                               m_per_group=r if G > 1 else 0, b1_mn_ofs_per_mgroup=0 if shared_x else K)
    if form == "dB":   # gB_g += dy_gᵀ·u_g
        return T["dy"], T["u"], T["gB"], dict(M=G * Ng, N=r, K1=M, a1_mn=True, b1_mn=True, accumulate=True, split_k=split_k,
                                              m_per_group=Ng if G > 1 else 0, b1_mn_ofs_per_mgroup=r if G > 1 else 0)
    raise ValueError(form)


def lora_group_composition(form, T, *, G, K, Ng, r, s, drop, bias=True, residual=True):
    """The same product written group by group in fp64 torch, as the executors' docstrings state it."""
    d = lambda t: t.to(torch.float64)  # noqa: E731
    xd = lambda g: d(T["xd"][:, g * K:(g + 1) * K] if drop else T["xd"])  # noqa: E731
    rows = lambda t, g, n: d(t[g * n:(g + 1) * n])  # noqa: E731
    cols = lambda t, g, n: d(t[:, g * n:(g + 1) * n])  # noqa: E731
    if form == "u":
        return torch.cat([s * xd(g) @ rows(T["A"], g, r).t() for g in range(G)], 1)
    if form == "y":
        y = torch.cat([d(T["xn"]) @ rows(T["W"], g, Ng).t() + cols(T["u"], g, r) @ rows(T["B"], g, Ng).t() for g in range(G)], 1)
        return y + (d(T["bias"]) if bias else 0) + (d(T["res"]) if residual else 0)
    if form == "du":
        return torch.cat([s * cols(T["dy"], g, Ng) @ rows(T["B"], g, Ng) for g in range(G)], 1)
    if form == "parts":
        return torch.cat([cols(T["du"], g, r) @ rows(T["A"], g, r) for g in range(G)], 1)
    if form == "dA":
        return d(T["gA"]) + torch.cat([cols(T["du"], g, r).t() @ xd(g) for g in range(G)], 0)
    if form == "dB":
        return d(T["gB"]) + torch.cat([cols(T["dy"], g, Ng).t() @ cols(T["u"], g, r) for g in range(G)], 0)
    raise ValueError(form)
