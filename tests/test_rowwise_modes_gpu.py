"""The norm, rotary, activation, loss, embedding, dropout, fp8 and optimizer kernels element by element against the fp64
references of their contracts (ops/reference.py, row-wise section): every branch of each kernel on guarded buffers, and an audit
of every such call the fused executors and update() issue (H100: -m gpu).

Operands sit inside NaN-filled buffers; outputs sit inside buffers whose guard region holds a sentinel that must survive bit for
bit, and start as NaN (accumulated outputs start at non-zero values), so an element that is never written fails too.  Every
call goes through _Checker: it clones the inputs after a device synchronise, runs the kernel, synchronises, checks every output
against the reference and records the mode the call took.  The sweep and the executor audit share it."""
import math

import pytest
import torch

from guarded_buffers import Guarded
from relora_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
BF, F32 = torch.bfloat16, torch.float32
SENTINEL = 1234.0
WORST = {}  # worst error/tolerance ratio per family (printed at the end of the module with -s)
CALIB = {}  # share of the empirical coefficient each family used (rowwise_excess)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for fam, (w, case) in sorted(WORST.items()):
        print(f"[rowwise modes] {fam}: worst ratio {w:.3g} ({case})")
    for fam, (w, case) in sorted(CALIB.items()):
        print(f"[rowwise modes] calibration {fam}: {w:.3g} ({case})")


def _note(table, family, worst, case=""):
    if worst > table.get(family, (-1.0, ""))[0]:
        table[family] = (worst, case)


@pytest.fixture(scope="module")
def C():
    from relora_b200.ops import native

    return native.require()


# ----------------------------------------------------------------------------------------------- the checker
_SIGS = {  # positional parameters of the extension's entry points, with the defaults the bindings declare
    "rmsnorm_fwd": ("x w y rstd eps xd seed keys p q8 q_inv_scale q_amax", dict(q8=None, q_inv_scale=None, q_amax=None)),
    "rmsnorm_bwd": ("dy x w rstd dx_add dx dw ws ticket", {}),
    "dropout_expand": ("x xd seed keys p q8 q_inv_scale q_amax", dict(q8=None, q_inv_scale=None, q_amax=None)),
    "dropout_combine": ("base parts out seed keys p", {}),
    "fp8_quantize_weight": ("w w8 scratch scale inv_scale w8t", dict(w8t=None)),
    "fp8_quantize_act": ("x x8 inv_scale amax_cur e5m2", dict(amax_cur=None, e5m2=False)),
    "fp8_prep": ("state w_scale inv_sx alpha_main alpha_inv margin n_e4m3", dict(n_e4m3=-1)),
    "rope_inplace": ("buf T n_rot_heads hd rotary_dim cos sin backward pos0", {}),
    "rope_pack_bwd": ("dq dk dv out rotary_dim cos sin pos0 nkv", dict(nkv=-1)),
    "swiglu_fwd": ("gu h hd seed key p q8 q_inv_scale q_amax", dict(hd=None, seed=None, key=0, p=0.0, q8=None, q_inv_scale=None,
                                                                    q_amax=None)),
    "swiglu_bwd": ("dh gu dgu", {}),
    "layernorm_fwd": ("x w b y mean rstd eps w2 b2 y2 xd xd2 seed keys p", dict(w2=None, b2=None, y2=None, xd=None, xd2=None, seed=None,
                                                                             keys=(), p=0.0)),
    "layernorm_bwd": ("dy x w mean rstd dx dw db dres dy2 w2 dw2 db2 dres_sum dres_sum2", dict(dres=None, dy2=None, w2=None, dw2=None,
                                                                                            db2=None, dres_sum=None, dres_sum2=None)),
    "gelu_fwd": ("z a tanh_approx xd seed key p", dict(xd=None, seed=None, key=0, p=0.0)),
    "gelu_bwd": ("da z dz tanh_approx dbias", dict(dbias=None)),
    "colsum": ("x out", {}),
    "neox_rope": ("qkv T nh hd rot cos sin pos0 inverse", {}),
    "embedding_fwd": ("ids table out", {}),
    "embedding_bwd": ("ids dout dtable padding_idx", {}),
    "embedding_bwd_sorted": ("sorted_ids perm dout dtable padding_idx", {}),
    "cross_entropy_fwd_bwd": ("logits labels V grad_scale ignore_index loss_sum count", {}),
    "cast_f32_to_bf16": ("inp out scale", {}),
    "adamw_flat": ("p g m v lr b1 b2 eps wd step grad_scale grad_scale_host skip step_dev", {}),
    "sumsq": ("x out", {}),
    "transpose": ("inp out", {}),
    "seed_advance": ("seed", {}),
}


def _bind(name, args, kw):
    names, defaults = _SIGS[name]
    names = names.split()
    a = dict(defaults)
    a.update(zip(names, args))
    a.update(kw)
    missing = [n for n in names if n not in a]
    assert not missing, f"{name}: missing arguments {missing}"
    return a


def _clone(v):
    return v.clone() if torch.is_tensor(v) else v


def _rows(t, H):
    return t.reshape(-1, H)


def _same_bits(x, y):
    return bool(torch.equal(ref._bits(x), ref._bits(y)))


class _Checker:
    """Runs extension calls checked against the row-wise references; records the mode of each call and the worst ratio."""

    def __init__(self, C):
        self.C = C
        self.orig = {n: getattr(C, n) for n in _SIGS}
        self.modes, self.worst = {}, 0.0
        self.case = ""

    def install(self, monkeypatch):
        for n in _SIGS:
            monkeypatch.setattr(self.C, n, (lambda name: lambda *a, **k: self.call(name, *a, **k))(n))

    def call(self, name, *args, **kw):
        a = _bind(name, args, kw)
        torch.cuda.synchronize()
        b = {k: _clone(v) for k, v in a.items()}
        self.orig[name](*args, **kw)
        torch.cuda.synchronize()
        mode = getattr(self, "_" + name)(b, a)
        self.modes[mode] = self.modes.get(mode, 0) + 1
        return mode

    # ---- helpers
    def close(self, family, got, r, b):
        w = ref.assert_rowwise_close(family, got, r, b)
        self.worst = max(self.worst, w)
        _note(WORST, family, w, self.case)
        _note(CALIB, family, ref.rowwise_excess(got, r, b), self.case)

    def exact(self, family, got, expected):
        ref.assert_bitwise_equal(family, got, expected)

    def fp8_copy(self, name, y, b, a):
        if a.get("q8") is None:
            return ""
        q, amax = ref.fp8_copy_exact(y, b["q_inv_scale"], b["q_amax"])
        self.exact(f"{name} q8", a["q8"].view(torch.uint8), q)
        self.exact(f"{name} amax", a["q_amax"].reshape(-1)[:1], amax)
        return " e4m3"

    # ---- RMSNorm
    def _rmsnorm_fwd(self, b, a):
        H = b["x"].shape[-1]
        x = _rows(b["x"], H)
        M = x.shape[0]
        rstd = a["rstd"].reshape(-1)[:M]
        r = ref.rmsnorm_fwd_ref(x, b["w"], b["eps"], rstd)
        self.close("rmsnorm_fwd rstd", rstd, *r["rstd"])
        y = _rows(a["y"], H)
        self.exact("rmsnorm_fwd y", y, r["y"])
        G = 0
        if b["xd"] is not None:
            G = len(b["keys"])
            xd = a["xd"].reshape(M, G, H)
            for g in range(G):
                self.exact(f"rmsnorm_fwd xd[{g}]", xd[:, g], ref.dropout_copy_exact(y, b["seed"], b["keys"][g], b["p"]))
        e4 = self.fp8_copy("rmsnorm_fwd", y, b, a)
        path = f"warp VPL={_vpl(H // 8)}" if H <= 2048 else f"block VPT={_vpt(H // 8)}"
        return f"rmsnorm_fwd {path} G={G}{e4}"

    def _rmsnorm_bwd(self, b, a):
        H = b["x"].shape[-1]
        x = _rows(b["x"], H)
        M = x.shape[0]
        add = None if b["dx_add"] is None else _rows(b["dx_add"], H)
        r = ref.rmsnorm_bwd_ref(_rows(b["dy"], H), x, b["w"], b["rstd"].reshape(-1)[:M], add, b["dw"])
        self.close("rmsnorm_bwd dx", _rows(a["dx"], H), *r["dx"])
        self.close("rmsnorm_bwd dw", a["dw"], *r["dw"])
        warp = H <= 2048 and a["dw"].data_ptr() % 16 == 0
        v = _vpl(H // 8)
        path = f"warp VPL={v}{' prefetch' if v <= 4 else ''}" if warp else f"block VPT={_vpt(H // 8)}"
        return f"rmsnorm_bwd {path}{' dx_add' if add is not None else ''}"

    # ---- LayerNorm
    def _layernorm_fwd(self, b, a):
        x = b["x"]
        M, H = x.shape
        norms = [(b["w"], b["b"])] + ([(b["w2"], b["b2"])] if b["y2"] is not None else [])
        r = ref.layernorm_fwd_ref(x, b["eps"], a["mean"].reshape(-1), a["rstd"].reshape(-1), norms)
        self.close("layernorm_fwd mean", a["mean"].reshape(-1), *r["mean"])
        self.close("layernorm_fwd rstd", a["rstd"].reshape(-1), *r["rstd"])
        tags = []
        for n, (yk, xk) in enumerate((("y", "xd"), ("y2", "xd2"))):
            if a[yk] is None:
                continue
            self.close("layernorm_fwd y", a[yk], *r[f"y{n}"])
            if a[xk] is not None:
                self.exact(f"layernorm_fwd {xk}", a[xk], ref.dropout_copy_exact(a[yk], b["seed"], b["keys"][n], b["p"]))
                tags.append(xk)
        bias = "bias" if b["b"] is not None else "nobias"
        return f"layernorm_fwd VPL={_vpl(H // 8, 16)} {bias}{' dual' if b['y2'] is not None else ''}{''.join(' ' + t for t in tags)}"

    def _layernorm_bwd(self, b, a):
        M, H = b["x"].shape
        norms = [(b["dy"], b["w"], b["dw"], b["db"])]
        outs = [("dw0", a["dw"]), ("db0", a["db"])]
        if b["dy2"] is not None:
            norms.append((b["dy2"], b["w2"], b["dw2"], b["db2"]))
            outs += [("dw1", a["dw2"]), ("db1", a["db2"])]
        sums = [s for s in (b["dres_sum"], b["dres_sum2"]) if s is not None]
        r = ref.layernorm_bwd_ref(b["x"], b["mean"], b["rstd"], norms, b["dres"], sums)
        self.close("layernorm_bwd dx", a["dx"], *r["dx"])
        for k, got in outs:
            if got is not None:
                self.close(f"layernorm_bwd {k[:2]}", got, *r[k])
        for k, got in enumerate((a["dres_sum"], a["dres_sum2"])):
            if got is not None:
                self.close("layernorm_bwd dres_sum", got, *r[f"dres_sum{k}"])
        if len(sums) == 2 and _same_bits(b["dres_sum"], b["dres_sum2"]):
            assert _same_bits(a["dres_sum"], a["dres_sum2"]), "layernorm_bwd: the two dres_sum outputs started equal and ended apart"
        dual = b["dres"] is not None or b["dy2"] is not None or b["dres_sum"] is not None
        tags = ("dual" if dual else "module", "bias" if b["db"] is not None else "nobias", "two" if b["dy2"] is not None else "",
                "dres" if b["dres"] is not None else "", "sum" if b["dres_sum"] is not None else "",
                "sum2" if b["dres_sum2"] is not None else "")
        return f"layernorm_bwd VPL={_vpl(H // 8)} " + " ".join(t for t in tags if t)

    # ---- cross-entropy
    def _cross_entropy_fwd_bwd(self, b, a):
        V = int(b["V"])
        lg = a["logits"]
        r = ref.cross_entropy_ref(b["logits"], b["labels"], V, b["grad_scale"], b["ignore_index"], b["loss_sum"], b["count"])
        self.close("ce grad", lg[:, :V], *r["grad"])
        self.exact("ce padding columns", lg[:, V:], b["logits"][:, V:])
        self.close("ce loss_sum", a["loss_sum"].reshape(-1)[:1], *r["loss_sum"])
        self.exact("ce count", a["count"].reshape(-1)[:1], r["count"])
        ign = bool((b["labels"] == b["ignore_index"]).any())
        return f"ce V%8={V % 8}{' ignored' if ign else ''}{' scaled' if b['grad_scale'] != 1.0 else ''}"

    # ---- rotary
    def _rope_inplace(self, b, a):
        buf = b["buf"]
        mask, rv, bd = ref.rope_inplace_ref(buf, b["T"], b["n_rot_heads"], b["hd"], b["rotary_dim"], b["cos"], b["sin"], b["backward"],
                                            b["pos0"])
        self.close("rope_inplace buf", a["buf"][mask], rv[mask], bd[mask])
        self.exact("rope_inplace untouched", a["buf"][~mask], buf[~mask])
        half = b["rotary_dim"] // 2
        vec = half % 8 == 0 and b["hd"] % 8 == 0 and a["buf"].stride(0) % 8 == 0 and a["buf"].data_ptr() % 16 == 0
        return (f"rope_inplace {'vec' if vec else 'scalar'} {'bwd' if b['backward'] else 'fwd'}"
                f"{' partial' if b['rotary_dim'] < b['hd'] else ''}{' pos0' if b['pos0'] else ''}")

    def _rope_pack_bwd(self, b, a):
        exact, rv, bd = ref.rope_pack_bwd_ref(b["dq"], b["dk"], b["dv"], b["rotary_dim"], b["cos"], b["sin"], b["pos0"])
        out = a["out"]
        self.close("rope_pack_bwd out", out[~exact], rv[~exact], bd[~exact])
        self.exact("rope_pack_bwd copies", out[exact], rv[exact].to(BF))
        gqa = b["dk"].shape[1] != b["dq"].shape[1]
        return (f"rope_pack_bwd {'gqa' if gqa else 'mha'}{' partial' if b['rotary_dim'] < b['dq'].shape[3] else ''}"
                f"{' pos0' if b['pos0'] else ''}")

    def _neox_rope(self, b, a):
        mask, rv, bd = ref.neox_rope_ref(b["qkv"], b["T"], b["nh"], b["hd"], b["rot"], b["cos"], b["sin"], b["pos0"], b["inverse"])
        self.close("neox_rope qkv", a["qkv"][mask], rv[mask], bd[mask])
        self.exact("neox_rope untouched", a["qkv"][~mask], b["qkv"][~mask])
        return f"neox_rope {'inverse' if b['inverse'] else 'fwd'}{' pos0' if b['pos0'] else ''}"

    # ---- activations
    def _swiglu_fwd(self, b, a):
        F = a["h"].shape[1]
        h = a["h"]
        self.close("swiglu_fwd h", h, *ref.swiglu_fwd_ref(b["gu"], F))
        if a["hd"] is not None:
            self.exact("swiglu_fwd hd", a["hd"], ref.dropout_copy_exact(h, b["seed"], b["key"], b["p"]))
        e4 = self.fp8_copy("swiglu_fwd", h, b, a)
        return f"swiglu_fwd{' dropout' if a['hd'] is not None else ''}{e4}"

    def _swiglu_bwd(self, b, a):
        F = b["dh"].shape[1]
        r = ref.swiglu_bwd_ref(b["dh"], b["gu"], F)
        self.close("swiglu_bwd dg", a["dgu"][:, :F], *r["dg"])
        self.close("swiglu_bwd du", a["dgu"][:, F:2 * F], *r["du"])
        return "swiglu_bwd"

    def _gelu_fwd(self, b, a):
        self.close("gelu_fwd a", a["a"], *ref.gelu_fwd_ref(b["z"], b["tanh_approx"]))
        if a["xd"] is not None:
            N = b["z"].shape[-1]
            self.exact("gelu_fwd xd", _rows(a["xd"], N), ref.dropout_copy_exact(_rows(a["a"], N), b["seed"], b["key"], b["p"]))
        return f"gelu_fwd {'tanh' if b['tanh_approx'] else 'erf'}{' dropout' if a['xd'] is not None else ''}"

    def _gelu_bwd(self, b, a):
        self.close("gelu_bwd dz", a["dz"], *ref.gelu_bwd_ref(b["da"], b["z"], b["tanh_approx"]))
        if a["dbias"] is not None:
            N = b["z"].shape[-1]
            self.close("gelu_bwd dbias", a["dbias"], *ref.colsum_ref(_rows(a["dz"], N), b["dbias"]))
        return f"gelu_bwd {'tanh' if b['tanh_approx'] else 'erf'}{' dbias' if a['dbias'] is not None else ''}"

    def _colsum(self, b, a):
        self.close("colsum out", a["out"], *ref.colsum_ref(b["x"], b["out"]))
        return "colsum"

    # ---- embedding
    def _embedding_fwd(self, b, a):
        self.exact("embedding_fwd", a["out"].reshape(-1, b["table"].shape[1]), b["table"][b["ids"].reshape(-1)])
        return "embedding_fwd"

    def _embedding_bwd(self, b, a):
        self.close("embedding_bwd dtable", a["dtable"], *ref.embedding_bwd_ref(b["ids"], b["dout"], b["dtable"], b["padding_idx"]))
        return "embedding_bwd atomic"

    def _embedding_bwd_sorted(self, b, a):
        self.exact("embedding_bwd_sorted", a["dtable"],
                   ref.embedding_bwd_sorted_exact(b["sorted_ids"], b["perm"], b["dout"], b["dtable"], b["padding_idx"]))
        return "embedding_bwd sorted"

    # ---- dropout
    def _dropout_expand(self, b, a):
        H = b["x"].shape[-1]
        x = _rows(b["x"], H)
        G = len(b["keys"])
        xd = a["xd"].reshape(x.shape[0], G, H)
        for g in range(G):
            self.exact(f"dropout_expand xd[{g}]", xd[:, g], ref.dropout_copy_exact(x, b["seed"], b["keys"][g], b["p"]))
        return f"dropout_expand G={G}{self.fp8_copy('dropout_expand', x, b, a)}"

    def _dropout_combine(self, b, a):
        M, H = a["out"].shape
        G = len(b["keys"])
        P = b["parts"]
        groups = [P[g] for g in range(G)] if P.dim() == 3 else [P[:, g * H:(g + 1) * H] for g in range(G)]
        self.close("dropout_combine out", a["out"], *ref.dropout_combine_ref(b["base"], groups, b["seed"], b["keys"], b["p"]))
        return f"dropout_combine G={G}{' base' if b['base'] is not None else ''}"

    # ---- fp8
    def _fp8_quantize_act(self, b, a):
        x = b["x"]
        inv = ref._f32(b["inv_scale"].reshape(-1)[:1])
        self.exact("fp8_quantize_act x8", a["x8"].view(torch.uint8), ref.fp8_saturate(ref._f32(x) * inv, b["e5m2"]))
        if b["amax_cur"] is not None:
            amax = torch.maximum(b["amax_cur"].reshape(-1)[:1], ref._f32(x).abs().max().reshape(1))
            self.exact("fp8_quantize_act amax", a["amax_cur"].reshape(-1)[:1], amax)
        return f"fp8_quantize_act {'e5m2' if b['e5m2'] else 'e4m3'}{' amax' if b['amax_cur'] is not None else ''}"

    def _fp8_quantize_weight(self, b, a):
        amax, scale, inv, q, qt = ref.fp8_quantize_weight_exact(b["w"])
        self.exact("fp8_quantize_weight amax", a["scratch"].reshape(-1)[:1], amax)
        self.exact("fp8_quantize_weight scale", a["scale"].reshape(-1)[:1], scale)
        self.exact("fp8_quantize_weight inv_scale", a["inv_scale"].reshape(-1)[:1], inv)
        self.exact("fp8_quantize_weight w8", a["w8"].view(torch.uint8), q)
        if a["w8t"] is not None:
            self.exact("fp8_quantize_weight w8t", a["w8t"].view(torch.uint8), qt)
        return f"fp8_quantize_weight{' transposed' if a['w8t'] is not None else ''}"

    def _fp8_prep(self, b, a):
        n = b["w_scale"].numel()
        r = ref.fp8_prep_exact(b["state"], b["w_scale"], b["margin"], n if b["n_e4m3"] < 0 else b["n_e4m3"])
        for k in ("state", "inv_sx", "alpha_main", "alpha_inv"):
            self.exact(f"fp8_prep {k}", a[k].reshape(-1), r[k].reshape(-1))
        return "fp8_prep"

    # ---- misc
    def _cast_f32_to_bf16(self, b, a):
        self.exact("cast_f32_to_bf16", a["out"], (b["inp"] * torch.tensor(b["scale"], dtype=F32)).to(BF).reshape(a["out"].shape))
        return "cast_f32_to_bf16"

    def _transpose(self, b, a):
        self.exact("transpose", a["out"], b["inp"].t())
        return "transpose"

    def _seed_advance(self, b, a):
        s = (int(b["seed"].reshape(-1)[0].item()) + 0x9E3779B9) & 0xFFFFFFFF
        want = int(ref._lowbias32(torch.tensor([s], dtype=torch.int64))[0])
        got = int(a["seed"].reshape(-1)[0].item()) & 0xFFFFFFFF
        assert got == want, f"seed_advance: got {got:#x}, expected {want:#x}"
        return "seed_advance"

    # ---- optimizer
    def _adamw_flat(self, b, a):
        gs = float(b["grad_scale_host"]) * (float(b["grad_scale"].reshape(-1)[0]) if b["grad_scale"] is not None else 1.0)
        skip = b["skip"] is not None and float(b["skip"].reshape(-1)[0]) != 0.0
        step = b["step"] if b["step_dev"] is None else max(float(b["step_dev"].reshape(-1)[0]), 1.0)
        mode = (f"adamw_flat g={'f32' if b['g'].dtype == F32 else 'bf16'} s={'f32' if b['m'].dtype == F32 else 'bf16'} "
                f"step={'dev' if b['step_dev'] is not None else 'host'}")
        gs32 = float(torch.tensor(float(b["grad_scale_host"]), dtype=F32)) * (float(b["grad_scale"].reshape(-1)[0]) if b["grad_scale"]
                                                                               is not None else 1.0)
        if skip or not math.isfinite(gs32):
            for k in ("p", "m", "v"):
                self.exact(f"adamw_flat {k} (skipped)", a[k], b[k])
            return mode + " skipped"
        r = ref.adamw_ref(b["p"], b["g"], b["m"], b["v"], lr=b["lr"], b1=b["b1"], b2=b["b2"], eps=b["eps"], wd=b["wd"], step=step,
                          grad_scale=gs)
        for k in ("p", "m", "v"):
            self.close(f"adamw_flat {k}", a[k], *r[k])
        return mode

    def _sumsq(self, b, a):
        self.close("sumsq out", a["out"].reshape(-1)[:1], *ref.sumsq_ref(b["x"], b["out"]))
        return f"sumsq {'f32' if b['x'].dtype == F32 else 'bf16'}"


def _vpl(nvec, top=8):
    need = (nvec + 31) // 32
    for v in (1, 2, 3, 4, 8, 16):
        if need <= v and v <= top:
            return v
    return 0


def _vpt(nvec):
    return 1 if nvec <= 256 else (2 if nvec <= 512 else 4)


@pytest.fixture
def K(C):
    return _Checker(C)


# ----------------------------------------------------------------------------------------------- guarded buffers
def _operand(t, pitch_multiple=8):
    return Guarded(t, float("nan"), pitch_multiple=pitch_multiple).view


def _flat_operand(t):
    """A contiguous operand: the 1-D guarded form reshaped."""
    return Guarded(t.reshape(-1).contiguous(), float("nan")).view.view(t.shape)


def _output(shape, dtype, start=float("nan"), flat=False):
    """An output inside a sentinel guard, starting at ``start`` (one-byte outputs: guard 0xA5, row pitch a multiple of 16)."""
    t = torch.full(shape, start, dtype=dtype, device="cuda")
    fill = 0xA5 if dtype == torch.uint8 else SENTINEL
    if flat or len(shape) != 2:
        g = Guarded(t.reshape(-1), fill)
        return g, g.view.view(shape)
    g = Guarded(t, fill, pitch_multiple=16 if dtype == torch.uint8 else 8)
    return g, g.view


def _accum_fill(shape, gen, scale):
    """An accumulated fp32 output in a 1-D guarded buffer, starting at non-zero values."""
    t = torch.randn(shape, generator=gen, device="cuda") * scale
    g = Guarded(t.reshape(-1), SENTINEL)
    return g, g.view.view(shape)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _intact(*gs):
    for g in gs:
        assert g.guards_intact(), "a kernel wrote outside its output"


# ----------------------------------------------------------------------------------------------- RMSNorm
RMS_H = [8, 136, 256, 264, 520, 776, 1032, 2048, 2056, 2560, 4096, 4104, 8192]


@pytest.mark.parametrize("M", [1, 7, 8, 9, 1500])
@pytest.mark.parametrize("H", RMS_H)
def test_rmsnorm(K, H, M):
    """Every VPL branch of the warp kernels (H <= 2048) and VPT branch of the block kernels, each boundary and one vector past
    it.  Forward with G = 0..4 dropout copies (by M) and the E4M3 copy (warp kernels); backward with and without dx_add.  Warps
    that loop over several rows are test_norm_backward_loops_over_rows."""
    g = _gen(H * 7 + M)
    K.case = f"M={M} H={H}"
    x = _flat_operand((torch.randn(M, H, generator=g, device="cuda") * 2.0 + 0.1).to(BF))
    w = _flat_operand((1.0 + 0.3 * torch.randn(H, generator=g, device="cuda")).to(BF))
    G = M % 5
    gy, y = _output((M, H), BF, flat=True)
    gr, rstd = _output((M,), F32)
    outs = [gy, gr]
    xd = seed = None
    keys = []
    if G:
        gx, xd = _output((M, G * H), BF, flat=True)
        outs.append(gx)
        seed = torch.tensor([1234567 + M], dtype=torch.int32, device="cuda")
        keys = [11 * k + 3 for k in range(G)]
    q8 = ()
    if H <= 2048 and M != 8:
        gq, q = _output((M, H), torch.uint8, start=0, flat=True)
        inv = torch.tensor([3.5], device="cuda")
        amax = torch.tensor([0.25], device="cuda")
        q8 = (q, inv, amax)
        outs.append(gq)
    K.call("rmsnorm_fwd", x, w, y, rstd, 1e-5, xd, seed, keys, 0.1 if G else 0.0, *q8)
    _intact(*outs)
    _rmsnorm_bwd_forms(K, x, w, rstd, g, (M % 2 == 1,))


def _rmsnorm_bwd_forms(K, x, w, rstd, g, with_add):
    M, H = x.shape
    dy = _flat_operand(torch.randn(M, H, generator=g, device="cuda").to(BF))
    for a in with_add:
        add = _flat_operand(torch.randn(M, H, generator=g, device="cuda").to(BF)) if a else None
        gdx, dx = _output((M, H), BF, flat=True)
        gdw, dw = _accum_fill((H,), g, 3.0)
        K.call("rmsnorm_bwd", dy, x, w, rstd, add, dx, dw, None, None)
        _intact(gdx, gdw)


def test_rmsnorm_shapes_of_the_earlier_sweep(K):
    for M, H in [(64, 768), (300, 2048), (17, 4096), (5, 128)]:
        g = _gen(M + H)
        K.case = f"M={M} H={H}"
        x = _flat_operand(torch.randn(M, H, generator=g, device="cuda").to(BF))
        w = _flat_operand((1.0 + 0.1 * torch.randn(H, generator=g, device="cuda")).to(BF))
        gy, y = _output((M, H), BF, flat=True)
        gr, rstd = _output((M,), F32)
        K.call("rmsnorm_fwd", x, w, y, rstd, 1e-6, None, None, [], 0.0)
        dy = _flat_operand(torch.randn(M, H, generator=g, device="cuda").to(BF))
        gdx, dx = _output((M, H), BF, flat=True)
        gdw, dw = _accum_fill((H,), g, 1.0)
        K.call("rmsnorm_bwd", dy, x, w, rstd, None, dx, dw, None, None)
        _intact(gy, gr, gdx, gdw)


# ----------------------------------------------------------------------------------------------- LayerNorm
LN_H = [8, 136, 256, 264, 520, 776, 1032, 2048, 2056, 2560, 4096]


@pytest.mark.parametrize("offset", [0.0, 64.0])
@pytest.mark.parametrize("M", [1, 9, 700])
@pytest.mark.parametrize("H", LN_H)
def test_layernorm(K, H, M, offset):
    """Forward at VPL 1..16 (bias or none, one or two norms, the dropout copies of each); backward up to 2048 in the module form
    and the executor's dual forms (dres, Σ dres into one or two outputs).  ``offset``: inputs with a large mean."""
    g = _gen(H * 3 + M + int(offset))
    K.case = f"M={M} H={H} offset={offset}"
    x = _flat_operand((torch.randn(M, H, generator=g, device="cuda") + offset).to(BF))
    w1 = _flat_operand((1.0 + 0.3 * torch.randn(H, generator=g, device="cuda")).to(BF))
    b1 = _flat_operand((0.2 * torch.randn(H, generator=g, device="cuda")).to(BF)) if M != 9 else None
    w2 = _flat_operand((1.0 + 0.3 * torch.randn(H, generator=g, device="cuda")).to(BF))
    b2 = _flat_operand((0.2 * torch.randn(H, generator=g, device="cuda")).to(BF))
    gy, y = _output((M, H), BF, flat=True)
    gm, mean = _output((M,), F32)
    gr, rstd = _output((M,), F32)
    K.call("layernorm_fwd", x, w1, b1, y, mean, rstd, 1e-5)
    _intact(gy, gm, gr)
    gy1, y1 = _output((M, H), BF, flat=True)
    gy2, y2 = _output((M, H), BF, flat=True)
    gx1, xd1 = _output((M, H), BF, flat=True)
    gx2, xd2 = _output((M, H), BF, flat=True)
    seed = torch.tensor([777 + H], dtype=torch.int32, device="cuda")
    K.call("layernorm_fwd", x, w1, b1, y1, mean, rstd, 1e-5, w2=w2, b2=b2, y2=y2, xd=xd1, xd2=xd2, seed=seed, keys=[5, 9], p=0.1)
    _intact(gy1, gy2, gx1, gx2, gm, gr)
    if H <= 2048:
        _layernorm_bwd_forms(K, x, w1, b1, w2, mean, rstd, g)


def _layernorm_bwd_forms(K, x, w1, b1, w2, mean, rstd, g):
    """The module form and the executor's dual forms: dres with Σ dres into one output, two norms with Σ dres into two outputs
    (ln_add_total) that start at the same non-zero values."""
    M, H = x.shape
    dy1 = _flat_operand(torch.randn(M, H, generator=g, device="cuda").to(BF))
    dy2 = _flat_operand(torch.randn(M, H, generator=g, device="cuda").to(BF))
    dres = _flat_operand(torch.randn(M, H, generator=g, device="cuda").to(BF))
    gdx, dx = _output((M, H), BF, flat=True)
    acc = [_accum_fill((H,), g, 2.0) for _ in range(4)]
    K.call("layernorm_bwd", dy1, x, w1, mean, rstd, dx, acc[0][1], acc[1][1] if b1 is not None else None)
    _intact(gdx, *(a[0] for a in acc))
    gdx, dx = _output((M, H), BF, flat=True)
    K.call("layernorm_bwd", dy1, x, w1, mean, rstd, dx, acc[0][1], acc[1][1], dres=dres, dres_sum=acc[2][1])
    _intact(gdx)
    gdx, dx = _output((M, H), BF, flat=True)
    gs1, s1 = _accum_fill((H,), g, 2.0)
    gs2, s2 = _accum_fill((H,), g, 2.0)
    s2.copy_(s1)
    K.call("layernorm_bwd", dy1, x, w1, mean, rstd, dx, acc[0][1], acc[1][1], dres=dres, dy2=dy2, w2=w2, dw2=acc[2][1], db2=acc[3][1],
           dres_sum=s1, dres_sum2=s2)
    _intact(gdx, gs1, gs2, *(a[0] for a in acc))


def _loop_rows():
    """Rows enough for every warp of the norm backward kernels to take at least three: 8 warps per block and at most 8 resident
    blocks per SM (2048 threads), while the grids are capped at one resident wave (RMSNorm) or 2 blocks per SM (LayerNorm)."""
    return 3 * 8 * 8 * torch.cuda.get_device_properties(0).multi_processor_count + 5


@pytest.mark.parametrize("H", [136, 264, 520, 776, 2048, 2560])
def test_norm_backward_loops_over_rows(K, H):
    """The backward kernels' per-warp row loops: dw / db / Σ dres carried across rows, and (RMSNorm VPL <= 4) the next row
    prefetched while the current one is reduced.  H covers RMSNorm VPL 1, 2, 3, 4, 8 and the block kernel, LayerNorm VPL 1..8."""
    M = _loop_rows()
    g = _gen(H + M)
    K.case = f"M={M} H={H}"
    x = _flat_operand((torch.randn(M, H, generator=g, device="cuda") * 2.0 + 0.1).to(BF))
    w = _flat_operand((1.0 + 0.3 * torch.randn(H, generator=g, device="cuda")).to(BF))
    gy, y = _output((M, H), BF, flat=True)
    gr, rstd = _output((M,), F32)
    K.call("rmsnorm_fwd", x, w, y, rstd, 1e-5, None, None, [], 0.0)
    _intact(gy, gr)
    _rmsnorm_bwd_forms(K, x, w, rstd, g, (True, False))
    if H > 2048:
        return
    b = _flat_operand((0.2 * torch.randn(H, generator=g, device="cuda")).to(BF))
    w2 = _flat_operand((1.0 + 0.3 * torch.randn(H, generator=g, device="cuda")).to(BF))
    gy, y = _output((M, H), BF, flat=True)
    gm, mean = _output((M,), F32)
    gr, rstd = _output((M,), F32)
    K.call("layernorm_fwd", x, w, b, y, mean, rstd, 1e-5)
    _intact(gy, gm, gr)
    _layernorm_bwd_forms(K, x, w, b, w2, mean, rstd, g)


def test_layernorm_shapes_of_the_earlier_sweep(K):
    for M, H, bias in [(300, 512, True), (257, 2048, True), (64, 768, False), (33, 1000, True)]:
        g = _gen(M + H)
        K.case = f"M={M} H={H}"
        x = _flat_operand(torch.randn(M, H, generator=g, device="cuda").to(BF))
        w = _flat_operand((1.0 + 0.1 * torch.randn(H, generator=g, device="cuda")).to(BF))
        b = _flat_operand((0.1 * torch.randn(H, generator=g, device="cuda")).to(BF)) if bias else None
        gy, y = _output((M, H), BF, flat=True)
        gm, mean = _output((M,), F32)
        gr, rstd = _output((M,), F32)
        K.call("layernorm_fwd", x, w, b, y, mean, rstd, 1e-5)
        dy = _flat_operand(torch.randn(M, H, generator=g, device="cuda").to(BF))
        gdx, dx = _output((M, H), BF, flat=True)
        gdw, dw = _accum_fill((H,), g, 1.0)
        gdb, db = _accum_fill((H,), g, 1.0)
        K.call("layernorm_bwd", dy, x, w, mean, rstd, dx, dw, db if bias else None)
        _intact(gy, gm, gr, gdx, gdw, gdb)


# ----------------------------------------------------------------------------------------------- cross-entropy
CE_V = [8, 1000, 1001, 1002, 1003, 1004, 1005, 1006, 1007, 32100, 50257, 102391]


@pytest.mark.parametrize("regime", ["random", "equal", "dominant", "huge"])
@pytest.mark.parametrize("V", CE_V)
def test_cross_entropy(K, V, regime):
    """Vocabulary tails V % 8 = 0..7 up to ~100 K (shared-memory limit of the single-pass kernel), labels at column 0, V − 1 and
    in the tail, ignored rows, grad_scale != 1; logits random, all equal, one dominant, |x| in the thousands.  The logits sit at
    a row pitch above V: the columns past V must keep their bits."""
    M = 11
    g = _gen(V + len(regime))
    K.case = f"V={V} {regime}"
    x = torch.randn(M, V, generator=g, device="cuda") * 2.0
    if regime == "equal":
        x = torch.full((M, V), 0.75, device="cuda")
    elif regime == "dominant":
        x[torch.arange(M), torch.arange(M) * 7 % V] += 40.0
    elif regime == "huge":
        x = x * 1500.0
    lab = torch.randint(0, V, (M,), generator=g, device="cuda")
    lab[0], lab[1], lab[2] = 0, V - 1, V - 1 - (V % 8) // 2
    lab[3] = -100
    lab[7] = -100
    logits = Guarded(x.to(BF), SENTINEL, pitch_multiple=8)
    loss = torch.tensor([2.5], device="cuda")
    count = torch.tensor([3.0], device="cuda")
    K.call("cross_entropy_fwd_bwd", logits.view, lab, V, 0.37 if V % 2 else 1.0, -100, loss, count)
    assert logits.guards_intact(), "cross_entropy wrote outside the logits"


# ----------------------------------------------------------------------------------------------- rotary
def _tables(rot, n_pos, fp32=False, base=10000.0):
    cos, sin = ref.rope_tables(rot, n_pos, base, device="cuda")
    return (cos, sin) if fp32 else (cos.to(BF).contiguous(), sin.to(BF).contiguous())


@pytest.mark.parametrize("pos0", [0, 37])
@pytest.mark.parametrize("nh,nkv", [(4, 4), (4, 2), (8, 1)])
@pytest.mark.parametrize("hd,rot", [(48, 48), (64, 64), (64, 16), (64, 8), (128, 128), (128, 16), (256, 256), (256, 8)])
def test_rope(K, hd, rot, nh, nkv, pos0):
    """rope_inplace forward and backward on the packed [q | k | v] buffer at a row pitch above the width (rotary_dim = 8 forces
    the scalar kernel); rope_pack_bwd from strided [B, T, heads, hd] views (the layout the executors pass) into a guarded dQKV."""
    B, T = 2, 45
    g = _gen(hd * 13 + rot + nh + nkv + pos0)
    K.case = f"hd={hd} rot={rot} nh={nh} nkv={nkv} pos0={pos0}"
    W = (nh + 2 * nkv) * hd
    cos, sin = _tables(rot, T + pos0 + 3)
    for backward in (False, True):
        buf = Guarded(torch.randn(B * T, W, generator=g, device="cuda").to(BF), SENTINEL, pitch_multiple=8)
        K.call("rope_inplace", buf.view, T, nh + nkv, hd, rot, cos, sin, backward, pos0)
        assert buf.guards_intact()
    if rot % 16:
        return
    def heads(n, parts=1):  # strided [B, n, T, hd] views of a [B·T, parts·n·hd] guarded buffer, as the executors pass them
        t = _operand(torch.randn(B * T, parts * n * hd, generator=g, device="cuda").to(BF)).view(B, T, parts, n, hd)
        return [t[:, :, i].transpose(1, 2) for i in range(parts)]

    if nkv == nh:  # one stride set for all three
        dq, dk, dv = heads(nh, 3)
    else:
        (dq,), (dk, dv) = heads(nh), heads(nkv, 2)
    out = Guarded(torch.full((B * T, W), float("nan"), device="cuda").to(BF), SENTINEL, pitch_multiple=8)
    K.call("rope_pack_bwd", dq, dk, dv, out.view, rot, cos, sin, pos0, nkv=nkv)
    assert out.guards_intact()


@pytest.mark.parametrize("nh,hd,rot", [(8, 64, 16), (4, 128, 32), (2, 256, 64), (4, 64, 64), (4, 80, 20)])
@pytest.mark.parametrize("pos0", [0, 5])
def test_neox_rope(K, nh, hd, rot, pos0):
    T, B = 33, 3
    g = _gen(nh + hd + rot + pos0)
    K.case = f"nh={nh} hd={hd} rot={rot} pos0={pos0}"
    cos, sin = _tables(rot, T + pos0, fp32=True)
    for inverse in (False, True):
        buf = Guarded(torch.randn(B * T, nh * 3 * hd, generator=g, device="cuda").to(BF), SENTINEL, pitch_multiple=8)
        K.call("neox_rope", buf.view, T, nh, hd, rot, cos, sin, pos0, inverse)
        assert buf.guards_intact()


# ----------------------------------------------------------------------------------------------- SwiGLU / GELU
def _wide_z(M, N, g, top=90.0):
    z = torch.randn(M, N, generator=g, device="cuda") * 3.0
    z[0] = torch.linspace(-top, top, N, device="cuda")
    return z


@pytest.mark.parametrize("M,F", [(1, 8), (3, 264), (77, 1000), (300, 2048), (1029, 1376)])
def test_swiglu(K, M, F):
    g = _gen(M + F)
    K.case = f"M={M} F={F}"
    gu = _operand(torch.cat([_wide_z(M, F, g), torch.randn(M, F, generator=g, device="cuda")], 1).to(BF))
    gh, h = _output((M, F), BF)
    ghd, hd = _output((M, F), BF)
    gq, q = _output((M, F), torch.uint8, start=0)
    seed = torch.tensor([99 + M], dtype=torch.int32, device="cuda")
    K.call("swiglu_fwd", gu, h, hd, seed, 17, 0.1, q, torch.tensor([2.0], device="cuda"), torch.tensor([0.5], device="cuda"))
    gh2, h2 = _output((M, F), BF)
    K.call("swiglu_fwd", gu, h2)
    dh = _operand(torch.randn(M, F, generator=g, device="cuda").to(BF))
    gd, dgu = _output((M, 2 * F), BF)
    K.call("swiglu_bwd", dh, gu, dgu)
    _intact(gh, ghd, gq, gh2, gd)


@pytest.mark.parametrize("tanh_approx", [False, True])
@pytest.mark.parametrize("M,N", [(1, 8), (5, 264), (300, 1024), (97, 4104), (2000, 768)])
def test_gelu(K, M, N, tanh_approx):
    g = _gen(M + N + int(tanh_approx))
    K.case = f"M={M} N={N} tanh={tanh_approx}"
    z = _flat_operand(_wide_z(M, N, g).to(BF))
    ga, a = _output((M, N), BF, flat=True)
    K.call("gelu_fwd", z, a, tanh_approx)
    gx, xd = _output((M, N), BF, flat=True)
    ga2, a2 = _output((M, N), BF, flat=True)
    K.call("gelu_fwd", z, a2, tanh_approx, xd=xd, seed=torch.tensor([5], dtype=torch.int32, device="cuda"), key=3, p=0.1)
    da = _flat_operand(torch.randn(M, N, generator=g, device="cuda").to(BF))
    gdz, dz = _output((M, N), BF, flat=True)
    K.call("gelu_bwd", da, z, dz, tanh_approx)
    gdz2, dz2 = _output((M, N), BF, flat=True)
    gdb, db = _accum_fill((N,), g, 1.0)
    K.call("gelu_bwd", da, z, dz2, tanh_approx, dbias=db)
    gcs, cs = _accum_fill((N,), g, 1.0)
    K.call("colsum", da, cs)
    _intact(ga, gx, ga2, gdz, gdz2, gdb, gcs)


# ----------------------------------------------------------------------------------------------- embedding, dropout, misc
@pytest.mark.parametrize("M,H,V", [(1, 8, 3), (300, 256, 50), (4099, 264, 1000)])
def test_embedding(K, M, H, V):
    g = _gen(M + H + V)
    K.case = f"M={M} H={H} V={V}"
    ids = torch.randint(0, V, (M,), generator=g, device="cuda")
    ids[::5] = 1  # a frequent id and the padding id
    table = _flat_operand(torch.randn(V, H, generator=g, device="cuda").to(BF))
    go, out = _output((M, H), BF, flat=True)
    K.call("embedding_fwd", ids, table, out)
    dout = _flat_operand(torch.randn(M, H, generator=g, device="cuda").to(BF))
    for pad in (-1, 1):
        gt, dt = _accum_fill((V, H), g, 1.0)
        K.call("embedding_bwd", ids, dout, dt, pad)
        srt = torch.sort(ids, stable=True)
        gt2, dt2 = _accum_fill((V, H), g, 1.0)
        keep = dt2.clone()
        K.call("embedding_bwd_sorted", srt.values, srt.indices, dout, dt2, pad)
        first = dt2.clone()
        dt2.copy_(keep)
        K.call("embedding_bwd_sorted", srt.values, srt.indices, dout, dt2, pad)
        assert torch.equal(first, dt2), "embedding_bwd_sorted is not bit-reproducible"
        _intact(gt, gt2)
    _intact(go)


@pytest.mark.parametrize("M,H,G", [(1, 8, 1), (37, 264, 2), (300, 1024, 3), (129, 2048, 4)])
def test_dropout_expand_and_combine(K, M, H, G):
    g = _gen(M + H + G)
    K.case = f"M={M} H={H} G={G}"
    x = _flat_operand(torch.randn(M, H, generator=g, device="cuda").to(BF))
    seed = torch.tensor([31337 + G], dtype=torch.int32, device="cuda")
    keys = [101 + k for k in range(G)]
    gxd, xd = _output((M, G * H), BF, flat=True)
    gq, q = _output((M, H), torch.uint8, start=0)
    K.call("dropout_expand", x, xd, seed, keys, 0.25, q, torch.tensor([16.0], device="cuda"), torch.tensor([1.0], device="cuda"))
    parts2 = _operand(torch.randn(M, G * H, generator=g, device="cuda").to(BF))
    parts3 = _flat_operand(torch.randn(G, M, H, generator=g, device="cuda").to(BF))
    for parts, base in ((parts2, x), (parts3, None)):
        go, out = _output((M, H), BF, flat=True)
        K.call("dropout_combine", base, parts, out, seed, keys, 0.25)
        _intact(go)
    _intact(gxd, gq)


@pytest.mark.parametrize("R,C_", [(16, 16), (200, 272), (1024, 768)])
def test_fp8_quantisers(K, R, C_):
    g = _gen(R + C_)
    K.case = f"{R}x{C_}"
    w = _operand((torch.randn(R, C_, generator=g, device="cuda") * 0.05).to(BF))
    gq, q = _output((R, C_), torch.uint8, start=0)
    gt, qt = _output((C_, R), torch.uint8, start=0)
    sc = [torch.full((1,), 7.0, device="cuda") for _ in range(3)]
    K.call("fp8_quantize_weight", w, q, sc[0], sc[1], sc[2], qt)
    x = _operand((torch.randn(R, C_, generator=g, device="cuda") * 100.0).to(BF))  # saturates at inv = 8
    for e5m2, inv in ((False, 8.0), (True, 400.0)):
        gx, x8 = _output((R, C_), torch.uint8, start=0)
        K.call("fp8_quantize_act", x, x8, torch.tensor([inv], device="cuda"), torch.tensor([3.0], device="cuda"), e5m2)
        _intact(gx)
    n = 13
    state = torch.rand(n, 2, generator=g, device="cuda") * 10
    state[::3, 1] = 0.0
    K.call("fp8_prep", state, torch.rand(n, generator=g, device="cuda") + 0.01, torch.empty(n, device="cuda"),
           torch.empty(n, device="cuda"), torch.empty(n, device="cuda"), 1.25, 9)
    _intact(gq, gt)


def test_cast_and_transpose(K):
    g = _gen(4)
    x = _flat_operand(torch.randn(1000, 264, generator=g, device="cuda") * 1e3)
    go, out = _output((1000, 264), BF, flat=True)
    K.call("cast_f32_to_bf16", x, out, 0.37)
    src = _operand(torch.randn(77, 45, generator=g, device="cuda").to(BF))
    gt, t = _output((45, 77), BF)
    K.call("transpose", src, t)
    _intact(go, gt)


# ----------------------------------------------------------------------------------------------- optimizer
_PASS = 132 * 8 * 256 * 8  # elements one grid-stride pass of adamw_flat covers on 132 SMs


@pytest.mark.parametrize("gdt,sdt", [(BF, BF), (F32, BF), (F32, F32)])
@pytest.mark.parametrize("n", [8000, 3 * _PASS + 8 * 37])
def test_adamw_flat(K, gdt, sdt, n):
    """Step 1 and step 10⁴ from the host, and from the device step counter with a device grad scale; v = 0 rows (denominator eps)
    and tiny gradients; n past several grid-stride passes."""
    g = _gen(n + (gdt == F32) + 2 * (sdt == F32))
    K.case = f"n={n} g={gdt} s={sdt}"
    for step, dev in ((1, False), (10000, False), (7, True)):
        p = _flat_operand(torch.randn(n, generator=g, device="cuda").to(BF))
        grad = torch.randn(n, generator=g, device="cuda") * 0.01
        grad[:64] = 1e-10  # √v' far below eps
        grad = _flat_operand(grad.to(gdt))
        m = _flat_operand((torch.randn(n, generator=g, device="cuda") * 0.01).to(sdt))
        v = (torch.rand(n, generator=g, device="cuda") * 1e-4)
        v[:64] = 0.0
        v = _flat_operand(v.to(sdt))
        gs = torch.tensor([0.8], device="cuda") if dev else None
        step_dev = torch.tensor([float(step)], device="cuda") if dev else None
        K.call("adamw_flat", p, grad, m, v, 1e-3, 0.9, 0.999, 1e-8, 0.1, step, gs, 1.0 if dev else 0.5, None, step_dev)
    p = _flat_operand(torch.randn(n, generator=g, device="cuda").to(BF))
    grad = _flat_operand(torch.randn(n, generator=g, device="cuda").to(gdt))
    m = _flat_operand(torch.zeros(n, device="cuda").to(sdt))
    v = _flat_operand(torch.zeros(n, device="cuda").to(sdt))
    assert K.call("adamw_flat", p, grad, m, v, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, None, 1.0, torch.ones(1, device="cuda"), None).endswith("skipped")
    for bad in (float("nan"), float("inf")):  # a non-finite gradient norm upstream poisons the scale: the update is skipped
        assert K.call("adamw_flat", p, grad, m, v, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, torch.tensor([bad], device="cuda"), 1.0, None,
                      None).endswith("skipped")


@pytest.mark.parametrize("dtype", [BF, F32])
@pytest.mark.parametrize("n", [1, 777, 1024 * 256 + 99, 5_000_003])
def test_sumsq(K, n, dtype):
    g = _gen(n)
    K.case = f"n={n} {dtype}"
    x = _flat_operand(torch.randn(n, generator=g, device="cuda").to(dtype))
    outs = []
    for _ in range(2):
        o = torch.tensor([1.5], device="cuda")
        K.call("sumsq", x, o)
        outs.append(o)
    assert torch.equal(outs[0], outs[1]), "sumsq is not bit-reproducible"


# ----------------------------------------------------------------------------------------------- host refusals
def test_rope_refuses_misaligned_or_mismatched_operands(C):
    """The scalar rotary kernel makes 4-byte accesses and rope_pack_bwd 16-byte ones: views that break that alignment, tables
    too short for T + pos0 or not rotary_dim wide are refused on the host, before any launch."""
    T, nh, hd = 16, 2, 64
    cos, sin = _tables(hd, T)
    base = torch.zeros(T, 3 * nh * hd + 2, dtype=BF, device="cuda")
    with pytest.raises(RuntimeError, match="aligned"):
        C.rope_inplace(base[:, 1:1 + 3 * nh * hd], T, 2 * nh, hd, 8, *_tables(8, T), False, 0)
    with pytest.raises(RuntimeError, match="rotary table"):
        C.rope_inplace(base[:, :3 * nh * hd], T, 2 * nh, hd, hd, cos, sin, False, 5)
    dq = torch.zeros(1, nh, T, hd, dtype=BF, device="cuda")
    out = torch.zeros(T, 3 * nh * hd + 8, dtype=BF, device="cuda")
    with pytest.raises(RuntimeError, match="rotary table"):
        C.rope_pack_bwd(dq, dq, dq, out[:, :3 * nh * hd], hd, cos, sin, 1)
    with pytest.raises(RuntimeError, match="rotary_dim"):
        C.rope_pack_bwd(dq, dq, dq, out[:, :3 * nh * hd], 32, cos, sin, 0)
    with pytest.raises(RuntimeError, match="aligned"):
        C.rope_pack_bwd(dq, dq, dq, out[:, 4:4 + 3 * nh * hd], hd, cos, sin, 0)
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------- executor audit
def _info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")


def _relora_llama(nkv=4, inter=512, dropout=0.1):
    from relora_b200.models import LlamaForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cfg = SimpleConfig(model_type="llama", vocab_size=1000, hidden_size=256, intermediate_size=inter, num_hidden_layers=2,
                       num_attention_heads=4, num_key_value_heads=nkv, rope_theta=10000.0, rms_norm_eps=1e-6, pad_token_id=-1,
                       max_position_embeddings=256)
    torch.manual_seed(0)
    w = ReLoRaModel(LlamaForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=dropout, target_modules=["attn", "mlp"],
                    init_lora_a="kaiming")
    for mod in w.relora_modules():
        torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
    return w.cuda().to(BF)


def _pythia(parallel):
    from relora_b200.models import GPTNeoXForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cfg = SimpleConfig(model_type="gpt_neox", vocab_size=1000, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                       intermediate_size=1024, rotary_pct=0.25, max_position_embeddings=128, layer_norm_eps=1e-5,
                       use_parallel_residual=parallel, hidden_act="gelu", rotary_emb_base=10000, tie_word_embeddings=False)
    torch.manual_seed(0)
    w = ReLoRaModel(GPTNeoXForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=0.1, target_modules=["attn", "attention", "mlp"],
                    init_lora_a="kaiming")
    with torch.no_grad():
        for mod in w.relora_modules():
            torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
            torch.nn.init.normal_(mod.bias, std=0.02)
    return w.cuda().to(BF).train()


_CONFIGS = ["llama_mha", "llama_p0", "llama_gqa", "llama_ragged_f", "llama_fp8", "llama_atomic_embedding", "pythia_parallel",
            "pythia_sequential"]
_AUDIT = {  # configuration -> the call forms of one micro-step, one eval_loss and one update(); a path that starts issuing
    # another form shows up here
    'llama_mha': {
        'adamw_flat g=f32 s=bf16 step=dev', 'ce V%8=0 ignored scaled', 'dropout_expand G=1', 'embedding_bwd sorted',
        'embedding_fwd', 'rmsnorm_bwd warp VPL=1 prefetch', 'rmsnorm_bwd warp VPL=1 prefetch dx_add',
        'rmsnorm_fwd warp VPL=1 G=0', 'rmsnorm_fwd warp VPL=1 G=2', 'rmsnorm_fwd warp VPL=1 G=3', 'rope_inplace vec bwd',
        'rope_inplace vec fwd', 'seed_advance', 'swiglu_bwd', 'swiglu_fwd', 'swiglu_fwd dropout',
    },
    'llama_p0': {
        'adamw_flat g=f32 s=bf16 step=dev', 'ce V%8=0 ignored scaled', 'embedding_bwd sorted', 'embedding_fwd',
        'rmsnorm_bwd warp VPL=1 prefetch', 'rmsnorm_bwd warp VPL=1 prefetch dx_add', 'rmsnorm_fwd warp VPL=1 G=0',
        'rope_inplace vec bwd', 'rope_inplace vec fwd', 'seed_advance', 'swiglu_bwd', 'swiglu_fwd',
    },
    'llama_gqa': {
        'adamw_flat g=f32 s=bf16 step=dev', 'ce V%8=0 ignored scaled', 'dropout_expand G=1', 'embedding_bwd sorted',
        'embedding_fwd', 'rmsnorm_bwd warp VPL=1 prefetch', 'rmsnorm_bwd warp VPL=1 prefetch dx_add',
        'rmsnorm_fwd warp VPL=1 G=0', 'rmsnorm_fwd warp VPL=1 G=2', 'rmsnorm_fwd warp VPL=1 G=3', 'rope_inplace vec bwd',
        'rope_inplace vec fwd', 'seed_advance', 'swiglu_bwd', 'swiglu_fwd', 'swiglu_fwd dropout',
    },
    'llama_ragged_f': {
        'adamw_flat g=f32 s=bf16 step=dev', 'ce V%8=0 ignored scaled', 'dropout_expand G=1', 'embedding_bwd sorted',
        'embedding_fwd', 'rmsnorm_bwd warp VPL=1 prefetch', 'rmsnorm_bwd warp VPL=1 prefetch dx_add',
        'rmsnorm_fwd warp VPL=1 G=0', 'rmsnorm_fwd warp VPL=1 G=2', 'rmsnorm_fwd warp VPL=1 G=3', 'rope_inplace vec bwd',
        'rope_inplace vec fwd', 'seed_advance', 'swiglu_bwd', 'swiglu_fwd', 'swiglu_fwd dropout',
    },
    'llama_fp8': {
        'adamw_flat g=f32 s=bf16 step=dev', 'ce V%8=0 ignored scaled', 'dropout_expand G=1 e4m3', 'embedding_bwd sorted',
        'embedding_fwd', 'fp8_prep', 'fp8_quantize_act e4m3 amax', 'rmsnorm_bwd warp VPL=1 prefetch',
        'rmsnorm_bwd warp VPL=1 prefetch dx_add', 'rmsnorm_fwd warp VPL=1 G=0', 'rmsnorm_fwd warp VPL=1 G=2 e4m3',
        'rmsnorm_fwd warp VPL=1 G=3 e4m3', 'rope_inplace vec bwd', 'rope_inplace vec fwd', 'seed_advance', 'swiglu_bwd',
        'swiglu_fwd dropout e4m3', 'swiglu_fwd e4m3',
    },
    'llama_atomic_embedding': {
        'adamw_flat g=f32 s=bf16 step=dev', 'ce V%8=0 ignored scaled', 'dropout_expand G=1', 'embedding_bwd atomic',
        'embedding_fwd', 'rmsnorm_bwd warp VPL=1 prefetch', 'rmsnorm_bwd warp VPL=1 prefetch dx_add',
        'rmsnorm_fwd warp VPL=1 G=0', 'rmsnorm_fwd warp VPL=1 G=2', 'rmsnorm_fwd warp VPL=1 G=3', 'rope_inplace vec bwd',
        'rope_inplace vec fwd', 'seed_advance', 'swiglu_bwd', 'swiglu_fwd', 'swiglu_fwd dropout',
    },
    'pythia_parallel': {
        'adamw_flat g=f32 s=bf16 step=dev', 'ce V%8=0 ignored scaled', 'colsum', 'dropout_expand G=1', 'embedding_bwd sorted',
        'embedding_fwd', 'gelu_bwd erf dbias', 'gelu_fwd erf', 'gelu_fwd erf dropout',
        'layernorm_bwd VPL=1 dual bias two dres sum sum2', 'layernorm_bwd VPL=1 module bias', 'layernorm_fwd VPL=1 bias',
        'layernorm_fwd VPL=1 bias dual', 'layernorm_fwd VPL=1 bias dual xd xd2', 'neox_rope fwd', 'neox_rope inverse',
        'seed_advance',
    },
    'pythia_sequential': {
        'adamw_flat g=f32 s=bf16 step=dev', 'ce V%8=0 ignored scaled', 'colsum', 'dropout_expand G=1', 'embedding_bwd sorted',
        'embedding_fwd', 'gelu_bwd erf dbias', 'gelu_fwd erf', 'gelu_fwd erf dropout', 'layernorm_bwd VPL=1 dual bias dres sum',
        'layernorm_bwd VPL=1 module bias', 'layernorm_fwd VPL=1 bias', 'layernorm_fwd VPL=1 bias xd', 'neox_rope fwd',
        'neox_rope inverse', 'seed_advance',
    },
}


@pytest.mark.parametrize("config", _CONFIGS)
def test_executor_rowwise_calls_match_the_reference(C, config, monkeypatch):
    """Every non-GEMM, non-attention call of one training micro-step, one evaluation and one update (CUDA graphs off, 3 x 97
    tokens) checked against its reference; the set of modes seen must be the expected one."""
    from relora_b200.ops import fused

    dev = torch.device("cuda", 0)
    monkeypatch.setenv("RELORA_B200_ATOMIC_EMBEDDING", "1" if config == "llama_atomic_embedding" else "0")
    if config.startswith("pythia"):
        from relora_b200.engine.fused_pythia import FusedPythiaStepper

        st = FusedPythiaStepper(_pythia(config == "pythia_parallel"), _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=False)
    else:
        from relora_b200.engine.fused_llama import FusedLlamaStepper

        model = _relora_llama(nkv=2 if config == "llama_gqa" else 4, inter=440 if config == "llama_ragged_f" else 512,
                              dropout=0.0 if config == "llama_p0" else 0.1)
        st = FusedLlamaStepper(model, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=False, fp8=config == "llama_fp8",
                               weight_decay=0.01)
    ids = torch.randint(0, 1000, (3, 97), device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    fused.seed_state.set(dev, 4321)
    audit = _Checker(C)
    audit.case = config
    audit.install(monkeypatch)
    loss = st.micro_step(ids)
    ev = st.eval_loss(ids)
    st.update()
    torch.cuda.synchronize()
    assert torch.isfinite(loss) and torch.isfinite(ev)
    calls = sum(audit.modes.values())
    print(f"[rowwise modes] audit {config}: {calls} calls, worst ratio {audit.worst:.3g}, modes {dict(sorted(audit.modes.items()))}")
    _note(WORST, "audit", audit.worst, config)
    assert set(audit.modes) == _AUDIT[config]
