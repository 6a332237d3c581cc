"""The block-scaled MXFP8 kernels (csrc/gemm_mx.cu) against the exact contract of ops/reference.py (block-scaled MXFP8
section): the quantisers byte for byte, the dequantiser bit for bit and gemm_mx element by element with assert_gemm_close, on
guarded buffers, plus an audit of every such call one forward, backward and merge of a quantised Llama issues (H100: -m gpu).

Operands have a power-of-two magnitude of their own per 32-block (rows) or 32 x 32 tile (weights), so a scale read from the
wrong row group, k column or layout changes the result.  Byte operands sit inside 0x7F (E4M3 NaN) and scale arrays inside 0xFF
(Inf scale), so a read past the extents given shows as NaN; outputs start as NaN inside a sentinel that must survive.  Every
call goes through _Checker: it clones the inputs after a device synchronise, runs the kernel, synchronises and checks every
output.  The GEMM operands are built by the reference quantisers, so a GEMM check does not depend on the CUDA quantisers."""
import pytest
import torch

from guarded_buffers import Guarded
from relora_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
SENTINEL = 1234.0
WORST = {}  # worst error/tolerance ratio per gemm_mx mode (printed at the end of the module with -s)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for mode, (w, case) in sorted(WORST.items()):
        print(f"[mx modes] {mode}: worst ratio {w:.3g} ({case})")


@pytest.fixture(scope="module")
def C():
    from relora_b200.ops import native

    return native.require()


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cap_threads():
    """Threads of the capped grid of the quantise / dequantise kernels (num_sms·16 blocks of 256)."""
    return _num_sms() * 16 * 256


def _pad(n):
    return (n + 127) // 128 * 128


# ----------------------------------------------------------------------------------------------- the checker
_SIGS = {
    "mx_quantize_rows": ("x q sf", {}),
    "mx_quantize_weight_2d": ("w delta q sf_fwd sf_bwd N K", {}),
    "mx_dequantize_weight": ("q sf_fwd out", {}),
    "gemm_mx": ("a sfa b sfb out M N K b_mn_major a2 b2 residual", dict(b_mn_major=False, a2=None, b2=None, residual=None)),
}


def _bind(name, args, kw):
    names, defaults = _SIGS[name]
    a = dict(defaults)
    a.update(zip(names.split(), args))
    a.update(kw)
    return a


def _same_or_both_nan(name, got, want):
    """bf16 results equal bit for bit, a NaN matching any NaN."""
    g, w = got.float(), want.to(got.device).float()
    nan = torch.isnan(w)
    assert torch.equal(torch.isnan(g), nan), f"{name}: NaN where none is expected, or a NaN missing"
    ref.assert_bitwise_equal(name, got[~nan], want.to(got.device)[~nan])


class _Checker:
    """Runs extension calls checked against the exact MXFP8 contract; records the mode of each call and the worst ratio."""

    def __init__(self, C):
        self.C = C
        self.orig = {n: getattr(C, n) for n in _SIGS}
        self.modes, self.worst, self.case = {}, 0.0, ""

    def install(self, monkeypatch):
        for n in _SIGS:
            monkeypatch.setattr(self.C, n, (lambda name: lambda *a, **k: self.call(name, *a, **k))(n))

    def call(self, name, *args, **kw):
        a = _bind(name, args, kw)
        torch.cuda.synchronize()
        b = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in a.items()}
        self.orig[name](*args, **kw)
        torch.cuda.synchronize()
        mode = getattr(self, "_" + name)(b, a)
        self.modes[mode] = self.modes.get(mode, 0) + 1
        return mode

    def _mx_quantize_rows(self, b, a):
        M, K = b["x"].shape
        q, sf = ref.mx_quantize_rows_exact(b["x"])
        ref.assert_e4m3_bytes_equal("mx_quantize_rows q", a["q"][:M, :_pad(K)], q)
        ref.assert_bitwise_equal("mx_quantize_rows sf", a["sf"].reshape(-1)[:sf.numel()], sf)
        loops = _pad(M) * (_pad(K) // 128) * 32 > _cap_threads()
        return f"quantize_rows{' grid-stride' if loops else ''}"

    def _mx_quantize_weight_2d(self, b, a):
        N, K = int(b["N"]), int(b["K"])
        if b["w"] is not None:
            q, f, bw = ref.mx_quantize_weight_2d_exact(b["w"], delta=b["delta"], N=N, K=K)
        else:
            q, f, bw = ref.mx_quantize_weight_2d_exact(q_old=b["q"], sf_old=b["sf_fwd"], delta=b["delta"], N=N, K=K)
        ref.assert_e4m3_bytes_equal("mx_quantize_weight_2d q", a["q"][:_pad(N), :_pad(K)], q)
        ref.assert_bitwise_equal("mx_quantize_weight_2d sf_fwd", a["sf_fwd"].reshape(-1)[:f.numel()], f)
        ref.assert_bitwise_equal("mx_quantize_weight_2d sf_bwd", a["sf_bwd"].reshape(-1)[:bw.numel()], bw)
        loops = (_pad(N) // 32) * (_pad(K) // 32) * 32 > _cap_threads()
        return f"quantize_weight_2d {'bf16' if b['w'] is not None else 'merge'}{' grid-stride' if loops else ''}"

    def _mx_dequantize_weight(self, b, a):
        N, K = a["out"].shape
        want = ref.mx_decode_weight(b["q"], b["sf_fwd"], N, K).float().to(BF)
        _same_or_both_nan("mx_dequantize_weight", a["out"], want)
        return f"dequantize_weight{' grid-stride' if N * K // 4 > _cap_threads() else ''}"

    def _gemm_mx(self, b, a):
        M, N, K = int(b["M"]), int(b["N"]), int(b["K"])
        r, bound = ref.gemm_mx_ref(b["a"], b["sfa"], b["b"], b["sfb"], M, N, K, b["b_mn_major"], b["a2"], b["b2"], b["residual"])
        out = a["out"][:M, :N]
        fin = torch.isfinite(r)
        assert torch.equal(torch.isfinite(out.float()), fin), "gemm_mx: non-finite outputs differ from the reference's"
        o = torch.where(fin, out, torch.zeros((), dtype=out.dtype, device=out.device))
        z = torch.zeros((), dtype=r.dtype, device=r.device)
        w = ref.assert_gemm_close(o, torch.where(fin, r, z), torch.where(fin, bound, z), fp8=True)
        tiles = -(-M // 128) * -(-N // 128)
        k2 = 0 if b["a2"] is None else b["a2"].shape[1]
        mode = (f"gemm_mx {'MN' if b['b_mn_major'] else 'K'}-major K2={k2}{' residual' if b['residual'] is not None else ''}"
                f"{' persistent' if tiles > _num_sms() else ''}")
        self.worst = max(self.worst, w)
        if w > WORST.get(mode, (-1.0, ""))[0]:
            WORST[mode] = (w, self.case)
        return mode


@pytest.fixture
def K_(C):
    return _Checker(C)


# ----------------------------------------------------------------------------------------------- operands
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def block_scaled(rows, cols, g, tile_rows, spread=5):
    """bf16 ``[rows, cols]``; block (i, j) of ``tile_rows`` x 32 has magnitude 2^((i + 2j) mod spread - spread // 2)."""
    i = torch.arange(rows, device="cuda").unsqueeze(1) // tile_rows
    j = torch.arange(cols, device="cuda").unsqueeze(0) // 32
    e = ((i + 2 * j) % spread - spread // 2).float()
    return (torch.randn(rows, cols, generator=g, device="cuda") * torch.exp2(e)).to(BF)


def _bf16_neighbours(x):
    b = int(torch.tensor([x], dtype=torch.float32).to(BF).view(torch.int16))
    return [float(torch.tensor([b + d], dtype=torch.int16).view(BF).float()) for d in (-1, 0, 1)]


def with_boundaries(x, tile_rows):
    """Put block maxima exactly on 448·2^e and on its bf16 neighbours, one block of bf16 subnormals and one zero block."""
    R, Kc = x.shape
    for t in range(min(R // tile_rows, 30)):
        r = t * tile_rows + (t % tile_rows)
        v = _bf16_neighbours(448.0 * 2.0 ** (t % 10 - 2))[t % 3]
        x[r, (t * 7) % Kc] = -v if t % 2 else v
    x[-1, :32] = torch.tensor(_bf16_neighbours(2.0 ** -131) * 10 + [0.0, -(2.0 ** -133)], device="cuda")[:min(32, Kc)].to(BF)
    if R > 2:
        x[R // 2, :32] = 0
    return x


def _operand(t):
    return Guarded(t, float("nan"), pitch_multiple=8).view


def _bytes(t):
    return Guarded(t, 0x7F, pitch_multiple=16).view


def _scales(t):
    return Guarded(t, 0xFF).view


def _out(shape, dtype):
    if dtype == torch.uint8:
        start, fill = (0xFF, 0xA5) if len(shape) == 1 else (0x7F, 0xA5)
        g = Guarded(torch.full(shape, start, dtype=dtype, device="cuda"), fill, pitch_multiple=16)
    else:
        g = Guarded(torch.full(shape, float("nan"), dtype=dtype, device="cuda"), SENTINEL, pitch_multiple=8)
    return g, g.view


def _intact(*gs):
    for g in gs:
        assert g.guards_intact(), "a kernel wrote outside its output"


def _quantize_rows(K_, x):
    M, K = x.shape
    gq, q = _out((M, _pad(K)), torch.uint8)
    gs, sf = _out((ref.mx_sf_bytes(M, K),), torch.uint8)
    K_.call("mx_quantize_rows", _operand(x), q, sf)
    _intact(gq, gs)
    return q, sf


def _quantize_weight(K_, w):
    N, K = w.shape
    gq, q = _out((_pad(N), _pad(K)), torch.uint8)
    gf, f = _out((ref.mx_sf_bytes(N, K),), torch.uint8)
    gb, bw = _out((ref.mx_sf_bytes(K, N),), torch.uint8)
    K_.call("mx_quantize_weight_2d", _operand(w), None, q, f, bw, N, K)
    _intact(gq, gf, gb)
    return (gq, q), (gf, f), (gb, bw)


def _dequantize(K_, q, f, N, K):
    go, out = _out((N, K), BF)
    K_.call("mx_dequantize_weight", q, f, out)
    _intact(go)
    return out


# ----------------------------------------------------------------------------------------------- quantisers
SHAPES = [1, 127, 129, 300]
KS = [8, 32, 328, 768]


@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("M", SHAPES)
def test_mx_quantize_rows(K_, M, K):
    K_.case = f"M={M} K={K}"
    x = with_boundaries(block_scaled(M, K, _gen(M * 31 + K), 1), 1)
    _quantize_rows(K_, x)


@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("N", SHAPES)
def test_mx_quantize_weight_merge_and_dequantize(K_, N, K):
    """bf16 source, dequantisation, the merge in place against the exact requantisation, and a zero-delta merge that leaves
    every dequantised value bit-identical."""
    K_.case = f"N={N} K={K}"
    g = _gen(N * 17 + K)
    w = with_boundaries(block_scaled(N, K, g, 32), 32)
    (gq, q), (gf, f), (gb, bw) = _quantize_weight(K_, w)
    before = _dequantize(K_, q, f, N, K)
    delta = _operand(block_scaled(N, K, g, 32).float() * 0.05)
    K_.call("mx_quantize_weight_2d", None, delta, q, f, bw, N, K)
    merged = _dequantize(K_, q, f, N, K)
    assert not torch.equal(merged, before)
    K_.call("mx_quantize_weight_2d", None, _operand(torch.zeros(N, K, device="cuda")), q, f, bw, N, K)
    again = _dequantize(K_, q, f, N, K)
    nz = merged != 0  # the fp32 add of a zero delta turns -0 into +0 (x + 0 in IEEE arithmetic)
    assert bool((again[~nz] == 0).all())
    ref.assert_bitwise_equal("zero-delta merge", again[nz], merged[nz])
    _intact(gq, gf, gb)


def test_mx_quantisers_run_their_grid_stride_loops(K_):
    """Each kernel at a shape past its num_sms·16·256-thread grid: every thread runs its loop at least once more."""
    cap = _cap_threads()
    K = 768
    M = 2 * cap // (32 * (K // 128)) + 37
    assert _pad(M) * (K // 128) * 32 > cap
    K_.case = f"rows M={M} K={K}"
    _quantize_rows(K_, with_boundaries(block_scaled(M, K, _gen(1), 1), 1))
    N = 4100
    Kw = (cap // 32 // (_pad(N) // 32) + 1) * 32 + 8
    assert (_pad(N) // 32) * (_pad(Kw) // 32) * 32 > cap and N * Kw // 4 > cap
    K_.case = f"weight N={N} K={Kw}"
    g = _gen(2)
    (gq, q), (gf, f), (gb, bw) = _quantize_weight(K_, with_boundaries(block_scaled(N, Kw, g, 32), 32))
    K_.call("mx_quantize_weight_2d", None, block_scaled(N, Kw, g, 32).float() * 0.05, q, f, bw, N, Kw)
    _dequantize(K_, q, f, N, Kw)
    _intact(gq, gf, gb)
    assert {"quantize_rows grid-stride", "quantize_weight_2d bf16 grid-stride", "quantize_weight_2d merge grid-stride",
            "dequantize_weight grid-stride"} <= set(K_.modes)


def test_mx_weight_survives_a_cuda_cpu_cuda_round_trip():
    """A packed CUDA weight moved to the CPU layout (1 x 32 blocks, ops/quant.py) and back keeps every value: each 1 x 32 block
    takes a scale no larger than its tile's, which holds every value of the tile exactly."""
    from relora_b200.relora import ReLoRaLinear

    w = block_scaled(264, 328, _gen(3), 32).cpu()
    lin = ReLoRaLinear(328, 264, r=8, lora_alpha=16, bias=False, weight_data=w.clone(), quantize="mxfp8", lora_dropout=0.0).to("cuda", BF)
    before = lin.weight.float()
    lin.to("cpu")
    lin.to("cuda")
    ref.assert_bitwise_equal("round trip", lin.weight.float(), before)


# ----------------------------------------------------------------------------------------------- gemm_mx
GEMM_SHAPES = [(1, 8, 8), (129, 136, 40), (300, 264, 328), (4096, 768, 776)]  # (M, N, K) of the call


def _gemm_operands(M, N, K, b_mn, seed):
    """x [M, K] (rows) and the weight (K-major: W [N, K]; MN-major: W [K, N], read transposed), quantised by the reference."""
    g = _gen(seed)
    xq, sfx = ref.mx_quantize_rows_exact(block_scaled(M, K, g, 1))
    if b_mn:
        wq, _, sfb = ref.mx_quantize_weight_2d_exact(block_scaled(K, N, g, 32))
    else:
        wq, sfb, _ = ref.mx_quantize_weight_2d_exact(block_scaled(N, K, g, 32))
    return g, _bytes(xq), _scales(sfx), _bytes(wq), _scales(sfb)


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
@pytest.mark.parametrize("b_mn", [False, True], ids=["kmajor", "mnmajor"])
def test_gemm_mx(K_, b_mn, M, N, K):
    """B K-major (forward) / MN-major (input gradient) x LoRA segment K2 in {0, 64, 128} x residual on / off.  The last shape
    has more tiles than SMs: the persistent loop's second tile per CTA and its stage / phase carry."""
    g, a, sfa, b, sfb = _gemm_operands(M, N, K, b_mn, M + N + K + b_mn)
    for k2 in (0, 64, 128):
        for res in (False, True):
            K_.case = f"M={M} N={N} K={K} K2={k2} res={res}"
            a2 = _operand((torch.randn(M, k2, generator=g, device="cuda") * 0.5).to(BF)) if k2 else None
            b2 = _operand((torch.randn(N, k2, generator=g, device="cuda") * 0.1).to(BF)) if k2 else None
            r = _operand(torch.randn(M, N, generator=g, device="cuda").to(BF)) if res else None
            go, out = _out((M, N), BF)
            K_.call("gemm_mx", a, sfa, b, sfb, out, M, N, K, b_mn, a2, b2, r)
            _intact(go)
    if -(-M // 128) * -(-N // 128) > _num_sms():
        assert any(m.endswith("persistent") for m in K_.modes), K_.modes


# ----------------------------------------------------------------------------------------------- non-finite inputs
def test_nan_or_inf_in_x_makes_only_its_output_rows_non_finite(K_):
    M, N, K = 300, 264, 328
    g = _gen(11)
    x = block_scaled(M, K, g, 1)
    x[5, 100] = float("nan")
    x[77, 3] = float("inf")
    x[78, 327] = float("-inf")
    _, _, _, wb, sfb = _gemm_operands(M, N, K, False, 12)
    xq, sfx = _quantize_rows(K_, x)
    go, out = _out((M, N), BF)
    K_.call("gemm_mx", xq, sfx, wb, sfb, out, M, N, K, False)
    bad = torch.zeros(M, dtype=torch.bool, device="cuda")
    bad[[5, 77, 78]] = True
    fin = torch.isfinite(out.float())
    assert not bool(fin[bad].any()) and bool(fin[~bad].all())
    _intact(go)


def test_inf_in_dy_makes_dx_non_finite(K_):
    """dx = dy·W: an Inf in one row of dy must not come out as a finite row (the non-finite check of the trainer relies on it)."""
    M, N, K = 300, 264, 328  # dy [M, N], W [N, K], dx [M, K]
    g = _gen(13)
    dy = block_scaled(M, N, g, 1)
    dy[9, 40] = float("inf")
    wq, _, sf_bwd = ref.mx_quantize_weight_2d_exact(block_scaled(N, K, g, 32))
    dq, sfd = _quantize_rows(K_, dy)
    go, dx = _out((M, K), BF)
    K_.call("gemm_mx", dq, sfd, _bytes(wq), _scales(sf_bwd), dx, M, K, N, True)
    fin = torch.isfinite(dx.float())
    assert not bool(fin[9].any()) and bool(fin[:9].all()) and bool(fin[10:].all())
    _intact(go)


def test_nan_or_inf_in_the_merge_delta_stays_in_its_tile(K_):
    N, K = 264, 328
    g = _gen(14)
    (gq, q), (gf, f), (gb, bw) = _quantize_weight(K_, block_scaled(N, K, g, 32))
    delta = block_scaled(N, K, g, 32).float() * 0.05
    delta[40, 70] = float("inf")
    delta[200, 300] = float("nan")
    K_.call("mx_quantize_weight_2d", None, delta, q, f, bw, N, K)
    d = _dequantize(K_, q, f, N, K)
    bad = torch.zeros(N, K, dtype=torch.bool, device="cuda")
    bad[32:64, 64:96] = True
    bad[200, 300] = True
    fin = torch.isfinite(d.float())
    assert not bool(fin[bad].any()) and bool(fin[~bad].all())
    # the forward GEMM: every output column that reads the Inf tile is non-finite, the rest are checked against the reference
    M = 77
    xq, sfx = ref.mx_quantize_rows_exact(block_scaled(M, K, g, 1))
    go, out = _out((M, N), BF)
    K_.call("gemm_mx", _bytes(xq), _scales(sfx), q, f, out, M, N, K, False)
    col = torch.isfinite(out.float()).all(0)
    assert not bool(col[32:64].any()) and not bool(col[200]) and int(col.sum()) == N - 33
    _intact(gq, gf, gb, go)


# ----------------------------------------------------------------------------------------------- host refusals
def test_mx_bindings_refuse_misaligned_or_undersized_operands(C):
    """mx_quantize_rows makes 8-byte loads, mx_quantize_weight_2d 16-byte ones, mx_dequantize_weight reads q / sf_fwd over the
    extent of out: operands that break that are refused on the host, before any launch."""
    q = torch.zeros(16, 128, dtype=torch.uint8, device="cuda")
    sf = torch.zeros(512, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="aligned"):
        C.mx_quantize_rows(torch.zeros(16, 40, dtype=BF, device="cuda")[:, 1:33], q, sf)
    with pytest.raises(RuntimeError, match="pitch"):
        C.mx_quantize_rows(torch.zeros(16, 42, dtype=BF, device="cuda")[:, :32], q, sf)
    wq = torch.zeros(128, 128, dtype=torch.uint8, device="cuda")
    f, bw = sf.clone(), sf.clone()
    with pytest.raises(RuntimeError, match="aligned"):
        C.mx_quantize_weight_2d(torch.zeros(16, 48, dtype=BF, device="cuda")[:, 4:36], None, wq, f, bw, 16, 32)
    with pytest.raises(RuntimeError, match="pitch"):
        C.mx_quantize_weight_2d(torch.zeros(16, 44, dtype=BF, device="cuda")[:, :32], None, wq, f, bw, 16, 32)
    out = torch.empty(128, 128, dtype=BF, device="cuda")
    with pytest.raises(RuntimeError, match="smaller"):
        C.mx_dequantize_weight(torch.zeros(64, 128, dtype=torch.uint8, device="cuda"), sf, out)
    with pytest.raises(RuntimeError, match="smaller"):
        C.mx_dequantize_weight(wq, sf, torch.empty(130, 128, dtype=BF, device="cuda"))
    with pytest.raises(RuntimeError, match="aligned"):
        C.mx_dequantize_weight(wq, sf, torch.empty(64, 132, dtype=BF, device="cuda")[:, 2:130])
    with pytest.raises(RuntimeError, match="pitch"):
        C.mx_dequantize_weight(wq, sf, torch.empty(64, 130, dtype=BF, device="cuda")[:, :128])
    with pytest.raises(RuntimeError, match="aligned"):
        C.mx_dequantize_weight(torch.zeros(64, 132, dtype=torch.uint8, device="cuda")[:, 2:130], sf, torch.empty(64, 128, dtype=BF,
                                                                                                              device="cuda"))
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------- module audit
def test_module_path_mx_calls_match_the_reference(C, monkeypatch):
    """Every MXFP8 call of building, one forward + backward and one merge of a 2-layer Llama with quantize="mxfp8", checked
    against the reference; the set of modes seen must be the expected one."""
    from relora_b200.models import LlamaForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    audit = _Checker(C)
    audit.case = "llama mxfp8"
    audit.install(monkeypatch)
    cfg = SimpleConfig(model_type="llama", vocab_size=1000, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                       num_attention_heads=4, num_key_value_heads=4, rope_theta=10000.0, rms_norm_eps=1e-6, pad_token_id=-1,
                       max_position_embeddings=256)
    torch.manual_seed(0)
    model = ReLoRaModel(LlamaForCausalLM(cfg), r=64, lora_alpha=32, lora_dropout=0.0, target_modules=["attn", "mlp"],
                        init_lora_a="kaiming", quantize="mxfp8")
    for mod in model.relora_modules():
        torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
    model = model.cuda().to(BF)
    ids = torch.randint(0, 1000, (2, 97), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    loss = model(input_ids=ids, labels=ids).loss
    loss.backward()
    for mod in model.relora_modules():
        mod.merge_and_reinit()
    torch.cuda.synchronize()
    assert torch.isfinite(loss)
    print(f"[mx modes] audit: {sum(audit.modes.values())} calls, worst ratio {audit.worst:.3g}, modes {dict(sorted(audit.modes.items()))}")
    assert {"quantize_rows", "quantize_weight_2d bf16", "quantize_weight_2d merge", "gemm_mx K-major K2=0",
            "gemm_mx MN-major K2=0"} <= set(audit.modes)
    assert audit.modes["quantize_weight_2d merge"] == len(list(model.relora_modules()))
