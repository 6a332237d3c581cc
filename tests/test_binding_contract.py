"""Source check of the binding layer (relora_b200/csrc/bindings.cpp): every tensor argument of every binding goes through the one
operand check, no operand rule is checked anywhere else in the file, and every binding is either exercised by
tests/test_binding_contract_gpu.py or exempt for a stated reason."""
import os
import re

from test_binding_contract_gpu import CASES, EXEMPT

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "relora_b200", "csrc", "bindings.cpp")
# the helpers that check operands: arg() itself and the two that hand their tensors to it
HELPERS = ("arg", "dropout", "fp8_out", "comm_ctx")
# what a TORCH_CHECK condition on an operand reads: a tensor's metadata or data
# (a tensor's size() takes a dimension; a std::vector's takes none)
OPERAND_READ = re.compile(r"(\.|->)(size\([^)]|(sizes|stride|strides|numel|dim|is_cuda|is_contiguous|scalar_type|element_size|device|data_ptr)\()")


def _source():
    with open(SRC) as f:
        return f.read()


def _code(src):
    """src with every string literal emptied, so that brackets in messages do not count."""
    return re.sub(r'"(?:\\.|[^"\\])*"', '""', src)


def _functions(src):
    """name -> (parameter text, body) of every top-level function in the anonymous namespace."""
    out = {}
    for m in re.finditer(r"^[\w:<>*&\s]+?\b(\w+)\(((?:[^;{]|\{\})*?)\)\s*\{", src, re.M | re.S):
        depth, i = 1, m.end()
        while depth:
            depth += {"{": 1, "}": -1}.get(src[i], 0)
            i += 1
        out[m.group(1)] = (m.group(2), src[m.end():i - 1])
    return out


def _calls(body, name):
    """Argument texts of every call of `name` (template arguments allowed) in body."""
    res = []
    for m in re.finditer(rf"\b{name}(<[^>]*>)?\(", body):
        depth, i = 1, m.end()
        while depth:
            depth += {"(": 1, ")": -1}.get(body[i], 0)
            i += 1
        res.append(body[m.end():i - 1])
    return res


def _args(text):
    """Top-level comma-separated arguments of a call's argument text."""
    out, depth, start = [], 0, 0
    for i, ch in enumerate(text):
        depth += {"(": 1, "[": 1, "{": 1, ")": -1, "]": -1, "}": -1}.get(ch, 0)
        if ch == "," and depth == 0:
            out.append(text[start:i].strip())
            start = i + 1
    return out + [text[start:].strip()]


def _first_arg(text):
    return _args(text)[0]


def _bindings(src):
    """Python name -> C++ function of every m.def that binds a function of this file."""
    return dict(re.findall(r'm\.def\("(\w+)",\s*&([\w:]+)', src))


def _tensor_params(params):
    return re.findall(r"(?:const\s+)?(?:Tensor|OptTensor)&\s*(\w+)", params)


# Byte alignment of base and row pitch that each vector- or TMA-accessed operand's kernel needs (16-byte bf16x8 / uint4 /
# float4 loads and stores, 8-byte E4M3 stores, 4-byte element pairs), by binding and C++ parameter.
ALIGN = {
    "gemm": dict(a1=16, b1=16, a2=16, b2=16),
    "rmsnorm_fwd": dict(x=16, w=16, y=16, xd=16),
    "rmsnorm_bwd": dict(dy=16, x=16, w=16, dx_add=16, dx=16),
    "dropout_expand": dict(x=16, xd=16),
    "dropout_combine": dict(base=16, parts=16, out=16),
    "fp8_out": dict(q8=8),
    "fp8_quantize_weight": dict(w=16, w8=16),
    "fp8_quantize_act": dict(x=16, x8=16),
    "lora_dx": dict(dy=16, w=16, du=16, a=16, out=16, base=16),
    "attention_fwd": dict(qkv=16, out=16),
    "attention_bwd": dict(qkv=16, out=16, dout=16, dqkv=16),
    "rope_inplace": dict(buf=4, cos=4, sin=4),
    "rope_pack_bwd": dict(dq=16, dk=16, dv=16, out=16, cos=16, sin=16),
    "swiglu_fwd": dict(gu=16, h=16, hd=16),
    "swiglu_bwd": dict(dh=16, gu=16, dgu=16),
    "mx_quantize_rows": dict(x=8, q=4),
    "mx_quantize_weight_2d": dict(w=16, q=4),
    "mx_dequantize_weight": dict(q=4, out=8),
    "gemm_mx": dict(a=16, b=16, a2=16, b2=16, out=16, residual=16),
    "layernorm_fwd": dict(x=16, w=16, b=16, y=16, xd=16, w2=16, b2=16, y2=16, xd2=16),
    "layernorm_bwd": dict(dy=16, x=16, w=16, dx=16, dres=16, dy2=16, w2=16),
    "gelu_fwd": dict(z=16, a=16, xd=16),
    "gelu_bwd": dict(da=16, z=16, dz=16, dbias=16),
    "colsum": dict(x=16, out=16),
    "embedding_fwd": dict(table=16, out=16),
    "embedding_bwd": dict(dout=16),
    "embedding_bwd_sorted": dict(dout=16, dtable=16),
    "cross_entropy_fwd_bwd": dict(logits=16),
    "add": dict(a=16, b=16, out=16),
    "cast_f32_to_bf16": {"in": 16, "out": 16},
    "adamw_flat": dict(p=16),
}


def test_vector_accessed_operands_are_checked_for_alignment():
    funcs = _functions(_code(_source()))
    for fn, want in ALIGN.items():
        found = {}
        for call in _calls(funcs[fn][1], "arg"):
            a = _args(call)
            found[a[1].lstrip("*")] = int(a[5]) if len(a) > 5 and a[5].isdigit() else 1
        for p, align in want.items():
            assert p in found, f"{fn}: {p} does not go through arg()"
            assert found[p] >= align, f"{fn}: {p} is checked for {found[p]}-byte alignment, its kernel needs {align}"


def test_every_binding_is_exercised_or_exempt():
    src = _source()
    names = set(re.findall(r'm\.def\("(\w+)"', src))
    cases = {c.split("-")[0] for c in CASES}  # case ids: binding[-form]
    assert not cases & set(EXEMPT)
    assert names == cases | set(EXEMPT), (sorted(names - cases - set(EXEMPT)), sorted(cases | set(EXEMPT) - names))
    assert all(EXEMPT.values()), "every exemption gives its reason"


def test_every_tensor_argument_goes_through_the_operand_check():
    src = _source()
    funcs = _functions(_code(src))
    checked = 0
    for py, cpp in _bindings(src).items():
        if cpp.startswith("rb::"):
            continue
        params, body = funcs[cpp]
        for p in _tensor_params(params):
            hits = [a for h in HELPERS for a in _calls(body, h) if re.search(rf"(^|[\s(,*]){p}\s*(,|\)|$)", a)]
            assert hits, f"{py}: tensor argument {p} is not checked by arg()"
            checked += 1
    assert checked > 100


def test_no_operand_check_outside_the_helpers():
    funcs = _functions(_code(_source()))
    bad = []
    for name, (_, body) in funcs.items():
        if name in HELPERS:
            continue
        for cond in _calls(body, "TORCH_CHECK"):
            if OPERAND_READ.search(_first_arg(cond)):
                bad.append(f"{name}: TORCH_CHECK({cond[:80]}")
    assert not bad, "\n".join(bad)
