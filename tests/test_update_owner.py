"""The data-parallel update has one owner (`parallel.grad_sync`): the transport decision and the reduce / clip / AdamW / zero sequence
behind every stepper's `update()`.  No GPU: symmetric memory is stubbed and the update runs on a gloo world of one."""
import copy
import pathlib
import re
import types

import pytest
import torch
import torch.distributed as dist

from relora_b200.parallel import grad_sync, symm
from relora_b200.parallel.dist import DistInfo

PKG = pathlib.Path(grad_sync.__file__).resolve().parents[1]


def _info(world):
    return DistInfo(0, 0, world, torch.device("cpu"), "gloo")


# ---------------------------------------------------------------------- the transport decision
@pytest.fixture
def warnings_seen(monkeypatch):
    import relora_b200.obs as obs

    seen = []
    monkeypatch.setattr(obs, "logger", types.SimpleNamespace(warning=seen.append))
    return seen


def _stub_symm(monkeypatch, available, comm):
    """`comm`: what `SymmComm()` returns, or the exception it raises."""
    def make():
        if isinstance(comm, Exception):
            raise comm
        return comm

    monkeypatch.setattr(symm, "symmetric_memory_available", lambda: available)
    monkeypatch.setattr(symm, "SymmComm", make)


def test_auto_uses_peer_memory_when_it_is_there_and_nccl_when_it_is_not(monkeypatch, warnings_seen):
    comm = object()
    _stub_symm(monkeypatch, True, comm)
    assert grad_sync.peer_transport(_info(2), "auto") is comm
    assert grad_sync.peer_transport(_info(2), "p2p") is comm
    assert grad_sync.peer_transport(_info(2), "nccl") is None
    assert grad_sync.peer_transport(_info(2), "auto", eligible=False) is None
    _stub_symm(monkeypatch, False, comm)
    assert grad_sync.peer_transport(_info(2), "auto") is None
    assert warnings_seen == []


def test_auto_warns_and_falls_back_when_the_constructor_raises(monkeypatch, warnings_seen):
    _stub_symm(monkeypatch, True, OSError("no peer access"))
    assert grad_sync.peer_transport(_info(2), "auto") is None
    assert warnings_seen == ["peer-memory collectives unavailable (OSError: no peer access); using NCCL"]
    with pytest.raises(OSError, match="no peer access"):
        grad_sync.peer_transport(_info(2), "p2p")


def test_p2p_names_what_is_missing(monkeypatch):
    _stub_symm(monkeypatch, False, object())
    with pytest.raises(RuntimeError, match=r"^--comm p2p needs torch symmetric memory over an NCCL process group$"):
        grad_sync.peer_transport(_info(2), "p2p")
    _stub_symm(monkeypatch, True, object())
    with pytest.raises(RuntimeError, match=r"^--comm p2p needs bf16 parameters on CUDA$"):
        grad_sync.peer_transport(_info(2), "p2p", eligible=False)


@pytest.mark.parametrize("asked", ["auto", "p2p", "nccl"])
def test_a_single_rank_has_no_transport(monkeypatch, asked):
    _stub_symm(monkeypatch, True, RuntimeError("must not be constructed"))
    assert grad_sync.peer_transport(_info(1), asked) is None
    assert grad_sync.peer_transport(_info(1), asked, eligible=False) is None
    from relora_b200.parallel.flat import FlatParamStore

    store = FlatParamStore([("w", torch.nn.Parameter(torch.zeros(4)))])
    assert grad_sync.GradSync(store, _info(1), transport=asked).transport == "none"
    assert grad_sync.GradSync(store, _info(2), transport="nccl").transport == "nccl"


# ---------------------------------------------------------------------- the update sequence
@pytest.fixture
def gloo_world_of_one(tmp_path):
    """A group of this process alone; the one an earlier in-process trainer run left behind serves as well."""
    mine = not dist.is_initialized()
    if mine:
        dist.init_process_group("gloo", store=dist.FileStore(str(tmp_path / "rendezvous"), 1), rank=0, world_size=1)
    assert dist.get_world_size() == 1 and dist.get_backend() == "gloo"
    yield _info(1)
    if mine:
        dist.destroy_process_group()


def _steppers(info, clip):
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.models import LlamaForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cfg = SimpleConfig(model_type="llama", vocab_size=64, hidden_size=32, intermediate_size=48, num_hidden_layers=2,
                       num_attention_heads=2, rms_norm_eps=1e-6, pad_token_id=-1, max_position_embeddings=32)
    torch.manual_seed(0)
    model = ReLoRaModel(LlamaForCausalLM(cfg), r=4, lora_alpha=8, lora_dropout=0.0, target_modules=["attn", "mlp"],
                        keep_original_weights=True)
    kw = dict(lr=1e-2, weight_decay=0.1, clip_grad_norm=clip, zero=True)
    return ModuleStepper(copy.deepcopy(model), info, **kw), ModuleStepper(model, info, **kw)


def _by_hand(st, skip):
    st.sync.reduce()
    total, scale = st.sync.grad_norm_and_scale(st.clip)
    st.optimizer.step(grad_scale=scale, skip=skip)
    st.sync.gather_params()
    st.optimizer.zero_grad()
    return total


@pytest.mark.parametrize("clip", [1e-3, 0.0])
def test_update_is_reduce_norm_step_zero(gloo_world_of_one, clip):
    """`update()` against the sequence written out by hand on a copy: bit-identical parameters, moments and norm; a skipped update
    and one with a NaN gradient change nothing but the gradients, which are zeroed."""
    a, b = _steppers(gloo_world_of_one, clip)
    g = torch.Generator().manual_seed(1)
    for kind in ("plain", "skip", "plain", "nan", "plain"):
        ids = torch.randint(0, 64, (2, 16), generator=g)
        assert torch.equal(a.micro_step(ids), b.micro_step(ids))
        if kind == "nan":
            a.store.grads[3] = b.store.grads[3] = float("nan")
        before = a.store.params.clone(), a.optimizer.exp_avg.clone()
        skip = torch.tensor(1.0) if kind == "skip" else None
        info = a.update(skip=skip)
        total = _by_hand(b, skip)
        assert torch.equal(info.grad_norm, total) or (kind == "nan" and torch.isnan(info.grad_norm) and torch.isnan(total))
        assert info.mean_loss is None and info.skip_count is None
        for x, y in ((a.store.params, b.store.params), (a.optimizer.exp_avg, b.optimizer.exp_avg),
                     (a.optimizer.exp_avg_sq, b.optimizer.exp_avg_sq), (a.optimizer._step_t, b.optimizer._step_t)):
            assert torch.equal(x, y)
        unchanged = torch.equal(a.store.params, before[0]) and torch.equal(a.optimizer.exp_avg, before[1])
        assert unchanged == (kind != "plain")
        assert not a.store.grads.any()
    assert a.optimizer.step_count == b.optimizer.step_count == 3


def test_a_non_finite_norm_can_be_made_an_error(gloo_world_of_one):
    a, _ = _steppers(gloo_world_of_one, 1.0)
    a.micro_step(torch.randint(0, 64, (2, 16)))
    a.store.grads[0] = float("inf")
    with pytest.raises(RuntimeError, match=r"The total norm of order 2\.0 for gradients is non-finite \(inf\), so it cannot be clipped\."):
        a.update(error_if_nonfinite=True)


# ---------------------------------------------------------------------- one copy in the source
def test_the_policy_is_written_once():
    src = {p: p.read_text() for d in ("engine", "parallel") for p in sorted((PKG / d).glob("*.py"))}
    assert sum(t.count("so it cannot be clipped") for t in src.values()) == 1
    assert sum(t.count("SymmComm()") for t in src.values()) == 1
    for p, t in src.items():
        if p.name != "grad_sync.py":
            assert not re.search(r"\.transport\s*=[^=]", t), p
            assert "peer_memory_update" not in t, p
