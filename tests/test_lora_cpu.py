"""LoRA merge / unmerge (easyanimate_b200.lora) without a GPU: `ops.lora_merge` is the reference's torch formula
(`lora_merge_stand_in` below) and the staging device is the host.  The layer resolver and the merged weights against the reference's own
merge_lora / unmerge_lora (utils/lora_utils.py:369-494, lifted unmodified), every weight storage and memory mode, invalidation
of the transformer's derived weights, and the errors that must leave every parameter unchanged."""
import ast
import copy
import os
import types
from collections import defaultdict

import pytest
import torch
import torch.nn as nn

from tests import cpu_ops
from tests.test_offload_cpu import CFG, LogStreamer, _forward, _inputs, _model

bf16, e4m3 = torch.bfloat16, torch.float8_e4m3fn
REF_LORA = "/root/reference/easyanimate/utils/lora_utils.py"
need_ref = pytest.mark.skipif(not os.path.exists(REF_LORA), reason="/root/reference not present")


def lora_merge_stand_in(w, up, down, scale):
    """include/ea_b200.h ea_lora_merge as the reference's torch formula (utils/lora_utils.py:424-430): the weight cast to the
    factors' dtype, += scale * mm(up, down), cast back into its own storage."""
    wc = w.to(up.dtype)
    wc += scale * torch.mm(up, down)
    w.copy_(wc.to(w.dtype))


@pytest.fixture
def host(monkeypatch):
    """Stand-ins for the kernels (the LoRA merge's among them), and the host as the device that stages host-resident
    weights."""
    from easyanimate_b200 import lora, ops
    cpu_ops.use_stand_ins(monkeypatch)
    monkeypatch.setattr(ops, "lora_merge", lora_merge_stand_in)
    monkeypatch.setattr(lora, "_work_device", lambda pipeline: torch.device("cpu"))
    return lora


def _reference():
    from safetensors.torch import load_file
    fns = [n for n in ast.parse(open(REF_LORA).read()).body if isinstance(n, ast.FunctionDef) and n.name in ("merge_lora", "unmerge_lora")]
    ns = {"torch": torch, "defaultdict": defaultdict, "load_file": load_file}
    exec(compile(ast.Module(body=fns, type_ignores=[]), REF_LORA, "exec"), ns)
    return ns["merge_lora"], ns["unmerge_lora"]


class _Qwen2Named(nn.Module):
    """A text encoder with Qwen2's module names (model.layers.N.self_attn.q_proj, mlp.gate_proj, lm_head, ...) and one 1x1
    convolution, whose LoRA factors are 4-D."""

    def __init__(self, h=32):
        super().__init__()
        self.model = nn.Module()
        self.model.embed_tokens = nn.Embedding(16, h)
        self.model.layers = nn.ModuleList()
        for _ in range(2):
            layer = nn.Module()
            layer.self_attn, layer.mlp = nn.Module(), nn.Module()
            for n in ("q_proj", "k_proj", "v_proj", "o_proj"):
                setattr(layer.self_attn, n, nn.Linear(h, h, bias=n != "o_proj"))
            layer.mlp.gate_proj, layer.mlp.up_proj, layer.mlp.down_proj = nn.Linear(h, 2 * h), nn.Linear(h, 2 * h), nn.Linear(2 * h, h)
            self.model.layers.append(layer)
        self.lm_head = nn.Linear(h, 16, bias=False)
        self.visual_merger = nn.Conv2d(h, h, 1)


def _text_encoder(seed=3):
    torch.manual_seed(seed)
    return _Qwen2Named().to(bf16)


def _factors(weight, g, rank, alpha, fdtype):
    o, i = weight.shape[:2]
    up, down = torch.randn(o, rank, generator=g) * 0.2, torch.randn(rank, i, generator=g) * 0.2
    if weight.dim() == 4:
        up, down = up[:, :, None, None], down[:, :, None, None]
    out = {"lora_up.weight": up.to(fdtype), "lora_down.weight": down.to(fdtype)}
    if alpha is not None:
        out["alpha"] = torch.tensor(float(alpha))
    return out


def _lora_file(t, te, g, rank=4, alpha=None, fdtype=torch.float32, block_names=None):
    """A LoRA in the reference training's key format (lora_unet__<module path>, lora_te_<module path>)."""
    sd = {}
    names = [n for n, m in t.named_modules() if isinstance(m, nn.Linear)]
    if block_names is not None:
        names = [n for n in names if any(n.startswith(b) for b in block_names)]
    for n in names:
        if n in ("text_proj_t5.1", "text_proj_t5"):
            continue  # the reference's walk cannot reach text_proj_t5 (see test_resolver_matches_the_reference)
        for k, v in _factors(t.get_submodule(n).weight, g, rank, alpha, fdtype).items():
            sd[f"lora_unet__{n.replace('.', '_')}.{k}"] = v
    if te is not None:
        for n in ("model.layers.0.self_attn.q_proj", "model.layers.1.mlp.down_proj", "lm_head", "visual_merger"):
            for k, v in _factors(te.get_submodule(n).weight, g, rank, alpha, fdtype).items():
                sd[f"lora_te_{n.replace('.', '_')}.{k}"] = v
    return sd


def _bits(m):
    return {k: v.detach().clone().view(torch.uint8) if v.dtype.itemsize == 1 else v.detach().clone() for k, v in m.state_dict().items()}


def _same(a, b):
    assert set(a) == set(b)
    for k in a:
        assert a[k].dtype == b[k].dtype and torch.equal(a[k].view(torch.uint8), b[k].view(torch.uint8)), k


# ---- resolver ---------------------------------------------------------------------------------------------------------
@need_ref
@pytest.mark.parametrize("extra", [dict(add_norm_text_encoder=True, text_embed_dim_t5=128, ref_channels=16, clip_channels=32),
                                   dict(add_norm_text_encoder=False, text_embed_dim_t5=128)])
@pytest.mark.parametrize("form", ["training", "single"])
def test_resolver_matches_the_reference(host, monkeypatch, extra, form):
    """For every nn.Linear of the product transformer and of the Qwen2-named encoder, the module the reference's merge_lora
    edits is the one the native merge edits; where the reference's walk fails, or lands on a module of another shape, the
    native merge raises ValueError before any change."""
    from easyanimate_b200 import lora
    ref_merge, _ = _reference()
    t, te = _model(**extra), _text_encoder()
    pipe = types.SimpleNamespace(transformer=t, text_encoder=te)
    touched = []
    orig_to = nn.Module.to

    def to(self, *a, **k):
        touched.append(self)
        return orig_to(self, *a, **k)
    g = torch.Generator().manual_seed(1)
    cases = [("lora_unet" + ("__" if form == "training" else "_") + n.replace(".", "_"), m)
             for n, m in t.named_modules() if isinstance(m, nn.Linear)]
    cases += [("lora_te_" + n.replace(".", "_"), m) for n, m in te.named_modules() if isinstance(m, (nn.Linear, nn.Conv2d))]
    outcomes = set()
    for layer, m in cases:
        sd = {f"{layer}.{k}": v for k, v in _factors(m.weight, g, 2, None, torch.float32).items()}
        del touched[:]
        monkeypatch.setattr(nn.Module, "to", to)
        try:
            ref_merge(copy.copy(pipe), None, 1.0, state_dict=sd)
            ref_ok = True
        except Exception:
            ref_ok = False
        monkeypatch.setattr(nn.Module, "to", orig_to)
        ref_module = touched[0] if touched else None
        if ref_ok:
            edits = lora._plan(pipe, sd, 1.0, torch.float32, False, 1.0)
            assert ref_module is m and [e.weight for e in edits] == [m.weight], layer
            outcomes.add("same module")
        else:
            with pytest.raises(ValueError):
                lora._plan(pipe, sd, 1.0, torch.float32, False, 1.0)
            outcomes.add("refused")
    assert "same module" in outcomes


# ---- weights against the reference ----------------------------------------------------------------------------------
@need_ref
@pytest.mark.parametrize("dtype", [torch.float32, bf16])
@pytest.mark.parametrize("alpha", [None, 3.0])
def test_merge_and_round_trip_equal_the_reference(host, tmp_path, dtype, alpha):
    from safetensors.torch import save_file
    from easyanimate_b200 import merge_lora, unmerge_lora
    ref_merge, ref_unmerge = _reference()
    t, te = _model(add_norm_text_encoder=True), _text_encoder()
    g = torch.Generator().manual_seed(7)
    sd = _lora_file(t, te, g, rank=7, alpha=alpha, fdtype=bf16 if alpha is None else torch.float32)
    path = str(tmp_path / "lora.safetensors")
    save_file(sd, path)
    ref = types.SimpleNamespace(transformer=copy.deepcopy(t), text_encoder=copy.deepcopy(te))
    ours = types.SimpleNamespace(transformer=copy.deepcopy(t), text_encoder=copy.deepcopy(te))
    ref_merge(ref, path, 0.7, dtype=dtype)
    assert merge_lora(ours, path, 0.7, dtype=dtype) is ours
    for a, b in ((ours.transformer, ref.transformer), (ours.text_encoder, ref.text_encoder)):
        _same(_bits(a), _bits(b))
    assert not torch.equal(ours.text_encoder.visual_merger.weight, te.visual_merger.weight)  # the 4-D factors landed
    ref_unmerge(ref, path, 0.7, dtype=dtype)
    unmerge_lora(ours, path, 0.7, dtype=dtype)
    for a, b in ((ours.transformer, ref.transformer), (ours.text_encoder, ref.text_encoder)):
        _same(_bits(a), _bits(b))


@need_ref
def test_e4m3_storage_equals_the_reference(host):
    ref_merge, _ = _reference()
    t = _model(e4m3)
    sd = _lora_file(t, None, torch.Generator().manual_seed(8), rank=5, alpha=2.0)
    ref, ours = types.SimpleNamespace(transformer=copy.deepcopy(t)), types.SimpleNamespace(transformer=copy.deepcopy(t))
    ref_merge(ref, None, 1.3, state_dict=sd, transformer_only=True)
    from easyanimate_b200 import merge_lora
    merge_lora(ours, None, 1.3, state_dict=sd, transformer_only=True)
    _same(_bits(ours.transformer), _bits(ref.transformer))
    assert not torch.equal(_bits(ours.transformer)["proj_out.weight"], _bits(t)["proj_out.weight"])


# ---- memory modes ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [bf16, e4m3])
def test_every_mode_merges_what_the_resident_merge_does(host, tmp_path, dtype):
    from easyanimate_b200 import EasyAnimatePipeline, merge_lora, unmerge_lora
    from tests import test_native_pipelines_cpu as N
    base = _model(dtype)
    sd = _lora_file(base, None, torch.Generator().manual_seed(9), rank=6, alpha=4.0)
    resident = types.SimpleNamespace(transformer=copy.deepcopy(base), text_encoder=None)
    merge_lora(resident, None, 0.9, state_dict=sd)
    want = _bits(resident.transformer)
    assert not torch.equal(want["transformer_blocks.1.attn1.to_v.weight"], _bits(base)["transformer_blocks.1.attn1.to_v.weight"])

    log = []
    seq = copy.deepcopy(base).enable_sequential_cpu_offload("cpu", streamer=LogStreamer(log))
    packs = list(seq._offload.packs)
    hosts = [pk.host.data_ptr() for pk in packs]
    ptrs = {k: p.data_ptr() for k, p in seq.named_parameters()}
    merge_lora(types.SimpleNamespace(transformer=seq), None, 0.9, state_dict=sd)
    _same(_bits(seq), want)
    assert all(a is b for a, b in zip(packs, seq._offload.packs)) and [pk.host.data_ptr() for pk in packs] == hosts
    assert {k: p.data_ptr() for k, p in seq.named_parameters()} == ptrs  # the same views: nothing was repacked

    t, v = copy.deepcopy(base), N._modules()[1]
    pipe = EasyAnimatePipeline(vae=v, transformer=t, tokenizer=N._FakeTokenizer(),
                               text_encoder=N._FakeTextEncoder(128).to(bf16)).enable_model_cpu_offload("cpu")
    devices = {k: p.device for k, p in t.named_parameters()}
    merge_lora(pipe, None, 0.9, state_dict=sd)
    _same(_bits(t), want)
    assert {k: p.device for k, p in t.named_parameters()} == devices
    # the unmerge in each mode equals the resident unmerge too
    from safetensors.torch import save_file
    path = str(tmp_path / "lora.safetensors")
    save_file(sd, path)
    unmerge_lora(resident, path, 0.9)
    unmerge_lora(types.SimpleNamespace(transformer=seq), path, 0.9)
    unmerge_lora(pipe, path, 0.9)
    back = _bits(resident.transformer)
    _same(_bits(seq), back)
    _same(_bits(t), back)


# ---- derived weights -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [bf16, e4m3])
@pytest.mark.parametrize("offloaded", [False, True])
def test_forward_after_merge_equals_a_fresh_model_with_the_merged_weights(host, tmp_path, dtype, offloaded):
    """A forward before the merge (which builds the fused q/k/v and, for e4m3, the bf16 staging head), then one after it: the
    second equals a fresh model loaded with the merged state dict; the same after the unmerge.  The LoRA covers text_proj,
    which the fp8 staging head's cache key does not follow."""
    from easyanimate_b200 import merge_lora, unmerge_lora
    from easyanimate_b200.transformer3d import EasyAnimateTransformer3DModel
    m = _model(dtype)
    if offloaded:
        m.enable_sequential_cpu_offload("cpu", streamer=LogStreamer([]))
    sd = _lora_file(m, None, torch.Generator().manual_seed(10), rank=4, alpha=8.0,
                    block_names=("transformer_blocks.0.attn1", "transformer_blocks.1.attn2", "text_proj", "proj_out"))
    lat, enc, rope = _inputs(B=1)
    pipe = types.SimpleNamespace(transformer=m)

    def fresh():
        f = EasyAnimateTransformer3DModel(**CFG).to(dtype)
        f.load_state_dict({k: v.clone() for k, v in m.state_dict().items()})
        return f
    before = _forward(m, lat, 600, enc, rope)
    merge_lora(pipe, None, 1.0, state_dict=sd)
    after = _forward(m, lat, 600, enc, rope)
    assert torch.equal(after, _forward(fresh(), lat, 600, enc, rope)) and not torch.equal(after, before)

    from safetensors.torch import save_file
    save_file(sd, str(tmp_path / "lora.safetensors"))
    unmerge_lora(pipe, str(tmp_path / "lora.safetensors"), 1.0)
    again = _forward(m, lat, 600, enc, rope)
    assert torch.equal(again, _forward(fresh(), lat, 600, enc, rope)) and not torch.equal(again, after)


# ---- errors ----------------------------------------------------------------------------------------------------------
def test_errors_leave_every_parameter_unchanged(host):
    from easyanimate_b200 import merge_lora
    t, te = _model(), _text_encoder()
    good = _lora_file(t, None, torch.Generator().manual_seed(11), rank=3, block_names=("transformer_blocks.0",))
    d = t.inner_dim
    cases = {
        "no module": {"lora_unet__transformer_blocks_0_attn9_to_q.lora_up.weight": torch.zeros(d, 2),
                      "lora_unet__transformer_blocks_0_attn9_to_q.lora_down.weight": torch.zeros(2, d)},
        "does not make": {"lora_unet__proj_out.lora_up.weight": torch.zeros(d, 2),
                          "lora_unet__proj_out.lora_down.weight": torch.zeros(2, d)},
        "text encoder": {"lora_te_lm_head.lora_up.weight": torch.zeros(16, 2), "lora_te_lm_head.lora_down.weight": torch.zeros(2, 32)},
        "lora_down": {"lora_unet__proj_out.lora_up.weight": torch.zeros(64, 2)},
    }
    for what, bad in cases.items():
        for pipe in (types.SimpleNamespace(transformer=t, text_encoder=None), types.SimpleNamespace(transformer=t)):
            before = _bits(t)
            with pytest.raises(ValueError, match=what):
                merge_lora(pipe, None, 1.0, state_dict={**good, **bad})  # the good layers come first in the file
            _same(_bits(t), before)
    before = _bits(t), _bits(te)
    with pytest.raises(ValueError, match="dtype"):
        merge_lora(types.SimpleNamespace(transformer=t, text_encoder=te), None, 1.0, state_dict=good, dtype=torch.float16)
    _same(_bits(t), before[0])
    # transformer_only skips the text encoder's layers instead of refusing them
    merge_lora(types.SimpleNamespace(transformer=t, text_encoder=None), None, 1.0,
               state_dict={**good, **cases["text encoder"]}, transformer_only=True)
    _same(_bits(te), before[1])
