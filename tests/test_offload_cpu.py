"""CPU-offload memory modes without a GPU: the packed host layout of the sequentially offloaded transformer, the order in which
it issues copies and waits (through an injected streamer that logs), its forward on the kernel stand-ins against the resident
forward, the module moves of the pipelines' model offload, load_pipeline's GPU_memory_mode, and the e4m3 text encoder against
the reference's own fp8 helpers."""
import copy
import importlib.util
import os

import pytest
import torch

from tests import cpu_ops

bf16, e4m3 = torch.bfloat16, torch.float8_e4m3fn
CFG = dict(num_attention_heads=2, attention_head_dim=64, in_channels=16, out_channels=16, patch_size=2, num_layers=3, mmdit_layers=2,
           time_embed_dim=64, add_norm_text_encoder=True, text_embed_dim=128, text_embed_dim_t5=None)
REF_FP8 = "/root/reference/easyanimate/utils/fp8_optimization.py"


class LogStreamer:
    """offload.CudaBlockStreamer's interface on host tensors: copies and expansions happen at once, every call is logged."""
    pin_memory = False

    def __init__(self, log):
        self.log = log

    def begin(self):
        self.log.append(("begin",))

    def copy(self, slot, index, dst, src):
        self.log.append(("copy", slot, index))
        dst[:src.numel()].copy_(src)

    def acquire(self, slot, index):
        self.log.append(("acquire", slot, index))

    def release(self, slot, index):
        self.log.append(("release", slot, index))

    def segment_table(self, segments):
        return list(segments)

    def expand(self, src, table):
        self.log.append(("expand",))
        for off, dst in table:
            dst.copy_(src[off:off + dst.numel()].view(e4m3).to(bf16).view(dst.shape))

    def drain(self):
        pass


@pytest.fixture
def log(monkeypatch):
    entries = []

    def qkv(*a, **k):  # marks the compute of a block in the log
        entries.append(("compute",))
        return cpu_ops.qkv_gemm_ln_rope(*a, **k)
    cpu_ops.use_stand_ins(monkeypatch, qkv_gemm_ln_rope=qkv)
    return entries


def _model(dtype=bf16, seed=5, **kw):
    from easyanimate_b200.transformer3d import EasyAnimateTransformer3DModel
    torch.manual_seed(seed)
    m = EasyAnimateTransformer3DModel(**dict(CFG, **kw))
    with torch.no_grad():
        for p in m.parameters():  # LayerNorm affines and biases away from 1 / 0, so that a misplaced one shows
            p.add_(torch.randn_like(p) * 0.05)
    return m.to(bf16).to(dtype)


def _inputs(seed=6, B=2):
    from easyanimate_b200.pipeline import rope_table
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(B, 16, 2, 8, 8, generator=g).to(bf16)
    enc = (torch.randn(B, 9, 128, generator=g) * 3).to(bf16)
    return lat, enc, rope_table(64, 64, 2)


def _forward(m, lat, t, enc, rope):
    return m(lat, torch.full((lat.shape[0],), float(t)), encoder_hidden_states=enc, image_rotary_emb=rope, return_dict=False)[0]


@pytest.mark.parametrize("dtype", [bf16, e4m3])
def test_packing_round_trips_every_parameter(log, dtype):
    from easyanimate_b200 import offload
    m = _model(dtype)
    before = {k: v.clone() for k, v in m.state_dict().items()}
    m.enable_sequential_cpu_offload("cpu", streamer=LogStreamer(log))
    after = m.state_dict()
    assert set(after) == set(before)
    for k, v in before.items():
        assert after[k].dtype == v.dtype and torch.equal(after[k].view(torch.uint8), v.view(torch.uint8)), k
    for i, blk in enumerate(m.transformer_blocks):
        pk = m._offload.packs[i]
        lo, hi = pk.host.data_ptr(), pk.host.data_ptr() + pk.host.nbytes
        for name, p in blk.named_parameters():  # the block's parameters are views of its packed buffer
            assert lo <= p.data_ptr() < hi and p.data_ptr() % offload.ALIGN == 0, name
        for a in ("attn1", "attn2"):
            if getattr(blk, a) is None:
                continue
            w, b = offload.fused_qkv_views(pk.host, pk.layout, a)  # the fused projection operand, straight from the packed rows
            at = getattr(blk, a)
            assert torch.equal(w.view(torch.uint8), torch.cat([at.to_q.weight, at.to_k.weight, at.to_v.weight]).view(torch.uint8))
            assert torch.equal(b.view(torch.uint8), torch.cat([at.to_q.bias, at.to_k.bias, at.to_v.bias]).view(torch.uint8))
    # edits through .data land in the packed buffer; load_state_dict too
    two = torch.full(m.transformer_blocks[1].ff.net[2].bias.shape, 2.0).to(dtype)
    m.transformer_blocks[1].ff.net[2].bias.data.copy_(two)
    pk = m._offload.packs[1]
    assert torch.equal(offload._views(pk.host, pk.layout)["ff.net.2.bias"].view(torch.uint8), two.view(torch.uint8))
    m.load_state_dict(before)
    for k, v in before.items():
        assert torch.equal(m.state_dict()[k].view(torch.uint8), v.view(torch.uint8)), k


@pytest.mark.parametrize("dtype", [bf16, e4m3])
def test_copies_are_issued_ahead_and_slots_rewritten_after_their_reader(log, dtype):
    m = _model(dtype)
    m.enable_sequential_cpu_offload("cpu", streamer=LogStreamer(log))
    lat, enc, rope = _inputs()
    del log[:]
    _forward(m, lat, 500, enc, rope)
    n = len(m.transformer_blocks)
    copies = [e for e in log if e[0] == "copy"]
    assert [c[2] for c in copies] == list(range(n)) and all(c[1] == c[2] % 2 for c in copies)
    pos = {e: i for i, e in enumerate(log)}
    for i in range(n):
        first_compute = next(j for j in range(pos[("acquire", i % 2, i)], len(log)) if log[j] == ("compute",))
        if i + 1 < n:
            assert pos[("copy", (i + 1) % 2, i + 1)] < first_compute  # block i+1 is on its way before block i computes
        if i >= 2:  # the slot is refilled only after its previous reader's release
            assert pos[("release", i % 2, i - 2)] < pos[("copy", i % 2, i)]
        if dtype == bf16:  # a bf16 slot is read by the block itself: released after its compute
            assert first_compute < pos[("release", i % 2, i)]


@pytest.mark.parametrize("dtype", [bf16, e4m3])
def test_offloaded_forward_equals_resident_forward(log, dtype):
    resident = _model(dtype)
    off = copy.deepcopy(resident).enable_sequential_cpu_offload("cpu", streamer=LogStreamer(log))
    coeffs = [1.07862322, -4.19362456, 3.06725828, 0.33161686, 0.02374758]
    for m in (resident, off):
        m.enable_teacache(4, 0.3, coefficients=coeffs)
    lat, enc, rope = _inputs()  # CFG batch of 2
    for t in (999, 900, 880, 500):
        want, got = _forward(resident, lat, t, enc, rope), _forward(off, lat, t, enc, rope)
        assert torch.equal(got, want), t
    assert off.teacache.skipped == resident.teacache.skipped > 0


def test_offload_follows_to_and_invalidate_weight_caches(log):
    m = _model()
    m.enable_sequential_cpu_offload("cpu", streamer=LogStreamer(log))
    resident = copy.deepcopy(m)
    resident._offload = None
    lat, enc, rope = _inputs(B=1)
    packs = list(m._offload.packs)
    m.to(torch.float32).to(bf16)  # replaces every parameter: the blocks are repacked on the next forward
    assert torch.equal(_forward(m, lat, 700, enc, rope), _forward(resident, lat, 700, enc, rope))
    assert all(a is not b for a, b in zip(packs, m._offload.packs))
    packs = list(m._offload.packs)
    with torch.no_grad():  # the reference's LoRA merge: .data edits, then the hand-shake
        for mod in (m, resident):
            mod.transformer_blocks[0].attn1.to_k.weight.data += 0.25
            mod.invalidate_weight_caches()
    assert torch.equal(_forward(m, lat, 700, enc, rope), _forward(resident, lat, 700, enc, rope))
    assert all(a is b for a, b in zip(packs, m._offload.packs))  # the edits landed in the packed buffers: no repack


def test_opting_in_drops_what_a_resident_forward_derived(log):
    m = _model()
    lat, enc, rope = _inputs(B=1)
    _forward(m, lat, 700, enc, rope)
    assert all(b.attn1._fused is not None for b in m.transformer_blocks)
    m.enable_sequential_cpu_offload("cpu", streamer=LogStreamer(log))
    assert all(b.attn1._fused is None for b in m.transformer_blocks)


def test_a_module_without_opt_in_refuses_host_parameters():
    from easyanimate_b200 import _lib
    m = _model()
    lat, enc, rope = _inputs(B=1)
    with pytest.raises(_lib.EaError, match="CUDA"):
        _forward(m, lat, 700, enc, rope)


# ---- pipelines ----------------------------------------------------------------------------------------------------------
def _pipeline_modules(monkeypatch, in_channels=16):
    from tests import test_native_pipelines_cpu as N
    cpu_ops.use_stand_ins(monkeypatch)
    return N._modules(in_channels=in_channels, **({} if in_channels == 16 else dict(resize_inpaint_mask_directly=True,
                                                                                  enable_clip_in_inpaint=False)))


def _log_moves(monkeypatch, modules, moves):
    for name, mod in modules.items():
        orig = type(mod).to

        def to(self, *a, _name=name, _orig=orig, **k):
            moves.append((_name, str(a[0]) if a else str(k)))
            return _orig(self, *a, **k)
        monkeypatch.setattr(mod, "to", to.__get__(mod))


def test_model_cpu_offload_moves_each_module_while_it_is_used(monkeypatch):
    from easyanimate_b200 import EasyAnimateInpaintPipeline, EasyAnimatePipeline
    from tests import test_native_pipelines_cpu as N
    t, v = _pipeline_modules(monkeypatch, in_channels=33)
    tok, enc = N._FakeTokenizer(), N._FakeTextEncoder(128).to(bf16)
    g = torch.Generator().manual_seed(3)
    video = torch.rand(1, 3, N.FRAMES, N.H, N.W, generator=g)
    mask = torch.zeros_like(video[:, :1])
    mask[:, :, 1:] = 255
    kw = dict(prompt="a cat", negative_prompt="blurry", video_length=N.FRAMES, video=video, mask_video=mask, height=N.H,
              width=N.W, num_inference_steps=2, guidance_scale=6.0)
    want = EasyAnimateInpaintPipeline(vae=v, transformer=t, tokenizer=tok, text_encoder=enc)(
        generator=torch.Generator().manual_seed(4), **kw).frames
    pipe = EasyAnimateInpaintPipeline(vae=v, transformer=t, tokenizer=tok, text_encoder=enc).enable_model_cpu_offload("cpu")
    moves = []
    _log_moves(monkeypatch, {"text_encoder": enc, "vae": v, "transformer": t}, moves)
    got = pipe(generator=torch.Generator().manual_seed(4), **kw).frames
    assert torch.equal(got, want)
    # moves come in pairs, to(device) then to("cpu") of the same module: each goes back before the next one comes up
    assert len(moves) % 2 == 0 and all(moves[i][0] == moves[i + 1][0] for i in range(0, len(moves), 2))
    assert [m[1] for m in moves[1::2]] == ["cpu"] * (len(moves) // 2)
    names = [m[0] for m in moves[::2]]
    # two prompts, the masked video encoded (the mask is resized directly), the loop, the decode
    assert names == ["text_encoder", "text_encoder", "vae", "transformer", "vae"]
    # the text-to-video pipeline: prompt, loop, decode
    t16, v16 = _pipeline_modules(monkeypatch)
    moves2 = []
    pipe = EasyAnimatePipeline(vae=v16, transformer=t16, tokenizer=tok, text_encoder=enc).enable_model_cpu_offload("cpu")
    _log_moves(monkeypatch, {"text_encoder": enc, "vae": v16, "transformer": t16}, moves2)
    pipe(prompt="a cat", video_length=N.FRAMES, height=N.H, width=N.W, num_inference_steps=2, guidance_scale=6.0,
         generator=torch.Generator().manual_seed(5))
    assert [m[0] for m in moves2[::2]] == ["text_encoder", "text_encoder", "transformer", "vae"]


def test_load_pipeline_validates_the_memory_mode(tmp_path):
    from easyanimate_b200 import load_pipeline
    from easyanimate_b200.pipelines import GPU_MEMORY_MODES
    assert GPU_MEMORY_MODES == ("model_full_load", "model_cpu_offload", "model_cpu_offload_and_qfloat8", "sequential_cpu_offload")
    with pytest.raises(ValueError, match="GPU_memory_mode"):
        load_pipeline(str(tmp_path), GPU_memory_mode="sequential")


def test_load_pipeline_qfloat8_stores_the_transformer_as_e4m3(tmp_path, monkeypatch):
    import json
    from safetensors.torch import save_file
    from easyanimate_b200 import load_pipeline
    t, v = _pipeline_modules(monkeypatch)
    for name, module in (("transformer", t), ("vae", v)):
        d = tmp_path / name
        d.mkdir()
        (d / "config.json").write_text(json.dumps(dict(module.config)))
        save_file({k: x.detach().contiguous() for k, x in module.state_dict().items()}, str(d / "diffusion_pytorch_model.safetensors"))
    pipe = load_pipeline(str(tmp_path), device="cpu", GPU_memory_mode="model_cpu_offload_and_qfloat8")
    assert pipe.transformer.dtype == e4m3 and pipe._model_offload and pipe._execution_device == torch.device("cpu")
    for k, x in t.state_dict().items():
        assert torch.equal(pipe.transformer.state_dict()[k], x.to(e4m3) if x.is_floating_point() else x), k


# ---- the e4m3 text encoder of sequential_cpu_offload --------------------------------------------------------------------
def _tiny_qwen2_vl():
    transformers = pytest.importorskip("transformers")
    cfg = transformers.Qwen2VLConfig(
        text_config=dict(vocab_size=256, hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                         num_key_value_heads=2, max_position_embeddings=128,
                         rope_scaling={"type": "mrope", "mrope_section": [2, 3, 3]}),
        vision_config=dict(depth=1, embed_dim=32, hidden_size=64, num_heads=2, in_chans=3, patch_size=2, spatial_merge_size=2,
                           temporal_patch_size=2))
    torch.manual_seed(0)
    return transformers.Qwen2VLForConditionalGeneration(cfg).to(bf16).eval()


@pytest.mark.skipif(not os.path.exists(REF_FP8), reason="/root/reference not present")
def test_e4m3_text_encoder_equals_the_reference_conversion():
    """store_text_encoder_e4m3 against the reference's convert_model_weight_to_float8 + convert_weight_dtype_wrapper, imported
    unmodified: same parameter dtypes, the same hidden_states[-2] bit for bit - and not those of the bf16 encoder."""
    from easyanimate_b200.pipelines import _drop_visual_tower, store_text_encoder_e4m3
    spec = importlib.util.spec_from_file_location("reference_fp8_optimization", REF_FP8)
    ref_fp8 = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_fp8)
    base = _tiny_qwen2_vl()
    _drop_visual_tower(base)
    assert "visual" not in base.model._modules
    ref, ours = copy.deepcopy(base), copy.deepcopy(base)
    ref_fp8.convert_model_weight_to_float8(ref)
    ref_fp8.convert_weight_dtype_wrapper(ref, bf16)
    store_text_encoder_e4m3(ours, bf16)
    assert {n: p.dtype for n, p in ours.named_parameters()} == {n: p.dtype for n, p in ref.named_parameters()}
    ids = torch.randint(0, 256, (2, 12), generator=torch.Generator().manual_seed(1))
    mask = torch.ones_like(ids)
    mask[1, 9:] = 0
    with torch.no_grad():
        h = [m(input_ids=ids, attention_mask=mask, output_hidden_states=True).hidden_states[-2] for m in (base, ref, ours)]
    assert torch.equal(h[2], h[1])
    assert not torch.equal(h[2], h[0])
    assert {p.dtype for n, p in ours.named_parameters() if "embed_tokens" not in n} == {e4m3}  # back to e4m3 after the call
