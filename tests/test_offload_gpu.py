"""CPU-offload memory modes on the GPU: the packed e4m3 expansion kernel against per-parameter ea_dequant_e4m3, the sequentially
offloaded transformer forward against the resident forward (bit for bit, bf16 and e4m3 storage, CFG batch 2, TeaCache, three
blocks so both slots are reused), the device memory it holds, and the native pipelines under model_cpu_offload and
sequential_cpu_offload against model_full_load."""
import copy

import numpy as np
import pytest
import torch

from tests.test_offload_cpu import _forward, _inputs, _model

bf16, e4m3 = torch.bfloat16, torch.float8_e4m3fn


@pytest.mark.gpu
def test_packed_expansion_equals_per_parameter_dequant():
    from easyanimate_b200 import ops
    g = torch.Generator().manual_seed(0)
    counts = [256, 17, 4096 * 3, 1, 640, 8192 + 5]  # every e4m3 code (NaN included) in the first one, ragged tails
    offs, o = [], 0
    for n in counts:
        offs.append(o)
        o += (n + 15) // 16 * 16
    src = torch.randint(0, 256, (o,), generator=g, dtype=torch.uint8)
    src[:256] = torch.arange(256, dtype=torch.uint8)
    src = src.cuda()
    got = [torch.full((n,), 7.0, dtype=bf16, device="cuda") for n in counts]
    ops.expand_e4m3_segments(src, ops.e4m3_segment_table(list(zip(offs, got))))
    for off, n, x in zip(offs, counts, got):
        want = torch.empty((n,), dtype=bf16, device="cuda")
        ops.dequant_e4m3(src[off:off + n].view(e4m3).contiguous(), want)
        assert torch.equal(x.view(torch.int16), want.view(torch.int16)), (off, n)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [bf16, e4m3])
def test_offloaded_forward_is_bit_identical_to_resident(dtype):
    host = _model(dtype)
    resident = copy.deepcopy(host).to("cuda")
    off = host.enable_sequential_cpu_offload("cuda")
    coeffs = [1.07862322, -4.19362456, 3.06725828, 0.33161686, 0.02374758]
    for m in (resident, off):
        m.enable_teacache(4, 0.3, coefficients=coeffs)
    lat, enc, (c, s) = _inputs()
    lat, enc, rope = lat.cuda(), enc.cuda(), (c.cuda(), s.cuda())
    for t in (999, 900, 880, 500):
        want, got = _forward(resident, lat, t, enc, rope), _forward(off, lat, t, enc, rope)
        assert torch.equal(got, want), t
    assert off.teacache.skipped == resident.teacache.skipped > 0
    assert all(p.device.type == "cpu" and p.is_pinned() for p in off.transformer_blocks.parameters())
    with pytest.raises(Exception, match="CUDA graph"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            _forward(off, lat, 500, enc, rope)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [bf16, e4m3])
def test_device_parameter_memory_is_bounded(dtype):
    kw = dict(num_attention_heads=4, num_layers=5, mmdit_layers=5)
    lat, enc, (c, s) = _inputs(B=2)
    lat, enc, rope = lat.cuda(), enc.cuda(), (c.cuda(), s.cuda())
    torch.cuda.synchronize()

    def measure(m):
        _forward(m, lat, 500, enc, rope)  # derived copies (fused q/k/v, staging, slots) exist from here on
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        _forward(m, lat, 500, enc, rope)
        torch.cuda.synchronize()
        return base, torch.cuda.max_memory_allocated() - base

    resident = _model(dtype, **kw).to("cuda")
    r_base, r_act = measure(resident)
    del resident
    torch.cuda.empty_cache()
    zero = torch.cuda.memory_allocated()
    off = _model(dtype, **kw).enable_sequential_cpu_offload("cuda")
    o_base, o_act = measure(off)
    held = o_base - zero

    def alloc(tensors):  # bytes the caching allocator hands out for them (512-byte granules)
        return sum((t.nbytes + 511) // 512 * 512 for t in tensors)
    head = alloc(p for n, p in off.named_parameters() if not n.startswith("transformer_blocks."))
    block = off._offload.packs[0].host.nbytes
    slots = off._offload.device_bytes()
    assert slots == 2 * block
    patch = alloc([off.proj.weight.to(bf16)])  # the [d, 4C] patch-embed GEMM operand
    bound = head + slots + patch
    if dtype == e4m3:  # the bf16 copies of the non-block parameters and the one bf16 staging block (+ its fused q/k/v)
        staging = off._fp8[1]
        st = staging._blocks[True]
        assert list(staging._blocks) == [True]
        bound += alloc(staging.head.parameters()) + alloc(st.parameters())
        bound += alloc(t for a in (st.attn1, st.attn2) for t in a._fused_static)
    assert held <= bound, (held, bound)
    assert held < sum(p.nbytes for p in off.transformer_blocks.parameters())  # the blocks are not resident
    assert o_act <= r_act + (1 << 20), (o_act, r_act)  # activations: no more than the resident forward's


class _DeviceTokens(dict):
    input_ids = property(lambda self: self["input_ids"])
    attention_mask = property(lambda self: self["attention_mask"])

    def to(self, device):
        return _DeviceTokens({k: v.to(device) for k, v in self.items()})


def _tokenizer():
    from tests import test_native_pipelines_cpu as N

    class Tokenizer(N._FakeTokenizer):  # whose tokens follow the text encoder to the GPU
        def __call__(self, *a, **k):
            t = super().__call__(*a, **k)
            return _DeviceTokens(input_ids=t.input_ids, attention_mask=t.attention_mask)
    return Tokenizer()


def _pipelines(in_channels):
    from tests import test_native_pipelines_cpu as N
    kw = {} if in_channels == 16 else dict(resize_inpaint_mask_directly=True, enable_clip_in_inpaint=False)
    return N._modules(in_channels=in_channels, seeds=(61, 62), **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["model_cpu_offload", "sequential_cpu_offload"])
@pytest.mark.parametrize("in_channels", [16, 33])
def test_offloaded_pipeline_frames_equal_full_load(mode, in_channels):
    from easyanimate_b200 import EasyAnimateInpaintPipeline, EasyAnimatePipeline
    from tests import test_native_pipelines_cpu as N
    kind = EasyAnimatePipeline if in_channels == 16 else EasyAnimateInpaintPipeline
    g = torch.Generator().manual_seed(3)
    kw = dict(prompt="a cat", negative_prompt="blurry", video_length=N.FRAMES, height=N.H, width=N.W, num_inference_steps=2,
              guidance_scale=6.0)
    if in_channels == 33:
        video = torch.rand(1, 3, N.FRAMES, N.H, N.W, generator=g)
        mask = torch.zeros_like(video[:, :1])
        mask[:, :, 1:] = 255
        kw.update(video=video, mask_video=mask)
    torch.manual_seed(0)
    enc = N._FakeTextEncoder(128).to(bf16)
    t, v = _pipelines(in_channels)
    full = kind(vae=v, transformer=t, tokenizer=_tokenizer(), text_encoder=copy.deepcopy(enc)).to("cuda")
    want = full(generator=torch.Generator().manual_seed(4), **kw).frames
    t, v = _pipelines(in_channels)
    pipe = kind(vae=v, transformer=t, tokenizer=_tokenizer(), text_encoder=enc)
    pipe = pipe.enable_model_cpu_offload("cuda") if mode == "model_cpu_offload" else pipe.enable_sequential_cpu_offload("cuda")
    got = pipe(generator=torch.Generator().manual_seed(4), **kw).frames
    assert np.array_equal(got, want)
    assert all(p.device.type == "cpu" for p in enc.parameters())
    if mode == "model_cpu_offload":
        assert all(p.device.type == "cpu" for m in (t, v) for p in m.parameters())
    else:
        assert all(p.is_pinned() for p in t.transformer_blocks.parameters()) and next(v.parameters()).is_cuda
