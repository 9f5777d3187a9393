"""LoRA merge on the H100: ea_lora_merge bit for bit against a host emulation of its specified arithmetic (fp32 FMA chain in
ascending k from +0, then the rounding points of include/ea_b200.h), every e4m3 store code against torch's own CUDA cast, a
bench-shaped two-block model, and every weight storage / memory mode against the resident merge."""
import copy
import types

import numpy as np
import pytest
import torch

from tests.test_offload_cpu import _forward, _inputs, _model

bf16, e4m3 = torch.bfloat16, torch.float8_e4m3fn


def _rnd(x: np.ndarray, dtype) -> np.ndarray:
    """fp32 array rounded to `dtype` (torch's casts) and back to fp32; identity for fp32."""
    if dtype == torch.float32:
        return x
    return torch.from_numpy(np.ascontiguousarray(x)).to(dtype).float().numpy()


def emulate(w: torch.Tensor, up: torch.Tensor, down: torch.Tensor, scale: float) -> torch.Tensor:
    """The merged weight in w's storage dtype, in numpy fp32: the exact products up[:, k] * down[k, :] added to an accumulator
    that starts at +0 in ascending k (what a chain of fp32 FMAs gives when the products are exact), then
    d = rnd_c(acc), d2 = rnd_c(scale * d), w = rnd_c(W + d2), stored with torch's cast."""
    c = up.dtype
    U, D = up.cpu().float().numpy(), down.cpu().float().numpy()
    acc = np.zeros((U.shape[0], D.shape[1]), dtype=np.float32)
    tmp = np.empty_like(acc)
    for k in range(U.shape[1]):
        np.multiply(U[:, k, None], D[None, k, :], out=tmp)
        np.add(acc, tmp, out=acc)
    d = _rnd(acc, c)
    d2 = _rnd(np.float32(scale) * d, c)
    wv = _rnd(w.cpu().float().numpy() + d2, c)
    return torch.from_numpy(wv).to(w.dtype)


def emulate_on_gpu(w: torch.Tensor, up: torch.Tensor, down: torch.Tensor, scale: float) -> torch.Tensor:
    """emulate() with torch's elementwise CUDA ops (one rounding each, like numpy's), for the large models."""
    c = up.dtype
    U, D = up.cuda().float(), down.cuda().float()
    acc = torch.zeros((U.shape[0], D.shape[1]), dtype=torch.float32, device="cuda")
    for k in range(U.shape[1]):
        acc = acc + U[:, k, None] * D[None, k, :]
    rnd = (lambda x: x) if c == torch.float32 else (lambda x: x.to(c).float())
    d = rnd(acc)
    d2 = rnd(torch.tensor(scale, dtype=torch.float32, device="cuda") * d)
    return rnd(w.cuda().float() + d2).to(w.dtype).cpu()


def _same(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.cpu().view(torch.uint8), b.cpu().view(torch.uint8))


def _factors(rows, rank, cols, compute, g, exact_f32=True, mag=1.0):
    up, down = torch.randn(rows, rank, generator=g) * mag, torch.randn(rank, cols, generator=g) * mag
    if compute == torch.float32 and exact_f32:  # fp16-representable: every product is exact in fp32
        up, down = up.half().float(), down.half().float()
    return up.to(compute), down.to(compute)


CASES = (
    # (rows, cols, rank, compute, storage, ldw pad, scale)
    [(100, 36, r, c, bf16, 0, 0.37) for r in (1, 4, 13, 64, 128, 320) for c in (bf16, torch.float32)]
    + [(100, 36, r, torch.float32, e4m3, 5, -1.7) for r in (1, 13, 320)]
    + [(shape[0], shape[1], 13, c, s, pad, sc) for shape, pad, sc in (((3072, 3072), 0, 0.5), ((12288, 3072), 0, -0.25),
                                                                        ((3072, 12288), 8, 0.125), ((1, 8), 3, -2.0))
       for c, s in ((bf16, bf16), (torch.float32, e4m3))]
    + [(3072, 3072, 128, bf16, bf16, 0, 0.25), (3072, 3072, 320, torch.float32, bf16, 1, -0.5), (3072, 3072, 64, bf16, e4m3, 0, 3.0)]
)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols,rank,compute,storage,pad,scale", CASES)
def test_kernel_equals_the_emulation(rows, cols, rank, compute, storage, pad, scale):
    from easyanimate_b200 import ops
    g = torch.Generator().manual_seed(rows * 7 + cols * 3 + rank)
    w0 = (torch.randn(rows, cols + pad, generator=g) * 4)
    if storage == e4m3:  # some weights near the top of the e4m3 range, where the sum can round past 448 to NaN
        w0[::7] = w0[::7].sign() * 448
    w0 = w0.to(storage)
    up, down = _factors(rows, rank, cols, compute, g, mag=4.0 if storage == e4m3 else 1.0)
    want = emulate(w0[:, :cols], up, down, scale)
    if rows * cols * rank < 10 ** 8:  # the GPU emulation of the model test agrees with this one
        assert _same(emulate_on_gpu(w0[:, :cols], up, down, scale), want)
    w = w0.cuda()
    ops.lora_merge(w[:, :cols], up.cuda(), down.cuda(), scale)
    torch.cuda.synchronize()
    assert _same(w[:, :cols], want)
    assert _same(w[:, cols:], w0[:, cols:])  # the row padding beyond cols is untouched
    if storage == e4m3 and rows * cols >= 3600:
        assert torch.isnan(w.float()).any()  # overflow past 448 stored NaN, as torch's cast does


@pytest.mark.gpu
def test_every_e4m3_store_code_is_torchs_cast():
    """Rank 1, up = 1, W = 0: the stored byte is the cast of down (each of the 65 536 bf16 patterns) for every non-NaN input,
    compared with torch's own CUDA cast of the same fp32 value.  -0 becomes +0 on the way (the sum starts at +0)."""
    from easyanimate_b200 import ops
    down = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(bf16).reshape(1, -1).cuda()
    up = torch.ones((1, 1), dtype=bf16, device="cuda")
    w = torch.zeros((1, 65536), dtype=e4m3, device="cuda")
    ops.lora_merge(w, up, down, 1.0)
    value = down.float() + 0.0  # the accumulator's value: down itself, -0 turned +0
    want = value.to(e4m3)
    nan = torch.isnan(value)
    got, ref = w.view(torch.uint8), want.view(torch.uint8)
    assert torch.equal(got[~nan], ref[~nan])
    assert torch.isnan(w[nan].float()).all()
    assert (ref == 0x7f).any() and (ref == 0xff).any()  # finite overflow reached NaN in both signs


def _merged_state(m, sd, multiplier, compute):
    """The emulated merge of `sd` (lora_unet__<path> keys) into the state dict of m."""
    out = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    layers = {k.split(".", 1)[0] for k in sd}
    for layer in layers:
        path = layer[len("lora_unet__"):]
        name = next(n for n, _ in m.named_modules() if n.replace(".", "_") == path) + ".weight"
        up, down = sd[layer + ".lora_up.weight"], sd[layer + ".lora_down.weight"]
        s = float(torch.tensor(multiplier * sd[layer + ".alpha"].item() / up.shape[1], dtype=torch.float32))
        out[name] = emulate_on_gpu(out[name], up.to(compute), down.to(compute), s)
    return out


def _lora_for(m, rank, g, scale=0.05):
    sd = {}
    for n, mod in m.named_modules():
        if isinstance(mod, torch.nn.Linear):
            o, i = mod.weight.shape
            key = "lora_unet__" + n.replace(".", "_")
            sd[key + ".lora_up.weight"] = (torch.randn(o, rank, generator=g) * scale).to(bf16)
            sd[key + ".lora_down.weight"] = (torch.randn(rank, i, generator=g) * scale).to(bf16)
            sd[key + ".alpha"] = torch.tensor(float(rank // 2))
    return sd


@pytest.mark.gpu
def test_bench_shaped_model_merge_and_forward():
    """Two blocks at d = 3072 (48 heads), a rank-64 LoRA on every Linear: the merged parameters equal the emulation, and a
    forward before the merge then one after it equals a fresh model loaded with the emulated state dict."""
    from easyanimate_b200 import merge_lora
    from easyanimate_b200.transformer3d import EasyAnimateTransformer3DModel
    cfg = dict(num_attention_heads=48, attention_head_dim=64, in_channels=16, out_channels=16, patch_size=2, num_layers=2,
               time_embed_dim=512, add_norm_text_encoder=True, text_embed_dim=256, text_embed_dim_t5=None)
    torch.manual_seed(0)
    m = EasyAnimateTransformer3DModel(**cfg).to(bf16)
    sd = _lora_for(m, 64, torch.Generator().manual_seed(1))
    want = _merged_state(m, sd, 0.8, bf16)
    m = m.cuda()
    g = torch.Generator().manual_seed(2)
    lat = torch.randn(1, 16, 2, 16, 16, generator=g).to(bf16).cuda()
    enc = (torch.randn(1, 12, 256, generator=g) * 3).to(bf16).cuda()
    from easyanimate_b200.pipeline import rope_table
    rope = tuple(x.cuda() for x in rope_table(128, 128, 2))
    _forward(m, lat, 500, enc, rope)
    merge_lora(types.SimpleNamespace(transformer=m), None, 0.8, state_dict=sd, dtype=bf16)
    got = m.state_dict()
    for k, v in want.items():
        assert _same(got[k], v), k
    after = _forward(m, lat, 500, enc, rope)
    fresh = EasyAnimateTransformer3DModel(**cfg).to(bf16)
    fresh.load_state_dict(want)
    assert torch.equal(after, _forward(fresh.cuda(), lat, 500, enc, rope))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [bf16, e4m3])
def test_every_mode_equals_the_resident_merge(dtype):
    from easyanimate_b200 import EasyAnimatePipeline, merge_lora
    from tests import test_native_pipelines_cpu as N
    host = _model(dtype)
    sd = _lora_for(host, 8, torch.Generator().manual_seed(3), scale=0.2)
    lat, enc, (c, s) = _inputs()
    lat, enc, rope = lat.cuda(), enc.cuda(), (c.cuda(), s.cuda())

    resident = copy.deepcopy(host).cuda()
    _forward(resident, lat, 700, enc, rope)
    merge_lora(types.SimpleNamespace(transformer=resident), None, 1.1, state_dict=sd)
    want = {k: v.detach().cpu().clone() for k, v in resident.state_dict().items()}
    assert not _same(want["transformer_blocks.0.attn1.to_q.weight"], host.state_dict()["transformer_blocks.0.attn1.to_q.weight"])
    want_out = _forward(resident, lat, 700, enc, rope)

    seq = copy.deepcopy(host).enable_sequential_cpu_offload("cuda")
    _forward(seq, lat, 700, enc, rope)
    hosts = [pk.host.data_ptr() for pk in seq._offload.packs]
    seq.invalidate_weight_caches()  # what the forward derived on the device goes; the merge itself must leave nothing behind
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    merge_lora(types.SimpleNamespace(transformer=seq), None, 1.1, state_dict=sd)
    assert torch.cuda.memory_allocated() == before
    assert [pk.host.data_ptr() for pk in seq._offload.packs] == hosts
    assert all(p.is_pinned() for p in seq.transformer_blocks.parameters())
    for k, v in seq.state_dict().items():
        assert _same(v, want[k]), k
    assert torch.equal(_forward(seq, lat, 700, enc, rope), want_out)

    t, v = copy.deepcopy(host), N._modules()[1]
    pipe = EasyAnimatePipeline(vae=v, transformer=t, tokenizer=N._FakeTokenizer(),
                               text_encoder=N._FakeTextEncoder(128).to(bf16)).enable_model_cpu_offload("cuda")
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    merge_lora(pipe, None, 1.1, state_dict=sd)
    assert torch.cuda.memory_allocated() == before
    assert all(p.device.type == "cpu" for p in t.parameters())
    for k, x in t.state_dict().items():
        assert _same(x, want[k]), k
    assert torch.equal(_forward(t.cuda(), lat, 700, enc, rope), want_out)
