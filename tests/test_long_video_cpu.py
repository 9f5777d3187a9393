"""`generate_long_video` (easyanimate_b200/long_video.py) against the reference's "Long Video Generation" loop (ui.py:485-552,
restated in tests/long_video_oracle.py over the reference's own EasyAnimateInpaintPipeline, PIL for the chained frames), both
over the same tiny product modules with the kernels replaced by the torch stand-ins of tests/cpu_ops.py.  Where the reference is
not installed the frames are compared with a stored sample of the reference's (tests/golden/long_video_ref.safetensors)."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import ref_pipeline
from tests import cpu_ops, long_video_oracle, refgold
from tests.test_native_pipelines_cpu import _embeds, _mask_kw, _modules, on_cpu  # noqa: F401  (on_cpu is a fixture)

LIVE = ref_pipeline.available()
GOLD = refgold.Store("long_video_ref")
H, W, STEPS = 64, 96, 2
INP = dict(in_channels=33, seeds=(73, 74), resize_inpaint_mask_directly=True, enable_clip_in_inpaint=False,
           add_noise_in_inpaint_model=True)


def frames_out_blend(video, out, overlap):
    """ea_frames_out_blend as the reference's tensor ops (pipeline_easyanimate.py:738-741, then ui.py:524-531)."""
    f = (video.clamp(-1, 1) / 2 + 0.5).clamp(0, 1).float()
    if overlap:
        r = torch.tensor([float(i) / float(overlap) for i in range(overlap)], dtype=torch.float32).view(1, 1, -1, 1, 1)
        out[:, :, :overlap] = out[:, :, :overlap] * (1 - r) + f[:, :, :overlap] * r
    out[:, :, overlap:] = f[:, :, overlap:]
    return out


@pytest.fixture
def lv_cpu(on_cpu, monkeypatch):  # noqa: F811
    from easyanimate_b200 import vae_ops
    monkeypatch.setattr(vae_ops, "frames_out_blend", frames_out_blend)
    return on_cpu


@pytest.fixture(scope="module", autouse=True)
def _save_minted():
    yield
    GOLD.save()


def _images(seed, n):
    g = torch.Generator().manual_seed(seed)
    return [Image.fromarray(torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8).numpy()) for _ in range(n)]


CASES = {  # name: (video_length, partial_video_length, overlap_video_length, start images, end images)
    "no_start": (13, 9, 4, None, None),
    "start": (13, 9, 4, 1, None),
    "start_end": (20, 9, 4, 1, 1),
    "overlap_1": (14, 5, 1, 1, None),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_long_video_equals_the_reference_loop(lv_cpu, case):
    from easyanimate_b200 import EasyAnimateInpaintPipeline, generate_long_video
    length, partial, ov, n_start, n_end = CASES[case]
    t, v = _modules(lv_cpu, **INP)
    pe, ne = _embeds(torch.Generator().manual_seed(50))
    start = None if n_start is None else _images(51, n_start)
    end = None if n_end is None else _images(52, n_end)
    kw = dict(num_inference_steps=STEPS, guidance_scale=6.0, **_mask_kw(pe, ne))
    got = generate_long_video(EasyAnimateInpaintPipeline(vae=v, transformer=t), video_length=length, partial_video_length=partial,
                              overlap_video_length=ov, start_image=start, end_image=end, height=H, width=W,
                              generator=torch.Generator().manual_seed(53), **kw).frames
    want = windows = None
    if LIVE:
        want, windows = long_video_oracle.long_video(
            ref_pipeline.reference_inpaint_pipeline(t, v), length_slider=length, partial_video_length=partial,
            overlap_video_length=ov, start_image=start, end_image=end, height=H, width=W,
            generator=torch.Generator().manual_seed(53), **kw)
    windows = GOLD.value(f"{case}.windows", (lambda: [list(w) for w in windows]) if LIVE else None)
    assert len(windows) > 1 and got.shape == (1, 3, windows[-1][0] + windows[-1][1], H, W) and got.dtype == torch.float32
    GOLD.same_sample(case, got, want)


def test_window_schedule_equals_the_reference_loop():
    """Window starts and lengths, including the 1 + 4m rounding of the last window and a rest that rounds to no frame."""
    from easyanimate_b200.long_video import long_video_windows

    class Shape:
        def __call__(self, video_length, **kw):
            return type("Out", (), {"frames": torch.zeros(1, 3, video_length, 2, 2)})()

    for length, partial, ov, cache in [(97, 49, 4, True), (139, 49, 4, True), (49, 49, 4, True), (30, 49, 4, True),
                                       (14, 5, 1, True), (13, 9, 4, True), (50, 25, 3, True), (47, 25, 4, True),
                                       (52, 24, 4, False), (2, 8, 4, False)]:
        want = long_video_oracle.long_video(Shape(), length_slider=length, partial_video_length=partial, overlap_video_length=ov,
                                            start_image=None, end_image=None, height=2, width=2, cache_mag_vae=cache)[1]
        assert long_video_windows(length, partial, ov, 4, cache) == want, (length, partial, ov, cache)
    assert long_video_windows(97, 49, 4) == [(0, 49), (45, 49), (90, 5)]


def test_long_video_refuses_what_the_reference_refuses(lv_cpu):
    from easyanimate_b200 import EasyAnimateInpaintPipeline, EasyAnimatePipeline, generate_long_video
    t, v = _modules(lv_cpu, **INP)
    t16, _ = _modules(lv_cpu)
    pe, ne = _embeds(torch.Generator().manual_seed(54))
    ok = dict(video_length=13, partial_video_length=9, height=H, width=W, num_inference_steps=STEPS, guidance_scale=6.0,
              **_mask_kw(pe, ne))
    for pipe in (EasyAnimatePipeline(vae=v, transformer=t16), EasyAnimateInpaintPipeline(vae=v, transformer=t16)):
        with pytest.raises(ValueError, match="image to video pretrained model"):
            generate_long_video(pipe, **ok)
    pipe = EasyAnimateInpaintPipeline(vae=v, transformer=t)
    with pytest.raises(ValueError, match="Video to Video is not Support"):
        generate_long_video(pipe, video=torch.zeros(1, 3, 9, H, W), **ok)
    with pytest.raises(ValueError, match="specify a starting image"):
        generate_long_video(pipe, end_image=_images(55, 1), **ok)
    bad = [dict(overlap_video_length=0), dict(overlap_video_length=9), dict(partial_video_length=8),
           dict(video_length=20, partial_video_length=5, overlap_video_length=3), dict(mask_video=torch.zeros(1, 1, 9, H, W)),
           dict(start_image=torch.zeros(3, H, W + 16, dtype=torch.uint8))]
    for extra in bad:
        with pytest.raises(ValueError):
            generate_long_video(pipe, **{**ok, **extra})


def test_tensor_images_condition_like_pil_images(lv_cpu):
    """uint8 tensors [n,3,H,W] give the frames the same pictures give as PIL images."""
    from easyanimate_b200 import EasyAnimateInpaintPipeline, generate_long_video
    t, v = _modules(lv_cpu, **INP)
    pe, ne = _embeds(torch.Generator().manual_seed(56))
    start, end = _images(57, 2), _images(58, 1)
    as_tensor = [torch.stack([torch.from_numpy(np.array(im)).permute(2, 0, 1) for im in ims]) for ims in (start, end)]
    kw = dict(video_length=13, partial_video_length=9, overlap_video_length=4, height=H, width=W, num_inference_steps=STEPS,
              guidance_scale=6.0, **_mask_kw(pe, ne))
    pipe = EasyAnimateInpaintPipeline(vae=v, transformer=t)
    a = generate_long_video(pipe, start_image=start, end_image=end[0], generator=torch.Generator().manual_seed(59), **kw).frames
    b = generate_long_video(pipe, start_image=as_tensor[0], end_image=as_tensor[1][0], generator=torch.Generator().manual_seed(59),
                            **kw).frames
    assert torch.equal(a, b)


def _dist_worker(rank, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE="2")
    dist.init_process_group("gloo", rank=rank, world_size=2)
    mp = pytest.MonkeyPatch()
    try:
        q.put((rank, _run_cfg_pair(mp, dist.new_group([0, 1]))))
        dist.barrier()
    finally:
        mp.undo()
        dist.destroy_process_group()


def _run_cfg_pair(mp, group):
    import easyanimate_b200.autoencoder_magvit as A
    from easyanimate_b200 import EasyAnimateInpaintPipeline, generate_long_video, ops, vae_ops
    cpu_ops.install(mp)
    cpu_ops.install_vae(mp)
    mp.setattr(ops, "cfg_euler_step", cpu_ops.cfg_euler_step)
    mp.setattr(A, "_require_cuda", lambda t, what: None)
    mp.setattr(vae_ops, "frames_out_blend", frames_out_blend)
    t, v = _modules(A, **INP)
    pe, ne = _embeds(torch.Generator().manual_seed(60))
    pipe = EasyAnimateInpaintPipeline(vae=v, transformer=t, cfg_group=group)
    return generate_long_video(pipe, video_length=13, partial_video_length=9, overlap_video_length=4, start_image=_images(61, 1),
                               height=H, width=W, num_inference_steps=STEPS, guidance_scale=6.0,
                               generator=torch.Generator().manual_seed(62), **_mask_kw(pe, ne)).frames


def test_cfg_parallel_pair_gives_the_single_process_video():
    """A gloo CFG pair (each rank one guidance branch, pipeline.py): both ranks return the whole video, equal to one process."""
    import torch.multiprocessing as tmp
    ctx = tmp.get_context("spawn")
    q = ctx.Queue()
    port = 29100 + (os.getpid() % 400)
    procs = [ctx.Process(target=_dist_worker, args=(r, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=600) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    mp = pytest.MonkeyPatch()
    try:
        single = _run_cfg_pair(mp, None)
    finally:
        mp.undo()
    assert torch.equal(got[0], got[1]) and torch.equal(got[0], single)


def test_gpu_prelude_runs_without_a_gpu():
    from tests import test_long_video_gpu as T
    pipe, kw, start = T.prelude_long_video(device="cpu")
    assert pipe.transformer.config.in_channels == 33 and start.size == (T.W, T.H) and kw["num_inference_steps"] == 3


def test_pil_resize_to_its_own_size_is_a_copy():
    """ui.py:540-544 chains the frames through `Image.fromarray` and get_image_to_video_latent's `.resize` to the size the image
    has: the pixels come back unchanged, so generate_long_video conditions the next window on the uint8 frames directly."""
    g = torch.Generator().manual_seed(63)
    for h, w in ((H, W), (512, 512), (48, 80)):
        a = torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).numpy()
        assert np.array_equal(np.array(Image.fromarray(a).resize([w, h])), a)
