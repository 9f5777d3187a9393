"""Long-video cost on one GPU: ms per output frame of `generate_long_video` (three 49-frame windows, 4-frame overlap:
video_length 139 -> 139 frames) against one 49-frame `EasyAnimateInpaintPipeline` call, on a random-init 7B-shaped InP model
(bench.py's R512_7B preset with in_channels 33) at 512x512, and the GPU idle time ("host gap") inside the long-video call from
a torch.profiler trace taken in a separate run.  Prints one JSON line; the trace goes to --out.

    python tools/bench_long_video.py [--steps 8] [--out DIR]   (DIR defaults to a new temporary directory)
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from easyanimate_b200 import EasyAnimateInpaintPipeline, generate_long_video  # noqa: E402

H = W = 512
PARTIAL, OVERLAP, LONG = 49, 4, 139


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def build_inp_model(preset, dev, seed=1234):
    """bench.build_model with the V5.1 InP transformer settings (predict_i2v.py's config: the mask resized to the latent grid,
    no CLIP branch, noise on the conditioning video)."""
    from easyanimate_b200.transformer3d import EasyAnimateTransformer3DModel
    torch.manual_seed(seed)
    with torch.device(dev):
        model = EasyAnimateTransformer3DModel(**bench.model_cfg(preset), resize_inpaint_mask_directly=True,
                                              enable_clip_in_inpaint=False, add_noise_in_inpaint_model=True).to(torch.bfloat16)
    with torch.no_grad():
        for name, prm in model.named_parameters():
            prm.normal_(1.0 if prm.dim() == 1 and name.endswith("weight") else 0.0, 0.02)
    return model


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--out", default=None, help="where the trace goes (default: a new temporary directory)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda")
    preset = dict(bench.PRESETS["R512_7B"], inpaint=True)
    pipe = EasyAnimateInpaintPipeline(vae=bench.build_vae(dev), transformer=build_inp_model(preset, dev))
    g = torch.Generator().manual_seed(0)
    pe = torch.randn(1, bench.S_TEXT, bench.E_TEXT, generator=g).to(dev, torch.bfloat16)
    ne = torch.randn(1, bench.S_TEXT, bench.E_TEXT, generator=g).to(dev, torch.bfloat16)
    ones = torch.ones(1, bench.S_TEXT, dtype=torch.long, device=dev)
    start = torch.randint(0, 256, (3, H, W), generator=g, dtype=torch.uint8)
    kw = dict(prompt_embeds=pe, negative_prompt_embeds=ne, prompt_attention_mask=ones, negative_prompt_attention_mask=ones,
              prompt_embeds_2=pe, prompt_attention_mask_2=ones, height=H, width=W, num_inference_steps=args.steps,
              guidance_scale=bench.GUIDANCE, noise_aug_strength=0.0563)

    def one_window():
        return generate_long_video(pipe, video_length=PARTIAL, partial_video_length=PARTIAL, overlap_video_length=OVERLAP,
                                   start_image=start, generator=torch.Generator(device=dev).manual_seed(1), **kw).frames

    def long_video():
        return generate_long_video(pipe, video_length=LONG, partial_video_length=PARTIAL, overlap_video_length=OVERLAP,
                                   start_image=start, generator=torch.Generator(device=dev).manual_seed(1), **kw).frames

    def timed(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        frames = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1e3, frames.shape[2]

    # per-phase host times of one long video: every denoise loop and decode is bracketed by synchronisations, the rest of the
    # call (conditioning, VAE encode, cross-fade into host memory, chained frames) is what lies between them
    phases = {"denoise": 0.0, "decode": 0.0}

    def bracket(name, fn):
        def run(*a, **k):
            torch.cuda.synchronize()
            t = time.perf_counter()
            r = fn(*a, **k)
            torch.cuda.synchronize()
            phases[name] += (time.perf_counter() - t) * 1e3
            return r
        return run

    timed(one_window)  # warm-up of every shape
    timed(long_video)
    runs = {"single": [], "long": []}
    for _ in range(2):
        runs["single"].append(timed(one_window))
        runs["long"].append(timed(long_video))
    pipe._denoise = bracket("denoise", pipe._denoise)
    pipe.vae.decode_scaled_video = bracket("decode", pipe.vae.decode_scaled_video)
    bracketed_ms, _ = timed(long_video)
    del pipe._denoise, pipe.vae.decode_scaled_video

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        timed(long_video)
    args.out = args.out or tempfile.mkdtemp(prefix="ea_long_video_")
    os.makedirs(args.out, exist_ok=True)
    trace = os.path.join(args.out, "long_video_trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        events = json.load(f)["traceEvents"]
    dev_ev = sorted((e["ts"], e["ts"] + e["dur"], e["name"]) for e in events
                    if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset") and "dur" in e)
    idle, end, gaps = 0.0, dev_ev[0][1], []
    for t0, t1, name in dev_ev[1:]:
        if t0 > end:
            idle += t0 - end
            gaps.append((t0 - end, name))
        end = max(end, t1)
    span_ms = (dev_ev[-1][1] - dev_ev[0][0]) / 1e3
    single_ms = min(ms for ms, _ in runs["single"])
    long_ms = min(ms for ms, _ in runs["long"])
    n_single, n_long = runs["single"][0][1], runs["long"][0][1]
    print(json.dumps({
        "card": card(), "model": "random-init 7B-shaped InP transformer (28 layers, 48 heads, in_channels 33) + MagViT VAE",
        "size": f"{H}x{W}", "steps": args.steps, "guidance": bench.GUIDANCE,
        "single_call": {"frames": n_single, "ms": [round(ms, 1) for ms, _ in runs["single"]], "ms_per_frame": round(single_ms / n_single, 2)},
        "long_video": {"frames": n_long, "windows": [PARTIAL] * 3, "overlap": OVERLAP,
                       "ms": [round(ms, 1) for ms, _ in runs["long"]], "ms_per_frame": round(long_ms / n_long, 2)},
        "long_video_phases_ms": {"total_bracketed": round(bracketed_ms, 1), "denoise": round(phases["denoise"], 1),
                                 "decode": round(phases["decode"], 1),
                                 "rest": round(bracketed_ms - phases["denoise"] - phases["decode"], 1)},
        "profiler": {"device_span_ms": round(span_ms, 1), "device_idle_ms": round(idle / 1e3, 1),
                     "largest_idle_gaps_ms_before": [[round(d / 1e3, 2), n[:60]] for d, n in sorted(gaps, reverse=True)[:8]],
                     "trace": trace},
    }))


if __name__ == "__main__":
    main()
