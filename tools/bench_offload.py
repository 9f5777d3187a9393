"""Sequential CPU offload of the MMDiT on one GPU: CFG-step time (one transformer forward on the CFG batch of 2) of resident
execution and of the offloaded forward with bf16 and with e4m3 host storage, alternated in one run; device memory; host-to-device
bytes per step; and, in a separate torch.profiler pass, the time the compute stream sits idle during an offloaded forward.
Device memory of a mode is everything it holds on the device - its parameters, the slots, and every copy derived from them on
the first forward (fused q/k/v operands, the e4m3 staging block and bf16 non-block copies) - measured with memory_allocated()
from before the mode's model is built, plus the peak of max_memory_allocated() above that during its forward.
--e2e adds one end-to-end text-to-video call of the native pipeline under model_cpu_offload with the UNTILED VAE decode
(bench.py's VAE), which the resident model rules out at 720p.  Random-init models of bench.py's shapes.  Prints one JSON line
per shape (and writes them all to --out when given).

    python tools/bench_offload.py [--presets R512_7B R720_7B R720_12B] [--reps 3] [--e2e R720_7B] [--out FILE]
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from easyanimate_b200.pipeline import rope_table  # noqa: E402
from easyanimate_b200.transformer3d import EasyAnimateTransformer3DModel  # noqa: E402

bf16 = torch.bfloat16


def host_copy(resident, dtype, offload=True):
    """The resident model's weights in a host model stored as `dtype`, sequentially offloaded (or moved to the device)."""
    with torch.device("meta"):
        m = EasyAnimateTransformer3DModel(**{k: v for k, v in resident.config.items() if not k.startswith("_")})
    m = m.to_empty(device="cpu").to(bf16)
    m.load_state_dict(resident.state_dict())
    m = m.to(dtype)
    return m.enable_sequential_cpu_offload("cuda") if offload else m.to("cuda")


def idle_ms(fn):
    """Sum of the gaps between consecutive kernels of the compute stream during fn() (torch.profiler, a run of its own)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    spans = sorted((e.time_range.start, e.time_range.end) for e in prof.events()
                   if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
                   and "memset" not in e.name.lower())
    gap, end = 0.0, spans[0][1]
    for s, e in spans[1:]:
        gap += max(0.0, s - end)
        end = max(end, e)
    return gap / 1e3, (spans[-1][1] - spans[0][0]) / 1e3


def e2e(name, steps, dev, smi):
    """One text-to-video call of the native pipeline under model_cpu_offload (prompt given as embeddings): the transformer
    visits the GPU for the loop, then the VAE for the untiled decode."""
    from easyanimate_b200 import EasyAnimatePipeline
    p = bench.PRESETS[name]
    t = bench.build_model(p, dev).to("cpu")
    v = bench.build_vae(dev, tiled=False).to("cpu")
    torch.cuda.empty_cache()
    pipe = EasyAnimatePipeline(vae=v, transformer=t).enable_model_cpu_offload(dev)
    g = torch.Generator().manual_seed(1)
    pe, ne = ((torch.randn(1, bench.S_TEXT, bench.E_TEXT, generator=g) * 3).to(bf16) for _ in range(2))
    ones = torch.ones((1, bench.S_TEXT), dtype=torch.long)
    frames = 4 * (p["F"] - 1) + 1
    kw = dict(video_length=frames, height=p["h"] * 8, width=p["w"] * 8, num_inference_steps=steps, guidance_scale=bench.GUIDANCE,
              prompt_embeds=pe, negative_prompt_embeds=ne, prompt_attention_mask=ones, negative_prompt_attention_mask=ones,
              prompt_embeds_2=pe, prompt_attention_mask_2=ones, generator=torch.Generator().manual_seed(2))
    gc.collect()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    video = pipe(**kw).frames
    torch.cuda.synchronize()
    sec = time.perf_counter() - t0
    on_host = all(not q.is_cuda for m in (t, v) for q in m.parameters())
    return {"e2e": f"EasyAnimatePipeline under model_cpu_offload, {name} transformer, {frames} frames x {kw['height']}x{kw['width']}, "
                   f"{steps} steps with CFG, untiled VAE decode", "gpu": smi, "call_s": sec,
            "device_peak_gb": (torch.cuda.max_memory_allocated() - before) / 1e9, "frames_shape": list(video.shape),
            "frames_finite": bool(torch.isfinite(torch.as_tensor(video)).all()), "modules_back_on_host": on_host}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--presets", nargs="*", default=["R512_7B", "R720_7B", "R720_12B"])
    ap.add_argument("--e2e", default=None, help="preset of the end-to-end model_cpu_offload call (untiled decode)")
    ap.add_argument("--e2e-steps", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="JSON file for all shapes' results")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_offload needs a CUDA device"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    dev = torch.device("cuda:0")
    out = []
    for name in args.presets:
        p = bench.PRESETS[name]
        g = torch.Generator().manual_seed(0)
        F, h, w = p["F"], p["h"], p["w"]
        lat = torch.randn(2, 16, F, h, w, generator=g).to(dev, bf16)
        enc = (torch.randn(2, bench.S_TEXT, bench.E_TEXT, generator=g) * 3).to(dev, bf16)
        rope = rope_table(h * 8, w * 8, F, device=dev)
        t = torch.full((2,), 500.0, device=dev)

        def fwd(m):
            return m(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope, return_dict=False)[0]

        held, modes = {}, {}
        for k, make in (("resident", lambda: bench.build_model(p, dev)),
                        ("offload_bf16", lambda: host_copy(modes["resident"], bf16)),
                        ("offload_e4m3", lambda: host_copy(modes["resident"], torch.float8_e4m3fn)),
                        # the same e4m3 weights, resident: the reference for offload_e4m3's output
                        ("resident_e4m3", lambda: host_copy(modes["resident"], torch.float8_e4m3fn, offload=False))):
            gc.collect()  # device tensors of unreachable cycles would otherwise be freed inside the window
            torch.cuda.synchronize()
            before = torch.cuda.memory_allocated()
            m = make()
            fwd(m)  # derives what the mode keeps on the device
            gc.collect()
            torch.cuda.synchronize()
            held[k] = torch.cuda.memory_allocated() - before
            modes[k] = m
        ref = {"resident": fwd(modes["resident"]), "resident_e4m3": fwd(modes["resident_e4m3"])}
        same = {"offload_bf16 == resident": bool(torch.equal(fwd(modes["offload_bf16"]), ref["resident"])),
                "offload_e4m3 == resident_e4m3": bool(torch.equal(fwd(modes["offload_e4m3"]), ref["resident_e4m3"]))}
        del modes["resident_e4m3"], ref
        torch.cuda.empty_cache()
        times = {k: [] for k in modes}
        peak, h2d = {}, {}
        for _ in range(args.reps):
            for k, m in modes.items():
                gc.collect()
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                b0 = m._offload.h2d_bytes if m._offload else 0
                t0 = time.perf_counter()
                fwd(m)
                torch.cuda.synchronize()
                times[k].append(time.perf_counter() - t0)
                peak[k] = held[k] + torch.cuda.max_memory_allocated() - base
                h2d[k] = (m._offload.h2d_bytes if m._offload else 0) - b0
        idle = {k: idle_ms(lambda m=m: fwd(m)) for k, m in modes.items()}
        row = {"preset": name, "shape": f"{F} latent frames x {h * 8}x{w * 8}, CFG batch 2, {p['layers']} blocks d={p['heads'] * 64}",
               "gpu": smi, "bit_identical": same, "device_held_gb": {k: v / 1e9 for k, v in held.items()},
               "cfg_step_s_median": {k: sorted(v)[len(v) // 2] for k, v in times.items()},
               "cfg_step_s_all": times, "device_peak_gb": {k: v / 1e9 for k, v in peak.items()},
               "h2d_gb_per_step": {k: v / 1e9 for k, v in h2d.items()},
               "idle_ms_profiled": {k: v[0] for k, v in idle.items()}, "span_ms_profiled": {k: v[1] for k, v in idle.items()},
               "packed_block_mb": {k: m._offload.packs[0].host.nbytes / 1e6 for k, m in modes.items() if m._offload}}
        print(json.dumps(row), flush=True)
        out.append(row)
        del modes, m
        torch.cuda.empty_cache()
    if args.e2e:
        row = e2e(args.e2e, args.e2e_steps, dev, smi)
        print(json.dumps(row), flush=True)
        out.append(row)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
