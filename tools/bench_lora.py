"""LoRA merge + unmerge time on one GPU, per memory mode, for random-init models of bench.py's MMDiT shapes (7B: 28 blocks, 12B:
48 blocks, d = 3072) with a LoRA of rank 64 and 128 on every nn.Linear.  Each timing is one merge_lora plus one unmerge_lora
(dtype float32, the reference's default) ending in a device synchronise, from a LoRA state dict already in host memory.
Modes: resident bf16 (model_full_load), resident e4m3, sequential offload with bf16 and e4m3 packs, and model CPU offload
(the weights in host memory, staged through the GPU).  The resident merge is compared with the torch formula on the same
device, W = bf16(float(W) + s * (U @ D)) per layer and its inverse, alternated with it in the same process.  Reps are alternated
too and medians reported.  Prints one JSON line per (model, rank) and writes them all to --out when given.

    python tools/bench_lora.py [--presets R720_7B R720_12B] [--ranks 64 128] [--reps 3] [--out FILE]
"""
import argparse
import copy
import gc
import json
import os
import statistics
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from easyanimate_b200 import merge_lora, unmerge_lora  # noqa: E402
from easyanimate_b200 import lora as lora_mod  # noqa: E402

bf16, e4m3 = torch.bfloat16, torch.float8_e4m3fn


def lora_state(model, rank, seed=5):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for n, m in model.named_modules():
        if isinstance(m, torch.nn.Linear):
            o, i = m.weight.shape
            key = "lora_unet__" + n.replace(".", "_")
            sd[key + ".lora_up.weight"] = (torch.randn(o, rank, generator=g) * 0.01).to(bf16)
            sd[key + ".lora_down.weight"] = (torch.randn(rank, i, generator=g) * 0.01).to(bf16)
            sd[key + ".alpha"] = torch.tensor(float(rank))
    return sd


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def native(pipe, sd):
    """merge_lora + unmerge_lora (unmerge reads a file in the reference's signature: it is handed the same state dict)."""
    def run():
        merge_lora(pipe, None, 1.0, state_dict=sd)
        orig = lora_mod._load
        lora_mod._load = lambda path: sd
        try:
            unmerge_lora(pipe, "in-memory", 1.0)
        finally:
            lora_mod._load = orig
    return run


def torch_formula(model, sd):
    """The reference's arithmetic on the GPU, one layer at a time: W.float() += s * (U @ D), cast back; then -=."""
    layers = sorted({k.split(".", 1)[0] for k in sd})
    mods = {n.replace(".", "_"): m for n, m in model.named_modules()}
    plan = []
    for layer in layers:
        m = mods[layer[len("lora_unet__"):]]
        up, down = sd[layer + ".lora_up.weight"], sd[layer + ".lora_down.weight"]
        plan.append((m.weight, up, down, sd[layer + ".alpha"].item() / up.shape[1]))

    def run():
        with torch.no_grad():
            for sign in (1.0, -1.0):
                for w, up, down, s in plan:
                    u, d = up.to("cuda", torch.float32), down.to("cuda", torch.float32)
                    w32 = w.data.float()
                    w32 += sign * s * torch.mm(u, d)
                    w.data.copy_(w32.to(w.dtype))
                    del u, d, w32
        torch.cuda.empty_cache()
    return run


def host_model(resident, dtype):
    with torch.device("meta"):
        m = type(resident)(**{k: v for k, v in resident.config.items() if not k.startswith("_")})
    m = m.to_empty(device="cpu").to(bf16)
    m.load_state_dict(resident.state_dict())
    return m.to(dtype)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--presets", nargs="+", default=["R720_7B", "R720_12B"])
    ap.add_argument("--ranks", nargs="+", type=int, default=[64, 128])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_lora.py needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    results = []
    for name in args.presets:
        p = bench.PRESETS[name]
        resident = bench.build_model(p, "cuda")
        n_linear = sum(m.weight.numel() for m in resident.modules() if isinstance(m, torch.nn.Linear))
        for rank in args.ranks:
            sd = lora_state(resident, rank)
            res = {"model": name, "blocks": p["layers"], "rank": rank, "linear_weights": n_linear, "gpu": smi,
                   "flop_per_merge": 2 * rank * n_linear, "ms": {}}
            ms = {"resident_bf16": [], "torch_formula_bf16": []}
            pipe = types.SimpleNamespace(transformer=resident)
            for _ in range(args.reps):  # alternated
                ms["resident_bf16"].append(timed(native(pipe, sd)))
                ms["torch_formula_bf16"].append(timed(torch_formula(resident, sd)))
            modes = {
                "resident_e4m3": lambda: resident_e4m3(resident),
                "sequential_bf16": lambda: host_model(resident, bf16).enable_sequential_cpu_offload("cuda"),
                "sequential_e4m3": lambda: host_model(resident, e4m3).enable_sequential_cpu_offload("cuda"),
                "model_cpu_offload_bf16": lambda: host_model(resident, bf16),
            }
            for mode, make in modes.items():
                m = make()
                pipe_m = types.SimpleNamespace(transformer=m)
                gc.collect()
                torch.cuda.synchronize()
                before = torch.cuda.memory_allocated()
                ms[mode] = [timed(native(pipe_m, sd)) for _ in range(args.reps)]
                res.setdefault("device_bytes_unchanged", {})[mode] = torch.cuda.memory_allocated() == before
                del m, pipe_m
                gc.collect()
                torch.cuda.empty_cache()
            res["ms"] = {k: {"median": statistics.median(v), "all": [round(x, 2) for x in v]} for k, v in ms.items()}
            med = res["ms"]["resident_bf16"]["median"]
            # merge + unmerge = two products: achieved fp32 FMA rate of the native resident run
            res["resident_tflops"] = 2 * res["flop_per_merge"] / (med * 1e-3) / 1e12
            print(json.dumps(res), flush=True)
            results.append(res)
        del resident
        gc.collect()
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


def resident_e4m3(resident):
    m = copy.deepcopy(resident).to(e4m3)
    return m


if __name__ == "__main__":
    main()
