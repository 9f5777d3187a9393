"""Micro-benchmarks of individual kernels (CUDA events, L2-flushed between reps). Usage: python tools/bench_kernels.py gemm|attn|conv"""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

bf16 = torch.bfloat16


def timeit(fn, reps=10, warmup=3, flush=True):
    scratch = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda") if flush else None
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        if flush:
            scratch.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record(); torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def bench_gemm():
    from easyanimate_b200 import ops, _lib as L
    shapes = [(8192, 8192, 8192), (46800, 3072, 3072), (46800, 12288, 3072), (46800, 3072, 12288), (46800, 9216, 3072),
              (512, 3072, 3072), (4096, 4096, 4096)]
    for M, N, K in shapes:
        a = torch.randn(M, K, device="cuda").to(bf16)
        w = (torch.randn(N, K, device="cuda") * 0.02).to(bf16)
        b = torch.randn(N, device="cuda").to(bf16)
        out = torch.empty(M, N, device="cuda", dtype=bf16)
        med, best = timeit(lambda: ops.gemm(a, w, b, out=out))
        medt, bestt = timeit(lambda: torch.nn.functional.linear(a, w, b))
        fl = 2.0 * M * N * K
        print(json.dumps({"kernel": "gemm_bias", "M": M, "N": N, "K": K, "ms": round(med, 4), "tflops": round(fl / med / 1e9, 1),
                          "best_tflops": round(fl / best / 1e9, 1), "torch_ms": round(medt, 4),
                          "torch_tflops": round(fl / medt / 1e9, 1)}), flush=True)


def bench_attn():
    from easyanimate_b200 import ops
    variant = int(os.environ.get("EA_ATTN_VARIANT", "0x217c"), 0)
    compare = not os.environ.get("EA_ATTN_NO_COMPARE")
    shapes = [(1, 48, 13312 + 256, 256), (1, 48, 47056, 256)]
    if os.environ.get("EA_ATTN_SMALL"):
        shapes = [(1, 16, 8192 + 256, 256)]
    if os.environ.get("EA_ATTN_SHAPE"):  # "B,H,S,S_text", e.g. the bench step's 2,48,47056,256
        shapes = [tuple(int(x) for x in os.environ["EA_ATTN_SHAPE"].split(","))]
    for (B, H, S, St) in shapes:
        q = torch.randn(B, H, S, 64, device="cuda").to(bf16)
        k = torch.randn(B, H, S, 64, device="cuda").to(bf16)
        v = torch.randn(B, H, S, 64, device="cuda").to(bf16)
        fl = 4.0 * B * H * S * S * 64
        med, best = timeit(lambda: ops.attention(q, k, v, St, variant=variant), reps=5, warmup=2)
        res = {"kernel": "attn_fwd", "variant": variant, "B": B, "H": H, "S": S, "ms": round(med, 3), "tflops": round(fl / med / 1e9, 1)}
        if not compare:
            print(json.dumps(res), flush=True)
            continue
        try:
            medt, _ = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(q, k, v), reps=5, warmup=2)
            res.update({"torch_sdpa_ms": round(medt, 3), "torch_sdpa_tflops": round(fl / medt / 1e9, 1)})
        except Exception as e:  # noqa
            res["torch_sdpa_error"] = str(e)[:100]
        try:
            from flash_attn import flash_attn_func
            qf, kf, vf = [t.transpose(1, 2).contiguous() for t in (q, k, v)]
            medf, _ = timeit(lambda: flash_attn_func(qf, kf, vf), reps=5, warmup=2)
            res.update({"flash_attn2_ms": round(medf, 3), "flash_attn2_tflops": round(fl / medf / 1e9, 1)})
        except Exception as e:  # noqa
            res["flash_attn2_error"] = str(e)[:100]
        print(json.dumps(res), flush=True)


def vae_conv_flops(F_lat, h, w, boc=(128, 256, 512, 512), mid_attn=True):
    """conv FLOPs of one untiled decode."""
    T1, T2, T3 = F_lat, 2 * F_lat - 1, 4 * F_lat - 3
    c0, c1, c2, c3 = boc  # 128,256,512,512
    def conv(T, H, W, cin, cout, k=27): return 2.0 * T * H * W * cout * cin * k
    fl = conv(T1, h, w, 16, c3)                                  # conv_in
    fl += 4 * conv(T1, h, w, c3, c3)                             # mid block: 2 res blocks
    fl += 6 * conv(T1, h, w, c3, c3) + conv(T1, 2 * h, 2 * w, c3, c3)          # up0 + spatial upsampler
    fl += 6 * conv(T1, 2 * h, 2 * w, c3, c3) + conv(T1, 4 * h, 4 * w, c3, c3)  # up1 (+temporal x2 after conv)
    fl += conv(T2, 4 * h, 4 * w, c3, c1) + 5 * conv(T2, 4 * h, 4 * w, c1, c1) + conv(T2, 4 * h, 4 * w, c3, c1, 1)
    fl += conv(T2, 8 * h, 8 * w, c1, c1)                         # up2 upsampler
    fl += conv(T3, 8 * h, 8 * w, c1, c0) + 5 * conv(T3, 8 * h, 8 * w, c0, c0) + conv(T3, 8 * h, 8 * w, c1, c0, 1)
    fl += conv(T3, 8 * h, 8 * w, c0, 3)                          # conv_out
    return fl


def bench_vae():
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    shapes = [(13, 48, 48, False), (13, 64, 64, False), (13, 90, 160, False), (13, 90, 160, True)]
    only = os.environ.get("EA_VAE_SHAPES")
    with torch.device("cuda"):
        vae = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True, mid_block_attention_type="spatial",
                                  mini_batch_decoder=1, scaling_factor=0.7125).to(bf16)
    with torch.no_grad():
        for n, p in vae.named_parameters():
            if p.dim() >= 2:
                p.normal_(0, (1.0 / p[0].numel()) ** 0.5)
            elif "norm" in n and n.endswith("weight"):
                p.normal_(1.0, 0.05)
            else:
                p.normal_(0, 0.05)
    for F_lat, h, w, tiled in shapes:
        if only and f"{h}x{w}" not in only:
            continue
        vae.use_tiling = tiled
        z = torch.randn(1, 16, F_lat, h, w, device="cuda").to(bf16)
        out = vae.decode(z).sample
        torch.cuda.synchronize()
        med, best = timeit(lambda: vae.decode(z), reps=3, warmup=1, flush=False)
        mpix = out.shape[2] * out.shape[3] * out.shape[4] / 1e6
        fl = vae_conv_flops(F_lat, h, w)
        print(json.dumps({"kernel": "vae_decode", "z": [1, 16, F_lat, h, w], "tiled": tiled, "frames": out.shape[2], "ms": round(med, 2),
                          "mpix_per_s": round(mpix / med * 1e3, 1), "untiled_conv_tflop": round(fl / 1e12, 1),
                          "conv_tflops_if_untiled": round(fl / med / 1e9, 1), "finite": bool(torch.isfinite(out).all())}), flush=True)


if __name__ == "__main__":
    which = sys.argv[1] if len(sys.argv) > 1 else "gemm"
    {"gemm": bench_gemm, "attn": bench_attn, "vae": bench_vae}[which]()

