"""Multi-GPU checks (run under torchrun on a multi-GPU H100 machine, world 2 / 4 / 8):
  1. CFG-parallel sampler == single-GPU batch-of-2 sampler (world 2 only), bit for bit;
  2. sequence-parallel forward over ALL ranks == single-GPU forward, bit for bit, for both exchange implementations:
     the fused peer-store exchange (`p2p`: QKV-epilogue / attention-epilogue stores into CUDA-IPC-mapped peer buffers) and
     the NCCL all-to-all form (`nccl`); plus a TeaCache sequence under sequence parallelism;
  3. tile-parallel VAE tiled_decode == single-GPU tiled_decode, bit for bit; strip-parallel UNTILED decode vs the single-GPU
     untiled decode (GroupNorm sums associate differently: reported as max error / fraction of differing elements);
  4. timing at the benchmark's width (d=3072, 48 heads, 4 blocks, 46 800 + 256 tokens): single GPU vs nccl vs p2p.
Usage:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29533 tools/test_multigpu.py
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

from easyanimate_b200 import AutoencoderKLMagvit, EasyAnimateSampler, EasyAnimateTransformer3DModel, rope_table

bf16 = torch.bfloat16


def make_model(cfg, dev, std=0.05):
    with torch.device(dev):
        model = EasyAnimateTransformer3DModel(**cfg).to(bf16)
    torch.manual_seed(0)
    with torch.no_grad():
        for n, p in model.named_parameters():
            p.normal_(1.0 if (p.dim() == 1 and n.endswith("weight")) else 0.0, std)
    return model


def set_sp(model, group, mode):
    os.environ["EA_SP_MODE"] = mode
    model.set_sequence_parallel_group(group)


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dev = torch.device("cuda", lr)
    dist.init_process_group("nccl", device_id=dev)
    grp = dist.new_group(list(range(world)))
    res = {"world": world}
    heads = 8 if world <= 4 else 16
    cfg = dict(num_attention_heads=heads, attention_head_dim=64, in_channels=16, out_channels=16, patch_size=2, num_layers=2,
               time_embed_dim=128, add_norm_text_encoder=True, text_embed_dim=256, text_embed_dim_t5=None)
    model = make_model(cfg, dev)
    g = torch.Generator(device=dev).manual_seed(5)
    lat = torch.randn((1, 16, 3, 16, 32), device=dev, generator=g).to(bf16)  # 3*8*16 = 384 video tokens
    emb = (torch.randn((2, 40, 256), device=dev, generator=g) * 3).to(bf16)
    rope = rope_table(128, 256, 3, device=dev)

    # ---- 1. CFG-parallel pair vs batch of 2
    if world == 2:
        single = EasyAnimateSampler(model, guidance_scale=6.0)
        pair = EasyAnimateSampler(model, guidance_scale=6.0, cfg_group=grp)
        single.set_timesteps(4, device="cpu"); pair.set_timesteps(4, device="cpu")
        a, b = lat.clone(), lat.clone()
        for i in range(4):
            a = single.step(a, i, emb, rope)
            b = pair.step(b, i, emb, rope)
        torch.cuda.synchronize()
        res["cfg_parallel_max_abs_diff"] = (a.float() - b.float()).abs().max().item()
        model.set_cfg_parallel_group(None)

    # ---- 2. sequence parallelism over all ranks vs the single-GPU forward
    t = torch.tensor([937.0], device=dev).to(bf16)
    one = model(lat, t, encoder_hidden_states=emb[:1], image_rotary_emb=rope, return_dict=False)[0]
    for mode in ("p2p", "nccl"):
        set_sp(model, grp, mode)
        sp = model(lat, t, encoder_hidden_states=emb[:1], image_rotary_emb=rope, return_dict=False)[0]
        sp2 = model(lat, t, encoder_hidden_states=emb[:1], image_rotary_emb=rope, return_dict=False)[0]  # buffers reused
        torch.cuda.synchronize()
        res[f"sequence_parallel_{mode}_max_abs_diff"] = max((one.float() - sp.float()).abs().max().item(),
                                                            (one.float() - sp2.float()).abs().max().item())
    # TeaCache decisions under sequence parallelism (p2p): same outputs as single GPU over a 6-call sequence
    coeffs = [1.07862322, -4.19362456, 3.06725828, 0.33161686, 0.02374758]
    outs = {}
    for mode in (None, "p2p"):
        if mode is None:
            model.set_sequence_parallel_group(None)
        else:
            set_sp(model, grp, mode)
        model.enable_teacache(6, 0.08, coefficients=coeffs)
        seq = []
        for i in range(6):
            x = (lat.float() * (1.0 - 0.01 * i)).to(bf16)
            tt = torch.tensor([900.0 - 30 * i], device=dev).to(bf16)
            seq.append(model(x, tt, encoder_hidden_states=emb[:1], image_rotary_emb=rope, return_dict=False)[0])
        outs[mode] = (torch.stack(seq), model.teacache.skipped)
        model.teacache = None
    model.set_sequence_parallel_group(None)
    torch.cuda.synchronize()
    res["teacache_sp_max_abs_diff"] = (outs[None][0].float() - outs["p2p"][0].float()).abs().max().item()
    res["teacache_skipped"] = [outs[None][1], outs["p2p"][1]]

    # ---- 3. VAE: tile-parallel tiled decode vs single-GPU tiled decode
    with torch.device(dev):
        vae = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True,
                                  mid_block_attention_type="spatial", block_out_channels=[64, 64, 128, 128],
                                  use_tiling=True, tile_sample_min_size=64).to(bf16)
    torch.manual_seed(1)
    with torch.no_grad():
        for n, p in vae.named_parameters():
            if p.dim() >= 2:
                p.normal_(0, (1.0 / p[0].numel()) ** 0.5)
            elif "norm" in n and n.endswith("weight"):
                p.normal_(1.0, 0.05)
            else:
                p.normal_(0, 0.05)
    z = torch.randn((1, 16, 2, 14, 20), device=dev, generator=g).to(bf16)
    ref = vae.decode(z).sample
    vae.set_tile_parallel_group(grp)
    par = vae.decode(z).sample
    torch.cuda.synchronize()
    res["tile_parallel_max_abs_diff"] = (ref.float() - par.float()).abs().max().item()
    # ---- 3b. strip-parallel UNTILED decode (vae_strips.py) vs the single-GPU untiled decode: convolutions bit-identical, the
    # per-frame GroupNorm sums are added per rank and then in rank order (fp64), so an occasional bf16 flip is possible
    vae.set_tile_parallel_group(None)
    vae.use_tiling = False
    zs = torch.randn((1, 16, 3, 4 * world + 3, 20), device=dev, generator=g).to(bf16)
    ref_u = vae.decode(zs).sample
    vae.set_strip_parallel_group(grp)
    par_u = vae.decode(zs).sample
    vae.set_strip_parallel_group(None)
    torch.cuda.synchronize()
    du = (ref_u.float() - par_u.float()).abs()
    res["strip_parallel_max_abs_err"] = du.max().item()
    res["strip_parallel_frac_differing"] = (du > 0).float().mean().item()
    res["strip_parallel_output_scale"] = ref_u.float().abs().max().item()
    del vae

    # ---- 4. timing at the benchmark's width: 4 blocks of d=3072 / 48 heads on 46 800 + 256 tokens, batch 1
    if os.environ.get("EA_MG_TIMING", "1") == "1" and 48 % world == 0 and 46800 % world == 0:
        del model
        torch.cuda.empty_cache()
        big = dict(num_attention_heads=48, attention_head_dim=64, in_channels=16, out_channels=16, patch_size=2, num_layers=4,
                   time_embed_dim=512, add_norm_text_encoder=True, text_embed_dim=3584, text_embed_dim_t5=None)
        model = make_model(big, dev, std=0.02)
        lat = torch.randn((1, 16, 13, 90, 160), device=dev, generator=g).to(bf16)
        emb = (torch.randn((1, 256, 3584), device=dev, generator=g) * 10).to(bf16)
        rope = rope_table(720, 1280, 13, device=dev)

        def timed(reps=3):
            for _ in range(2):
                out = model(lat, t, encoder_hidden_states=emb, image_rotary_emb=rope, return_dict=False)[0]
            dist.barrier(); torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                out = model(lat, t, encoder_hidden_states=emb, image_rotary_emb=rope, return_dict=False)[0]
            e1.record()
            dist.barrier(); torch.cuda.synchronize()
            ms = torch.tensor([e0.elapsed_time(e1) / reps], device=dev)
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
            return float(ms), out
        ms1, o1 = timed()
        timing = {"single_gpu_ms": ms1}
        for mode in ("p2p", "nccl"):
            set_sp(model, grp, mode)
            ms, o = timed()
            timing[f"sp{world}_{mode}_ms"] = ms
            timing[f"sp{world}_{mode}_speedup"] = ms1 / ms
            timing[f"sp{world}_{mode}_max_abs_diff"] = (o.float() - o1.float()).abs().max().item()
        model.set_sequence_parallel_group(None)
        res["timing_4_blocks_R720"] = timing

    keys = [k for k in res if k.endswith("max_abs_diff")]
    # (whether the synthetic drift makes TeaCache skip at all depends on the model width: it does at 8 heads, not at 16 -
    #  what is checked is that the decisions and the outputs are those of one GPU)
    ok_local = all(res[k] == 0.0 for k in keys) and res["teacache_skipped"][0] == res["teacache_skipped"][1]
    ok_local = ok_local and res["strip_parallel_max_abs_err"] <= 0.05 * res["strip_parallel_output_scale"] \
        and res["strip_parallel_frac_differing"] < 0.05
    ok = torch.tensor([float(ok_local)], device=dev)
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    res["ok"] = bool(ok.item())
    if rank == 0:
        print(json.dumps(res))
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok.item() else 1)


if __name__ == "__main__":
    main()
