"""world_size-2 gloo test of the CFG-parallel host logic (rank -> branch assignment, all_gather layout, identical
latents on both ranks, equality with the single-process batch-of-2 evaluation).  The transformer and the
CFG+Euler kernel are replaced by CPU stand-ins: this exercises the N>1 plumbing, not the kernels."""
import pytest
import torch
import torch.distributed as dist

from tests import cpu_ops
from tests.gloo import run_ranks

bf16 = torch.bfloat16


class FakeTransformer(torch.nn.Module):
    """Deterministic stand-in with the transformer call signature; depends on latents, timestep and the embeds row."""

    def forward(self, hidden_states, timestep, encoder_hidden_states=None, image_rotary_emb=None, inpaint_latents=None,
                return_dict=True):
        bias = encoder_hidden_states.float().mean(dim=(1, 2)).view(-1, 1, 1, 1, 1)
        out = hidden_states.float() * 0.5 + bias + timestep.float().view(-1, 1, 1, 1, 1) * 1e-3
        return (out.to(hidden_states.dtype),)


def _sampler_run(cfg_group=None):
    from easyanimate_b200.pipeline import EasyAnimateSampler
    g = torch.Generator().manual_seed(0)
    lat, emb = torch.randn(1, 4, 2, 4, 4, generator=g).to(bf16), torch.randn(2, 3, 8, generator=g).to(bf16)
    with pytest.MonkeyPatch.context() as mp:
        cpu_ops.use_stand_ins(mp)
        s = EasyAnimateSampler(FakeTransformer(), guidance_scale=6.0, cfg_group=cfg_group)
        s.set_timesteps(4, device="cpu")
        for i in range(4):
            lat = s.step(lat, i, emb, None)
    return lat.float()


def _cfg_pair(rank):
    return _sampler_run(dist.new_group([0, 1]))


def test_cfg_parallel_pair_matches_single_process():
    got = run_ranks(_cfg_pair, 2, timeout=120)
    ref = _sampler_run()
    assert torch.equal(got[0], got[1]), "both ranks of a CFG pair must hold identical latents"
    assert torch.equal(got[0], ref), "CFG-parallel must reproduce the batch-of-2 evaluation bit for bit"


def test_scheduler_mirror_matches_oracle():
    from oracle import dit
    from easyanimate_b200.scheduler import FlowMatchEulerDiscreteScheduler
    for shift, dyn in ((1.0, False), (3.0, False), (1.0, True)):
        ours = FlowMatchEulerDiscreteScheduler(shift=shift, use_dynamic_shifting=dyn)
        ref = dit.FlowMatchEulerScheduler(shift=shift, use_dynamic_shifting=dyn)
        for n in (25, 30, 50):
            ours.set_timesteps(n, device="cpu", mu=1.0)
            ref.set_timesteps(n, mu=1.0)
            assert torch.equal(ours.sigmas, ref.sigmas) and torch.equal(ours.timesteps, ref.timesteps)
    with pytest.raises(ValueError):
        FlowMatchEulerDiscreteScheduler(use_dynamic_shifting=True).set_timesteps(10)


def test_rope_table_mirror_matches_oracle():
    from oracle import dit
    from easyanimate_b200.pipeline import rope_table
    for (hh, ww, f) in ((720, 1280, 13), (512, 512, 13), (64, 64, 1), (384, 672, 7)):
        a, b = rope_table(hh, ww, f), dit.rope_for_video(hh, ww, f)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


# ---- TeaCache under CFG-parallel: the skip decision is the reference's joint-batch decision on both ranks ----
_TC_CFG = dict(num_attention_heads=2, attention_head_dim=64, in_channels=33, out_channels=16, patch_size=2, num_layers=2,
               time_embed_dim=64, add_norm_text_encoder=True, text_embed_dim=128, text_embed_dim_t5=None)
_TC_COEFFS = [1.07862322, -4.19362456, 3.06725828, 0.33161686, 0.02374758]


def _teacache_sampler_run(cfg_group=None, steps=8, thresh=0.15):
    """8 sampler steps with TeaCache on; returns (latents, skipped-forward count)."""
    from oracle import dit
    from easyanimate_b200.pipeline import EasyAnimateSampler, rope_table
    from easyanimate_b200.transformer3d import EasyAnimateTransformer3DModel
    ob = dit.init_weights_(dit.OracleTransformer3D(**_TC_CFG), 11).to(bf16)
    m = EasyAnimateTransformer3DModel(**_TC_CFG).to(bf16)
    m.load_state_dict(ob.state_dict(), strict=True)
    m.enable_teacache(steps, thresh, coefficients=_TC_COEFFS)
    g = torch.Generator().manual_seed(8)
    lat = torch.randn(1, 16, 3, 8, 12, generator=g).to(bf16)
    emb = torch.cat([torch.randn(1, 9, 128, generator=g) * 0.2, torch.randn(1, 9, 128, generator=g) * 8.0]).to(bf16)
    # TeaCache looks at block 0's modulated VIDEO input, which the text does not reach: the branches differ there only through
    # their conditioning latents.  Give the two branches very different ones, so that per-rank decisions would differ from
    # the joint-batch decision (with identical conditioning the per-branch means equal the joint mean and nothing is tested).
    inp = torch.cat([torch.zeros(1, 17, 3, 8, 12), torch.randn(1, 17, 3, 8, 12, generator=g) * 4.0]).to(bf16)
    rope = rope_table(64, 96, 3)
    with pytest.MonkeyPatch.context() as mp, torch.no_grad():
        cpu_ops.use_stand_ins(mp)
        s = EasyAnimateSampler(m, guidance_scale=6.0, cfg_group=cfg_group)
        s.set_timesteps(steps, device="cpu")
        for i in range(steps):
            lat = s.step(lat, i, emb, rope, inpaint_latents=inp)
    return lat.float(), m.teacache.skipped


def _teacache_cfg_pair(rank):
    return _teacache_sampler_run(dist.new_group([0, 1]))


def test_teacache_with_cfg_parallel_takes_the_joint_batch_decision():
    """With cfg_group each rank sees one branch (B=1); the reference decides skip/compute once per step
    from the rel-L1 means over the batch of 2 (transformer3d.py:1563-1586).  The (num, den) sums are all-reduced over the
    CFG pair, so both ranks skip exactly where the single-process batch-of-2 run skips and the latents agree bit for bit."""
    res = run_ranks(_teacache_cfg_pair, 2, timeout=180)
    single, skipped = _teacache_sampler_run(None)
    assert skipped >= 1, "the test must exercise the cached path"
    assert res[0][1] == res[1][1] == skipped, (res[0][1], res[1][1], skipped)
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][0], single)


# ---- the native pipeline call (easyanimate_b200.pipelines) on a CFG pair: same frames on both ranks and as one process ----
class _PipeTransformer(FakeTransformer):
    def __init__(self):
        super().__init__()
        from easyanimate_b200.config import FrozenConfig
        self.w = torch.nn.Parameter(torch.zeros(1, dtype=bf16))
        self.config = FrozenConfig(in_channels=4, attention_head_dim=64, patch_size=2, enable_text_attention_mask=True)

    dtype = property(lambda self: self.w.dtype)


class _PipeVae(torch.nn.Module):
    cache_mag_vae, mini_batch_encoder, mini_batch_decoder = True, 4, 1

    def __init__(self):
        super().__init__()
        from easyanimate_b200.config import FrozenConfig
        self.config = FrozenConfig(block_out_channels=[8, 8, 8, 8], scaling_factor=0.5, latent_channels=4)

    def decode_scaled(self, latents, out=None, dtype=torch.float32, to_host=True):
        return (latents.float() / self.config.scaling_factor).clamp(-1, 1).mul(0.5).add(0.5).repeat_interleave(2, dim=1)[:, :3]


def _pipeline_call(cfg_group=None):
    from easyanimate_b200.pipelines import EasyAnimatePipeline
    g = torch.Generator().manual_seed(3)
    pe, ne = torch.randn(1, 3, 8, generator=g).to(bf16), torch.randn(1, 3, 8, generator=g).to(bf16)
    ones = torch.ones(1, 3, dtype=torch.long)
    pipe = EasyAnimatePipeline(vae=_PipeVae(), transformer=_PipeTransformer(), cfg_group=cfg_group)
    with pytest.MonkeyPatch.context() as mp:
        cpu_ops.use_stand_ins(mp)
        return pipe(video_length=5, height=32, width=32, num_inference_steps=3, guidance_scale=6.0,
                    generator=torch.Generator().manual_seed(4), prompt_embeds=pe, negative_prompt_embeds=ne,
                    prompt_attention_mask=ones, negative_prompt_attention_mask=ones, prompt_embeds_2=pe,
                    prompt_attention_mask_2=ones).frames


def _pipeline_cfg_pair(rank):
    return _pipeline_call(dist.new_group([0, 1]))


def test_native_pipeline_call_on_a_cfg_pair_matches_single_process():
    got = run_ranks(_pipeline_cfg_pair, 2, timeout=120)
    ref = _pipeline_call()
    assert ref.shape == (1, 3, 2, 4, 4)
    assert torch.equal(got[0], got[1]) and torch.equal(got[0], ref)
