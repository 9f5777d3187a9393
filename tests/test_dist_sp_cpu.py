"""world_size-2 gloo check of the Ulysses sequence-parallel exchanges (easyanimate_b200/sequence_parallel.py): head scatter /
token gather before attention, the reverse after it, the replicated text rows, and the token shard / gather of the
per-token streams - against single-process attention over all tokens.  Attention itself is a CPU stand-in."""
import pytest
import torch
import torch.distributed as dist

from tests import cpu_ops
from tests.gloo import run_ranks

B, H, S_T, S_V = 2, 4, 5, 12


def _attention_cpu(q, k, v, S_t):  # the ops.attention contract: (out_text [B,S_t,h*64], out_video [B,S-S_t,h*64])
    b, h, s, hd = q.shape
    o = torch.nn.functional.scaled_dot_product_attention(q.float(), k.float(), v.float()).transpose(1, 2).reshape(b, s, h * hd)
    return o[:, :S_t].contiguous(), o[:, S_t:].contiguous()


def _global_qkv():
    g = torch.Generator().manual_seed(3)
    return [torch.randn(B, H, S_T + S_V, 64, generator=g) for _ in range(3)]


def _exchanges(rank):
    from easyanimate_b200.sequence_parallel import UlyssesAttention
    sp = UlyssesAttention(dist.new_group([0, 1]))
    s0, s1 = sp.local_range(S_V)
    q, k, v = _global_qkv()
    local = [torch.cat([t[:, :, :S_T], t[:, :, S_T + s0:S_T + s1]], dim=2).contiguous() for t in (q, k, v)]
    with pytest.MonkeyPatch.context() as mp:
        cpu_ops.use_stand_ins(mp, attention=_attention_cpu)
        o_t, o_v = sp.attention(local[0], local[1], local[2], S_T)
    # token shard / gather round trip of a per-token stream
    x = torch.arange(B * S_V * 3, dtype=torch.float32).view(B * S_V, 3)
    x_loc = sp.shard_tokens(x, B, S_V)
    back = sp.gather_tokens(x_loc, B, s1 - s0)
    return o_t, o_v, bool(torch.equal(back, x)), tuple(x_loc.shape)


def test_ulysses_exchanges_match_single_process_attention():
    res = run_ranks(_exchanges, 2, timeout=120)
    q, k, v = _global_qkv()
    full_t, full_v = _attention_cpu(q, k, v, S_T)
    n = S_V // 2
    for rank, (o_t, o_v, roundtrip, shape) in enumerate(res):
        assert roundtrip and shape == (B * n, 3)
        torch.testing.assert_close(o_t, full_t, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(o_v, full_v[:, rank * n:(rank + 1) * n], rtol=1e-5, atol=1e-6)


# ---- the whole transformer forward under sequence parallelism (host logic; CUDA entry points replaced by tests/cpu_ops.py) ----
CFG = dict(num_attention_heads=2, attention_head_dim=64, in_channels=16, out_channels=16, patch_size=2, num_layers=2,
           time_embed_dim=64, add_norm_text_encoder=True, text_embed_dim=128, text_embed_dim_t5=None)


def _forward(sp_group=None, teacache=False):
    from oracle import dit
    from easyanimate_b200.transformer3d import EasyAnimateTransformer3DModel
    bf16 = torch.bfloat16
    ob = dit.init_weights_(dit.OracleTransformer3D(**CFG), 11).to(bf16)
    m = EasyAnimateTransformer3DModel(**CFG).to(bf16)
    m.load_state_dict(ob.state_dict(), strict=True)
    m.set_sequence_parallel_group(sp_group)
    g = torch.Generator().manual_seed(2)
    lat = torch.randn(2, 16, 3, 8, 12, generator=g).to(bf16)  # S_v = 3*4*6 = 72 video tokens, 2 heads
    enc = (torch.randn(2, 9, 128, generator=g) * 3).to(bf16)
    t = torch.tensor([937.0, 421.0]).to(bf16)
    rope = dit.rope_for_video(64, 96, 3)
    with pytest.MonkeyPatch.context() as mp, torch.no_grad():
        cpu_ops.use_stand_ins(mp)
        if not teacache:
            return m(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope, return_dict=False)[0]
        m.enable_teacache(6, 0.08, coefficients=[1.07862322, -4.19362456, 3.06725828, 0.33161686, 0.02374758])
        outs = []
        for i in range(6):
            x, tt = (lat.float() * (1.0 - 0.01 * i)).to(bf16), torch.tensor([900.0 - 30 * i] * 2).to(bf16)
            outs.append(m(x, tt, encoder_hidden_states=enc, image_rotary_emb=rope, return_dict=False)[0])
        assert m.teacache.skipped >= 1
        return torch.stack(outs)


def _sp_forwards(rank):
    grp = dist.new_group([0, 1])
    return _forward(grp).float(), _forward(grp, teacache=True).float()


def test_sequence_parallel_forward_equals_single_process_forward():
    res = run_ranks(_sp_forwards, 2, timeout=180)
    single = _forward(None).float()
    single_tc = _forward(None, teacache=True).float()
    # every per-token op sees the same rows and attention sees the same keys: identical, not just close
    assert torch.equal(res[0][0], res[1][0])
    assert torch.equal(res[0][0], single)
    # TeaCache under sequence parallelism: the rel-L1 pieces are summed over the group, so every rank takes the same
    # skip decisions as the single-process run (6 calls, at least one served from the cached residual)
    assert torch.equal(res[0][1], res[1][1]) and torch.equal(res[0][1], single_tc)


# ---- one video on 4 ranks: 2 CFG branches x 2 sequence-parallel ranks (the 8-GPU single-video topology at small scale) ----
def _sampler_run(sp_group=None, cfg_group=None):
    from oracle import dit
    from easyanimate_b200.pipeline import EasyAnimateSampler
    from easyanimate_b200.transformer3d import EasyAnimateTransformer3DModel
    bf16 = torch.bfloat16
    ob = dit.init_weights_(dit.OracleTransformer3D(**CFG), 11).to(bf16)
    m = EasyAnimateTransformer3DModel(**CFG).to(bf16)
    m.load_state_dict(ob.state_dict(), strict=True)
    m.set_sequence_parallel_group(sp_group)
    g = torch.Generator().manual_seed(8)
    lat = torch.randn(1, 16, 3, 8, 12, generator=g).to(bf16)
    emb = (torch.randn(2, 9, 128, generator=g) * 3).to(bf16)  # cat(negative, positive)
    from easyanimate_b200.pipeline import rope_table
    rope = rope_table(64, 96, 3)
    with pytest.MonkeyPatch.context() as mp, torch.no_grad():
        cpu_ops.use_stand_ins(mp)
        s = EasyAnimateSampler(m, guidance_scale=6.0, cfg_group=cfg_group)
        s.set_timesteps(3, device="cpu")
        for i in range(3):
            lat = s.step(lat, i, emb, rope)
    return lat.float()


def _cfg_pairs_times_sp(rank):
    sp_groups = [dist.new_group([0, 1]), dist.new_group([2, 3])]      # every rank creates every group
    cfg_pairs = [dist.new_group([0, 2]), dist.new_group([1, 3])]      # rank r (uncond branch) <-> rank r + 2 (text branch)
    return _sampler_run(sp_group=sp_groups[rank // 2], cfg_group=cfg_pairs[rank % 2])


def test_cfg_pairs_times_sequence_parallel_equals_single_process_sampler():
    res = run_ranks(_cfg_pairs_times_sp, 4, timeout=300)
    single = _sampler_run()
    for rank, out in enumerate(res):
        assert torch.equal(out, single), rank
