"""The sequence-parallel (Ulysses) stores fused into the q/k/v projection (ea_qkv_peers) and into the attention epilogue
(ea_attn_peers), run on one GPU: the peer tables are plain pointer tables, so every entry can point at a local buffer and
the stores can be compared bit for bit with the single-GPU calls.  Buffers start filled with a sentinel, so a store to the
wrong place (or one that should have been skipped) shows up as well as a missing one.  The IPC / NCCL set-up of
sequence_parallel.PeerExchange is not exercised here."""
import ctypes as C

import pytest
import torch

from tests.test_gemm_gpu import qkv_inputs

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
SENTINEL = -1024.0  # a bf16 value no LayerNorm / attention output here comes near


def _filled(shape):
    return torch.full(shape, SENTINEL, device="cuda", dtype=bf16)


def _untouched(*bufs):
    return all(bool((b == SENTINEL).all()) for b in bufs)


def _qkv_peers(bufs, heads_per_peer, only=None):
    """An ea_qkv_peers table over local (q, k, v) buffers; only = r leaves every entry but r NULL (the text part on rank r)."""
    from easyanimate_b200 import _lib as L
    pe = L.QkvPeers()
    pe.heads_per_peer = heads_per_peer
    for r, (q, k, v) in enumerate(bufs):
        if only is None or r == only:
            pe.q[r], pe.k[r], pe.v[r] = q.data_ptr(), k.data_ptr(), v.data_ptr()
    return pe


@pytest.mark.parametrize("d,heads_per_peer", [(512, 1), (512, 2), (512, 4), (384, 3)])
def test_qkv_peer_stores_match_the_single_gpu_projection(d, heads_per_peer):
    """Head h of every row lands in buffer h // heads_per_peer at local head h % heads_per_peer, bit-identical to the
    non-peer call; a text-part call with only entry r set (rank r) writes rank r's heads and nothing else."""
    from easyanimate_b200 import ops
    H = d // 64
    P = H // heads_per_peer
    B, S_t, S_v = 2, 77, 150
    S = S_t + S_v + 13  # rows after the video part belong to no call
    a, w, b, lnq, lnk, rope = qkv_inputs(B, S_v, d, True, seed=1)
    at, wt, bt, lnqt, lnkt, _ = qkv_inputs(B, S_t, d, False, seed=21)
    ref = [torch.zeros((B, H, S, 64), device="cuda", dtype=bf16) for _ in range(3)]
    ops.qkv_gemm_ln_rope(a, w, b, lnq, lnk, rope, *ref, rows_per_batch=S_v, seq_offset=S_t, eps=1e-6)
    ops.qkv_gemm_ln_rope(at, wt, bt, lnqt, lnkt, None, *ref, rows_per_batch=S_t, seq_offset=0, eps=1e-6)

    bufs = [tuple(_filled((B, heads_per_peer, S, 64)) for _ in range(3)) for _ in range(P)]
    expect = [tuple(_filled((B, heads_per_peer, S, 64)) for _ in range(3)) for _ in range(P)]

    def settle(rows, ranks):
        for r in ranks:
            heads = slice(r * heads_per_peer, (r + 1) * heads_per_peer)
            for i in range(3):
                expect[r][i][:, :, rows] = ref[i][:, heads, rows]
        for r in range(P):
            for i in range(3):
                assert torch.equal(bufs[r][i], expect[r][i]), (r, "qkv"[i])

    # the video rows of this rank: every head goes to its owner
    ops.qkv_gemm_ln_rope(a, w, b, lnq, lnk, rope, *bufs[0], rows_per_batch=S_v, seq_offset=S_t, eps=1e-6,
                         peers=_qkv_peers(bufs, heads_per_peer))
    settle(slice(S_t, S_t + S_v), range(P))
    # the replicated text rows: rank r projects them for its own heads only
    for r in range(P):
        ops.qkv_gemm_ln_rope(at, wt, bt, lnqt, lnkt, None, *bufs[0], rows_per_batch=S_t, seq_offset=0, eps=1e-6,
                             peers=_qkv_peers(bufs, heads_per_peer, only=r))
        settle(slice(0, S_t), [r])


def _attn_peers(P, S_loc, out_heads, head0, out_video, out_text):
    from easyanimate_b200 import _lib as L
    pe = L.AttnPeers()
    pe.n_peers, pe.tokens_per_peer, pe.out_heads, pe.head0 = P, S_loc, out_heads, head0
    for p in range(P):
        pe.out_video[p] = out_video[p].data_ptr()
        pe.out_text[p] = out_text[p].data_ptr() if out_text else None
    return pe


@pytest.mark.parametrize("S_t", [0, 77])
@pytest.mark.parametrize("S_loc", [40, 100, 300])
@pytest.mark.parametrize("P,H", [(2, 6), (3, 6), (8, 8)])
def test_attention_peer_stores_match_the_single_gpu_attention(P, H, S_loc, S_t):
    """P emulated ranks each run attention for their H/P heads over all tokens; afterwards every rank's video buffer holds
    its token slice of the single-call output and every rank's text buffer the whole text output, bit for bit.  With
    S_loc = 40 or 100 one 128-query tile spans several token owners."""
    from easyanimate_b200 import ops
    B, Hl = 2, H // P
    S = S_t + P * S_loc
    g = torch.Generator(device="cuda").manual_seed(1000 * P + S_loc + S_t)
    q, k, v = [torch.randn(B, H, S, 64, device="cuda", generator=g).to(bf16) for _ in range(3)]
    ot, ov = ops.attention(q, k, v, S_t)
    out_video = [_filled((B, S_loc, H * 64)) for _ in range(P)]
    out_text = [_filled((B, S_t, H * 64)) for _ in range(P)] if S_t else []
    for r in range(P):
        heads = slice(r * Hl, (r + 1) * Hl)
        got = ops.attention(q[:, heads].contiguous(), k[:, heads].contiguous(), v[:, heads].contiguous(), S_t,
                            peers=_attn_peers(P, S_loc, H, r * Hl, out_video, out_text))
        assert got == (None, None)
        # rank r filled its head columns and nothing of the ranks after it
        cols, later = slice(r * Hl * 64, (r + 1) * Hl * 64), slice((r + 1) * Hl * 64, H * 64)
        for p in range(P):
            assert torch.equal(out_video[p][..., cols], ov[:, p * S_loc:(p + 1) * S_loc, cols]), (r, p)
            assert _untouched(out_video[p][..., later]), (r, p)
        for p in range(len(out_text)):
            assert torch.equal(out_text[p][..., cols], ot[..., cols]), (r, p)
            assert _untouched(out_text[p][..., later]), (r, p)
    for p in range(P):
        assert torch.equal(out_video[p], ov[:, p * S_loc:(p + 1) * S_loc]), p
    for p in range(len(out_text)):
        assert torch.equal(out_text[p], ot), p


# ---- the library's own argument checks (the C entry points directly, not the asserts of easyanimate_b200.ops)

def _attn_call(pe, q, k, v, S_t):
    from easyanimate_b200 import _lib as L, ops
    B, H, S, _ = q.shape
    args = L.AttnArgs(q=q.data_ptr(), k=k.data_ptr(), v=v.data_ptr(), out_text=None, out_video=None, B=B, H=H, S=S,
                      S_text=S_t, S_pad=0, head_dim=64, scale=0.125, variant=ops.ATTN_VARIANT, peers=C.pointer(pe))
    rc = L.ea_attn_fwd(C.byref(args), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("bad", ["tokens_per_peer", "head_range", "null_video", "null_text", "n_peers_0", "n_peers_9"])
def test_attention_peer_table_rejections(bad):
    """ea_attn_fwd refuses an inconsistent ea_attn_peers table before anything is launched: it returns an error and the
    peers' buffers keep their sentinel.  The unmodified table is accepted first, so each rejection is the named field's."""
    from easyanimate_b200 import _lib as L
    B, Hl, out_heads, P, S_t, S_v = 1, 2, 4, 2, 16, 72
    S = S_t + S_v
    g = torch.Generator(device="cuda").manual_seed(5)
    q, k, v = [torch.randn(B, Hl, S, 64, device="cuda", generator=g).to(bf16) for _ in range(3)]
    out_video = [_filled((B, 9 * 8, out_heads * 64)) for _ in range(P)]  # large enough for any table below
    out_text = [_filled((B, S_t, out_heads * 64)) for _ in range(P)]
    assert _attn_call(_attn_peers(P, S_v // P, out_heads, Hl, out_video, out_text), q, k, v, S_t) == 0
    assert not _untouched(*out_video, *out_text)
    for t in out_video + out_text:
        t.fill_(SENTINEL)
    pe = _attn_peers(P, S_v // P, out_heads, Hl, out_video, out_text)
    if bad == "tokens_per_peer":
        pe.tokens_per_peer = S_v // P - 1  # tokens_per_peer * n_peers != S - S_text
    elif bad == "head_range":
        pe.head0 = out_heads - Hl + 1  # head0 + H > out_heads
    elif bad == "null_video":
        pe.out_video[1] = None
    elif bad == "null_text":
        pe.out_text[1] = None  # S_text > 0
    elif bad == "n_peers_0":
        pe.n_peers = 0
    elif bad == "n_peers_9":
        pe.n_peers, pe.tokens_per_peer = 9, S_v // 9  # 9 x 8 = 72 video tokens: only the peer count is wrong
    rc = _attn_call(pe, q, k, v, S_t)
    assert rc != 0 and b"ea_attn_fwd" in L.ea_last_error(), (rc, L.ea_last_error())
    assert _untouched(*out_video, *out_text)


@pytest.mark.parametrize("d,heads_per_peer", [(512, 3), (512, 0), (640, 1), (1024, 1)],
                         ids=["not_a_divisor", "zero", "10_groups", "16_groups"])
def test_qkv_peer_table_rejections(d, heads_per_peer):
    """ea_qkv_gemm_ln_rope refuses a heads_per_peer that does not split the heads into at most EA_MAX_PEERS equal groups."""
    from easyanimate_b200 import _lib as L
    B, S = 1, 96
    a, w, b, lnq, lnk, _ = qkv_inputs(B, S, d, False, seed=3)
    bufs = [tuple(_filled((B, 2, S, 64)) for _ in range(3)) for _ in range(L.MAX_PEERS)]
    pe = _qkv_peers(bufs, heads_per_peer)

    def call(peers):
        args = L.QkvArgs(a=a.data_ptr(), w=w.data_ptr(), bias=b.data_ptr(), ln_q_w=lnq[0].data_ptr(), ln_q_b=lnq[1].data_ptr(),
                         ln_k_w=lnk[0].data_ptr(), ln_k_b=lnk[1].data_ptr(), rope_cos=None, rope_sin=None, q=None, k=None,
                         v=None, M=B * S, d=d, lda=d, rows_per_batch=S, S=S, seq_offset=0, ln_eps=1e-6,
                         peers=C.pointer(peers))
        rc = L.ea_qkv_gemm_ln_rope(C.byref(args), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return rc

    rc = call(pe)
    assert rc != 0 and b"heads_per_peer" in L.ea_last_error(), (rc, L.ea_last_error())
    assert _untouched(*[t for group in bufs for t in group])
    # the same call with a valid split goes through
    H = d // 64
    hpp = next(h for h in range(1, H + 1) if H % h == 0 and H // h <= L.MAX_PEERS)
    ok_bufs = [tuple(_filled((B, hpp, S, 64)) for _ in range(3)) for _ in range(H // hpp)]
    assert call(_qkv_peers(ok_bufs, hpp)) == 0
    assert not _untouched(*[t for group in ok_bufs for t in group])
