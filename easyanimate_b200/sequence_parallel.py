"""Sequence parallelism for ONE video across the ranks of a group.  The reference has no multi-GPU inference code at this
commit; joint text+video attention (processor.py:287-289) makes a
per-block exchange unavoidable once one video spans more than the two CFG branches, and this module
is this framework's own design for it (Ulysses-style): every rank owns a contiguous slice of the video tokens for the
per-token work (AdaLN, projections, feed-forward) and, inside attention, all tokens of a slice of the HEADS.  The text
tokens are few (256) and replicated.

Two implementations of the two exchanges per block:

* `PeerExchange` (the product path on NVLink-connected GPUs, `mode="p2p"`): NO separate exchange pass.  The q/k/v buffers
  [B, H/P, S, 64] and the attention-output buffers of every rank are mapped into every other rank (CUDA IPC); the QKV
  projection's epilogue stores head h of its rows straight into the buffer of the rank that owns h, and the attention
  epilogue stores each token's row straight into the token-major buffer of the rank that owns the token
  (include/ea_b200.h `ea_qkv_peers` / `ea_attn_peers`: 128-byte NVLink stores issued from the same kernels as the wgmma
  tiles).  The only collectives left are two 4-byte all-reduces per block that order the kernels of different GPUs.
* NCCL collectives (`mode="nccl"`, also what the gloo CPU tests run): two `all_to_all_single` + one `all_gather` per block
  plus the permute copies around them - the baseline the fused path is measured against.

    q/k/v  [B, H, S_t + S_loc, 64]  --exchange-->  [B, H/P, S_t + S_v, 64]      (before attention)
    out    [B, S_v, (H/P)*64]       --exchange-->  [B, S_loc, H*64]  (+ the text rows on every rank)

Host logic of the collective form is covered by world_size-2/4 gloo tests against single-process attention / forward /
sampler (tests/test_dist_sp_cpu.py); both forms are checked on GPUs against the single-GPU forward by tools/test_multigpu.py.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Optional, Tuple

import torch
import torch.distributed as dist


def group_size(group) -> int:
    return dist.get_world_size(group)


def all_reduce_floats(values, group) -> list:
    """Sum a short list of Python floats over `group` (TeaCache's rel-L1 pieces); fp64 on the wire."""
    t = torch.tensor(list(values), dtype=torch.float64)
    if dist.get_backend(group) == "nccl":
        t = t.cuda()
    dist.all_reduce(t, group=group)
    return [float(v) for v in t.cpu()]


# A device allocation can be imported once per process: torch's caching allocator hands the same allocation (hence the same
# handle) to successive exchanges, so the mappings are cached by handle and reference-counted.
_IPC_OPEN = {}  # handle bytes -> [mapped base address, users]


def _ipc_open(handle: bytes) -> int:
    from . import _lib as L
    ent = _IPC_OPEN.get(handle)
    if ent is None:
        mapped = L.vp()
        if len(handle) != 64:
            raise ValueError(f"a cudaIpcMemHandle_t is 64 bytes, got {len(handle)}")
        L.check(L.ea_ipc_open((C.c_char * 64).from_buffer_copy(handle), C.byref(mapped)), "ea_ipc_open")
        ent = _IPC_OPEN[handle] = [mapped.value, 0]
    ent[1] += 1
    return ent[0]


def _ipc_close(handle: bytes) -> None:
    from . import _lib as L
    ent = _IPC_OPEN.get(handle)
    if ent is None:
        return
    ent[1] -= 1
    if ent[1] <= 0:
        del _IPC_OPEN[handle]
        L.check(L.ea_ipc_close(ent[0]), "ea_ipc_close")


class PeerExchange:
    """Symmetric q/k/v and attention-output buffers of one (B, H, S_t, S_loc) problem, mapped into every rank of the group,
    and the pointer tables the fused kernels take.  Built once per shape and reused by every block of every step."""

    def __init__(self, group, B: int, H: int, S_t: int, S_loc: int, device):
        from . import _lib as L
        self.group, self.rank, self.world = group, dist.get_rank(group), dist.get_world_size(group)
        P = self.world
        if P > L.MAX_PEERS:
            raise ValueError(f"peer exchange supports up to {L.MAX_PEERS} ranks per group")
        if H % P:
            raise ValueError(f"sequence parallelism needs the head count ({H}) to divide by the group size ({P})")
        self.B, self.H, self.Hl, self.S_t, self.S_loc = B, H, H // P, S_t, S_loc
        S = S_t + P * S_loc
        bf16 = torch.bfloat16
        # ONE allocation for the five buffers: a CUDA IPC handle names a whole device allocation, so every peer opens one handle
        n_qkv = B * self.Hl * S * 64
        sizes = [n_qkv, n_qkv, n_qkv, B * S_loc * H * 64, B * S_t * H * 64]
        offs = [0]
        for n in sizes:
            offs.append(offs[-1] + (n * 2 + 1023) // 1024 * 1024)  # byte offsets, 1 KB aligned
        self._buf = torch.empty((offs[-1],), device=device, dtype=torch.uint8)

        def part(i, shape):
            return self._buf[offs[i]:offs[i] + sizes[i] * 2].view(bf16).view(shape)
        self.q, self.k, self.v = (part(i, (B, self.Hl, S, 64)) for i in range(3))
        self.out_video = part(3, (B, S_loc, H * 64))
        self.out_text = part(4, (B, S_t, H * 64))
        self._flag = torch.zeros((1,), device=device, dtype=torch.int32)
        # export: the cudaIpcMemHandle_t of the device allocation that holds the buffer and the buffer's byte offset inside it
        # (torch's caching allocator sub-allocates from cudaMalloc'ed segments).  The peers import it with ea_ipc_open on THEIR
        # device: a mapping opened under the exporter's device index - what torch's own storage sharing does - cannot be
        # dereferenced by a kernel of another device.
        hbuf, hoff = (C.c_char * 64)(), L.i64(0)
        L.check(L.ea_ipc_export(self._buf.data_ptr(), hbuf, C.byref(hoff)), "ea_ipc_export")
        handle, base_off = bytes(hbuf.raw), int(hoff.value)
        gathered = [None] * P
        dist.all_gather_object(gathered, (torch.cuda.current_device(), handle, base_off), group=group)
        self._opened = []  # mapped bases, closed by release()
        ptrs = []
        for r, (peer_dev, hnd, off) in enumerate(gathered):
            if r == self.rank:
                base = self._buf.data_ptr()
            else:
                L.check(L.ea_enable_peer_access(int(peer_dev)), "ea_enable_peer_access")
                base = _ipc_open(hnd) + off
                self._opened.append(hnd)
            ptrs.append([base + offs[i] for i in range(5)])
        self.qkv_video, self.qkv_text, self.attn = L.QkvPeers(), L.QkvPeers(), L.AttnPeers()
        self.qkv_video.heads_per_peer = self.qkv_text.heads_per_peer = self.Hl
        for r in range(P):
            self.qkv_video.q[r], self.qkv_video.k[r], self.qkv_video.v[r] = ptrs[r][0], ptrs[r][1], ptrs[r][2]
            self.attn.out_video[r], self.attn.out_text[r] = ptrs[r][3], ptrs[r][4]
        # text rows are replicated: every rank projects them itself and keeps its own heads only
        self.qkv_text.q[self.rank], self.qkv_text.k[self.rank], self.qkv_text.v[self.rank] = ptrs[self.rank][:3]
        self.attn.n_peers, self.attn.tokens_per_peer, self.attn.out_heads, self.attn.head0 = P, S_loc, H, self.rank * self.Hl
        dist.barrier(group=group)  # nobody stores into a peer before every mapping exists

    def release(self):
        """Unmap the peers' buffers (every rank, collectively, before the buffers are freed or replaced)."""
        from . import _lib as L
        if self._opened:
            torch.cuda.synchronize()
            dist.barrier(group=self.group)  # nobody is still storing into a buffer that is about to be unmapped
            for hnd in self._opened:
                _ipc_close(hnd)
            self._opened = []
            dist.barrier(group=self.group)

    def barrier(self):
        """Orders the kernels of different GPUs on the compute stream (no host synchronisation): the 4-byte all-reduce can
        only complete on a rank once every rank has launched it, i.e. once every rank's preceding kernel has finished."""
        dist.all_reduce(self._flag, group=self.group)


class UlyssesAttention:
    def __init__(self, group, attention_fn: Optional[Callable] = None, mode: Optional[str] = None):
        import os
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self._attention = attention_fn  # (q, k, v, S_t) -> (out_text [B,S_t,h*64], out_video [B,S-S_t,h*64]); default ops.attention
        mode = mode or os.environ.get("EA_SP_MODE", "p2p")
        # the fused peer-store exchange needs CUDA IPC between the ranks' GPUs; gloo (CPU tests) runs the collective form
        self.p2p = mode == "p2p" and dist.get_backend(group) == "nccl" and attention_fn is None
        self._px = {}

    def exchange(self, B: int, H: int, S_t: int, S_loc: int, device) -> PeerExchange:
        key = (B, H, S_t, S_loc, str(device))
        if key not in self._px:
            for old in self._px.values():  # one shape at a time: unmap and free the previous buffers
                old.release()
            self._px = {key: PeerExchange(self.group, B, H, S_t, S_loc, device)}
        return self._px[key]

    def release(self):
        """Unmap and drop the peer-store buffers (collective over the group); the next forward builds new ones."""
        for px in self._px.values():
            px.release()
        self._px = {}

    # ---- token sharding of the per-token streams ----------------------------------------------------------------
    def local_range(self, S_v: int) -> Tuple[int, int]:
        if S_v % self.world:
            raise ValueError(f"sequence parallelism needs the video token count ({S_v}) to divide by the group size ({self.world})")
        n = S_v // self.world
        return self.rank * n, (self.rank + 1) * n

    def shard_tokens(self, x: torch.Tensor, B: int, S_v: int) -> torch.Tensor:
        """x [B*S_v, c] (token-major per batch element) -> this rank's [B*S_loc, c]."""
        s0, s1 = self.local_range(S_v)
        return x.view(B, S_v, -1)[:, s0:s1].reshape(B * (s1 - s0), -1).contiguous()

    def gather_tokens(self, x_loc: torch.Tensor, B: int, S_loc: int) -> torch.Tensor:
        """[B*S_loc, c] of every rank -> [B*S_v, c] on every rank (rank order = token order)."""
        c = x_loc.shape[1]
        out = torch.empty((self.world * B * S_loc, c), device=x_loc.device, dtype=x_loc.dtype)
        dist.all_gather_into_tensor(out, x_loc.contiguous(), group=self.group)
        return out.view(self.world, B, S_loc, c).permute(1, 0, 2, 3).reshape(B * self.world * S_loc, c).contiguous()

    # ---- attention with the two exchanges -----------------------------------------------------------------------
    def attention(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, S_t: int):
        """q, k, v [B, H, S_t + S_loc, 64]: ALL heads, the replicated text rows first, then this rank's video tokens.
        Returns (out_text [B, S_t, H*64] - identical on every rank, out_video [B, S_loc, H*64])."""
        P = self.world
        B, H, S_in, hd = q.shape
        if H % P:
            raise ValueError(f"sequence parallelism needs the head count ({H}) to divide by the group size ({P})")
        Hl, S_loc = H // P, S_in - S_t
        S_v = P * S_loc
        h0 = self.rank * Hl
        # (1) video rows: heads scattered, tokens gathered.  send[p] = my tokens, the heads rank p will own
        send = torch.stack([q[:, :, S_t:], k[:, :, S_t:], v[:, :, S_t:]])               # [3, B, H, S_loc, hd]
        send = send.view(3, B, P, Hl, S_loc, hd).permute(2, 0, 1, 3, 4, 5).contiguous()  # [P, 3, B, Hl, S_loc, hd]
        recv = torch.empty_like(send)
        dist.all_to_all_single(recv, send, group=self.group)                             # recv[p] = rank p's tokens, my heads
        vid = recv.permute(1, 2, 3, 0, 4, 5).reshape(3, B, Hl, S_v, hd)                  # tokens back in rank (= token) order
        # (2) text rows are replicated: take this rank's heads
        qkv = torch.empty((3, B, Hl, S_t + S_v, hd), device=q.device, dtype=q.dtype)
        qkv[0, :, :, :S_t], qkv[1, :, :, :S_t], qkv[2, :, :, :S_t] = (t[:, h0:h0 + Hl, :S_t] for t in (q, k, v))
        qkv[:, :, :, S_t:] = vid
        # (3) local attention over all S tokens for Hl heads
        fn = self._attention
        if fn is None:
            from . import ops
            fn = ops.attention
        o_t, o_v = fn(qkv[0], qkv[1], qkv[2], S_t)                                       # [B,S_t,Hl*hd], [B,S_v,Hl*hd]
        # (4) video rows back: tokens scattered, heads gathered
        send2 = o_v.view(B, P, S_loc, Hl * hd).permute(1, 0, 2, 3).contiguous()          # [P, B, S_loc, Hl*hd]
        recv2 = torch.empty_like(send2)
        dist.all_to_all_single(recv2, send2, group=self.group)                           # recv2[p] = my tokens, rank p's heads
        out_video = recv2.permute(1, 2, 0, 3).reshape(B, S_loc, H * hd).contiguous()
        # (5) text rows: every rank needs all heads (the text stream is replicated)
        gath = torch.empty((P,) + tuple(o_t.shape), device=o_t.device, dtype=o_t.dtype)
        dist.all_gather_into_tensor(gath.view(P * B, S_t, Hl * hd), o_t.contiguous(), group=self.group)
        out_text = gath.permute(1, 2, 0, 3).reshape(B, S_t, H * hd).contiguous()
        return out_text, out_video
