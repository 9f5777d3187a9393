"""Sequential CPU offload of the MMDiT (the reference's `sequential_cpu_offload` GPU_memory_mode, predict_t2v.py:256-265):
each block's parameters live in ONE pinned host buffer, laid out the way the kernels consume them (q/k/v weights and biases
back to back, so that the fused projection operand is a plain view), and the block's parameters ARE views into it - edits
through `load_state_dict` or `.data` land in the buffer itself.  On the device stay the non-block parameters and a ring of two
slots: block i+1 is copied into one slot on a side stream (`ea_h2d_block`) while block i computes out of the other.  A bf16 slot
is used in place through a block whose parameters are views into it; an e4m3 slot is expanded by one `ea_expand_e4m3_segments`
launch into the one-block bf16 staging of `_Fp8Staging`.  What is computed is unchanged: the same kernels read the same bytes."""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from . import _lib as L
from . import ops

ALIGN = 16  # bytes: every parameter starts 16-byte aligned in a packed block (the vector width of the expansion kernel)


def pack_order(names: List[str]) -> List[str]:
    """Parameter names of a block in packed order: named_parameters() order, except that each attention's to_q/to_k/to_v
    weights follow one another, and so do their biases ([3d, d] and [3d] operands of the fused projection)."""
    out = []
    for n in names:
        parts = n.split(".")
        if len(parts) == 3 and parts[1] in ("to_q", "to_k", "to_v"):
            if parts[1] == "to_q":
                out += [f"{parts[0]}.{p}.{parts[2]}" for p in ("to_q", "to_k", "to_v")]
            continue
        out.append(n)
    return out


def block_layout(block: nn.Module) -> List[Tuple[str, Tuple[int, ...], torch.dtype, int, int]]:
    """[(name, shape, dtype, byte offset, bytes)] of the block's parameters in its packed buffer."""
    params = dict(block.named_parameters())
    layout, off = [], 0
    for name in pack_order(list(params)):
        p = params[name]
        nbytes = p.numel() * p.element_size()
        layout.append((name, tuple(p.shape), p.dtype, off, nbytes))
        off += (nbytes + ALIGN - 1) // ALIGN * ALIGN
    return layout


def layout_bytes(layout) -> int:
    name, shape, dtype, off, nbytes = layout[-1]
    return (off + nbytes + ALIGN - 1) // ALIGN * ALIGN


def _set_param(root: nn.Module, name: str, value: torch.Tensor, requires_grad: bool = False) -> None:
    *path, attr = name.split(".")
    m = root
    for p in path:
        m = getattr(m, p)
    m._parameters[attr] = nn.Parameter(value, requires_grad=requires_grad)


def _views(buf: torch.Tensor, layout) -> Dict[str, torch.Tensor]:
    return {name: buf[off:off + nbytes].view(dtype).view(shape) for name, shape, dtype, off, nbytes in layout}


def fused_qkv_views(buf: torch.Tensor, layout, attn: str) -> Tuple[torch.Tensor, torch.Tensor]:
    """The [3d, d] weight / [3d] bias of attention `attn` as views of its packed, back-to-back q/k/v rows in `buf`."""
    ent = {name: (shape, dtype, off, nbytes) for name, shape, dtype, off, nbytes in layout}
    out = []
    for kind in ("weight", "bias"):
        (shape, dtype, off, nbytes), (_, _, off_k, _), (_, _, off_v, _) = (ent[f"{attn}.{p}.{kind}"] for p in ("to_q", "to_k", "to_v"))
        assert off_k == off + nbytes and off_v == off_k + nbytes
        out.append(buf[off:off + 3 * nbytes].view(dtype).view((3 * shape[0],) + shape[1:]))
    return out[0], out[1]


class PackedBlock:
    """One block's parameters moved into one (pinned) host buffer; the block's parameters become views into it."""

    def __init__(self, block: nn.Module, pin: bool):
        self.layout = block_layout(block)
        self.host = torch.empty((layout_bytes(self.layout),), dtype=torch.uint8, pin_memory=pin)
        params = dict(block.named_parameters())
        for name, view in _views(self.host, self.layout).items():
            p = params[name]
            view.copy_(p.detach())
            _set_param(block, name, view, p.requires_grad)
        self.key = self.block_key(block)

    def block_key(self, block: nn.Module) -> tuple:
        params = dict(block.named_parameters())
        return tuple((params[n].data_ptr(), params[n].dtype) for n, *_ in self.layout)


class CudaBlockStreamer:
    """The CUDA side of the ring: a copy stream and, per slot, the events "slot ready" (recorded by the copy) and "slot free"
    (recorded on the compute stream after the slot's last reader)."""
    pin_memory = True

    def __init__(self, device):
        self.device = torch.device(device)
        with torch.cuda.device(self.device):
            self.stream = torch.cuda.Stream(self.device)
            self.ready = [torch.cuda.Event(), torch.cuda.Event()]
            self.free = [torch.cuda.Event(), torch.cuda.Event()]
            for e in self.ready + self.free:
                e.record()  # creates the cudaEvent_t the C ABI takes

    def begin(self):
        if torch.cuda.is_current_stream_capturing():
            raise L.EaError("a sequentially offloaded transformer cannot be captured in a CUDA graph: its block copies run on "
                            "a side stream, ordered by events, from host memory")

    def copy(self, slot: int, index: int, dst: torch.Tensor, src: torch.Tensor):
        ops.h2d_block(dst, src, self.free[slot], self.ready[slot], self.stream)

    def acquire(self, slot: int, index: int):
        torch.cuda.current_stream(self.device).wait_event(self.ready[slot])

    def release(self, slot: int, index: Optional[int]):
        self.free[slot].record(torch.cuda.current_stream(self.device))

    def segment_table(self, segments):
        return ops.e4m3_segment_table(segments)

    def expand(self, src: torch.Tensor, table):
        ops.expand_e4m3_segments(src, table)

    def drain(self):
        self.stream.synchronize()


class SequentialOffload:
    """The packed blocks of one transformer and the device ring they are streamed through (see the module docstring)."""

    def __init__(self, model, device="cuda", streamer=None):
        self.model = model
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.streamer = streamer if streamer is not None else CudaBlockStreamer(self.device)
        self.packs: List[Optional[PackedBlock]] = [None] * len(model.transformer_blocks)
        self._device_side = None
        self.owner = [None, None]
        self.h2d_bytes = 0  # bytes copied host -> device since construction (tools/bench_offload.py)
        self.sync()

    # -- host side ------------------------------------------------------------------------------------------------
    def _place_head(self):
        m = self.model
        for name, child in m.named_children():
            if name != "transformer_blocks":
                child.to(self.device)
        for name, b in list(m._buffers.items()):
            if b is not None and b.device != self.device:
                m._buffers[name] = b.to(self.device)

    def invalidate(self):
        """invalidate_weight_caches(): drop the device side (slot views, expansion tables), rebuilt on the next forward.  The
        packed buffers stay: they ARE the parameters, so `.data` edits (the LoRA hand-shake) are already in them, and a
        replaced parameter is caught by sync()."""
        self.streamer.drain()
        self._device_side = None

    def sync(self):
        """(Re)pack the blocks whose parameters are no longer the packed views (.to(...), .data = ..., a changed block
        count), and put the non-block parameters on the device."""
        self._place_head()
        blocks = self.model.transformer_blocks
        if len(self.packs) != len(blocks):
            self.streamer.drain()
            self.packs = [None] * len(blocks)
        changed = False
        for i, blk in enumerate(blocks):
            pk = self.packs[i]
            if pk is None or pk.block_key(blk) != pk.key:
                if not changed:
                    self.streamer.drain()
                changed = True
                self.packs[i] = PackedBlock(blk, self.streamer.pin_memory)
        if changed:
            self._device_side = None

    def packed_block(self, i: int) -> bool:
        """Whether block i's parameters are still the views of its packed buffer (no sync() needed since they were replaced)."""
        pk = self.packs[i] if i < len(self.packs) else None
        return pk is not None and pk.block_key(self.model.transformer_blocks[i]) == pk.key

    def edit_blocks(self, blocks, fn):
        """Edit packed blocks in place on the device (a LoRA merge): each block i of `blocks` is copied from its pinned buffer
        into one device scratch block, fn(i, {parameter name: view of the scratch}) enqueues its kernels on the current stream,
        and the scratch is copied back into the same buffer.  Parameters, PackedBlocks and host addresses stay as they are, so
        nothing is repacked.  Returns after the last copy back has landed."""
        blocks = sorted(set(blocks))
        if not blocks:
            return
        for i in blocks:
            if not self.packed_block(i):
                raise L.EaError(f"edit_blocks: block {i} is not packed (its parameters were replaced since the last forward)")
        self.streamer.drain()  # no slot copy still reads a buffer that is about to be rewritten
        scratch = torch.empty((max(self.packs[i].host.nbytes for i in blocks),), dtype=torch.uint8, device=self.device)
        for i in blocks:
            host = self.packs[i].host
            dev = scratch[:host.nbytes]
            dev.copy_(host, non_blocking=True)
            fn(i, _views(dev, self.packs[i].layout))
            host.copy_(dev, non_blocking=True)
        if self.device.type == "cuda":
            torch.cuda.current_stream(self.device).synchronize()
        self._device_side = None

    # -- device side ----------------------------------------------------------------------------------------------
    def _kind(self, i: int) -> bool:
        return self.model.transformer_blocks[i].attn2 is not None

    def _build_device_side(self):
        from .transformer3d import EasyAnimateDiTBlock
        dtypes = {pk.layout[0][2] for pk in self.packs}
        if len(dtypes) != 1 or next(iter(dtypes)) not in (torch.bfloat16, torch.float8_e4m3fn):
            raise L.EaError(f"sequential offload streams bf16 or float8_e4m3fn blocks, got {sorted(map(str, dtypes))}")
        size = max(layout_bytes(pk.layout) for pk in self.packs)
        slots = [torch.empty((size,), dtype=torch.uint8, device=self.device) for _ in range(2)]
        layouts = {self._kind(i): pk.layout for i, pk in enumerate(self.packs)}
        c = self.model.config
        d = c.num_attention_heads * c.attention_head_dim
        views = {}
        if next(iter(dtypes)) == torch.bfloat16:
            for s in range(2):
                for kind, layout in layouts.items():
                    with torch.device("meta"):
                        blk = EasyAnimateDiTBlock(d, c.num_attention_heads, c.attention_head_dim, c.time_embed_dim,
                                                  c.norm_elementwise_affine, c.norm_eps, is_mmdit_block=kind)
                    for name, t in _views(slots[s], layout).items():
                        _set_param(blk, name, t)
                    for a in ("attn1", "attn2"):
                        if getattr(blk, a) is not None:
                            getattr(blk, a)._fused_static = fused_qkv_views(slots[s], layout, a)
                    views[(s, kind)] = blk
        self._device_side = {"slots": slots, "layouts": layouts, "views": views, "tables": {}}

    def start(self):
        """Called at the start of every forward."""
        self.streamer.begin()
        self.sync()
        if self._device_side is None:
            self._build_device_side()
        for s in (0, 1):  # whatever read a slot before this forward is ahead of its next copy
            self.streamer.release(s, None)
        self.owner = [None, None]

    def _fetch(self, i: int):
        s = i % 2
        if self.owner[s] != i:
            pk = self.packs[i]
            self.streamer.copy(s, i, self._device_side["slots"][s], pk.host)
            self.h2d_bytes += pk.host.nbytes
            self.owner[s] = i

    def block(self, i: int, staging=None):
        """Block i ready to run on the compute stream; block i+1's copy is issued first so that it overlaps block i."""
        self._fetch(i)
        if i + 1 < len(self.packs):
            self._fetch(i + 1)
        s = i % 2
        self.streamer.acquire(s, i)
        ds = self._device_side
        kind = self._kind(i)
        if staging is None:
            return ds["views"][(s, kind)]
        st = staging._staging_block(kind)
        ent = ds["tables"].get((s, kind))
        if ent is None or ent[0] is not st:
            segs = [(off, staging.destination(st, name)) for name, shape, dtype, off, nbytes in ds["layouts"][kind]]
            ent = ds["tables"][(s, kind)] = (st, self.streamer.segment_table(segs))
        self.streamer.expand(ds["slots"][s], ent[1])
        self.streamer.release(s, i)  # the expansion was the slot's only reader
        return st

    def release(self, i: int):
        """Block i's kernels are enqueued: its slot may be refilled once they have run."""
        self.streamer.release(i % 2, i)

    def device_bytes(self) -> int:
        """Bytes of the two device slots."""
        return 0 if self._device_side is None else sum(t.nbytes for t in self._device_side["slots"])
