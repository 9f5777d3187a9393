"""Merge and unmerge LoRA weights: drop-ins for the reference's `merge_lora` / `unmerge_lora` (utils/lora_utils.py:369-432,
435-494) with the same signatures, file format and arithmetic, for any pipeline object with `.transformer` (and optionally
`.text_encoder`): the native pipelines, the reference's pipeline classes over these modules, or a SimpleNamespace.

- Keys: `<layer>.lora_up.weight`, `<layer>.lora_down.weight` and an optional `<layer>.alpha`.  A layer whose name contains
  `lora_te` belongs to the text encoder, every other one to the transformer.  2-D factors, and 1x1 4-D factors for a 1x1
  convolution, are accepted.
- Layer names are resolved by the reference's rule (`resolve_layer`).
- Every layer is validated before any weight changes: a key that resolves to no weight, factors whose product does not have
  the weight's shape, `lora_te` layers without a text encoder (unless `transformer_only`), or a merge dtype other than
  bfloat16 / float32 raise ValueError and leave every parameter as it was.
- The arithmetic is the reference's, always on the CUDA device, with one specified product order (include/ea_b200.h
  `ea_lora_merge`); `device` is accepted for signature compatibility only.
- Each weight is edited in place in the storage it lives in, bf16 or float8_e4m3fn: on the device; in a sequentially
  offloaded block's pinned buffer (copied to the device and back, EasyAnimateTransformer3DModel.enable_sequential_cpu_offload);
  or in host memory (model CPU offload, an offloaded text encoder), staged through the device.  Modules stay where they are.
- Afterwards the transformer's derived weight copies are invalidated (fused q/k/v, patch-embed operands, the fp8 staging),
  so the next forward uses the merged weights.  A CUDA graph captured before the merge still holds the old operands and must
  be captured again.
"""
from __future__ import annotations

from collections import defaultdict
from contextlib import nullcontext
from typing import Dict, List, NamedTuple

import torch
import torch.nn as nn

from . import ops

LORA_PREFIX_TRANSFORMER = "lora_unet"
LORA_PREFIX_TEXT_ENCODER = "lora_te"
_STORAGE = (torch.bfloat16, torch.float8_e4m3fn)
_MISSING = object()


class _Edit(NamedTuple):
    layer: str
    weight: torch.Tensor  # the parameter, edited in place
    up: torch.Tensor      # [out, rank], as stored in the file
    down: torch.Tensor    # [rank, in]
    scale: float          # fp32 value of multiplier * alpha / rank (negated for unmerge)


def _child(node, name: str):
    """What nn.Module.__getattr__ finds under `name` (a parameter, buffer or submodule), else _MISSING."""
    if isinstance(node, nn.Module):
        for table in (node._parameters, node._buffers, node._modules):
            if name in table:
                return table[name]
    return _MISSING


def resolve_layer(root: nn.Module, layer: str, prefix: str):
    """The module a LoRA layer name addresses, by the reference's rule.  The name after `<prefix>_` is split at "_" into
    segments.  The segments after the first, joined by "_", are first looked up as one attribute of `root` (files written by
    the reference's training start the name with "_", so that is the whole name).  Otherwise the walk starts at `root` with the
    first segment: a name that matches descends and the next segment starts a new name; one that does not is extended by
    "_" and the next segment.  Matching is what nn.Module.__getattr__ sees: parameters, buffers and submodules.  Raises
    ValueError when the segments run out before a match."""
    infos = layer.split(prefix + "_")[-1].split("_")
    hit = _child(root, "_".join(infos[1:]))
    if hit is not _MISSING:
        return hit
    node, name = root, infos.pop(0)
    while True:
        hit = _child(node, name)
        if hit is not _MISSING:
            node = hit
            if not infos:
                return node
            name = infos.pop(0)
        elif not infos:
            raise ValueError(f"LoRA layer {layer!r}: no module of the {type(root).__name__} matches this name")
        else:
            name = f"{name}_{infos.pop(0)}" if name else infos.pop(0)


def _plan(pipeline, state_dict, multiplier, dtype, transformer_only: bool, sign: float) -> List[_Edit]:
    """Resolve and check every layer of `state_dict`; nothing is modified."""
    if dtype not in (torch.bfloat16, torch.float32):
        raise ValueError(f"LoRA merge dtype must be torch.bfloat16 or torch.float32, got {dtype}")
    updates: Dict[str, dict] = defaultdict(dict)
    for key, value in state_dict.items():
        if "." not in key:
            raise ValueError(f"LoRA key {key!r} has no '.<element>' part")
        layer, elem = key.split(".", 1)
        updates[layer][elem] = value
    edits = []
    for layer, elems in updates.items():
        if LORA_PREFIX_TEXT_ENCODER in layer:
            if transformer_only:
                continue
            root, prefix = getattr(pipeline, "text_encoder", None), LORA_PREFIX_TEXT_ENCODER
            if root is None:
                raise ValueError(f"LoRA layer {layer!r} is for the text encoder and the pipeline has none "
                                 "(transformer_only=True skips such layers)")
        else:
            root, prefix = pipeline.transformer, LORA_PREFIX_TRANSFORMER
        module = resolve_layer(root, layer, prefix)
        weight = _child(module, "weight")
        if not isinstance(weight, torch.Tensor):
            raise ValueError(f"LoRA layer {layer!r} resolves to a {type(module).__name__}, which has no weight")
        if weight.dtype not in _STORAGE:
            raise ValueError(f"LoRA layer {layer!r}: the weight is {weight.dtype}; merges write bfloat16 or float8_e4m3fn storage")
        missing = [e for e in ("lora_up.weight", "lora_down.weight") if e not in elems]
        if missing:
            raise ValueError(f"LoRA layer {layer!r} has no {' / '.join(missing)}")
        up, down = elems["lora_up.weight"], elems["lora_down.weight"]
        four_d = up.dim() == 4
        ok = up.dim() == down.dim() and up.dim() in (2, 4) and up.shape[1] == down.shape[0]
        if ok and four_d:
            ok = tuple(up.shape[2:]) == (1, 1) and tuple(down.shape[2:]) == (1, 1)
        want = (up.shape[0], down.shape[1]) + ((1, 1) if four_d else ()) if ok else None
        if not ok or tuple(weight.shape) != want:
            raise ValueError(f"LoRA layer {layer!r}: lora_up {tuple(up.shape)} x lora_down {tuple(down.shape)} does not make "
                             f"the weight's shape {tuple(weight.shape)}")
        rank = up.shape[1]
        alpha = elems["alpha"].item() / rank if "alpha" in elems else 1.0
        scale = float(torch.tensor(multiplier * alpha, dtype=torch.float32))  # torch's scalar multiply rounds it to fp32
        edits.append(_Edit(layer, weight, up.reshape(up.shape[:2]), down.reshape(down.shape[:2]), sign * scale))
    return edits


def _work_device(pipeline) -> torch.device:
    """The GPU that stages host-resident weights: the pipeline's offload device, else the current CUDA device."""
    dev = getattr(pipeline, "_offload_device", None)
    if dev is not None and torch.device(dev).type == "cuda":
        return torch.device(dev)
    return torch.device("cuda", torch.cuda.current_device())


def _merge_into(w: torch.Tensor, e: _Edit, dtype) -> None:
    """One launch on the weight's storage `w` (on the compute device)."""
    up = e.up.to(dtype).to(w.device).contiguous()
    down = e.down.to(dtype).to(w.device).contiguous()
    ops.lora_merge(w.view(up.shape[0], down.shape[1]), up, down, e.scale)


def _apply(pipeline, edits: List[_Edit], dtype) -> None:
    transformer = pipeline.transformer
    off = getattr(transformer, "_offload", None)
    packed: Dict[int, list] = defaultdict(list)  # block index -> [(parameter name in the block, edit)], file order
    loose: List[_Edit] = []
    owner = {}
    if off is not None:
        for i, blk in enumerate(transformer.transformer_blocks):
            if off.packed_block(i):
                owner.update({id(p): (i, name) for name, p in blk.named_parameters()})
    for e in edits:
        hit = owner.get(id(e.weight))
        if hit is not None:
            packed[hit[0]].append((hit[1], e))
        else:
            loose.append(e)
    cuda = False
    if packed:
        def fn(i, views):
            for name, e in packed[i]:
                _merge_into(views[name], e, dtype)
        cuda |= off.device.type == "cuda"
        with torch.cuda.device(off.device) if off.device.type == "cuda" else nullcontext():
            off.edit_blocks(list(packed), fn)
    work = None
    for e in loose:
        w = e.weight.detach()
        if w.is_cuda:
            with torch.cuda.device(w.device):
                _merge_into(w, e, dtype)
        else:  # host memory: to the device, merge, back into the same storage
            work = work or _work_device(pipeline)
            staged = torch.empty_like(w, device=work).copy_(w)
            _merge_into(staged, e, dtype)
            w.copy_(staged)
            del staged
        cuda |= w.is_cuda or work.type == "cuda"
    for m in (transformer, getattr(pipeline, "text_encoder", None)):
        if m is not None and hasattr(m, "invalidate_weight_caches"):
            m.invalidate_weight_caches()
    if cuda:
        torch.cuda.synchronize()
        torch.cuda.empty_cache()  # the staging and factor copies go back to the driver (pipelines._to_host does the same)


def _load(lora_path: str) -> dict:
    from safetensors.torch import load_file
    return load_file(lora_path, device="cpu")


@torch.no_grad()
def merge_lora(pipeline, lora_path, multiplier, device="cpu", dtype=torch.float32, state_dict=None, transformer_only=False):
    """W += multiplier * alpha / rank * lora_up @ lora_down for every layer of the LoRA file at `lora_path` (or of
    `state_dict`), computed in `dtype` (bfloat16 or float32) and stored back in each weight's own dtype.  `device` is
    ignored: the arithmetic runs on the CUDA device.  `transformer_only` skips the text encoder's layers.  Returns
    `pipeline`."""
    sd = _load(lora_path) if state_dict is None else state_dict
    _apply(pipeline, _plan(pipeline, sd, multiplier, dtype, transformer_only, 1.0), dtype)
    return pipeline


@torch.no_grad()
def unmerge_lora(pipeline, lora_path, multiplier=1, device="cpu", dtype=torch.float32):
    """merge_lora's update subtracted again (the same rounding points, so a bf16 round trip drifts as the reference's does).
    `device` is ignored.  Returns `pipeline`."""
    _apply(pipeline, _plan(pipeline, _load(lora_path), multiplier, dtype, False, -1.0), dtype)
    return pipeline
