"""Stored results of the reference for the tests that compare with it, so that they keep comparing where the reference tree is
not installed.  Where it is installed the tests compute the reference's result live; `EA_MINT_GOLDEN=1` then also records it
into tests/golden/<name>.safetensors (tensors, or a fixed seeded sample of 4096 elements of a large one; other values as JSON
in the metadata).  Where only the stored results are available, tensors are compared within the drift that bf16 CPU
arithmetic shows across machines (same_sample)."""
import json
import os

import torch
from safetensors.torch import load_file, save_file

MINT = os.environ.get("EA_MINT_GOLDEN") == "1"
SAMPLE = 4096
MAX_DRIFT, MEAN_DRIFT = 2.0 ** -3, 2.0 ** -7  # stored comparisons on another machine: see same_sample


def sample(x: torch.Tensor) -> torch.Tensor:
    flat = x.detach().reshape(-1)
    if flat.numel() <= SAMPLE:
        return flat.clone()
    idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(0))[:SAMPLE]
    return flat[idx].clone()


class Store:
    def __init__(self, name: str):
        self.path = os.path.join(os.path.dirname(__file__), "golden", name + ".safetensors")
        self.tensors, self.values = {}, {}
        if not MINT and os.path.exists(self.path):
            from safetensors import safe_open
            self.tensors = load_file(self.path)
            with safe_open(self.path, "pt") as f:
                self.values = {k: json.loads(v) for k, v in (f.metadata() or {}).items()}

    def value(self, key, live):
        """`live()` where the reference exists (recorded when minting), else the stored value."""
        if live is not None:
            v = live()
            if MINT:
                self.values[key] = v
            return v
        return self.values[key]

    def same_sample(self, key, got: torch.Tensor, want: torch.Tensor = None):
        """got equals the reference's tensor: all of it, exactly, when `want` (computed live) is given; else the stored shape and
        sample, within the drift of bf16 CPU arithmetic across machines."""
        if want is not None:
            if MINT:
                self.tensors[key] = sample(want)
                self.values[key + ".shape"] = list(want.shape)
            assert got.shape == want.shape and got.dtype == want.dtype and torch.equal(got, want), key
            return
        assert list(got.shape) == self.values[key + ".shape"], key
        s = sample(got)
        assert s.dtype == self.tensors[key].dtype, key
        # torch's bf16 CPU kernels round differently on other instruction sets, and a few bf16 ulps of that drift compound over
        # the denoise steps (up to ~0.05 on frames in [0, 1]); a host-logic error (noise draw, schedule index, conditioning)
        # moves frames by 0.1-1.  The live comparison above stays exact.
        d = (s.double() - self.tensors[key].double()).abs()
        assert float(d.max()) <= MAX_DRIFT and float(d.mean()) <= MEAN_DRIFT, (key, float(d.max()), float(d.mean()))

    def save(self):
        if MINT:
            save_file({k: v.contiguous() for k, v in self.tensors.items()}, self.path,
                      metadata={k: json.dumps(v) for k, v in self.values.items()})
