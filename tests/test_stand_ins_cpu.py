"""The CPU half of tests/test_stand_ins_gpu.py: every stand-in of tests/cpu_ops.py has a contract case there, every case
builds its inputs and runs its stand-in here, and the exact-input ("linear") cases are exact: the stand-in equals the op
evaluated in fp64 with each bf16 rounding point applied once, and most outputs do pass through a rounding."""
import pytest
import torch

from tests import cpu_ops
from tests.test_stand_ins_gpu import CASES, _outs, _within, run, trials


def test_every_stand_in_has_a_contract_case():
    assert set(CASES) == set(cpu_ops.OPS + cpu_ops.VAE_OPS)


@pytest.mark.parametrize("name", CASES)
def test_stand_in_side_of_every_case(name):
    stand_in = getattr(cpu_ops, name)
    ts = trials(name)
    assert ts
    rounded, total = 0, 0
    for t in ts:
        want = run(t, stand_in, "cpu")
        if t.kind == "linear":
            exact, pre = t.exact64(t.make("cpu"))
            assert torch.equal(want, exact), f"{t.label}: the stand-in is not the fp64 evaluation rounded once"
            if pre is not None:  # (SCALE_F32 has no bf16 rounding point)
                rounded += int((pre != pre.to(torch.bfloat16).double()).sum())
                total += pre.numel()
        elif t.kind in ("rounded", "contract"):
            for w, bd in zip(_outs(want), _outs(t.bound(t.make("cpu"), want))):
                _within(w, w, bd, t.label)  # the bound evaluates and broadcasts against the outputs
    if total:  # the exact inputs do exercise the rounding points
        print(f"ROUNDED {name}: {rounded / total:.3f}")
        assert rounded > total / 2, f"{name}: only {rounded / total:.1%} of the outputs need more than 8 bits before rounding"


def test_layernorm_modulate_rounds_one_plus_scale_to_bf16():
    """norm.py:164 `x * (1 + scale)` on bf16 tensors: 1 + scale is a bf16 tensor before the product."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(64, 3072, generator=g).to(torch.bfloat16)
    shift, scale = (torch.randn(1, 3072, generator=g).to(torch.bfloat16) for _ in range(2))
    got = cpu_ops.layernorm_modulate(x, None, None, 1e-6, shift=shift, scale=scale, rows_per_batch=64)
    n = torch.nn.functional.layer_norm(x.float(), (3072,), eps=1e-6).to(torch.bfloat16)
    assert torch.equal(got, n * (1 + scale) + shift)  # the reference's bf16 tensor ops
