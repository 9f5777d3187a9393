"""Three-way parity criterion used by the GPU tests.

north_star asks for rtol=1e-3/atol=1e-4 "bf16", which is tighter than one bf16 ulp (2^-8 relative): two *correct*
bf16 implementations of the same network differ by more than that.  So every module-level test checks
  (1) ours vs the oracle evaluated in fp32 with the same bf16-rounded weights ("truth"): the error must not exceed
      the error the reference's own op-by-op bf16 execution (oracle in bf16) makes against that truth, times a slack;
  (2) the direct ours-vs-oracle-bf16 difference, reported as the fraction of elements within rtol/atol and bounded
      by a few bf16 ulps of the output scale.
"""
import torch


def rel_rms(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double(), b.double()
    return float((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-30))


def three_way(ours: torch.Tensor, ref_bf16: torch.Tensor, truth: torch.Tensor, slack: float = 1.5, floor: float = 2e-3,
              name: str = ""):
    ours, ref_bf16, truth = ours.detach().cpu().float(), ref_bf16.detach().cpu().float(), truth.detach().cpu().float()
    assert ours.shape == truth.shape == ref_bf16.shape, (ours.shape, ref_bf16.shape, truth.shape)
    assert torch.isfinite(ours).all(), f"{name}: non-finite output"
    e_ours, e_ref = rel_rms(ours, truth), rel_rms(ref_bf16, truth)
    scale = truth.abs().max().item()
    max_ours = (ours - truth).abs().max().item() / max(scale, 1e-30)
    max_ref = (ref_bf16 - truth).abs().max().item() / max(scale, 1e-30)
    close = torch.isclose(ours, ref_bf16, rtol=1e-3, atol=1e-4).float().mean().item()
    report = {"name": name, "rel_rms_ours": e_ours, "rel_rms_ref_bf16": e_ref, "max_ours": max_ours,
              "max_ref_bf16": max_ref, "frac_within_rtol1e-3_atol1e-4_of_ref_bf16": close}
    print("PARITY", report)
    assert e_ours <= slack * e_ref + floor, report
    assert max_ours <= 3.0 * max_ref + 4 * floor, report
    return report
