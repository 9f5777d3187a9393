"""Every CUDA entry point of easyanimate_b200.ops / vae_ops against its CPU stand-in in tests/cpu_ops.py.

Half of the suite runs the product's host logic on the CPU with those stand-ins swapped in (cpu_ops.use_stand_ins); the
tests here hold each stand-in to what its kernel computes, so that a CPU result says something about the GPU one.  CASES has
one entry per stand-in; every case builds seeded inputs on the CPU, calls the entry point on CUDA copies and the stand-in on
CPU copies, and compares the two by one of these criteria:

  exact    ops without a reduction (layout changes, elementwise arithmetic): torch.equal; NaN outputs compare by position.
  linear   the linear ops (conv3d_causal, prepare_latents, skinny_linear, gemm) on operands that are small integers times
           powers of two, chosen so that every fp32 partial sum is exact in any order (at most 20 significant bits, asserted
           from the shapes): the only rounding left is at the bf16 rounding points, which must then agree bit for bit,
           round-to-nearest-even ties included.  Most outputs are asserted to need more than bf16's 8 bits before rounding.
  rounded  reductions and transcendentals: at least MIN_BIT_EXACT of the outputs equal the stand-in bit for bit, and every
           output lies within a bound of one ulp at each rounding point, carried through the later ops.
  contract attention, spatial_attention and qkv_gemm_ln_rope, whose numerics have strict suites of their own
           (test_attn_exact_gpu.py, test_gemm_tiles_gpu.py): here only the calling contract (layouts, gates, offsets).

tests/test_stand_ins_cpu.py runs the CPU half of every case without a GPU.  Nothing here touches CUDA at import time."""
import pytest
import torch
import torch.nn.functional as F

from tests import cpu_ops
from tests.test_gemm_tiles_gpu import bit_exact_fraction

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
EPI_BIAS, EPI_BIAS_GELU, EPI_BIAS_GATE_RES, EPI_SCALE_F32, EPI_BIAS_RES = 0, 1, 2, 3, 4  # include/ea_b200.h
# Lowest fraction of outputs of a "rounded" case that must equal the stand-in bit for bit, as in test_gemm_tiles_gpu.py.
# A missing or extra bf16 rounding point moves a large share of the outputs; a different fp32 evaluation order of a
# reduction or a transcendental only moves the values that sit next to a rounding boundary.  Observed on H100 80GB HBM3
# (SXM, 132 SMs), the lowest fraction over each op's trials: layernorm_modulate 0.99995, rmsnorm 1.0, groupnorm 0.99604
# (the trials with a mean of 50; 0.99997 elsewhere), groupnorm_from_sums 0.99993, timestep_embedding 0.99891,
# skinny_linear with activations 1.0, gemm BIAS_GELU 0.99410, prepare_latents at in_scale != 1 1.0.  With 1 + scale left
# unrounded in the stand-in (the reference rounds it, norm.py:164), layernorm_modulate falls to 0.89 at d = 8.
MIN_BIT_EXACT = 0.99
LINEAR_BITS = 20  # largest significant-bit count of any partial sum in a "linear" case


class Trial:
    """One call of an op.  make(device) builds fresh inputs on `device` from CPU tensors seeded at construction and returns
    an env dict with "args" and "kw"; call(fn, env) runs the op (default: fn(*args, **kw)) and result(ret, env) picks what is
    compared (default: the return value).  bound(env, want) gives the admissible |error| of every output ("rounded",
    "contract").  exact64(env) -> (outputs, pre) is the op evaluated in fp64 with the header's rounding points, each applied
    once, and pre the fp64 values at its first bf16 rounding point ("linear"; checked on the CPU, test_stand_ins_cpu.py)."""

    def __init__(self, label, kind, make, result=None, bound=None, exact64=None, min_exact=MIN_BIT_EXACT, call=None):
        assert kind in ("exact", "linear", "rounded", "contract"), kind
        assert (exact64 is not None) == (kind == "linear") and (bound is not None) == (kind in ("rounded", "contract"))
        self.label, self.kind, self.make, self.bound, self.exact64, self.min_exact = label, kind, make, bound, exact64, min_exact
        self.result = result or (lambda ret, env: ret)
        self.call = call or (lambda fn, env: fn(*env["args"], **env.get("kw", {})))


def run(trial, fn, device):
    """fn(*args, **kw) on inputs built on `device`; the compared outputs, moved to the CPU."""
    env = trial.make(device)
    ret = trial.call(fn, env)
    if device == "cuda":
        torch.cuda.synchronize()
    return _cpu(trial.result(ret, env))


def _cpu(x):
    if isinstance(x, torch.Tensor):
        return x.cpu()
    if isinstance(x, (tuple, list)):
        return tuple(_cpu(v) for v in x)
    return x


def _outs(x):
    return list(x) if isinstance(x, tuple) else [x]


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _randn(shape, scale=1.0, seed=0, offset=0.0):
    return (torch.randn(shape, generator=_gen(seed)) * scale + offset).to(bf16)


def _ints(shape, amp, exp2, seed):
    """Integers in [-amp, amp] times 2**exp2, as bf16: exact for amp <= 256."""
    assert amp <= 256
    return (torch.randint(-amp, amp + 1, shape, generator=_gen(seed)).float() * 2.0 ** exp2).to(bf16)


def _budget(K, amp_a, amp_w, extra=0):
    """A sum of K products of integers up to amp_a and amp_w (in units of the product's power of two), plus `extra` such
    units of bias / residual, stays within LINEAR_BITS significant bits: every fp32 partial sum is exact in any order."""
    worst = K * amp_a * amp_w + extra
    assert worst < 2 ** LINEAR_BITS, (K, amp_a, amp_w, extra, worst)


def _d(device):
    """CPU tensor -> a fresh copy on `device`."""
    return lambda t: None if t is None else t.to(device, copy=True)


def _bf16_ulp(x):
    """One bf16 ulp at |x| (8 significant bits); 2^-133 (the smallest normal's ulp) at 0."""
    x = x.float()
    return torch.exp2((torch.frexp(x).exponent - 8).clamp_min(-133).float())


def _r(x):
    return x.to(bf16).float()


# ---------------------------------------------------------------------------------------------------------------------
# ops (easyanimate_b200.ops)
# ---------------------------------------------------------------------------------------------------------------------
def _gemm_exact64(env):
    (a, w, bias), kw = env["args"], env["kw"]
    acc = a.double() @ w.double().t()
    epi = kw["epilogue"]
    if epi == EPI_SCALE_F32:
        return (acc * kw["scale"]).float(), None
    pre = acc + bias.double()
    lin = _r(pre).double()
    if epi == EPI_BIAS_GATE_RES:
        g = kw["gate"].double().repeat_interleave(kw["rows_per_batch"], dim=0)
        return (kw["residual"].double() + _r(g * lin).double()).to(bf16), pre
    if epi == EPI_BIAS_RES:
        return (lin + kw["residual"].double()).to(bf16), pre
    return lin.to(bf16), pre


def _gelu_bound(env, want):
    (a, w, bias) = env["args"]
    lin = _r(a.float() @ w.float().t() + bias.float())  # exact operands: lin is the kernel's bit for bit
    return 2.0 ** -19 * lin.abs() + 2.0 ** -20 + _bf16_ulp(want)


def gemm_cases():
    out = []
    M, N, K, B = 300, 200, 1024, 3
    _budget(K, 15, 15, extra=256)  # products in units of 2^-9; the bias up to 256 of them
    for name, epi in (("bias", EPI_BIAS), ("bias_res", EPI_BIAS_RES), ("gate_res", EPI_BIAS_GATE_RES),
                      ("scale_f32", EPI_SCALE_F32), ("bias_gelu", EPI_BIAS_GELU)):
        a, w = _ints((M, K), 15, -3, 1), _ints((N, K), 15, -6, 2)
        bias = _ints((N,), 256, -9, 3)
        res, gate = _ints((M, N), 256, -5, 4), _ints((B, N), 8, -2, 5)

        def make(device, epi=epi, a=a, w=w, bias=bias, res=res, gate=gate):
            d = _d(device)
            kw = dict(epilogue=epi, rows_per_batch=M // B, scale=2.0 ** -5)
            if epi in (EPI_BIAS_RES, EPI_BIAS_GATE_RES):
                kw["residual"] = d(res)
            if epi == EPI_BIAS_GATE_RES:
                kw["gate"] = d(gate)
            return {"args": (d(a), d(w), None if epi == EPI_SCALE_F32 else d(bias)), "kw": kw}
        if epi == EPI_BIAS_GELU:
            out.append(Trial(f"gemm {name}", "rounded", make, bound=_gelu_bound))
        else:
            out.append(Trial(f"gemm {name}", "linear", make, exact64=_gemm_exact64))
    return out


def _skinny_exact64(env):
    x, w, bias = env["args"]
    pre = x.double() @ w.double().t() + (0 if bias is None else bias.double())
    return pre.to(bf16), pre


def _skinny_act_bound(env, want):
    (x, w, bias), kw = env["args"], env["kw"]
    xs = x.float()
    if kw.get("act_in"):
        xs = _r(F.silu(xs))  # one bf16 ulp per input where the kernel's __expf rounds the other way
    lin = _r(xs @ w.float().t() + (0 if bias is None else bias.float()))
    err = (_bf16_ulp(xs) @ w.float().abs().t() if kw.get("act_in") else 0) + _bf16_ulp(lin)
    if kw.get("act_out"):
        err = 1.1 * err + 2.0 ** -20 * want.float().abs() + _bf16_ulp(want)
    return err


def skinny_linear_cases():
    out = []
    for K, (amp_x, amp_w) in ((8, (255, 255)), (520, (63, 31)), (3072, (31, 10))):
        _budget(K, amp_x, amp_w)
        for N in (1, 7, 18432):
            w = _ints((N, K), amp_w, -5, 11)
            for M in ((1, 8, 9, 17) if N == 18432 else range(1, 18)):  # M = 8, K = 3072: the 96 KB shared-memory stage
                x = _ints((M, K), amp_x, -4, 10 + M)

                def make(device, x=x, w=w):
                    d = _d(device)
                    return {"args": (d(x), d(w), None), "kw": {}}
                out.append(Trial(f"skinny_linear M={M} K={K} N={N}", "linear", make, exact64=_skinny_exact64))
    for act_in, act_out in ((1, 0), (0, 1), (1, 1)):
        M, K, N = 3, 3072, 1536
        x, w, b = _randn((M, K), 1.0, 20), _randn((N, K), K ** -0.5, 21), _randn((N,), 0.5, 22)

        def make(device, x=x, w=w, b=b, act_in=act_in, act_out=act_out):
            d = _d(device)
            return {"args": (d(x), d(w), d(b)), "kw": {"act_in": act_in, "act_out": act_out}}
        out.append(Trial(f"skinny_linear act_in={act_in} act_out={act_out}", "rounded", make, bound=_skinny_act_bound))
    return out


def _ln_bound(env, want):
    """One ulp of the normalised value n (plus, after a first LayerNorm, the ulp of its output carried through the second
    one's 1/std), then through m = bf16(n * bf16(1 + scale)) and bf16(m + shift), one more ulp at each."""
    (x, w, b, eps), kw = env["args"], env["kw"]
    pre = kw.get("pre")
    n = cpu_ops.layernorm_modulate(x, w, b, eps, pre=pre).float()
    err = _bf16_ulp(n)
    if pre is not None:
        p = cpu_ops.layernorm_modulate(x, pre[0], pre[1], pre[2]).float()
        rstd = torch.rsqrt(p.var(dim=1, unbiased=False, keepdim=True) + eps)
        err = err + (1.0 if w is None else w.float().abs()) * rstd * _bf16_ulp(p)
    if kw.get("shift") is not None:
        batch = torch.arange(x.shape[0]) // kw["rows_per_batch"]
        s = _r(1 + kw["scale"].float()[batch])
        m = _r(n * s)
        err = s.abs() * err + _bf16_ulp(m) + _bf16_ulp(want)
    return err


def layernorm_modulate_cases():
    out = []
    B, S = 3, 77
    for d in (8, 64, 248, 256, 264, 1536, 1920, 3072, 4096):
        x = _randn((B * S, d + 64), 1.0, d, offset=0.3)
        x[5] = _randn((d + 64,), 1.0, d + 1, offset=100.0)  # mean 100, std 1: bf16 spacing 0.5 and a large mean to remove
        x[6] = 0.75  # a constant row: zero variance, eps alone
        w, b = 1 + _randn((d,), 0.1, d + 2), _randn((d,), 0.1, d + 3)
        mod = _randn((B, 6 * d), 1.0, d + 4)
        pre = (1 + _randn((d,), 0.2, d + 5), _randn((d,), 0.2, d + 6))

        def make(device, x=x, w=w, b=b, mod=mod, d=d, affine=True, pre_ln=None, strided_out=False):
            dv = _d(device)
            mm = dv(mod)
            kw = dict(shift=mm[:, :d], scale=mm[:, d:2 * d], rows_per_batch=S)
            if pre_ln is not None:
                kw["pre"] = (dv(pre_ln[0]), dv(pre_ln[1]), 1e-5)
            env = {"args": (dv(x)[:, :d], dv(w) if affine else None, dv(b) if affine else None, 1e-6), "kw": kw}
            if strided_out:
                env["buf"] = torch.full((B * S, d + 24), -3.0, dtype=bf16, device=device)
                kw["out"] = env["buf"][:, :d]
            return env
        out.append(Trial(f"layernorm_modulate d={d}", "rounded", make, bound=_ln_bound))
        if d in (264, 3072):
            out.append(Trial(f"layernorm_modulate d={d} no affine, pre, strided out", "rounded",
                             lambda device, make=make, pre=pre: make(device, affine=False, pre_ln=pre, strided_out=True),
                             result=lambda ret, env: env["buf"], bound=_ln_strided_bound))
    x = _randn((50, 1536), 2.0, 7)

    def make_plain(device):
        d = _d(device)
        return {"args": (d(x), None, None, 1e-6), "kw": {}}
    out.append(Trial("layernorm_modulate no modulation", "rounded", make_plain, bound=_ln_bound))
    return out


def _ln_strided_bound(env, want):
    """_ln_bound on the columns written; the pad columns of the strided output must stay as they were (bound 0)."""
    d = env["args"][0].shape[1]
    err = torch.zeros_like(want, dtype=torch.float32)
    err[:, :d] = _ln_bound(env, want[:, :d])
    return err


def _rms_bound(env, want):
    x, w, eps = env["args"]
    xf = x.float()
    y = _r(xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps))
    return w.float().abs() * _bf16_ulp(y) + _bf16_ulp(want)


def rmsnorm_cases():
    out = []
    for d in (8, 256, 3584, 4096):
        for size in (10.0, 1e-3):  # at 1e-3 the mean square (1e-6) is comparable to eps
            x, w = _randn((45, d), size, d), 1 + _randn((d,), 0.1, d + 1)

            def make(device, x=x, w=w):
                dv = _d(device)
                return {"args": (dv(x), dv(w), 1e-6)}
            out.append(Trial(f"rmsnorm d={d} size={size}", "rounded", make, bound=_rms_bound))
    return out


def _temb_bound(env, want):
    t = env["args"][0].float()[:, None]
    return t * 2.0 ** -20 + 2.0 ** -20 + _bf16_ulp(want)


def timestep_embedding_cases():
    out = []
    t = torch.arange(1000).float().to(bf16)  # every integer step 0..999 (bf16 rounds the larger ones, as the caller's does)
    for flip in (True, False):
        for shift in (0.0, 1.0):
            def make(device, flip=flip, shift=shift):
                return {"args": (_d(device)(t), 256, flip, shift)}
            out.append(Trial(f"timestep_embedding flip={flip} shift={shift}", "rounded", make, bound=_temb_bound))
    return out


def patchify_cases():
    out = []
    B, F_, H, W = 2, 1, 6, 10  # H/2, W/2 odd
    for C1, C2 in ((16, None), (16, 0), (16, 1), (16, 17), (3, 0)):
        x = _randn((B, C1, F_, H, W), 1.0, C1)
        x2 = None if C2 is None else _randn((B, C2, F_, H, W), 1.0, 50 + C2)

        def make(device, x=x, x2=x2):
            dv = _d(device)
            return {"args": (dv(x), dv(x2))}
        out.append(Trial(f"patchify C1={C1} C2={C2}", "exact", make))
    x = _randn((1, 16, 3, 8, 12), 1.0, 9)
    out.append(Trial("patchify F=3", "exact", lambda device: {"args": (_d(device)(x),)}))
    return out


def unpatchify_cases():
    B, C, F_, H, W = 2, 16, 3, 6, 10
    y = _randn((B * F_ * (H // 2) * (W // 2), 4 * C + 40), 1.0, 3)

    def make(device):
        return {"args": (_d(device)(y)[:, :4 * C + 8], B, C, F_, H, W)}  # a column slice: ldy = 4C + 40
    return [Trial("unpatchify strided", "exact", make)]


def cfg_euler_step_cases():
    out = []
    shape = (1, 16, 3, 7, 9)  # 3024 elements: not a multiple of 512
    lat = _randn(shape, 1.0, 1)
    pred = _randn((2,) + shape[1:], 1.0, 2)
    for use_cfg in (True, False):
        for g in (1.0, 6.0, 7.5):
            def make(device, use_cfg=use_cfg, g=g):
                dv = _d(device)
                return {"args": (dv(pred) if use_cfg else dv(pred[:1]), dv(lat), g, 0.9123, 0.8731, use_cfg)}
            out.append(Trial(f"cfg_euler_step cfg={use_cfg} g={g}", "exact", make))
    return out


def ew_add_cases():
    out = []
    a, b = _randn((7, 334), 1.0, 1), _randn((7, 334), 3.0, 2)  # n = 2338: even, not a multiple of 512
    for subtract in (False, True):
        for with_out in (False, True):
            def make(device, subtract=subtract, with_out=with_out):
                dv = _d(device)
                kw = {"subtract": subtract}
                if with_out:
                    kw["out"] = torch.full((7, 334), 5.0, dtype=bf16, device=device)
                return {"args": (dv(a), dv(b)), "kw": kw}
            out.append(Trial(f"ew_add subtract={subtract} out={with_out}", "exact", make))
    return out


def dequant_e4m3_cases():
    codes = torch.arange(256, dtype=torch.uint8).repeat(4)[:3 * 256 + 10]  # every code, n % 16 = 10: the tail loop

    def make(device):
        w8 = _d(device)(codes).view(torch.float8_e4m3fn)
        return {"args": (w8, torch.full((w8.numel(),), 9.0, dtype=bf16, device=device))}
    return [Trial("dequant_e4m3 all codes", "exact", make)]


def _l1_bound(env, want):
    """fp32 partials per thread over the grid-stride loop, then a 32-lane and an 8-warp fp32 sum per block (l1_sums_kernel):
    each term passes through at most `adds` fp32 additions, each off by at most 2^-24 of the running sum."""
    cur = env["args"][0]
    n = cur.numel()
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    blocks = min(-(-n // 2 // 256), 4 * sms)
    adds = 2 * -(-n // (2 * blocks * 256)) + 5 + 8 + 2
    num = (cur.float() - env["args"][1].float()).to(bf16).double().abs().sum().item()
    den = env["args"][1].double().abs().sum().item()
    return adds * 2.0 ** -24 * num, adds * 2.0 ** -24 * den


def l1_sums_cases():
    out = []
    for n in (4096, 1_000_002):  # the second one beyond one grid-stride pass of the 4-blocks-per-SM grid
        cur, prev = _randn((n,), 1.0, 1), _randn((n,), 1.0, 2)

        def make(device, cur=cur, prev=prev):
            dv = _d(device)
            return {"args": (dv(cur), dv(prev))}
        out.append(Trial(f"l1_sums n={n}", "rounded", make, bound=_l1_bound, min_exact=None))
    same = _randn((10_000,), 1.0, 3)
    out.append(Trial("l1_sums cur == prev", "rounded", lambda device: {"args": (_d(device)(same), _d(device)(same))},
                     bound=_l1_bound, min_exact=None))
    return out


def qkv_gemm_ln_rope_cases():
    out = []
    B, S_part, d, S_text = 2, 77, 192, 40
    H, S = d // 64, S_text + S_part + 13
    a, w, b = _randn((B * S_part, d), 1.0, 1), _randn((3 * d, d), 0.05, 2), _randn((3 * d,), 0.5, 3)
    lnq = (1 + _randn((64,), 0.1, 4), _randn((64,), 0.1, 5))
    lnk = (1 + _randn((64,), 0.1, 6), _randn((64,), 0.1, 7))
    ang = torch.rand((S_part, 32), generator=_gen(8)) * 6.28
    cos, sin = torch.cos(ang).repeat_interleave(2, dim=1), torch.sin(ang).repeat_interleave(2, dim=1)
    for rope in (True, False):
        def make(device, rope=rope):
            dv = _d(device)
            q, k, v = (torch.zeros((B, H, S, 64), dtype=bf16, device=device) for _ in range(3))
            return {"args": (dv(a), dv(w), dv(b), (dv(lnq[0]), dv(lnq[1])), (dv(lnk[0]), dv(lnk[1])),
                             (dv(cos), dv(sin)) if rope else None, q, k, v),
                    "kw": dict(rows_per_batch=S_part, seq_offset=S_text, eps=1e-6)}
        out.append(Trial(f"qkv_gemm_ln_rope rope={rope}", "contract", make, result=lambda ret, env: env["args"][6:9],
                         bound=lambda env, want: tuple(2e-2 + 2 ** -6 * t.float().abs() for t in want)))
    return out


def attention_cases():
    B, H, S, S_text = 2, 3, 300, 45
    q, k, v = (_randn((B, H, S, 64), 1.0, i) for i in (1, 2, 3))

    def make(device):
        dv = _d(device)
        return {"args": (dv(q), dv(k), dv(v), S_text), "kw": {"scale": 0.1}}
    return [Trial("attention", "contract", make,
                  bound=lambda env, want: tuple(2e-2 + 3e-2 * t.float().abs() for t in want))]


# ---------------------------------------------------------------------------------------------------------------------
# VAE ops (easyanimate_b200.vae_ops)
# ---------------------------------------------------------------------------------------------------------------------
def _conv64(env):
    """The causal convolution in fp64 with the header's rounding points applied once each (ea_conv3d_args)."""
    (x, w_packed, bias, cout), kw = env["args"], env["kw"]
    T, H, W, Cin = x.shape
    w = w_packed.double().view(w_packed.shape[0], 3, 3, 3, Cin).permute(0, 4, 1, 2, 3)[:cout]
    xin = F.pad(x.double().permute(3, 0, 1, 2)[None], (0, 0, 0, 0, 2, 0), mode="replicate")
    st = kw.get("stride_t", 1)
    if kw.get("stride_hw", 1) == 2:
        y = F.conv3d(F.pad(xin, (0, 1, 0, 1)), w, bias.double()[:cout], stride=(st, 2, 2))[0]
    else:
        y = F.conv3d(xin, w, bias.double()[:cout], padding=(0, 1, 1), stride=(st, 1, 1))[0]
    if kw.get("out_rows", 0) > 0:
        y = y[:, :, kw["out_row0"]:kw["out_row0"] + kw["out_rows"]]
    assert torch.equal(y, y.float().double()), "a pre-rounding value is not an fp32 value: the operands are not exact"
    pre = y
    y = y.to(bf16).double()
    if kw.get("residual") is not None:
        y = (y + kw["residual"].double().permute(3, 0, 1, 2)).to(bf16).double()
    if kw.get("dup_frames") and T > 1:
        y = y[:, [0] + [i for t in range(1, T) for i in (t, t)]]
    y = y.to(bf16)
    return (y.contiguous() if kw.get("out_planar") else y.permute(1, 2, 3, 0).contiguous()), pre


def conv3d_causal_cases():
    from easyanimate_b200.vae_ops import pack_conv_weight  # pure torch: no kernel
    out = []

    def conv_trial(label, T, H, W, Cin, Cout, seed, cin_real=None, cout_pad=0, **flags):
        cin_real = cin_real or Cin
        amp_x, amp_w = (63, 31) if 27 * cin_real <= 432 else ((15, 7) if 27 * cin_real <= 3456 else (9, 7))
        _budget(27 * cin_real, amp_x, amp_w, extra=64 + 256 * 4)
        x = _ints((T, H, W, Cin), amp_x, -3, seed)
        if cin_real < Cin:
            x[..., cin_real:] = 0  # conv_in: 16 latent channels zero-padded to 64
        w = pack_conv_weight(_ints((Cout, cin_real, 3, 3, 3), amp_w, -6, seed + 1), cin_pad=Cin, cout_pad=cout_pad)
        b = _ints((Cout,), 64, -9, seed + 2)
        rows = flags.get("out_rows") or (H // 2 if flags.get("stride_hw") == 2 else H)
        res = _ints((T, rows, W, Cout), 256, -7, seed + 3) if flags.pop("with_residual", False) else None

        def make(device):
            dv = _d(device)
            kw = dict(flags)
            if res is not None:
                kw["residual"] = dv(res)
            return {"args": (dv(x), dv(w), dv(b), Cout), "kw": kw}
        out.append(Trial(f"conv3d_causal {label} T={T} H={H} W={W} Cin={Cin} Cout={Cout}", "linear", make,
                         exact64=_conv64))

    conv_trial("plain", 2, 9, 7, 128, 256, 1)  # ragged: one partial 128-pixel tile per frame
    conv_trial("persistent tile loop", 3, 400, 250, 64, 128, 2)
    conv_trial("Cin=512 residual", 2, 8, 12, 512, 128, 3, with_residual=True)
    conv_trial("residual dup_frames", 3, 10, 20, 64, 128, 4, with_residual=True, dup_frames=True)
    conv_trial("planar cout_pad", 3, 16, 24, 128, 3, 5, cout_pad=32, out_planar=True)
    conv_trial("cin_pad 16->64", 3, 6, 10, 64, 64, 6, cin_real=16)
    conv_trial("stride_t=2", 5, 12, 16, 64, 64, 7, stride_t=2)
    conv_trial("stride_hw=2", 3, 14, 18, 64, 128, 8, stride_hw=2)
    conv_trial("stride_t=2 stride_hw=2", 4, 10, 12, 128, 64, 9, stride_t=2, stride_hw=2)
    conv_trial("row window residual dup_frames", 3, 23, 40, 64, 128, 10, out_row0=4, out_rows=13, with_residual=True,
               dup_frames=True)
    conv_trial("row window planar", 2, 11, 24, 128, 3, 11, cout_pad=32, out_planar=True, out_row0=1, out_rows=9)
    return out


def _prep_exact64(env):
    z, w, b, cpad, in_scale = env["args"]
    Cc = z.shape[0]
    y = torch.einsum("oc,cthw->thwo", w.double().reshape(Cc, Cc), z.double()) + b.double()
    out = torch.zeros(y.shape[:3] + (cpad,), dtype=bf16)
    out[..., :Cc] = y.to(bf16)
    return out, y


def _prep_bound(env, want):
    z, w, b, cpad, in_scale = env["args"]
    Cc = z.shape[0]
    zs = _r(z.float() * torch.tensor(in_scale, dtype=torch.float32))
    mag = torch.einsum("oc,cthw->thwo", w.float().reshape(Cc, Cc).abs(), zs.abs()) + b.float().abs()
    err = torch.zeros(want.shape)
    err[..., :Cc] = 2.0 ** -19 * mag
    return err + _bf16_ulp(want) * (want != 0)


def prepare_latents_cases():
    Cc, T, H, W = 16, 3, 6, 10
    _budget(Cc, 255, 255, extra=256 * 4)
    z, w, b = _ints((Cc, T, H, W), 255, -6, 1), _ints((Cc, Cc, 1, 1, 1), 255, -8, 2), _ints((Cc,), 256, -12, 3)
    zr, wr, br = _randn((Cc, T, H, W), 1.0, 4), _randn((Cc, Cc, 1, 1, 1), 0.25, 5), _randn((Cc,), 0.1, 6)

    def make(device, z=z, w=w, b=b, in_scale=1.0):
        dv = _d(device)
        return {"args": (dv(z), dv(w), dv(b), 64, in_scale)}
    return [Trial("prepare_latents in_scale=1", "linear", make, exact64=_prep_exact64),
            Trial("prepare_latents in_scale=1/0.7125", "rounded",
                  lambda device: make(device, zr, wr, br, 1 / 0.7125), bound=_prep_bound)]


def _gn_bound(env, want, silu, x, gamma, beta, groups, mean, rstd):
    """One ulp of y = bf16(a x + b) plus the fp32 error of the affine form, then through SiLU and one more ulp."""
    T, H, W, C = x.shape
    cpg = C // groups
    a = (rstd.float().repeat_interleave(cpg, dim=1) * gamma.float())[:, None, None, :]
    m = mean.float().repeat_interleave(cpg, dim=1)[:, None, None, :]
    bb = beta.float() - a * m
    y = _r(x.float() * a + bb)
    err = _bf16_ulp(y) + 2.0 ** -21 * ((x.float() * a).abs() + bb.abs())
    if silu:
        err = 1.1 * err + 2.0 ** -19 * want.float().abs() + _bf16_ulp(want)
    return err


def _gn_stats(x, groups, eps):
    T, H, W, C = x.shape
    xg = x.double().view(T, H * W, groups, C // groups)
    mean = xg.mean(dim=(1, 3))
    var = (xg * xg).mean(dim=(1, 3)) - mean * mean
    return mean, 1.0 / torch.sqrt(var.clamp_min(0) + eps)


def groupnorm_cases():
    out = []
    for C, silu, H, W, offset in ((64, True, 40, 37, 0.5), (128, True, 12, 20, 0.5), (256, False, 33, 35, 50.0),
                                  (512, True, 9, 11, 0.5), (128, False, 36, 31, 50.0)):
        x = _randn((3, H, W, C), 2.0 if offset < 1 else 1.0, C + H, offset=offset)
        g, b = 1 + _randn((C,), 0.1, C + 1), _randn((C,), 0.1, C + 2)

        def make(device, x=x, g=g, b=b, silu=silu):
            dv = _d(device)
            return {"args": (dv(x), dv(g), dv(b), 32, 1e-6, silu)}

        def bound(env, want, silu=silu):
            x, g, b = env["args"][:3]
            mean, rstd = _gn_stats(x, 32, 1e-6)
            return _gn_bound(env, want, silu, x, g, b, 32, mean, rstd)
        out.append(Trial(f"groupnorm C={C} H={H} W={W} mean={offset} silu={silu}", "rounded", make, bound=bound))
    return out


def groupnorm_sums_cases():
    out = []
    for C, H, W, offset in ((128, 21, 37, 0.5), (512, 9, 11, 50.0), (64, 40, 37, 0.0)):
        x = _randn((3, H, W, C), 2.0, C, offset=offset)

        def make(device, x=x):
            return {"args": (_d(device)(x), 32)}

        def bound(env, want):
            # 1e-6 of the sums of |x| and of x^2: fp32 partial sums per thread, fp64 from there on
            x = env["args"][0]
            T, H, W, C = x.shape
            xa = x.double().abs().view(T, H * W, 32, C // 32)
            return torch.stack([xa.sum(dim=(1, 3)), (xa * xa).sum(dim=(1, 3))], dim=-1) * 1e-6
        out.append(Trial(f"groupnorm_sums C={C} H={H} W={W}", "rounded", make, bound=bound, min_exact=None))
    return out


def groupnorm_from_sums_cases():
    out = []
    T, H, W, C, G = 3, 21, 16, 128, 32
    x = _randn((T, H, W, C), 2.0, 1, offset=0.5)
    g, b = 1 + _randn((C,), 0.1, 2), _randn((C,), 0.1, 3)
    count = float(H * W * (C // G))
    for parts in ((0, H), (0, 9, 12, H)):
        lo, hi = parts[0], parts[1]
        sums = torch.stack([cpu_ops.groupnorm_sums(x[:, p0:p1].contiguous(), G) for p0, p1 in zip(parts[:-1], parts[1:])])
        xs = x[:, lo:hi].contiguous()

        def make(device, xs=xs, sums=sums):
            dv = _d(device)
            return {"args": (dv(xs), dv(sums), count, dv(g), dv(b), G, 1e-6, True)}

        def bound(env, want):
            xs, sums = env["args"][:2]
            tot = sums.sum(0)
            mean = tot[..., 0] / count
            rstd = 1.0 / torch.sqrt((tot[..., 1] / count - mean * mean).clamp_min(0) + 1e-6)
            return _gn_bound(env, want, True, xs, g, b, G, mean, rstd)
        out.append(Trial(f"groupnorm_from_sums parts={len(parts) - 1}", "rounded", make, bound=bound))
    return out


def upsample2x_cases():
    x = _randn((1, 5, 7, 64), 1.0, 1)  # T = 1, odd H and W
    y = _randn((3, 4, 9, 128), 1.0, 2)
    return [Trial("upsample2x T=1", "exact", lambda device: {"args": (_d(device)(x),)}),
            Trial("upsample2x T=3", "exact", lambda device: {"args": (_d(device)(y),)})]


def spatial_attention_cases():
    T, H, W, C = 2, 6, 10, 128
    n, res = _randn((T * H * W, C), 1.0, 1), _randn((T * H * W, C), 1.0, 2)
    wq, bq = _randn((3 * C, C), C ** -0.5, 3), _randn((3 * C,), 0.1, 4)
    wo, bo = _randn((C, C), C ** -0.5, 5), _randn((C,), 0.1, 6)
    p0, p1 = 2 * W, 5 * W
    res_q = res.view(T, H * W, C)[:, p0:p1].reshape(-1, C).contiguous()
    tol = lambda env, want: 3e-2 + 3e-2 * want.float().abs()  # noqa: E731

    def make(device, q_rows=None):
        dv = _d(device)
        return {"args": (dv(n), dv(wq), dv(bq), dv(wo), dv(bo), dv(res if q_rows is None else res_q), T, C ** -0.5),
                "kw": {} if q_rows is None else {"q_rows": q_rows}}
    return [Trial("spatial_attention", "contract", make, bound=tol),
            Trial("spatial_attention q_rows", "contract", lambda device: make(device, (p0, p1)), bound=tol)]


def tile_blend_cases():
    out = []
    C, T = 3, 2
    for axis, extent, a_hw, b_hw in ((0, 6, (10, 16), (12, 16)), (0, 40, (9, 16), (12, 16)),  # extent clamped to 9
                                     (1, 6, (12, 10), (12, 14)), (1, 40, (12, 13), (12, 11))):  # tiles of different widths
        a = _randn((1, C, T) + a_hw, 1.0, axis * 10 + extent)
        b = _randn((1, C, T) + b_hw, 1.0, axis * 10 + extent + 1)

        def make(device, a=a, b=b, axis=axis, extent=extent):
            dv = _d(device)
            return {"args": (dv(a), dv(b), extent, axis)}
        out.append(Trial(f"tile_blend axis={axis} extent={extent} a={a_hw} b={b_hw}", "exact", make,
                         result=lambda ret, env: env["args"][1]))
    big = _randn((1, 3, 2, 20, 30), 1.0, 99)

    def make_view(device):
        dv = _d(device)
        return {"args": (dv(big)[..., 2:14, 3:20], dv(big)[..., 5:17, 1:12], 8, 1)}  # crop views of decoded tiles
    out.append(Trial("tile_blend crop views", "exact", make_view, result=lambda ret, env: env["args"][1]._base))
    return out


def copy2d_cases():
    src = _randn((1, 3, 2, 20, 30), 1.0, 1)
    dst = _randn((1, 3, 2, 25, 40), 1.0, 2)

    def make(device):
        dv = _d(device)
        return {"args": (dv(src)[..., 3:17, 4:25], dv(dst), 11, 17, 6, 9)}  # a strided crop into the middle of dst
    return [Trial("copy2d strided", "exact", make, result=lambda ret, env: env["args"][1])]


def corner_blend_cases():
    out = []
    C, T = 3, 2
    for Hc, Wc in ((12, 20), (20, 12), (1, 17), (17, 1), (64, 64)):
        src, dst = _randn((1, C, T, Hc, Wc), 1.0, Hc), _randn((1, C, T, Hc + 5, Wc + 9), 1.0, Wc)

        def make(device, src=src, dst=dst):
            dv = _d(device)
            return {"args": (dv(src), dv(dst))}
        out.append(Trial(f"corner_blend {Hc}x{Wc}", "exact", make, result=lambda ret, env: env["args"][1]))

    # every N x N corner from 2 to 512: each weight of torch.linspace(0, 1, N) sits on the diagonal, where it is min(wx, wy)
    sizes = range(2, 513)
    srcs = [_randn((1, 1, 1, n, n), 1.0, n) for n in sizes]
    dsts = [_randn((1, 1, 1, n + 2, n + 3), 1.0, n + 1000) for n in sizes]

    def sweep(fn, env):
        for s, d in zip(env["srcs"], env["dsts"]):
            fn(s, d)

    out.append(Trial("corner_blend every N from 2 to 512", "exact",
                     lambda device: {"srcs": [_d(device)(s) for s in srcs], "dsts": [_d(device)(d) for d in dsts]},
                     call=sweep, result=lambda ret, env: tuple(env["dsts"])))
    return out


def frames_out_cases():
    out = []
    # every bf16 value in [-1.1, 1.1] (so every k/255 boundary of the uint8 output has its neighbours on both sides),
    # exactly +-1, +-0, and (float32 only) NaN and +-inf; n % 8 != 0
    bits = torch.arange(0, 1 << 16, dtype=torch.int32).to(torch.int16).view(bf16)
    vals = bits[(bits.float().abs() <= 1.1)]
    special = torch.tensor([1.0, -1.0, 0.0, -0.0, float("inf"), float("-inf"), float("nan")], dtype=bf16)
    f32_in = torch.cat([vals, special, vals[:5]])
    u8_in = torch.cat([vals, special[:6], vals[:4]])
    assert f32_in.numel() % 8 != 0 and u8_in.numel() % 8 != 0
    for dtype, v in ((torch.float32, f32_in), (torch.uint8, u8_in)):
        for pinned in (False, True):
            def make(device, v=v, dtype=dtype, pinned=pinned):
                o = torch.full((v.numel(),), 7, dtype=dtype)
                if device == "cuda":
                    o = o.pin_memory() if pinned else o.to(device)
                return {"args": (_d(device)(v), o)}
            out.append(Trial(f"frames_out {dtype} pinned={pinned}", "exact", make, result=lambda ret, env: env["args"][1]))
    return out


def frames_out_blend_cases():
    out = []
    B, C, F_, H, W, total, t0 = 1, 3, 5, 6, 10, 12, 4
    video = _randn((B, C, F_, H, W), 0.7, 1)
    whole = torch.rand((B, C, total, H, W), generator=_gen(2))
    for overlap in (0, 1, F_):
        for pinned in (False, True):
            def make(device, overlap=overlap, pinned=pinned):
                w = whole.clone()
                if device == "cuda":
                    w = w.pin_memory() if pinned else w.to(device)
                return {"args": (_d(device)(video), w[:, :, t0:t0 + F_], overlap), "whole": w}
            out.append(Trial(f"frames_out_blend overlap={overlap} pinned={pinned}", "exact", make,
                             result=lambda ret, env: env["whole"]))
    return out


CASE_BUILDERS = {
    "gemm": gemm_cases, "skinny_linear": skinny_linear_cases, "layernorm_modulate": layernorm_modulate_cases,
    "rmsnorm": rmsnorm_cases, "timestep_embedding": timestep_embedding_cases, "patchify": patchify_cases,
    "unpatchify": unpatchify_cases, "qkv_gemm_ln_rope": qkv_gemm_ln_rope_cases, "attention": attention_cases,
    "ew_add": ew_add_cases, "l1_sums": l1_sums_cases, "cfg_euler_step": cfg_euler_step_cases,
    "dequant_e4m3": dequant_e4m3_cases, "conv3d_causal": conv3d_causal_cases, "prepare_latents": prepare_latents_cases,
    "groupnorm": groupnorm_cases, "groupnorm_sums": groupnorm_sums_cases, "groupnorm_from_sums": groupnorm_from_sums_cases,
    "upsample2x": upsample2x_cases, "spatial_attention": spatial_attention_cases, "tile_blend": tile_blend_cases,
    "copy2d": copy2d_cases, "corner_blend": corner_blend_cases, "frames_out": frames_out_cases,
    "frames_out_blend": frames_out_blend_cases,
}
CASES = sorted(CASE_BUILDERS)


def entry_point(name):
    from easyanimate_b200 import ops, vae_ops
    return getattr(ops if name in cpu_ops.OPS else vae_ops, name)


# ---------------------------------------------------------------------------------------------------------------------
# comparison
# ---------------------------------------------------------------------------------------------------------------------
def _same(got, want):
    """torch.equal, NaN outputs compared by position only (NaN payload and sign are not part of the contract)."""
    if got.dtype != want.dtype or got.shape != want.shape:
        return False
    if got.is_floating_point():
        nan = torch.isnan(got.float())
        if not torch.equal(nan, torch.isnan(want.float())):
            return False
        return torch.equal(got[~nan], want[~nan])
    return torch.equal(got, want)


def _within(got, want, bound, label):
    if isinstance(got, float):
        assert abs(got - want) <= bound, f"{label}: {got!r} vs {want!r}, bound {bound:.3g}"
        return
    assert got.shape == want.shape and got.dtype == want.dtype, (label, got.shape, want.shape, got.dtype, want.dtype)
    err = (got.double() - want.double()).abs()
    bad = ~(err <= torch.as_tensor(bound).double())  # NaN errors are bad too
    assert not bad.any(), (f"{label}: {int(bad.sum())} of {bad.numel()} outputs beyond the bound, worst "
                           f"{float((err - torch.as_tensor(bound).double())[bad].max()):.4g} over it")


def compare(trial, got, want):
    """Asserts `got` (the kernel's outputs) against `want` (the stand-in's) by the trial's criterion; returns the lowest
    bit-exact fraction of a "rounded" trial (None for the others)."""
    g, w = _outs(got), _outs(want)
    assert len(g) == len(w), trial.label
    if trial.kind in ("exact", "linear"):
        for i, (a, b) in enumerate(zip(g, w)):
            if not _same(a, b):
                diff = int((a.float() != b.float()).sum()) if a.shape == b.shape else "shape"
                raise AssertionError(f"{trial.label}: output {i} differs from the stand-in ({diff} of {b.numel()} elements)")
        return None
    bounds = _outs(trial.bound(trial.make("cpu"), want))
    frac = None
    for a, b, bd in zip(g, w, bounds):
        _within(a, b, bd, trial.label)
        if trial.kind == "rounded" and trial.min_exact is not None:
            f = bit_exact_fraction(a, b)
            frac = f if frac is None else min(frac, f)
            assert f >= trial.min_exact, f"{trial.label}: only {f:.4%} of the outputs equal the stand-in bit for bit"
    return frac


def trials(name):
    return CASE_BUILDERS[name]()


@pytest.mark.parametrize("name", CASES)
def test_kernel_equals_stand_in(name):
    kernel, stand_in = entry_point(name), getattr(cpu_ops, name)
    lowest = None
    for t in trials(name):
        got, want = run(t, kernel, "cuda"), run(t, stand_in, "cpu")
        f = compare(t, got, want)
        if f is not None:
            print(f"BIT_EXACT {t.label}: {f:.5f}")
            lowest = f if lowest is None else min(lowest, f)
    if lowest is not None:
        print(f"BIT_EXACT_LOWEST {name}: {lowest:.5f}")

