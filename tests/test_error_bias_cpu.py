"""CPU: the direction statistics of tests/error_stats.py catch what the element-wise allowances miss.  Each wrong
variant below is a small wrapper around the emulated op layer (tests/ops_emulator.py) with a systematic error as large
as the old verdicts let through: every old verdict passes it (the statistics switched off), and with the statistics on
at least one record fails, printed with -s as "old verdicts: pass; new: <statistic> = x > bound y".  The correct
emulation passes the same cases with the statistics on."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import attention_variants as av
from tests import error_stats as es
from tests import kernel_checks as kc
from tests import launch_checks as lc
from tests import ops_emulator as emu

BF16 = torch.bfloat16


@pytest.fixture(scope="module", autouse=True)
def _cpu_device():
    saved = kc.DEVICE
    kc.DEVICE = "cpu"
    torch.set_grad_enabled(False)
    yield
    kc.DEVICE = saved
    torch.set_grad_enabled(True)


_trunc = av.trunc_bf16


def _into(y, out):
    if out is None:
        return y
    out.copy_(y)
    return out


def _g(seed):
    return torch.Generator().manual_seed(seed)


# ---- cases: one verdict each, on whatever ops.X currently is --------------------------------------------------------
def _case_gemm():
    """bias epilogue, positive-mean operands so that a bias toward zero does not cancel across signs"""
    from ctrl_adapter_b200 import ops
    m, k, n = 512, 64, 256
    x = (torch.randn(m, k, generator=_g(1)) * 0.5 + 1.0).to(BF16)
    w = ((torch.randn(n, k, generator=_g(2)) * 0.5 + 1.0) / k).to(BF16)
    b = ops.bias_f32((torch.randn(n, generator=_g(3)) * 0.1).to(BF16))
    call = dict(x=x, w=w, bias=b, act=0, rowvec=None, rows_per_vec=0, residual=None, blend_src=None, blend_alpha=None,
                out_scale=1.0, out=None, out_fp32=False, bn=0)
    return kc.linear_verdict("gemm bias", call, ops.linear(**call), lambda **ch: ops.linear(**{**call, **ch}))


def _case_layernorm():
    from ctrl_adapter_b200 import ops
    x = (torch.randn(2048, 320, generator=_g(4)) * 1.5 + 0.2).to(BF16)
    gamma = torch.randn(320, generator=_g(5)) * 0.2 + 1.0
    beta = torch.randn(320, generator=_g(6)) * 0.2
    a = dict(x=x, gamma=gamma, beta=beta, eps=1e-5, add_rowvec=None, rows_per_vec=0, return_sum=False)
    return kc.layernorm_verdict("layernorm", a, ops.layer_norm(x, gamma, beta, 1e-5))


def _case_attention(spread):
    """b 2, h 2, L 256, d 64; `spread`: the std of the logits (scale included), in natural-log units"""
    from ctrl_adapter_b200 import ops
    b, h, lq, lk, d = 2, 2, 256, 256, 64
    q = (torch.randn(b, lq, h, d, generator=_g(7)) * spread).to(BF16)
    k = torch.randn(b, lk, h, d, generator=_g(8)).to(BF16)
    v = (torch.randn(b, lk, h, d, generator=_g(9)) + 0.5).to(BF16)
    out = ops.attention(q.reshape(b, lq, h * d), k.reshape(b, lk, h * d), v.reshape(b, lk, h * d), h, d, d ** -0.5)
    return kc._attn_verdict(f"attention spread {spread}", q, k, v, torch.arange(b), d ** -0.5,
                            out.reshape(b, lq, h, d))


def _case_groupnorm():
    return kc.check_groupnorm_offset(1, 32, 32, 128)


def _case_cfg_euler():
    """positive-mean guidance outputs and latents, a step that moves the latents by half"""
    from ctrl_adapter_b200 import ops
    shape = (4, 4, 128, 128)  # 64 blocks of 4096 elements
    eu = (torch.randn(*shape, generator=_g(10)) * 0.3 + 1.0).to(BF16)
    et = (torch.randn(*shape, generator=_g(11)) * 0.3 + 1.0).to(BF16)
    lat = (torch.randn(*shape, generator=_g(12)) * 0.5 + 4.0).to(BF16).float()
    row = torch.tensor([500.0, 3.2, 1.6, math.sqrt(1.6 ** 2 + 1.0)])
    call = dict(eps_uncond=eu, eps_text=et, latents=lat, guidance=1.5, step_row=row, latents_out=None,
                model_in_next=None, round_latents_bf16=True)
    return kc.cfg_euler_verdict("cfg_euler bf16 latents", call, ops.cfg_euler(**call), None)


def _case_silu():
    from ctrl_adapter_b200 import ops
    x = (torch.randn(64, 4096, generator=_g(13)) * 2.0).to(BF16)
    recs, _ = lc._v_silu({"x": x}, ops.silu(x), None)
    return recs


# ---- wrong variants ---------------------------------------------------------------------------------------------------
def _linear_trunc(x, w, bias=None, *, out=None, out_fp32=False, act=0, **kw):
    """bf16 output of the plain bias epilogue rounded toward zero"""
    if out_fp32 or act or any(kw.get(k) is not None for k in ("residual", "rowvec", "blend_src")):
        return emu.linear(x, w, bias, out=out, out_fp32=out_fp32, act=act, **kw)
    return _into(_trunc(emu.linear(x, w, bias, out_fp32=True, act=act, **kw)), out)


def _layernorm_trunc(x, gamma, beta, eps=1e-5, **kw):
    return _trunc(F.layer_norm(x.float(), (x.shape[-1],), gamma.float(), beta.float(), eps))


def _attention_scale(factor):
    def fn(q, k, v, heads, head_dim_pad, scale, out=None, kv_batch_div=1):
        return emu.attention(q, k, v, heads, head_dim_pad, scale * factor, out=out, kv_batch_div=kv_batch_div)
    return fn


def _groupnorm_gain(x, gamma, beta, eps, *, groups=32, silu=False, up2x=False, x2=None, imgs_per_sample=1, out=None):
    """rstd off by +-2^-10 per group (alternating): a one-pass variance that lost ~2^-9 of itself to cancellation"""
    xin = x if x2 is None else torch.cat([x, x2], dim=3)
    n, h, w, c = xin.shape
    t = xin.float().reshape(n // imgs_per_sample, -1, groups, c // groups)
    mean, var = t.mean(dim=(1, 3), keepdim=True), t.var(dim=(1, 3), unbiased=False, keepdim=True)
    gain = 1.0 + 2.0 ** -10 * (1.0 - 2.0 * (torch.arange(groups) % 2)).reshape(1, 1, groups, 1)
    y = ((t - mean) * torch.rsqrt(var + eps) * gain).reshape(n, h, w, c) * gamma.float() + beta.float()
    y = F.silu(y) if silu else y
    y = y.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2) if up2x else y
    return _into(y.to(BF16), out)


def _cfg_euler_trunc(eps_uncond, eps_text, latents, guidance, step_row, latents_out=None, model_in_next=None,
                     round_latents_bf16=True):
    """sigma * eps rounded toward zero"""
    _, sigma, sigma_next, next_div = (float(v) for v in step_row)
    u, c = eps_uncond.float(), eps_text.float()
    eps = emu._r(u + emu._r(guidance * emu._r(c - u)))
    x = latents.float()
    x0 = x - _trunc(emu._r(torch.tensor(sigma)) * eps).float()
    xn = x + (x - x0) / sigma * (sigma_next - sigma)
    xn = emu._r(xn) if round_latents_bf16 else xn
    if model_in_next is not None:
        model_in_next.copy_((xn / emu._r(torch.tensor(next_div))).to(BF16))
    return _into(xn, latents_out) if latents_out is not None else xn.to(latents.dtype)


def _silu_biased(x):
    """SiLU through a sigmoid 2^-9 too large"""
    return (x.float() * torch.sigmoid(x.float()) * (1.0 + 2.0 ** -9)).to(BF16)


# variant -> (case, {op: wrong function})
VARIANTS = {
    "GEMM epilogue: final rounding toward zero": (_case_gemm, {"linear": _linear_trunc}),
    "LayerNorm: output rounded toward zero": (_case_layernorm, {"layer_norm": _layernorm_trunc}),
    "attention: P truncated to bf16 before P.V": (lambda: _case_attention(1.0), {"attention": lambda *a, **k:
                                                                                  av.flash(av.p_trunc, *a, **k)}),
    "attention: softmax scale 0.3 % high": (lambda: _case_attention(0.5), {"attention": _attention_scale(1.003)}),
    "attention: exp2 from a degree-2 polynomial": (lambda: _case_attention(1.0), {"attention": lambda *a, **k:
                                                                                   av.flash(av.poly2_exp2(), *a, **k)}),
    "GroupNorm: per-group gain 1 +- 2^-10": (_case_groupnorm, {"group_norm": _groupnorm_gain}),
    "cfg_euler: sigma * eps rounded toward zero": (_case_cfg_euler, {"cfg_euler": _cfg_euler_trunc}),
    "SiLU: sigmoid 2^-9 too large": (_case_silu, {"silu": _silu_biased}),
}
CASES = sorted({id(c): c for c, _ in VARIANTS.values()}.values(), key=lambda c: c.__name__)


def _records(case, wrong=None):
    kc.RESULTS.clear()
    with emu.patched_ops() as ops:
        for name, fn in (wrong or {}).items():
            setattr(ops, name, fn)
        ret = case()
    recs = list(kc.RESULTS)
    for r in ret if isinstance(ret, list) else [ret]:  # _v_silu's records are not collected by kc.RESULTS alone
        if not any(r is x for x in recs):
            recs.append(r)
    return recs


def _no_direction(*args, **kw):
    return {"ok": True, "why": ""}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_direction_catches_what_old_verdicts_miss(variant, monkeypatch):
    case, wrong = VARIANTS[variant]
    with monkeypatch.context() as mp:
        mp.setattr(es, "direction", _no_direction)
        old = _records(case, wrong)
    old_bad = [f"{r['check']}: {r.get('why') or 'out of tolerance'}" for r in old if not r["ok"]]
    assert not old_bad, f"{variant}: an old verdict already fails it: {old_bad}"
    new = _records(case, wrong)
    why = [r["why"] for r in new if not r["ok"]]
    print(f"\n{variant}: old verdicts: pass; new: {' | '.join(why) or 'NOTHING'}")
    assert why, f"no direction statistic notices: {variant}"
    assert all(r["n_bad"] == 0 for r in new if "n_bad" in r)


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.__name__)
def test_correct_emulation_passes_direction(case):
    recs = _records(case)
    print("\n" + "\n".join(f"{r['check']}: bias {r.get('bias_ulp', 0):+.4f} / {r.get('bias_bound', 0):.3g} "
                           f"toward-zero {r.get('bias0_ulp', 0):+.4f}, gain {r.get('gain', 0):+.2e} / "
                           f"{r.get('gain_bound', 0):.2e}" + (f", rms {r['rms_ratio']:.2f}x eager" if "rms_ratio" in r
                                                              else "") for r in recs if "bias_ulp" in r))
    bad = [f"{r['check']}: {r.get('why')}" for r in recs if not r["ok"]]
    assert not bad, bad
    assert any("bias_ulp" in r for r in recs)


def test_statistics_on_synthetic_errors():
    """the statistics themselves: unbiased +-1 ulp flips pass; a quarter ulp toward zero and a 2^-10 gain fail, each
    naming its statistic; fewer than MIN_UNITS units leave the bound loose"""
    g = _g(20)
    ref = (torch.rand(256, 512, generator=g, dtype=torch.float64) + 0.5) * torch.sign(torch.randn(256, 512, generator=g))
    ulp = es.bf16_ulp(ref)
    flips = (torch.randint(0, 9, ref.shape, generator=g) - 4).clamp(-1, 1).to(torch.float64)
    assert es.direction(ref + flips * ulp, ref, 1e-3, units=(0,))["ok"]
    toward0 = torch.rand(ref.shape, generator=g, dtype=torch.float64) < 0.25
    rec = es.direction(ref - torch.sign(ref) * ulp * toward0, ref, 1e-3, units=(0,))
    assert not rec["ok"] and "toward zero" in rec["why"], rec
    rec = es.direction(ref * (1 + 2.0 ** -10), ref, 1e-3, units=(0,))
    assert not rec["ok"] and "gain" in rec["why"], rec
    assert es.direction(ref[:8] - ulp[:8] * 0.3, ref[:8], 1e-3, units=(0,))["bias_bound"] == math.inf


def test_attention_statistics_use_the_rounded_reference():
    """nearly one-hot temporal-attention rows over 4 frames: against the unrounded float64 output, correct round-to-nearest
    has a gain about the mean of V (the output snaps back to the dominant bf16 V value); the verdict's statistics use the
    reference rounded to bf16, against which the correct emulation has none"""
    clips, frames, hw, heads = 2, 4, 144, 20
    inner = heads * 64
    qkv = torch.randn(clips * frames * hw, 3 * inner, generator=_g(21))
    qkv[:, :inner] *= 6.0
    qkv = qkv.to(BF16)
    q, k, v = qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:]
    out = emu.temporal_attention(q, k, v, clips, frames, hw, heads, 0.125)
    rec = kc.temporal_attention_verdict("temporal attention 4 frames, one-hot rows", q, k, v, clips, frames, hw, heads,
                                        0.125, out)

    def seq(t):
        return t.double().reshape(clips, frames, hw, heads, 64).permute(0, 2, 3, 1, 4)
    exact = (torch.softmax(seq(q) @ seq(k).transpose(-1, -2) * 0.125, dim=-1) @ seq(v)).permute(0, 3, 1, 2, 4)
    vmean = seq(v).mean(dim=3, keepdim=True).permute(0, 3, 1, 2, 4)
    raw = es.direction(out.reshape(exact.shape), exact, 6e-3, units=(0, 2, 3), center=vmean)
    print(f"\ngain against the unrounded output {raw['gain']:+.2e}, against the rounded one {rec['gain']:+.2e}")
    assert rec["ok"] and abs(rec["gain"]) < 1e-6
    assert raw["gain"] > 5e-5
