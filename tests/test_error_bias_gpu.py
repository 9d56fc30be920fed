"""pytest -m gpu -s: the direction statistics of tests/error_stats.py on large samples of every kernel instantiation, with
inputs that expose direction: positive-mean operands (a bias toward zero or a floor cannot cancel across signs), logits
spread over several log2 units (the softmax temperature matters), GroupNorm groups whose mean is 10 and 80 times their
std.  Every case has at least 2^20 outputs and goes through the same per-launch verifier as the launch census
(launch_checks.VERIFIERS), so its float64 reference and element-wise verdict are the census's; -s prints one row per
record with each statistic, its bound and the eager yardstick where the verdict has one.

Then the power checks: the real output of one large GEMM, one attention and one GroupNorm, moved by a systematic error
the element-wise allowance accepts (one ulp toward zero on a random half of the elements; one group scaled by
1 + 2^-10 about beta), must fail its verdict with `why` naming the statistic."""
import inspect
import math

import pytest
import torch

from tests import attention_variants as av
from tests import error_stats as es
from tests import kernel_checks as kc
from tests import launch_checks as lc
from tests import ops_emulator as emu

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device is visible (there is no CPU fallback to test)")
    from ctrl_adapter_b200 import _lib
    _lib.check(_lib.load().ca_device_ok(), "ca_device_ok")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_grad_enabled(False)
    yield
    torch.set_grad_enabled(True)


def _ops():
    from ctrl_adapter_b200 import ops
    return ops


def _rand(*shape, mean=0.0, std=1.0, seed=0, dtype=BF16):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * std + mean).to(dtype)


def _args(op, **kw):
    """every argument of ops.<op>, defaults filled in"""
    a = inspect.signature(getattr(_ops(), op)).bind(**kw)
    a.apply_defaults()
    return dict(a.arguments)


def _verify(op, **kw):
    """ops.<op>(**kw) through the census verifier of the op -> records"""
    fn = getattr(_ops(), op)
    a = _args(op, **kw)
    out = fn(**a)
    torch.cuda.synchronize()
    recs, _ = lc.VERIFIERS[op](a, out, lambda **ch: fn(**{**a, **ch}))
    return recs


def _line(r):
    s = (f"{'ok  ' if r['ok'] else 'FAIL'} {r['check'][:58]:<58} n={r.get('n', 0):>8} units={r.get('bias_units', 0):>6} "
         f"bias {r['bias_ulp']:+.4f}/{r['bias_bound']:.3f} to0 {r['bias0_ulp']:+.4f}/{r['bias0_bound']:.3f} "
         f"gain {r['gain']:+.2e}/{r['gain_bound']:.1e} max|gain| {r['gain_max']:.1e}")
    if "gain_eager" in r:
        s += f" eager gain {r['gain_eager']:+.1e}"
    if "rms_ratio" in r:
        s += f" rms {r['rms']:.2e} = {r['rms_ratio']:.3f}x eager"
    return s + ("" if r["ok"] else f"  WHY {r.get('why')}")


def _check(recs):
    recs = [r for r in recs if "bias_ulp" in r]
    assert recs, "no record with direction statistics"
    print("\n" + "\n".join(_line(r) for r in recs))
    bad = [f"{r['check']}: {r.get('why') or 'out of tolerance'}" for r in recs if not r["ok"]]
    assert not bad, bad


# ---- GEMM: every BN x every bf16 epilogue x both drains, and fp32 output ------------------------------------------------
M, K, N = 1024, 320, 1280


def _gemm_call(kind, bn, seed=0):
    ops = _ops()
    parts = kind.split("_")
    geglu = kind == "geglu"
    x = _rand(M, K, mean=0.5, seed=seed + 1)
    w = _rand(2 * N if geglu else N, K, mean=0.3, std=1.0, seed=seed + 2) * K ** -0.5
    w = w.to(BF16)
    b = _rand(w.shape[0], mean=0.2, std=0.2, seed=seed + 3) if ("bias" in parts or geglu) else None
    if geglu:
        w, b = ops.pack_geglu_weight(w, b, 256)
    return dict(x=x, w=w, bias=ops.bias_f32(b), act=ops.ACT_GEGLU if geglu else ops.ACT_SILU if "silu" in parts else 0,
                out_scale=0.7 if "scale" in parts else 1.0,
                rowvec=_rand(M // 256, N, mean=0.5, seed=seed + 4) if "rowvec" in parts else None,
                rows_per_vec=256 if "rowvec" in parts else 0,
                residual=_rand(M, N, mean=1.0, seed=seed + 5) if "res" in parts else None,
                blend_src=_rand(M, N, mean=1.0, seed=seed + 6) if "blend" in parts else None,
                blend_alpha=torch.sigmoid(torch.tensor([0.3], device=DEV)).to(BF16).float() if "blend" in parts else None,
                bn=bn)


def _slot(t):
    """the same values in columns [4, 4 + n) of a wider buffer: the 8-byte offset sends the storers down the element-wise
    drain"""
    if t is None:
        return None
    buf = torch.zeros(t.shape[0], t.shape[1] + 16, device=DEV, dtype=t.dtype)
    buf[:, 4:4 + t.shape[1]] = t
    return buf[:, 4:4 + t.shape[1]]


GEMM_CASES = [(bn, kind, drain) for bn in (64, 128, 160, 256) for kind in kc.EPILOGUES
              if kind != "geglu" or bn == 256 for drain in ("aligned", "elementwise")]


@pytest.mark.parametrize("bn,kind,drain", GEMM_CASES, ids=[f"bn{b}-{k}-{d}" for b, k, d in GEMM_CASES])
def test_gemm_epilogue(bn, kind, drain):
    call = _gemm_call(kind, bn)
    if drain == "elementwise":
        call = {**call, **{k: _slot(call[k]) for k in ("rowvec", "residual", "blend_src")},
                "out": _slot(torch.empty(M, N, device=DEV, dtype=BF16))}
    _check(_verify("linear", **call))


@pytest.mark.parametrize("bn", [64, 128, 160, 256])
def test_gemm_fp32_output(bn):
    _check(_verify("linear", **{**_gemm_call("bias", bn), "out_fp32": True}))


# ---- convolutions ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out_fp32", [False, True])
def test_conv3x3(out_fp32):
    ops = _ops()
    n, h, w, c = 4, 64, 64, 320
    wt = (_rand(c, c, 3, 3, mean=0.3, seed=12).float() * (9 * c) ** -0.5).to(BF16)
    kw = {} if out_fp32 else dict(rowvec=_rand(n, c, mean=0.5, seed=13), residual=_rand(n, h, w, c, mean=1.0, seed=14))
    _check(_verify("conv2d", x=_rand(n, h, w, c, mean=0.5, seed=11), w_packed=ops.pack_conv_weight(wt),
                   bias=ops.bias_f32(_rand(c, mean=0.2, std=0.2, seed=15)), out_fp32=out_fp32, **kw))


def test_temporal_conv():
    ops = _ops()
    b, f, h, w, c = 1, 16, 32, 32, 320
    wt = (_rand(c, c, 3, 1, 1, mean=0.3, seed=22).float() * (3 * c) ** -0.5).to(BF16)
    _check(_verify("temporal_conv", x=_rand(b * f, h, w, c, mean=0.5, seed=21), w_packed=ops.pack_conv_weight(wt),
                   bias=ops.bias_f32(_rand(c, mean=0.2, std=0.2, seed=23)), frames=f,
                   rowvec=_rand(b * f, c, mean=0.5, seed=24), residual=_rand(b * f, h, w, c, mean=1.0, seed=25)))


# ---- attention: attention_kernel<DQ, NWG> (1, 2) (1, 3) (2, 2) (3, 2), flat and peaked logits, one KV tile and many ---
ATTN = [  # (label, b, heads, lq, d, lk): b * heads * lq * d >= 2^20
    ("DQ1 NWG2 one-tile", 2, 8, 1024, 64, 77), ("DQ1 NWG2 multi-tile", 2, 8, 1024, 64, 1024),
    ("DQ1 NWG3", 1, 4, 4096, 64, 1024),
    ("DQ2 NWG2 one-tile", 2, 4, 1024, 128, 77), ("DQ2 NWG2 multi-tile", 2, 4, 1024, 128, 1024),
    ("DQ3 NWG2 one-tile", 2, 3, 1024, 192, 77), ("DQ3 NWG2 multi-tile", 2, 3, 1024, 192, 1024)]
SPREADS = {"flat": 1.0, "peaked": 2.0}  # std of the logits (scale included), natural-log units


def _attn_inputs(b, heads, lq, d, lk, spread, seed=30):
    q = _rand(b, lq, heads * d, std=spread, seed=seed + 1)
    k = _rand(b, lk, heads * d, seed=seed + 2)
    v = _rand(b, lk, heads * d, mean=0.5, seed=seed + 3)
    return q, k, v


@pytest.mark.parametrize("spread", list(SPREADS))
@pytest.mark.parametrize("case", ATTN, ids=[c[0] for c in ATTN])
def test_attention(case, spread):
    from tests.abi_domain import attention_nwg
    label, b, heads, lq, d, lk = case
    assert f"NWG{attention_nwg(d, lq, lk)}" in label
    q, k, v = _attn_inputs(b, heads, lq, d, lk, SPREADS[spread])
    _check(_verify("attention", q=q, k=k, v=v, heads=heads, head_dim_pad=d, scale=d ** -0.5))


@pytest.mark.parametrize("frames", [4, 16, 32])
def test_temporal_attention(frames):
    """frames 4: nearly one-hot rows (query std 6), where round-to-nearest alone has a gain about the mean of V against
    the unrounded reference (error_stats docstring)"""
    clips, hw, heads = 2, 512, 5
    q, k, v = (_rand(clips * frames * hw, heads * 64, mean=m, std=s, seed=40 + i)
               for i, (m, s) in enumerate(((0.0, 6.0 if frames == 4 else 3.0), (0.0, 1.0), (0.5, 1.0))))
    _check(_verify("temporal_attention", q=q, k=k, v=v, clips=clips, frames=frames, hw=hw, heads=heads, scale=0.125))


def test_temporal_attention_offset_values():
    """Regression: 14 frames, logits of std ~1 and V rows sharing an offset (mean 2, std 0.3), as video activations do.
    With P rounded to bf16 before P.V, nearly equal probabilities lost their differences and the softmax flattened:
    a gain of -5e-4 about the mean of V (emulated; -3e-4 to -1.2e-3 on the video census launches).  The kernel now
    multiplies V by P split into two bf16 terms (emulated gain 6e-7)."""
    clips, frames, hw, heads = 2, 14, 576, 10
    q, k, v = (_rand(clips * frames * hw, heads * 64, mean=m, std=s, seed=45 + i)
               for i, (m, s) in enumerate(((0.0, 1.0), (0.0, 1.0), (2.0, 0.3))))
    _check(_verify("temporal_attention", q=q, k=k, v=v, clips=clips, frames=frames, hw=hw, heads=heads, scale=0.125))


# ---- norms ------------------------------------------------------------------------------------------------------------
LN_WIDTHS = [64, 128, 192, 256, 320, 384, 512, 640, 768, 1024, 1280, 1536, 1792, 2048]  # every (NV, L)
LN_CASES = [(c, rv, 0.0) for c in LN_WIDTHS for rv in (0, 1)] + [(c, 0, 40.0) for c in (320, 640, 1280)]


@pytest.mark.parametrize("c,rv,offset", LN_CASES, ids=[f"c{c}-rv{rv}-off{o:g}" for c, rv, o in LN_CASES])
def test_layernorm(c, rv, offset):
    from tests.abi_domain import layernorm_variant
    rows = -(-(1 << 20) // c) // 4 * 4 + 4
    kw = dict(add_rowvec=_rand(4, c, seed=52), rows_per_vec=rows // 4, return_sum=True) if rv else {}
    print(f"\n{layernorm_variant(c, rv)}", end="")
    _check(_verify("layer_norm", x=_rand(rows, c, mean=offset + 0.2, std=1.5, seed=50), gamma=_rand(
        c, mean=1.0, std=0.2, seed=53, dtype=torch.float32), beta=_rand(c, std=0.2, seed=54, dtype=torch.float32),
        eps=1e-5, **kw))


GN_RATIOS = {0: (0.0, 1.0), 10: (10.0, 1.0), 80: (40.0, 0.5)}  # mean / std: (mean, std)
GN_CASES = [(silu, up, ratio) for silu in (False, True) for up in (False, True) for ratio in GN_RATIOS]


def _gn_call(silu, up, ratio, seed=60):
    mean, std = GN_RATIOS[ratio]
    n, h, w, c = 2, 64, 64, 320
    return dict(x=_rand(n, h, w, c, mean=mean, std=std, seed=seed + 1),
                gamma=_rand(c, mean=1.0, std=0.2, seed=seed + 2, dtype=torch.float32),
                beta=_rand(c, std=0.2, seed=seed + 3, dtype=torch.float32), eps=1e-6, silu=silu, up2x=up)


@pytest.mark.parametrize("silu,up,ratio", GN_CASES, ids=[f"silu{int(s)}-up{int(u)}-mean/std{r}" for s, u, r in GN_CASES])
def test_groupnorm(silu, up, ratio):
    _check(_verify("group_norm", **_gn_call(silu, up, ratio)))


# ---- scheduler updates ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bf16_latents", [True, False], ids=["bf16", "fp32"])
@pytest.mark.parametrize("op", ["cfg_euler", "cfg_euler_v", "cfg_ddim"])
def test_scheduler_update(op, bf16_latents):
    shape = (4, 4, 4, 128, 128)  # 2^20 latents; cfg_euler_v reads axis 1 as frames
    eu, et = _rand(*shape, mean=1.0, std=0.5, seed=71), _rand(*shape, mean=1.2, std=0.5, seed=72)
    lat = _rand(*shape, mean=4.0, std=2.0, seed=73, dtype=torch.float32)
    if bf16_latents:
        lat = lat.to(BF16).float()
    nxt = torch.empty(shape, device=DEV, dtype=BF16)
    kw = dict(eps_uncond=eu, eps_text=et, latents=lat, model_in_next=nxt, round_latents_bf16=bf16_latents)
    if op == "cfg_ddim":
        kw.update(guidance=7.5, step_row=torch.tensor([500.0, 0.3, 0.45, 0.0], device=DEV))
    else:
        kw["step_row"] = torch.tensor([500.0, 3.2, 1.6, math.sqrt(1.6 ** 2 + 1.0)], device=DEV)
        if op == "cfg_euler":
            kw["guidance"] = 5.0
        else:
            kw.update(frames=4, guidance_per_frame=torch.linspace(1.0, 3.0, 4, device=DEV).to(BF16).float())
    _check(_verify(op, **kw))


# ---- small ops --------------------------------------------------------------------------------------------------------
def test_small_ops():
    ops = _ops()
    recs = []
    recs += _verify("frame_conv_small", x=_rand(4 * 16, 96, 96, 8, mean=0.5, seed=81),
                    w_host=(torch.randn(3, 3, 3, generator=torch.Generator().manual_seed(82)) * 0.5 + 0.2).to(
                        BF16).float().contiguous(), bias_host=torch.tensor([0.1, -0.2, 0.3]), frames=16, cin=3)
    recs += _verify("softmax_rows", x=_rand(256, 4096, std=3.0, seed=83, dtype=torch.float32))
    recs += _verify("router_merge", xs=[_rand(4, 64, 64, 64, mean=1.0, seed=84 + i) for i in range(3)],
                    w=ops.router_weights(_rand(1, 3, seed=87, dtype=torch.float32), None)[0].contiguous())
    t = torch.rand(4096, generator=torch.Generator(device=DEV).manual_seed(88), device=DEV) * 1000.0
    recs += _verify("timestep_embedding", t=t, dim=320, round_t_bf16=False)
    recs += _verify("silu", x=_rand(1024, 1024, std=3.0, seed=89))
    _check(recs)


# ---- power checks: systematic errors the element-wise allowance accepts -------------------------------------------------
def _toward_zero(y, seed):
    """y (bf16) moved one ulp toward zero on a random half of its nonzero elements"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    pick = (torch.rand(y.shape, generator=g, device=DEV) < 0.5) & (y != 0)
    bits = y.contiguous().view(torch.int16)
    return torch.where(pick, bits - 1, bits).view(BF16)


def _fails_with(recs, stat):
    recs = [r for r in recs if "bias_ulp" in r]
    print("\n" + "\n".join(_line(r) for r in recs))
    final = recs[-1]
    assert not final["ok"] and stat in final["why"], final.get("why")


def test_power_gemm_toward_zero():
    ops = _ops()
    a = _args("linear", **_gemm_call("bias", 0))
    out = _toward_zero(ops.linear(**a), 90)
    torch.cuda.synchronize()
    _fails_with(kc.linear_verdict("gemm bias, half toward zero", a, out, lambda **ch: ops.linear(**{**a, **ch})),
                "toward zero")


def test_power_attention_toward_zero():
    ops = _ops()
    b, heads, lq, d, lk = 2, 8, 1024, 64, 1024
    q, k, v = _attn_inputs(b, heads, lq, d, lk, 1.0)
    out = _toward_zero(ops.attention(q, k, v, heads, d, d ** -0.5), 91)
    torch.cuda.synchronize()
    recs, _ = lc.VERIFIERS["attention"](dict(q=q, k=k, v=v, heads=heads, head_dim_pad=d, scale=d ** -0.5,
                                             kv_batch_div=1), out, None)
    _fails_with(recs, "toward zero")


def test_power_groupnorm_group_gain():
    ops = _ops()
    call = _args("group_norm", **_gn_call(False, False, 10))
    out = ops.group_norm(**call)
    torch.cuda.synchronize()
    # group 5 of 32 over 320 channels scaled by 1 + 2^-10 about beta.  The step is below half an ulp of most outputs, so
    # plain rounding would undo it: each output moves one ulp the step's way with probability step / ulp instead
    ch = slice(5 * 10, 6 * 10)
    y = out[..., ch].contiguous()
    step = (y.double() - call["beta"][ch].double()) * 2.0 ** -10 / es.bf16_ulp(y)
    g = torch.Generator(device=DEV).manual_seed(92)
    move = torch.rand(y.shape, generator=g, device=DEV, dtype=torch.float64) < step.abs()
    up = (step > 0) == (y > 0)  # bits + 1: one ulp further from zero
    bits = y.view(torch.int16)
    wrong = out.clone()
    wrong[..., ch] = torch.where(move & (y != 0), bits + torch.where(up, 1, -1).to(torch.int16), bits).view(BF16)
    recs, _ = lc.VERIFIERS["group_norm"](call, wrong, None)
    _fails_with(recs, "gain")


# ---- wrong attention variants the old verdicts pass, against the GPU's SDPA: their gain fails, their RMS error ratio -----
@pytest.mark.parametrize("variant", ["scale 1.003", "exp2 degree-2 polynomial"])
def test_attention_rms_of_wrong_variants(variant):
    """prints each variant's statistics against the GPU's own SDPA yardstick (their RMS error matches SDPA's, which is
    why error_stats bounds no RMS ratio); asserts the direction verdict fails it"""
    b, heads, lq, d, lk = 2, 8, 1024, 64, 1024
    q, k, v = _attn_inputs(b, heads, lq, d, lk, 0.5 if variant.startswith("scale") else 1.0)
    if variant.startswith("scale"):
        out = emu.attention(q, k, v, heads, d, d ** -0.5 * 1.003)
    else:
        out = av.flash(av.poly2_exp2(), q, k, v, heads, d, d ** -0.5)
    recs, _ = lc.VERIFIERS["attention"](dict(q=q, k=k, v=v, heads=heads, head_dim_pad=d, scale=d ** -0.5,
                                             kv_batch_div=1), out, None)
    print("\n" + "\n".join(_line(r) for r in recs))
    assert not recs[-1]["ok"] and "gain" in recs[-1]["why"], recs[-1].get("why")
