"""CPU: the layout checks of tests/kernel_checks.py can fail.  At reduced sizes over the emulated op layer
(tests/ops_emulator.py) every check passes, which shows that its reference and tolerance accept a correct
implementation with a different summation order; and each deliberately wrong variant of an emulated op below is
flagged by at least one check, which shows that the check would notice that mistake in a kernel."""
import functools

import pytest
import torch
import torch.nn.functional as F

from tests import kernel_checks as kc
from tests import ops_emulator as emu

BF16 = torch.bfloat16
CASES = kc.layout_cases(small=True)


@pytest.fixture(scope="module", autouse=True)
def _cpu_device():
    saved = kc.DEVICE
    kc.DEVICE = "cpu"
    yield
    kc.DEVICE = saved


def _failing_checks():
    """run every layout check on the currently patched ops -> (names of the checks that flagged, result records)"""
    kc.RESULTS.clear()
    flagged = []
    for name, fn in CASES:
        n0 = len(kc.RESULTS)
        fn()
        if any(not r["ok"] for r in kc.RESULTS[n0:]):
            flagged.append(name)
    return flagged, list(kc.RESULTS)


def _into(y, out):
    if out is None:
        return y
    out.copy_(y)
    return out


# ---- wrong variants of the emulated ops (each a small wrapper around the correct emulation) ----
def _kv_clip_modulo(q, k, v, heads, head_dim_pad, scale, out=None, kv_batch_div=1):
    """query batch b reads the K/V of clip b % (B / kv_batch_div) instead of b // kv_batch_div"""
    idx = torch.arange(q.shape[0]) % (q.shape[0] // kv_batch_div)
    return emu.attention(q, k[idx], v[idx], heads, head_dim_pad, scale, out=out)


def _no_key_mask(q, k, v, heads, head_dim_pad, scale, out=None, kv_batch_div=1):
    """keys past lk (up to the 128-key tile) enter the softmax with score 0"""
    pad = -k.shape[1] % 128
    return emu.attention(q, F.pad(k, (0, 0, 0, pad)), F.pad(v, (0, 0, 0, pad)), heads, head_dim_pad, scale, out=out,
                         kv_batch_div=kv_batch_div)


def _swapped_heads(q, k, v, heads, head_dim_pad, scale, out=None, kv_batch_div=1):
    """heads 0 and 1 of the last batch trade places in the output"""
    y = emu.attention(q, k, v, heads, head_dim_pad, scale, kv_batch_div=kv_batch_div)
    y4 = y.reshape(y.shape[0], y.shape[1], heads, head_dim_pad)
    y4[-1, :, [0, 1]] = y4[-1, :, [1, 0]]
    return _into(y, out)


def _temporal_attention_keys(keys):
    """temporal attention whose keys / values per sequence are keys(t) of the F real ones ([..., frame, 64])"""
    def fn(q, k, v, clips, frames, hw, heads, scale, out=None, row_stride=None):
        def seq(t):
            return t.float().reshape(clips, frames, hw, heads, 64).permute(0, 2, 3, 1, 4)
        p = torch.softmax(seq(q) @ keys(seq(k)).transpose(-1, -2) * scale, dim=-1)
        y = (p @ keys(seq(v))).permute(0, 3, 1, 2, 4).reshape(clips * frames * hw, heads * 64).to(BF16)
        return _into(y, out)
    return fn


def _swapped_alpha(fn):
    """AlphaBlender with alpha and 1 - alpha exchanged"""
    @functools.wraps(fn)
    def wrapped(*args, blend_alpha=None, **kw):
        if blend_alpha is not None:
            blend_alpha = (1.0 - blend_alpha.float()).to(BF16).float()
        return fn(*args, blend_alpha=blend_alpha, **kw)
    return wrapped


def _late_scale(fn):
    """output scale applied after the residual instead of before it"""
    @functools.wraps(fn)
    def wrapped(*args, out_scale=1.0, out=None, out_fp32=False, **kw):
        if out_scale == 1.0 or kw.get("residual") is None:
            return fn(*args, out_scale=out_scale, out=out, out_fp32=out_fp32, **kw)
        y = fn(*args, out_fp32=out_fp32, **kw)
        y = y * out_scale if out_fp32 else (y.float() * out_scale).to(BF16)
        return _into(y, out)
    return wrapped


def _rowvec_per_clip(x, w_packed, bias, frames, *, rowvec=None, **kw):
    """temporal_conv adds row vector row `clip` to every frame of the clip instead of row `clip * F + frame`"""
    if rowvec is not None and rowvec.shape[0] > 1:
        rowvec = rowvec[torch.arange(x.shape[0]) // frames]
    return emu.temporal_conv(x, w_packed, bias, frames, rowvec=rowvec, **kw)


def _ddim_v_as_epsilon(*args, v_prediction=False, **kw):
    """v-prediction model output put through the epsilon formula"""
    return emu.cfg_ddim(*args, v_prediction=False, **kw)


VARIANTS = {
    "kv_batch_div: clip b % (B / div) instead of b // div": {"attention": _kv_clip_modulo},
    "attention: no key-tail mask (score 0 past lk)": {"attention": _no_key_mask},
    "attention: heads 0 and 1 swapped in one batch": {"attention": _swapped_heads},
    "temporal attention: one zero-padded frame admitted": {
        "temporal_attention": _temporal_attention_keys(lambda t: F.pad(t, (0, 0, 0, 1)))},
    "temporal attention: only the first 16 frames when F > 16": {
        "temporal_attention": _temporal_attention_keys(lambda t: t[..., :16, :])},
    "AlphaBlender: alpha and 1 - alpha swapped": {
        "linear": _swapped_alpha(emu.linear), "conv2d": _swapped_alpha(emu.conv2d),
        "temporal_conv": _swapped_alpha(emu.temporal_conv)},
    "output scale after the residual": {"linear": _late_scale(emu.linear), "conv2d": _late_scale(emu.conv2d)},
    "temporal_conv: row vector per clip instead of per frame": {"temporal_conv": _rowvec_per_clip},
    "cfg_ddim: v-prediction through the epsilon formula": {"cfg_ddim": _ddim_v_as_epsilon},
    "latent encoder: attention scale 1 instead of 4^-0.5": {
        "i2vgen_latent_encoder": functools.partial(emu.i2vgen_latent_encoder, attn_scale=1.0)},
}


def test_layout_checks_pass_on_emulator():
    with emu.patched_ops():
        flagged, recs = _failing_checks()
    bad = [r for r in recs if not r["ok"]]
    assert not flagged and not bad, f"layout checks fail a correct implementation: {flagged} {bad[:3]}"
    assert len(recs) >= len(CASES)


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_layout_checks_catch_wrong_variant(variant):
    with emu.patched_ops() as ops:
        for name, fn in VARIANTS[variant].items():
            setattr(ops, name, fn)
        flagged, _ = _failing_checks()
    print(f"{variant}: caught by {', '.join(flagged) or 'NOTHING'}")
    assert flagged, f"no layout check notices: {variant}"
