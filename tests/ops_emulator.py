"""TEST INFRASTRUCTURE: plain-PyTorch emulation of the `ctrl_adapter_b200.ops` entry points (same names, arguments,
packed-weight formats and bf16 rounding points as the CUDA kernels behind the C ABI), runnable on CPU.

Purpose: the host modules (layers / adapter / controlnet / unet_*) are pure composition logic over `ops`; with the
emulator patched in, that logic -- block wiring, skip / residual order, strides, per-clip broadcast rows, weight packing
-- is checked against the oracle on the CPU box (`tests/test_host_emulated_cpu.py`), where there is no GPU.  It is never
imported by the product (the product has no CPU path and fails loudly without the CUDA library); the numerics of the
kernels themselves are checked on the H100 by tests/kernel_checks.py.
"""
from __future__ import annotations

import contextlib
import math
from typing import Optional

import torch
import torch.nn.functional as F

BF16 = torch.bfloat16
ACT_NONE, ACT_SILU, ACT_GEGLU = 0, 1, 2


def _r(x: torch.Tensor) -> torch.Tensor:
    """round to bf16, keep computing in fp32"""
    return x.to(BF16).float()


def _epilogue(acc, bias, act, out_scale, rowvec, residual, blend_src, blend_alpha, out_fp32):
    v = acc if bias is None else acc + bias.float()
    if out_fp32:  # rounded to bf16 only after SiLU and after the row vector
        if act == ACT_SILU:
            v = _r(F.silu(v))
        v = v * out_scale if out_scale != 1.0 else v
        if rowvec is not None:
            v = _r(v + rowvec.float())
        return v if residual is None else v + residual.float()
    v = _r(v)
    if act == ACT_SILU:
        v = _r(F.silu(v))
    return _finish(v, out_scale, rowvec, residual, blend_src, blend_alpha)


def _finish(v, out_scale, rowvec, residual, blend_src, blend_alpha):
    """the bf16 chain after the activation: output scale, row vector, residual, AlphaBlender, each rounded"""
    if out_scale != 1.0:
        v = _r(v * out_scale)
    if rowvec is not None:
        v = _r(v + rowvec.float())
    if residual is not None:
        v = _r(v + residual.float())
    if blend_src is not None:
        a = blend_alpha.float().reshape(())
        v = _r(_r(a * blend_src.float()) + _r(_r(1.0 - a) * v))
    return v.to(BF16)


def linear(x, w, bias=None, *, act=ACT_NONE, residual=None, rowvec=None, rows_per_vec=0, blend_src=None, blend_alpha=None,
           out_scale=1.0, out=None, out_fp32=False, bn=0):
    m, k = x.shape
    xf, wf = x.float(), w.float()
    rv = None
    if rowvec is not None:
        assert rows_per_vec > 0 and m % rows_per_vec == 0 and rowvec.shape[0] == m // rows_per_vec
        rv = rowvec.repeat_interleave(rows_per_vec, dim=0)
    if act == ACT_GEGLU:
        # value and gate rows interleaved per N tile of bn (ops.pack_geglu_weight); bn 0 is ca_gemm's GEGLU tile, 256
        d, half = w.shape[0] // 2, (bn or 256) // 2
        wt = wf.reshape(d // half, 2, half, k)
        a = xf @ wt[:, 0].reshape(d, k).t()
        g = xf @ wt[:, 1].reshape(d, k).t()
        if bias is not None:
            bt = bias.float().reshape(d // half, 2, half)
            a = a + bt[:, 0].reshape(d)
            g = g + bt[:, 1].reshape(d)
        a, g = _r(a), _r(g)
        y = _finish(_r(a * _r(F.gelu(g))), out_scale, rv, residual, blend_src, blend_alpha)
    else:
        y = _epilogue(xf @ wf.t(), bias, act, out_scale, rv, residual, blend_src, blend_alpha, out_fp32)
    if out is not None:
        out.copy_(y)
        return out
    return y


def _unpack_conv_weight(w_packed, ntaps, kpt, cin):
    cout = w_packed.shape[0]
    return w_packed.float().reshape(cout, ntaps, kpt)[:, :, :cin]  # [Cout, taps, Cin]


def conv2d(x, w_packed, bias, *, ksize=3, stride=1, x2=None, act=ACT_NONE, out_scale=1.0, rowvec=None, residual=None,
           blend_src=None, blend_alpha=None, out=None, out_fp32=False, bn=0, k_per_tap=None, pad=None):
    """pad (0, 1) at stride 2: one zero row / column at the bottom / right, then an unpadded convolution"""
    n, h, w_, c = x.shape
    xin = x if x2 is None else torch.cat([x, x2], dim=3)
    cin = xin.shape[3]
    ntaps = ksize * ksize
    kpt = k_per_tap if k_per_tap is not None else w_packed.shape[1] // ntaps
    wt = _unpack_conv_weight(w_packed, ntaps, kpt, cin).permute(0, 2, 1).reshape(-1, cin, ksize, ksize)
    xf = xin.float().permute(0, 3, 1, 2)
    if pad is None or tuple(pad) == (ksize // 2,) * 2:
        acc = F.conv2d(xf, wt, None, stride=stride, padding=ksize // 2)
    else:
        assert tuple(pad) == (0, 1) and stride == 2, pad
        acc = F.conv2d(F.pad(xf, (0, 1, 0, 1)), wt, None, stride=2)
    acc = acc.permute(0, 2, 3, 1)
    rv = None
    if rowvec is not None:
        rv = rowvec.reshape(rowvec.shape[0], 1, 1, -1)
    y = _epilogue(acc, bias, act, out_scale, rv, residual, blend_src, blend_alpha, out_fp32).contiguous()
    if out is not None:
        out.copy_(y)
        return out
    return y


def temporal_conv(x, w_packed, bias, frames, *, rowvec=None, residual=None, blend_src=None, blend_alpha=None, out=None):
    bf, h, w_, c = x.shape
    b = bf // frames
    wt = _unpack_conv_weight(w_packed, 3, w_packed.shape[1] // 3, c)  # [Cout, 3, C]
    xf = F.pad(x.float().reshape(b, frames, h, w_, c), (0, 0, 0, 0, 0, 0, 1, 1))  # zero frames at both clip ends
    acc = sum(xf[:, t:t + frames] @ wt[:, t].t() for t in range(3)).reshape(bf, h, w_, -1)
    rv = None if rowvec is None else rowvec.reshape(rowvec.shape[0], 1, 1, -1)
    y = _epilogue(acc, bias, ACT_NONE, 1.0, rv, residual, blend_src, blend_alpha, False).contiguous()
    if out is not None:
        out.copy_(y)
        return out
    return y


def attention(q, k, v, heads, head_dim_pad, scale, out=None, kv_batch_div=1):
    b, lq, _ = q.shape
    qh = q.float().reshape(b, lq, heads, head_dim_pad).permute(0, 2, 1, 3)
    kb = torch.arange(b, device=q.device) // kv_batch_div
    kh = k.float().reshape(k.shape[0], k.shape[1], heads, head_dim_pad).permute(0, 2, 1, 3)[kb]
    vh = v.float().reshape(v.shape[0], v.shape[1], heads, head_dim_pad).permute(0, 2, 1, 3)[kb]
    p = torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1)
    y = (p @ vh).permute(0, 2, 1, 3).reshape(b, lq, heads * head_dim_pad).to(BF16)
    if out is not None:
        out.copy_(y)
        return out
    return y


def temporal_attention(q, k, v, clips, frames, hw, heads, scale, out=None, row_stride=None):
    def seq(t):  # rows (clip, frame, pixel) -> [clip, pixel, head, frame, 64]
        return t.float().reshape(clips, frames, hw, heads, 64).permute(0, 2, 3, 1, 4)
    p = torch.softmax(seq(q) @ seq(k).transpose(-1, -2) * scale, dim=-1)
    y = (p @ seq(v)).permute(0, 3, 1, 2, 4).reshape(clips * frames * hw, heads * 64).to(BF16)
    if out is not None:
        out.copy_(y)
        return out
    return y


def group_norm(x, gamma, beta, eps, *, groups=32, silu=False, up2x=False, x2=None, imgs_per_sample=1, out=None):
    xin = x if x2 is None else torch.cat([x, x2], dim=3)
    n, h, w_, c = xin.shape
    ns = n // imgs_per_sample
    t = xin.float().reshape(ns, imgs_per_sample * h * w_, groups, c // groups)
    mean = t.mean(dim=(1, 3), keepdim=True)
    var = t.var(dim=(1, 3), unbiased=False, keepdim=True)
    y = ((t - mean) * torch.rsqrt(var + eps)).reshape(n, h, w_, c) * gamma.float() + beta.float()
    if silu:
        y = F.silu(y)
    if up2x:
        y = y.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    y = y.to(BF16).contiguous()
    if out is not None:
        out.copy_(y)
        return out
    return y


def layer_norm(x, gamma, beta, eps=1e-5, *, add_rowvec=None, rows_per_vec=0, return_sum=False):
    c = x.shape[-1]
    xf = x.float()
    xs = None
    if add_rowvec is not None:
        rows = x.numel() // c
        rv = add_rowvec.float().repeat_interleave(rows_per_vec, dim=0)
        assert rv.shape[0] == rows, (rv.shape, rows, rows_per_vec)
        xf = _r(xf.reshape(rows, c) + rv).reshape(x.shape)
        xs = xf.to(BF16)
    y = F.layer_norm(xf, (c,), gamma.float(), beta.float(), eps).to(BF16)
    return (y, xs) if return_sum else y


def timestep_embedding(t, dim, *, flip_sin_to_cos=True, freq_shift=0.0, round_t_bf16=False):
    t = t.float()
    if round_t_bf16:
        t = _r(t)
    half = dim // 2
    exponent = -math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=t.device) / (half - freq_shift)
    emb = t[:, None] * torch.exp(exponent)[None, :]
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
    if flip_sin_to_cos:
        emb = torch.cat([emb[:, half:], emb[:, :half]], dim=-1)
    return F.pad(emb, (0, dim - 2 * half)).to(BF16)  # odd dim: a trailing zero column


def silu(x):
    return F.silu(x.float()).to(BF16)


def add(a, b, out=None):
    y = (a.float() + b.float()).to(BF16)
    if out is not None:
        out.copy_(y)
        return out
    return y


def nchw_to_nhwc(x, c_pad: Optional[int] = None):
    n, c, h, w_ = x.shape
    cp = c if c_pad is None else c_pad
    y = torch.zeros((n, h, w_, cp), dtype=BF16, device=x.device)
    y[..., :c] = x.permute(0, 2, 3, 1).to(BF16)
    return y


def nhwc_to_nchw(x, c: Optional[int] = None, fp32: bool = False):
    cc = x.shape[3] if c is None else c
    return x[..., :cc].permute(0, 3, 1, 2).contiguous().to(torch.float32 if fp32 else BF16)


def avgpool(x, oh, ow):
    return F.adaptive_avg_pool2d(x.float().permute(0, 3, 1, 2), (oh, ow)).permute(0, 2, 3, 1).contiguous().to(BF16)


def upsample2x(x):
    return x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).contiguous()


def i2vgen_latent_encoder(x, clips, frames, params, *, attn_scale=0.5):
    """x [clips*frames, H, W, Cs] (first 4 channels used); params fp32 [288], layout in include/ctrl_adapter_b200.h:
    per pixel over the frames of a clip: h = x + to_out(attn(LN(x))) with 2 heads x 4; y = h + W2 gelu(W1 h + b1) + b2.
    attn_scale: 4^-0.5 (head dim 4); other values only model a wrong kernel in tests/test_kernel_checks_cpu.py."""
    n, h, w_, cs = x.shape
    p = params.float()
    o = 0

    def take(k, shape):
        nonlocal o
        t = p[o:o + k].reshape(shape)
        o += k
        return t
    ln_w, ln_b = take(4, (4,)), take(4, (4,))
    wq, wk, wv = take(32, (8, 4)), take(32, (8, 4)), take(32, (8, 4))
    wo, bo = take(32, (4, 8)), take(4, (4,))
    w1, b1, w2, b2 = take(64, (16, 4)), take(16, (16,)), take(64, (4, 16)), take(4, (4,))
    xs = x[..., :4].float().reshape(clips, frames, h * w_, 4).permute(0, 2, 1, 3)  # [clip, pixel, frame, 4]
    xn = _r(F.layer_norm(xs, (4,), ln_w, ln_b, 1e-5))

    def heads(t):
        return t.reshape(*t.shape[:-1], 2, 4).transpose(-2, -3)  # [clip, pixel, head, frame, 4]
    q, k, v = (heads(_r(xn @ m.t())) for m in (wq, wk, wv))
    a = _r(torch.softmax(q @ k.transpose(-1, -2) * attn_scale, dim=-1) @ v)
    a = a.transpose(-2, -3).reshape(clips, h * w_, frames, 8)
    hcur = _r(_r(a @ wo.t() + bo) + xs)
    y = _r(_r(_r(F.gelu(_r(hcur @ w1.t() + b1))) @ w2.t() + b2) + hcur)
    out = torch.zeros_like(x)
    out[..., :4] = y.permute(0, 2, 1, 3).reshape(n, h, w_, 4).to(BF16)
    return out


def softmax_rows(x):
    return torch.softmax(x.float(), dim=-1).to(BF16)


def frame_conv_small(x, w_host, bias_host, frames, cin):
    bf, h, w_, cs = x.shape
    b = bf // frames
    xs = x[..., :cin].float().reshape(b, frames, h, w_, cin).permute(0, 4, 1, 2, 3)   # [B, Cin, F, H, W]
    wt = w_host.float().to(x.device)[:, :, :, None, None]
    y = F.conv3d(xs, wt, None if bias_host is None else bias_host.float().to(x.device), padding=(1, 0, 0))
    return y.permute(0, 2, 1, 3, 4).reshape(bf, -1, h, w_).to(BF16).contiguous()


def router_weights(logits, mask):
    lg = logits.float().clone()
    if mask is not None:
        lg[:, mask.to(torch.bool).logical_not()] = -1e6
    return torch.softmax(lg, dim=-1)


def router_merge(xs, w):
    y = None
    for x, wk in zip(xs, w.float()):
        term = _r(x.float() * _r(wk))
        y = term if y is None else _r(y + term)
    return y.to(BF16)


def cfg_euler(eps_uncond, eps_text, latents, guidance, step_row, latents_out=None, model_in_next=None,
              round_latents_bf16=True):
    _, sigma, sigma_next, next_div = (float(v) for v in step_row)
    u, c = eps_uncond.float(), eps_text.float()
    eps = _r(u + _r(guidance * _r(c - u)))
    x = latents.float()
    x0 = x - _r(_r(torch.tensor(sigma)) * eps)
    xn = x + (x - x0) / sigma * (sigma_next - sigma)
    if round_latents_bf16:
        xn = _r(xn)
    if latents_out is None:
        latents_out = torch.empty_like(latents)
    latents_out.copy_(xn)
    if model_in_next is not None:
        model_in_next.copy_((xn / _r(torch.tensor(next_div))).to(BF16))
    return latents_out


def cfg_euler_v(eps_uncond, eps_text, latents, guidance_per_frame, frames, step_row, latents_out=None,
                model_in_next=None, round_latents_bf16=True):
    _, sigma, sigma_next, next_div = (float(v) for v in step_row)
    g = guidance_per_frame.float().reshape(1, frames, *([1] * (latents.dim() - 2)))
    u, c = eps_uncond.float(), eps_text.float()
    mo = _r(u + _r(g * _r(c - u)))
    x = latents.float()
    c_out = _r(torch.tensor(-sigma / math.sqrt(sigma * sigma + 1.0)))
    x0 = _r(mo * c_out) + x / (sigma * sigma + 1.0)
    xn = x + (x - x0) / sigma * (sigma_next - sigma)
    if round_latents_bf16:
        xn = _r(xn)
    if latents_out is None:
        latents_out = torch.empty_like(latents)
    latents_out.copy_(xn)
    if model_in_next is not None:
        model_in_next.copy_((xn / _r(torch.tensor(next_div))).to(BF16))
    return latents_out


def cfg_ddim(eps_uncond, eps_text, latents, guidance, step_row, latents_out=None, model_in_next=None,
             round_latents_bf16=True, v_prediction=False):
    a_t, a_prev = float(step_row[1]), float(step_row[2])
    sa, sb, sap, sbp = (torch.tensor(v).sqrt() for v in (a_t, 1.0 - a_t, a_prev, 1.0 - a_prev))
    rr = _r if round_latents_bf16 else (lambda t: t)
    sa, sb, sap, sbp = rr(sa), rr(sb), rr(sap), rr(sbp)
    u, c = eps_uncond.float(), eps_text.float()
    mo = _r(u + _r(guidance * _r(c - u)))
    x = latents.float()
    if v_prediction:
        x0 = rr(rr(sa * x) - rr(sb * mo))
        eps = rr(rr(sa * mo) + rr(sb * x))
    else:
        x0 = rr(rr(x - rr(sb * mo)) / sa)
        eps = mo
    xn = rr(rr(sap * x0) + rr(sbp * eps))
    if latents_out is None:
        latents_out = torch.empty_like(latents)
    latents_out.copy_(xn)
    if model_in_next is not None:
        model_in_next.copy_(xn.to(BF16))
    return latents_out


def vae_latents(moments, layout=0, noise=None, frames=1, num_videos=1, scale=1.0):
    """ca_vae_latents: posterior of the quant_conv output (mean, logvar in channels 0-3 / 4-7), then the image-latent
    layout of the posterior (0), the I2VGen-XL loop (1) or the SVD loop (2); fp32 arithmetic, one rounding to bf16."""
    m = moments.float().permute(0, 3, 1, 2)
    v = m[:, :4]
    if noise is not None:
        v = v + torch.exp(0.5 * m[:, 4:].clamp(-30.0, 20.0)) * noise.float()
    if layout == 0:
        return v.to(BF16)
    if layout == 1:
        pos = [torch.full_like(v[:, :, None], k / (frames - 1)) for k in range(1, frames)]
        x = torch.cat([(v * scale)[:, :, None]] + pos, dim=2).repeat(num_videos, 1, 1, 1, 1)
        return torch.cat([x, x]).to(BF16)
    x = torch.cat([torch.zeros_like(v), v]).repeat(num_videos, 1, 1, 1)
    return x[:, None].repeat(1, frames, 1, 1, 1).to(BF16)


_EMULATED = ["linear", "conv2d", "temporal_conv", "attention", "temporal_attention", "group_norm", "layer_norm",
             "timestep_embedding", "silu", "add", "nchw_to_nhwc", "nhwc_to_nchw", "avgpool", "upsample2x", "i2vgen_latent_encoder",
             "softmax_rows", "frame_conv_small", "router_weights", "router_merge", "cfg_euler", "cfg_euler_v", "cfg_ddim",
             "vae_latents"]


@contextlib.contextmanager
def patched_ops():
    """Swap the CUDA-backed entry points of ctrl_adapter_b200.ops for the emulation above (restored on exit)."""
    import sys
    g = sys.modules[__name__].__dict__
    from ctrl_adapter_b200 import ops
    saved = {name: getattr(ops, name) for name in _EMULATED}
    try:
        for name in _EMULATED:
            setattr(ops, name, g[name])
        yield ops
    finally:
        for name, fn in saved.items():
            setattr(ops, name, fn)
