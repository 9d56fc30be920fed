"""GPU parity checks of every CUDA kernel against a plain PyTorch fp32 reference of the same op on the same
bf16-quantised inputs.  Used by tests/test_kernels_gpu.py (pytest -m gpu), by __graft_entry__.smoke() and as a
stand-alone report:  python -m tests.kernel_checks  [--json out.json]

Tolerances (stated per check, torch.testing semantics |out-ref| <= atol + rtol*|ref|):
  * fp32-output contractions: rtol 1e-3 / atol 1e-4 (north-star tolerance; fp32 accumulate on both sides)
  * bf16-output kernels: the fp32 reference is rounded to bf16 the same way; allowance = 1 bf16 ulp
    (rtol 2^-7) + atol 1e-3 for values that straddle a rounding boundary after a different summation order;
    epilogues with several rounding steps (conv -> +temb -> +residual) get 2 ulps (rtol 2^-6) of the largest
    intermediate magnitude, since two independent boundary flips can stack
  * attention: P is rounded to bf16 before the PV product (as in flash-attention / SDPA): rtol 2e-2 / atol 2e-3,
    and the error must not exceed 2x that of torch's own bf16 SDPA against the same fp32 reference.
"""
from __future__ import annotations

import json
import math
import sys

import torch
import torch.nn.functional as F

BF16 = torch.bfloat16
RESULTS = []


def _ops():
    from ctrl_adapter_b200 import ops
    return ops


def _rand(*shape, scale=1.0, seed=None, dtype=BF16):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed if seed is not None else (hash(shape) & 0xFFFF) + 17)
    return (torch.randn(*shape, generator=g, device="cuda", dtype=torch.float32) * scale).to(dtype)


def _report(name, out, ref, rtol, atol, extra=None, mag=None):
    """mag: magnitude of the largest intermediate of a multi-step bf16 epilogue (a 1-ulp flip of an intermediate is
    1 ulp of THAT magnitude, which can be several ulps of a smaller final value after cancellation)."""
    out = out.float()
    ref = ref.float()
    assert out.shape == ref.shape, f"{name}: shape {tuple(out.shape)} vs {tuple(ref.shape)}"
    err = (out - ref).abs()
    tol = atol + rtol * (ref.abs() if mag is None else torch.maximum(ref.abs(), mag.float().abs()))
    bad = (err > tol) | ~torch.isfinite(out)
    rec = {
        "check": name,
        "max_abs_err": float(err.max()),
        "max_ref": float(ref.abs().max()),
        "rel_fro": float((out - ref).norm() / ref.norm().clamp_min(1e-20)),
        "n_bad": int(bad.sum()),
        "n": out.numel(),
        "rtol": rtol,
        "atol": atol,
        "ok": bool(bad.sum() == 0),
    }
    if extra:
        rec.update(extra)
    RESULTS.append(rec)
    return rec


# ------------------------------------------------------------------------------------------------
# linear
# ------------------------------------------------------------------------------------------------
def check_linear(m, k, n, *, bn=0, bias=True, out_fp32=True, residual=False, act="none", seed=0):
    ops = _ops()
    x = _rand(m, k, seed=seed + 1)
    w = _rand(n, k, scale=1.0 / math.sqrt(k), seed=seed + 2)
    b = _rand(n, seed=seed + 3) if bias else None
    res = _rand(m, n, seed=seed + 4) if residual else None
    ref = x.float() @ w.float().t()
    if b is not None:
        ref = ref + b.float()
    if not out_fp32:
        ref = ref.to(BF16).float()
    if act == "silu":
        ref = F.silu(ref).to(BF16).float()
    mag = ref.abs().clone()
    if residual:
        ref = (ref + res.float()).to(BF16).float()
        mag = torch.maximum(mag, res.float().abs())
    out = ops.linear(x, w, ops.bias_f32(b), act=ops.ACT_SILU if act == "silu" else ops.ACT_NONE, residual=res,
                     out_fp32=out_fp32, bn=bn)
    torch.cuda.synchronize()
    rtol, atol = (1e-3, 1e-4) if out_fp32 else (2 ** -6 if residual else 2 ** -7, 1e-3)
    return _report(f"linear m{m} k{k} n{n} bn{bn} {'f32' if out_fp32 else 'bf16'} act={act} res={int(residual)}",
                   out, ref, rtol, atol, mag=mag)


def check_geglu(m, k, d, seed=0):
    ops = _ops()
    x = _rand(m, k, seed=seed + 1)
    w = _rand(2 * d, k, scale=1.0 / math.sqrt(k), seed=seed + 2)
    b = _rand(2 * d, seed=seed + 3)
    wi, bi = ops.pack_geglu_weight(w, b, 256)
    out = ops.linear(x, wi, ops.bias_f32(bi), act=ops.ACT_GEGLU, bn=256)
    # the same contraction (same kernel, tiles and summation order) with the fp32 pre-activation as output
    pre = ops.linear(x, wi, ops.bias_f32(bi), out_fp32=True, bn=256).reshape(m, d // 128, 2, 128)
    pre = torch.cat([pre[:, :, 0].reshape(m, d), pre[:, :, 1].reshape(m, d)], dim=1)  # undo the per-tile interleave
    torch.cuda.synchronize()
    # (1) the contraction against the exact (fp64) pre-activation at the fp32 GEMM tolerance of check_linear
    exact = (x.double() @ w.double().t() + b.double()).float()
    _report(f"geglu pre-activation m{m} k{k} d{2 * d}", pre, exact, 1e-3, 1e-4)
    # (2) the epilogue's bf16 rounding chain applied to the pre-activation the kernel accumulated.  A pre-activation
    # within an fp32 ulp or two of a bf16 rounding tie rounds either way depending on the summation order (cuBLAS's
    # own fp32 result rounds ~3300 of the 25.6 M pre-activations at m5000 away from the exact value), and GELU times
    # the value half magnifies that one-ulp flip beyond the output tolerance, so the epilogue is checked against the
    # input it was given.
    h = pre.to(BF16).float()
    a, g = h[:, :d], h[:, d:]
    ref = (a * F.gelu(g).to(BF16).float()).to(BF16).float()
    return _report(f"geglu m{m} k{k} d{d}", out, ref, 2 ** -6, 2e-3)


def check_linear_rowvec(m, k, n, rpv, seed=0):
    ops = _ops()
    x = _rand(m, k, seed=seed + 1)
    w = _rand(n, k, scale=1.0 / math.sqrt(k), seed=seed + 2)
    rv = _rand(m // rpv, n, seed=seed + 3)
    lin = (x.float() @ w.float().t()).to(BF16).float()
    ref = (lin + rv.float().repeat_interleave(rpv, dim=0)).to(BF16).float()
    out = ops.linear(x, w, None, rowvec=rv, rows_per_vec=rpv)
    torch.cuda.synchronize()
    return _report(f"linear+rowvec m{m} k{k} n{n} rpv{rpv}", out, ref, 2 ** -6, 1e-3, mag=lin)


def check_linear_blend(m, k, n, seed=0):
    ops = _ops()
    x = _rand(m, k, seed=seed + 1)
    w = _rand(n, k, scale=1.0 / math.sqrt(k), seed=seed + 2)
    res = _rand(m, n, seed=seed + 4)
    xs = _rand(m, n, seed=seed + 5)
    alpha = torch.sigmoid(torch.tensor([0.3], device="cuda")).to(BF16)
    lin = (x.float() @ w.float().t()).to(BF16).float()
    xt = (lin + res.float()).to(BF16)
    ref = ((alpha * xs).to(BF16) + ((1.0 - alpha).to(BF16) * xt).to(BF16)).float()
    out = ops.linear(x, w, None, residual=res, blend_src=xs, blend_alpha=alpha.float())
    torch.cuda.synchronize()
    mag = torch.maximum(torch.maximum(xt.float().abs(), res.float().abs()), xs.float().abs())
    mag = torch.maximum(mag, lin.abs())  # bf16(x @ w^T) is the first rounded intermediate of the epilogue
    return _report(f"linear+res+blend m{m} k{k} n{n}", out, ref, 2 ** -7, 1e-3, mag=mag)


# ------------------------------------------------------------------------------------------------
# convs
# ------------------------------------------------------------------------------------------------
def _nhwc(x_nchw):
    return x_nchw.permute(0, 2, 3, 1).contiguous()


def check_conv(n, h, w, cin, cout, *, ksize=3, stride=1, cin2=0, out_fp32=True, rowvec=False, residual=False,
               scale=1.0, seed=0):
    ops = _ops()
    x = _rand(n, cin, h, w, seed=seed + 1)
    x2 = _rand(n, cin2, h, w, seed=seed + 5) if cin2 else None
    ct = cin + cin2
    wt = _rand(cout, ct, ksize, ksize, scale=1.0 / math.sqrt(ct * ksize * ksize), seed=seed + 2)
    b = _rand(cout, seed=seed + 3)
    xin = x.float() if x2 is None else torch.cat([x.float(), x2.float()], dim=1)
    ref = F.conv2d(xin, wt.float(), b.float(), stride=stride, padding=(ksize - 1) // 2)
    if not out_fp32:
        ref = ref.to(BF16).float()
    if scale != 1.0:
        ref = (ref * scale).to(BF16).float()
    rv = res = None
    mag = ref.abs().clone()
    if rowvec:
        rv = _rand(n, cout, seed=seed + 6)
        ref = (ref + rv.float()[:, :, None, None]).to(BF16).float()
        mag = torch.maximum(mag, ref.abs())
    if residual:
        res = _rand(n, cout, ref.shape[2], ref.shape[3], seed=seed + 7)
        ref = (ref + res.float()).to(BF16).float()
        mag = torch.maximum(mag, res.float().abs())
    kpad = 64 if stride == 2 else 8
    wp = ops.pack_conv_weight(wt, kpad)
    out = ops.conv2d(_nhwc(x), wp, ops.bias_f32(b), ksize=ksize, stride=stride, x2=_nhwc(x2) if x2 is not None else None,
                     out_fp32=out_fp32, rowvec=rv, residual=_nhwc(res) if res is not None else None, out_scale=scale)
    torch.cuda.synchronize()
    rtol, atol = (1e-3, 1e-4) if out_fp32 else (2 ** -6 if (rowvec or residual) else 2 ** -7, 1e-3)
    return _report(f"conv{ksize}x{ksize} s{stride} n{n} {h}x{w} c{cin}+{cin2}->{cout} {'f32' if out_fp32 else 'bf16'}"
                   f" rv={int(rowvec)} res={int(residual)} sc={scale}", out.permute(0, 3, 1, 2), ref, rtol, atol, mag=mag)


def check_temporal_conv(b, f, h, w, c, cout, seed=0):
    ops = _ops()
    x = _rand(b, c, f, h, w, seed=seed + 1)
    wt = _rand(cout, c, 3, 1, 1, scale=1.0 / math.sqrt(3 * c), seed=seed + 2)
    bias = _rand(cout, seed=seed + 3)
    rv = _rand(b * f, cout, seed=seed + 4)
    ref = F.conv3d(x.float(), wt.float(), bias.float(), padding=(1, 0, 0)).to(BF16).float()
    mag = ref.abs().clone()
    ref = (ref + rv.float().reshape(b, f, cout).permute(0, 2, 1)[:, :, :, None, None]).to(BF16).float()
    xl = x.permute(0, 2, 3, 4, 1).reshape(b * f, h, w, c).contiguous()
    out = ops.temporal_conv(xl, ops.pack_conv_weight(wt), ops.bias_f32(bias), f, rowvec=rv)
    torch.cuda.synchronize()
    out5 = out.reshape(b, f, h, w, cout).permute(0, 4, 1, 2, 3)
    return _report(f"temporal_conv b{b} f{f} {h}x{w} c{c}->{cout}", out5, ref, 2 ** -6, 1e-3, mag=mag)


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def check_attention(b, heads, lq, lk, d, seed=0, ramp=0.0):
    ops = _ops()
    dp = (d + 63) // 64 * 64
    q = _rand(b, lq, heads, d, seed=seed + 1)
    k = _rand(b, lk, heads, d, seed=seed + 2)
    if ramp:
        # logits whose row max keeps growing along the key axis: drives the kernel's lazy O / l rescale path on most
        # KV tiles (iid scores almost never move the max by the 2^8 threshold)
        grow = 1.0 + ramp * torch.arange(lk, device=k.device, dtype=torch.float32) / lk
        k = (k.float() * grow[None, :, None, None]).to(k.dtype)
    v = _rand(b, lk, heads, d, seed=seed + 3)
    scale = d ** -0.5
    qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))
    p = torch.softmax(qf @ kf.transpose(-1, -2) * scale, dim=-1)
    ref = (p @ vf).permute(0, 2, 1, 3)  # [b, lq, h, d]
    sd = F.scaled_dot_product_attention(q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), v.permute(0, 2, 1, 3))
    sd_err = float((sd.permute(0, 2, 1, 3).float() - ref).abs().max())

    def pad(t):
        return F.pad(t, (0, dp - d)).reshape(t.shape[0], t.shape[1], heads * dp).contiguous()
    out = ops.attention(pad(q), pad(k), pad(v), heads, dp, scale)
    torch.cuda.synchronize()
    out = out.reshape(b, lq, heads, dp)[..., :d]
    # ramped logits give nearly one-hot rows: the output is a bf16-rounded V row (|v| up to ~4.6, half-ulp 9e-3), so the
    # absolute floor follows torch's own bf16 SDPA error instead of the iid-case 2e-3
    atol = 2e-3 if not ramp else max(2e-3, 1.25 * sd_err)
    rec = _report(f"attention b{b} h{heads} lq{lq} lk{lk} d{d}" + (f" ramp{ramp:g}" if ramp else ""), out, ref, 2e-2, atol,
                  {"sdpa_bf16_max_err": sd_err})
    if rec["max_abs_err"] > 2.0 * sd_err + 1e-3:
        rec["ok"] = False
        rec["why"] = "error larger than 2x torch bf16 SDPA"
    return rec


def check_softmax_rows(rows, cols, seed=0):
    ops = _ops()
    g = torch.Generator(device="cpu").manual_seed(seed + 9)
    x = (torch.randn(rows, cols, generator=g) * 4.0).cuda()
    x[0, :7] = 30.0  # a few dominant scores in one row
    out = ops.softmax_rows(x)
    torch.cuda.synchronize()
    return _report(f"softmax_rows {rows}x{cols}", out, torch.softmax(x, dim=-1), 2 ** -8, 1e-6)


def check_temporal_attention(clips, frames, hw, heads, seed=0):
    ops = _ops()
    c = heads * 64
    q = _rand(clips * frames, hw, c, seed=seed + 1)
    k = _rand(clips * frames, hw, c, seed=seed + 2)
    v = _rand(clips * frames, hw, c, seed=seed + 3)

    def to_seq(t):  # (b f) s (h d) -> (b s h) f d
        return t.float().reshape(clips, frames, hw, heads, 64).permute(0, 2, 3, 1, 4)
    p = torch.softmax(to_seq(q) @ to_seq(k).transpose(-1, -2) * 0.125, dim=-1)
    ref = (p @ to_seq(v)).permute(0, 3, 1, 2, 4).reshape(clips * frames, hw, c)
    out = ops.temporal_attention(q.reshape(-1, c), k.reshape(-1, c), v.reshape(-1, c), clips, frames, hw, heads, 0.125)
    torch.cuda.synchronize()
    # 16-key softmax with O(1) values: bf16 P rounding alone gives ~4e-3 absolute error
    return _report(f"temporal_attention b{clips} f{frames} hw{hw} h{heads}", out.reshape(ref.shape), ref, 2e-2, 6e-3)


# ------------------------------------------------------------------------------------------------
# norms & elementwise
# ------------------------------------------------------------------------------------------------
def check_groupnorm(n, h, w, c, *, c2=0, silu=True, up=False, imgs_per_sample=1, eps=1e-6, seed=0):
    ops = _ops()
    x = _rand(n, c, h, w, seed=seed + 1) * 2.0 + 0.5
    x2 = (_rand(n, c2, h, w, seed=seed + 4) - 0.3) if c2 else None
    ct = c + c2
    gamma = _rand(ct, seed=seed + 2, dtype=torch.float32) * 0.2 + 1.0
    beta = _rand(ct, seed=seed + 3, dtype=torch.float32) * 0.2
    xin = x.float() if x2 is None else torch.cat([x.float(), x2.float()], dim=1)
    if imgs_per_sample > 1:
        b = n // imgs_per_sample
        x5 = xin.reshape(b, imgs_per_sample, ct, h, w).permute(0, 2, 1, 3, 4)
        ref = F.group_norm(x5, 32, gamma, beta, eps).permute(0, 2, 1, 3, 4).reshape(n, ct, h, w)
    else:
        ref = F.group_norm(xin, 32, gamma, beta, eps)
    if silu:
        ref = F.silu(ref)
    if up:
        ref = F.interpolate(ref, scale_factor=2.0, mode="nearest")
    ref = ref.to(BF16).float()
    out = ops.group_norm(_nhwc(x), gamma, beta, eps, silu=silu, up2x=up, x2=_nhwc(x2) if x2 is not None else None,
                         imgs_per_sample=imgs_per_sample)
    torch.cuda.synchronize()
    return _report(f"groupnorm n{n} {h}x{w} c{c}+{c2} silu={int(silu)} up={int(up)} ips={imgs_per_sample}",
                   out.permute(0, 3, 1, 2), ref, 2 ** -7, 2e-3)


def check_layernorm(rows, c, *, add=False, seed=0):
    ops = _ops()
    x = _rand(rows, c, seed=seed + 1) * 1.5 + 0.2
    gamma = _rand(c, seed=seed + 2, dtype=torch.float32) * 0.2 + 1.0
    beta = _rand(c, seed=seed + 3, dtype=torch.float32) * 0.2
    xin = x.float()
    if add:
        rpv = rows // 4
        rv = _rand(4, c, seed=seed + 4)
        xin = (xin + rv.float().repeat_interleave(rpv, 0)).to(BF16).float()
        out, osum = ops.layer_norm(x, gamma, beta, 1e-5, add_rowvec=rv, rows_per_vec=rpv, return_sum=True)
        _report(f"layernorm-sum rows{rows} c{c}", osum, xin, 0.0, 0.0)
    else:
        out = ops.layer_norm(x, gamma, beta, 1e-5)
    ref = F.layer_norm(xin, (c,), gamma, beta, 1e-5).to(BF16).float()
    torch.cuda.synchronize()
    return _report(f"layernorm rows{rows} c{c} add={int(add)}", out, ref, 2 ** -7, 2e-3)


def check_frame_conv_small(clips, frames, h, w, cin=3, cout=3, seed=0):
    ops = _ops()
    x = _rand(clips * frames, h, w, 8, seed=seed + 1)
    wt = (_rand(cout, cin, 3, seed=seed + 2, dtype=torch.float32) * 0.5).to(BF16).float().cpu().contiguous()
    b = (_rand(cout, seed=seed + 3, dtype=torch.float32) * 0.3).to(BF16).float().cpu().contiguous()
    y = ops.frame_conv_small(x, wt, b, frames, cin)
    xs = x[..., :cin].float().reshape(clips, frames, h, w, cin).permute(0, 4, 1, 2, 3)
    ref = F.conv3d(xs, wt.cuda()[:, :, :, None, None], b.cuda(), padding=(1, 0, 0))
    ref = ref.permute(0, 2, 1, 3, 4).reshape(clips * frames, cout, h, w).to(BF16).float()
    torch.cuda.synchronize()
    return _report(f"frame_conv_small {clips}x{frames} frames {h}x{w} {cin}->{cout}", y, ref, 2 ** -7, 2e-3)


def check_timestep_embedding(seed=0):
    ops = _ops()
    t = torch.tensor([999.0, 981.0, 501.0, 1.0, 0.0, 13.0], device="cuda")
    recs = []
    for dim, round_t in ((320, False), (320, True), (1280, True), (256, False)):
        tt = t.to(BF16).float() if round_t else t
        half = dim // 2
        freq = torch.exp(-math.log(10000.0) * torch.arange(half, device="cuda", dtype=torch.float32) / half)
        arg = tt[:, None] * freq[None, :]
        ref = torch.cat([torch.cos(arg), torch.sin(arg)], dim=-1).to(BF16).float()
        out = ops.timestep_embedding(t, dim, flip_sin_to_cos=True, freq_shift=0.0, round_t_bf16=round_t)
        torch.cuda.synchronize()
        recs.append(_report(f"timestep_embedding dim{dim} round_t={int(round_t)}", out, ref, 2 ** -7, 4e-3))
    return recs[-1]


def check_layout_pool(seed=0):
    ops = _ops()
    x = _rand(3, 5, 12, 20, seed=seed + 1)
    y = ops.nchw_to_nhwc(x, 8)
    ref = F.pad(x.permute(0, 2, 3, 1), (0, 3))
    _report("nchw_to_nhwc pad8", y, ref, 0.0, 0.0)
    xf = _rand(2, 4, 16, 16, seed=seed + 2, dtype=torch.float32)
    _report("nchw_to_nhwc fp32 src", ops.nchw_to_nhwc(xf, 8)[..., :4], xf.to(BF16).permute(0, 2, 3, 1), 0.0, 0.0)
    back = ops.nhwc_to_nchw(y, 5)
    _report("nhwc_to_nchw", back, x, 0.0, 0.0)
    z = _rand(2, 8, 32, 32, seed=seed + 3)
    zp = ops.avgpool(_nhwc(z), 16, 16)
    _report("avgpool 32->16", zp.permute(0, 3, 1, 2), F.adaptive_avg_pool2d(z.float(), (16, 16)).to(BF16), 2 ** -7, 1e-3)
    zu = ops.upsample2x(_nhwc(z))
    _report("upsample2x", zu.permute(0, 3, 1, 2), F.interpolate(z.float(), scale_factor=2.0, mode="nearest"), 0.0, 0.0)
    a, b = _rand(1000, 64, seed=5), _rand(1000, 64, seed=6)
    _report("add", ops.add(a, b), (a.float() + b.float()).to(BF16), 0.0, 0.0)
    _report("silu", ops.silu(a), F.silu(a.float()).to(BF16), 2 ** -7, 1e-3)
    torch.cuda.synchronize()


def check_router(seed=0):
    ops = _ops()
    logits = _rand(13, 7, seed=seed + 1, dtype=torch.float32)
    mask = torch.tensor([1, 1, 0, 1, 0, 0, 0], dtype=torch.uint8, device="cuda")
    masked = logits.clone()
    masked[:, mask == 0] -= 1e6
    ref = torch.softmax(masked, dim=-1)
    out = ops.router_weights(logits, mask)
    _report("router_weights", out, ref, 1e-5, 1e-7)
    xs = [_rand(4, 8, 8, 64, seed=seed + 10 + i) for i in range(3)]
    w = torch.tensor([0.5, 0.3, 0.2], device="cuda")
    acc = None
    for x, wk in zip(xs, w.to(BF16)):
        term = (x * wk)
        acc = term if acc is None else acc + term
    out = ops.router_merge(xs, w)
    torch.cuda.synchronize()
    _report("router_merge", out, acc, 0.0, 0.0)


def check_cfg(seed=0):
    ops = _ops()
    eu, et = _rand(2, 4, 16, 16, seed=seed + 1), _rand(2, 4, 16, 16, seed=seed + 2)
    lat = _rand(2, 4, 16, 16, seed=seed + 3, dtype=torch.float32).to(BF16).float()
    g, sigma, sigma_next = 5.0, 3.2, 2.7
    div = math.sqrt(sigma_next ** 2 + 1)
    row = torch.tensor([981.0, sigma, sigma_next, div], device="cuda")
    eps = (eu + (g * (et - eu)).to(BF16)).to(BF16)
    x0 = lat - (torch.tensor(sigma, device="cuda") * eps).float()  # 0-dim fp32 * bf16 tensor -> bf16
    ref = (lat + (lat - x0) / sigma * (sigma_next - sigma)).to(BF16)
    nxt = torch.empty_like(eu)
    out = ops.cfg_euler(eu, et, lat, g, row, model_in_next=nxt)
    torch.cuda.synchronize()
    _report("cfg_euler (bf16 latents)", out, ref, 2 ** -7, 1e-3)
    _report("cfg_euler next_in", nxt, (ref / torch.tensor(div, device="cuda")).to(BF16), 2 ** -7, 1e-3)
    a_t, a_prev = 0.3, 0.45
    row = torch.tensor([500.0, a_t, a_prev, 1.0], device="cuda")
    epsf = eps.float()
    x0 = (lat - math.sqrt(1 - a_t) * epsf) / math.sqrt(a_t)
    ref = math.sqrt(a_prev) * x0 + math.sqrt(1 - a_prev) * epsf
    out = ops.cfg_ddim(eu, et, lat, g, row, round_latents_bf16=False)
    torch.cuda.synchronize()
    _report("cfg_ddim (fp32 latents)", out, ref, 1e-5, 1e-5)


# ------------------------------------------------------------------------------------------------
def smoke_check():
    """Tiny hot-path invocation used by __graft_entry__.smoke(): one conv, one linear, one attention."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    RESULTS.clear()
    check_linear(256, 64, 64)
    check_conv(2, 16, 16, 64, 64)
    check_attention(1, 2, 256, 256, 64)
    bad = [r for r in RESULTS if not r["ok"]]
    if bad:
        raise AssertionError(f"smoke parity failed: {bad}")


def run_all(stop_on_fail=False, group=None):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    RESULTS.clear()
    plan = [
        lambda: check_linear(256, 64, 64),
        lambda: check_linear(128, 128, 128, bias=False),
        lambda: check_linear(1000, 512, 320),
        lambda: check_linear(4096, 320, 512, out_fp32=False),
        lambda: check_linear(300, 2048, 1280, out_fp32=False, residual=True),
        lambda: check_linear(77 * 2, 768, 320, bn=64),
        lambda: check_linear(16, 320, 1280, out_fp32=False, act="silu"),
        lambda: check_linear(50000, 512, 640, out_fp32=False, bn=128),
        lambda: check_geglu(1024, 512, 2048),
        lambda: check_linear_rowvec(1024, 512, 512, 256),
        lambda: check_linear_rowvec(192, 320, 320, 64),
        lambda: check_linear_blend(512, 2048, 512),
        # lean epilogue specialisations (bias / bias+residual / GEGLU) over every BN and ragged edges
        lambda: check_linear(3000, 640, 640, out_fp32=False, residual=True),       # BN 160: 80-column warp shares
        lambda: check_linear(1100, 320, 1920, out_fp32=False),                      # BN 128, partial last M tile
        lambda: check_linear(2048, 1280, 1280, out_fp32=False, residual=True),      # BN 256, two units per warp
        lambda: check_linear(700, 256, 328, out_fp32=False, residual=True),         # n_out not a multiple of 64
        lambda: check_linear(520, 192, 40, out_fp32=False, bias=False),             # BN 64, single partial unit
        lambda: check_geglu(5000, 640, 2560),
        lambda: check_conv(2, 16, 16, 64, 64),
        lambda: check_conv(2, 32, 32, 320, 320),
        lambda: check_conv(3, 8, 8, 1280, 1280, out_fp32=False, rowvec=True, residual=True),
        lambda: check_conv(2, 64, 64, 320, 320, out_fp32=False, rowvec=True),
        lambda: check_conv(2, 16, 16, 640, 320, ksize=1, out_fp32=False, residual=True),
        lambda: check_conv(2, 16, 16, 640, 640, cin2=320, out_fp32=False),
        lambda: check_conv(2, 32, 32, 320, 320, stride=2),
        lambda: check_conv(2, 64, 64, 16, 32, stride=2),
        lambda: check_conv(2, 64, 64, 8, 16),
        lambda: check_conv(2, 24, 40, 96, 256, stride=2, out_fp32=False),
        lambda: check_conv(2, 18, 32, 128, 64),
        lambda: check_conv(2, 16, 16, 320, 320, ksize=1, out_fp32=False, scale=0.7),
        lambda: check_temporal_conv(2, 16, 8, 8, 128, 128),
        lambda: check_temporal_conv(1, 14, 16, 16, 320, 320),
        lambda: check_attention(1, 2, 256, 256, 64),
        lambda: check_attention(2, 5, 1024, 1024, 64),
        lambda: check_attention(2, 10, 1000, 77, 64),
        lambda: check_attention(1, 5, 4096, 4096, 64),
        lambda: check_attention(2, 8, 512, 512, 40),
        lambda: check_attention(2, 8, 256, 256, 80),
        lambda: check_attention(2, 8, 64, 77, 160),
        lambda: check_attention(3, 20, 64, 64, 64),
        lambda: check_attention(2, 5, 1024, 1024, 64, ramp=40.0),
        lambda: check_attention(1, 8, 300, 640, 160, ramp=20.0),
        lambda: check_attention(1, 4, 512, 2048, 64, ramp=4.0),
        # short-KV kernel (Lk <= 80, head dim <= 64): several work items per persistent CTA (ring / phase wrap-around,
        # deferred output write of the previous item), Lk = 80 / 33 / 1, partial last query tile, padded head dim
        lambda: check_attention(16, 20, 1024, 77, 64),
        lambda: check_attention(8, 16, 700, 80, 64),
        lambda: check_attention(6, 10, 1280, 33, 40),
        lambda: check_attention(4, 8, 640, 1, 64),
        lambda: check_temporal_attention(2, 16, 64, 5),
        lambda: check_temporal_attention(1, 14, 100, 10),
        lambda: check_groupnorm(2, 32, 32, 320),
        lambda: check_groupnorm(2, 16, 16, 640, up=True),
        lambda: check_groupnorm(2, 16, 16, 640, c2=320, eps=1e-5),
        lambda: check_groupnorm(4, 8, 8, 320, imgs_per_sample=2, silu=False),
        lambda: check_layernorm(1000, 512),
        lambda: check_layernorm(400, 320, add=True),
        lambda: check_layernorm(64, 1280),
        # more rows than resident warps: every warp walks several rows through its two-stage bulk-copy ring
        lambda: check_layernorm(30001, 1280),
        lambda: check_layernorm(70000, 640),
        lambda: check_layernorm(40000, 320, add=True),
        lambda: check_layernorm(9000, 2048),     # widest row: gamma / beta reloaded per row
        lambda: check_layernorm(5, 8),
        # lane groups: 8 lanes x 4 rows (C = 320), 16 x 2 (C = 640), short last step, row-vector change inside a step
        lambda: check_layernorm(40003, 320),
        lambda: check_layernorm(70001, 640),
        lambda: check_layernorm(40004, 320, add=True),
        lambda: check_layernorm(20004, 640, add=True),
        lambda: check_layernorm(3001, 256),
        lambda: check_layernorm(3001, 512),
        lambda: check_layernorm(3001, 768),
        lambda: check_layernorm(3001, 1024),
        lambda: check_layernorm(3001, 1288),
        lambda: check_layernorm(777, 72),
        lambda: check_frame_conv_small(2, 5, 16, 24),
        lambda: check_frame_conv_small(1, 1, 5, 7),          # one frame (both neighbours padded), odd pixel count
        lambda: check_frame_conv_small(3, 2, 9, 5, cin=4, cout=2),
        lambda: check_softmax_rows(300, 4096),
        lambda: check_softmax_rows(64, 16384),
        check_timestep_embedding,
        check_layout_pool,
        check_router,
        check_cfg,
    ]
    groups = {"gemm": (0, 18), "conv": (18, 32), "attn": (32, 49), "misc": (49, len(plan))}
    if group:
        lo, hi = groups[group]
        plan = plan[lo:hi]
    for fn in plan:
        n0 = len(RESULTS)
        try:
            fn()
        except Exception as e:  # keep going so that one report shows every failure
            RESULTS.append({"check": f"EXC in plan[{plan.index(fn)}]", "ok": False, "why": repr(e)[:400]})
            if stop_on_fail:
                raise
            if "CUDA error" in repr(e) or "illegal" in repr(e):
                break
        for r in RESULTS[n0:]:
            flag = "ok  " if r["ok"] else "FAIL"
            print(f"[{flag}] {r['check']}: " + ", ".join(f"{k}={v:.3g}" if isinstance(v, float) else f"{k}={v}"
                                                         for k, v in r.items() if k not in ("check", "ok")), flush=True)
    return RESULTS


if __name__ == "__main__":
    grp = sys.argv[sys.argv.index("--group") + 1] if "--group" in sys.argv else None
    res = run_all(group=grp)
    if "--json" in sys.argv:
        with open(sys.argv[sys.argv.index("--json") + 1], "w") as f:
            json.dump(res, f, indent=1)
    nbad = sum(1 for r in res if not r["ok"])
    print(f"{len(res) - nbad}/{len(res)} checks ok")
    sys.exit(1 if nbad else 0)
