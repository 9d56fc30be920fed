"""GPU parity checks of the CUDA kernels against a plain PyTorch fp32 reference of the same op on the same
bf16-quantised inputs.  Used by tests/test_kernels_gpu.py (pytest -m gpu), by __graft_entry__.smoke() and as a
stand-alone report:  python -m tests.kernel_checks  [--group attn|misc|layouts]  [--json out.json]
The GEMM kernel (linears and convolutions) is checked bit for bit by tests/test_gemm_epilogue_exact_gpu.py, its
accumulators against float64 with conv2d_ref / temporal_conv_ref below; check_linear and check_conv remain for smoke().

The `layouts` group (LAYOUT_CHECKS, run by tests/test_kernel_layouts_gpu.py) calls the kernels the way the pipelines
do -- Q/K/V as views of one fused projection, shared per-clip contexts, 17..32 frames, every bf16 GEMM epilogue
through both store paths -- against float64 references.  The checks run on DEVICE; tests/test_kernel_checks_cpu.py
sets it to "cpu" and runs them at reduced sizes over tests/ops_emulator.py to show that each one passes a correct
implementation and fails deliberately wrong ones.

The reference and verdict of each op the pipelines call live in per-launch functions that take a call's arguments and
what it wrote (linear_verdict, conv2d_verdict, temporal_conv_verdict, _attn_verdict, temporal_attention_verdict,
groupnorm_verdict, layernorm_verdict, cfg_ddim_verdict, cfg_euler_verdict, latent_encoder_verdict,
vae_latents_verdict): the layout checks call them, and so does the launch census of tests/launch_checks.py, which checks
every distinct launch of a real pipeline step with them.

Tolerances (stated per check, torch.testing semantics |out-ref| <= atol + rtol*|ref|):
  * fp32-output contractions: rtol 1e-3 / atol 1e-4 (north-star tolerance; fp32 accumulate on both sides)
    -- in the per-launch verdicts atol is raised to 2^-16 of sum |x_k w_k| where that is larger (_sum_floor)
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

from tests import error_stats as es
from tests.abi_domain import gemm_bn

BF16 = torch.bfloat16
F64 = torch.float64
RESULTS = []
DEVICE = "cuda"  # where inputs and references live (the CPU tests point this at "cpu" and patch in the emulator)


def _ops():
    from ctrl_adapter_b200 import ops
    return ops


def _sync():
    if torch.device(DEVICE).type == "cuda":
        torch.cuda.synchronize()


def _rand(*shape, scale=1.0, seed=None, dtype=BF16):
    g = torch.Generator(device=DEVICE)
    g.manual_seed(seed if seed is not None else (hash(shape) & 0xFFFF) + 17)
    return (torch.randn(*shape, generator=g, device=DEVICE, dtype=torch.float32) * scale).to(dtype)


def _report(name, out, ref, rtol, atol, extra=None, mag=None, dims=None, rows=None, units=None, gain=None, eager=None,
            unit_shape=None, stats_ref=None):
    """mag: magnitude of the largest intermediate of a multi-step bf16 epilogue (a 1-ulp flip of an intermediate is
    1 ulp of THAT magnitude, which can be several ulps of a smaller final value after cancellation).
    dims: names of out's axes -- the record then says where the worst error / tolerance ratio is; rows: the indices the
    first axis stands for when it holds a sample of a launch's images or batch entries.
    units: the axes of out that name its independent units (error_stats.BLOCKS: blocks of 4096 elements); with it the
    record also gets the direction statistics of tests/error_stats.py (bias, gain, RMS error) and fails on them, `why`
    naming the statistic.  gain: (axes of the gain groups, the gain's center or None, the axes its se clusters by or None
    for `units`); eager: an eager torch op's output on the same inputs (the gain's and RMS error's yardstick);
    unit_shape: the shape of out / ref (and eager) the axes refer to; stats_ref: the reference of the statistics when it
    differs from ref (attention: ref rounded at the kernel's output rounding, error_stats docstring)."""
    stats = None
    if units is not None:
        groups, center, gunits = gain if gain is not None else ((), None, None)
        o, r, e = out, ref if stats_ref is None else stats_ref, eager
        if unit_shape is not None:
            o, r = out.reshape(unit_shape), r.reshape(unit_shape)
            e = None if eager is None else eager.reshape(unit_shape)
        at = atol.reshape(unit_shape) if unit_shape is not None and torch.is_tensor(atol) and atol.dim() else atol
        stats = es.direction(o, r, at, units=units, gain_groups=groups, gain_units=gunits, center=center, eager=e)
    out = out.float()
    ref = ref.float()
    assert out.shape == ref.shape, f"{name}: shape {tuple(out.shape)} vs {tuple(ref.shape)}"
    err = (out - ref).abs()
    tol = atol + rtol * (ref.abs() if mag is None else torch.maximum(ref.abs(), mag.float().abs()))
    bad = (err > tol) | ~torch.isfinite(out)
    ratio = torch.where(torch.isfinite(out), torch.where(err == 0, 0.0, err / tol), math.inf)
    worst = int(ratio.argmax()) if ratio.numel() else 0
    where = None
    if dims is not None and ratio.numel():
        idx = [int(i) for i in torch.unravel_index(torch.tensor(worst), ratio.shape)]
        if rows is not None:
            idx[0] = int(rows[idx[0]])
        where = " ".join(f"{d}{i}" for d, i in zip(dims, idx))
    rec = {
        "check": name,
        "max_abs_err": float(err.max()),
        "max_ref": float(ref.abs().max()),
        "rel_fro": float((out - ref).norm() / ref.norm().clamp_min(1e-20)),
        "n_bad": int(bad.sum()),
        "n": out.numel(),
        "rtol": rtol,
        "atol": atol if isinstance(atol, float) else float(atol.max()),
        "max_err_over_tol": float(ratio.reshape(-1)[worst]) if ratio.numel() else 0.0,
        "ok": bool(bad.sum() == 0),
    }
    if where is not None:
        rec["where"] = where
    if extra:
        rec.update(extra)
    _add_direction(rec, stats)
    RESULTS.append(rec)
    return rec


def _add_direction(rec, stats):
    """the direction statistics' fields into a record; their failure fails it, `why` naming the statistic"""
    if stats is None:
        return
    ok, why = stats.pop("ok"), stats.pop("why")
    rec.update(stats)
    if not ok:
        rec["ok"] = False
        rec["why"] = "; ".join(w for w in (rec.get("why"), why) if w)


# ------------------------------------------------------------------------------------------------
# linear
# ------------------------------------------------------------------------------------------------
def check_linear(m, k, n, seed=0):
    """fp32-output linear with bias vs torch fp32 at rtol 1e-3 / atol 1e-4 (__graft_entry__.smoke)"""
    ops = _ops()
    x = _rand(m, k, seed=seed + 1)
    w = _rand(n, k, scale=1.0 / math.sqrt(k), seed=seed + 2)
    b = ops.bias_f32(_rand(n, seed=seed + 3))
    out = ops.linear(x, w, b, out_fp32=True)
    _sync()
    return _report(f"linear m{m} k{k} n{n} f32", out, x.float() @ w.float().t() + b, 1e-3, 1e-4)


# ------------------------------------------------------------------------------------------------
# convs
# ------------------------------------------------------------------------------------------------
def _nhwc(x_nchw):
    return x_nchw.permute(0, 2, 3, 1).contiguous()


def check_conv(n, h, w, cin, cout, seed=0):
    """fp32-output 3x3 conv with bias vs torch fp32 at rtol 1e-3 / atol 1e-4 (__graft_entry__.smoke)"""
    ops = _ops()
    x = _rand(n, cin, h, w, seed=seed + 1)
    wt = _rand(cout, cin, 3, 3, scale=1.0 / math.sqrt(cin * 9), seed=seed + 2)
    b = ops.bias_f32(_rand(cout, seed=seed + 3))
    ref = F.conv2d(x.float(), wt.float(), b, padding=1)
    out = ops.conv2d(_nhwc(x), ops.pack_conv_weight(wt), b, out_fp32=True)
    _sync()
    return _report(f"conv3x3 n{n} {h}x{w} c{cin}->{cout} f32", out.permute(0, 3, 1, 2), ref, 1e-3, 1e-4)


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
    _sync()
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
    x = (torch.randn(rows, cols, generator=g) * 4.0).to(DEVICE)
    x[0, :7] = 30.0  # a few dominant scores in one row
    out = ops.softmax_rows(x)
    _sync()
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
    _sync()
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
    _sync()
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
    _sync()
    return _report(f"layernorm rows{rows} c{c} add={int(add)}", out, ref, 2 ** -7, 2e-3)


def check_frame_conv_small(clips, frames, h, w, cin=3, cout=3, seed=0):
    ops = _ops()
    x = _rand(clips * frames, h, w, 8, seed=seed + 1)
    wt = (_rand(cout, cin, 3, seed=seed + 2, dtype=torch.float32) * 0.5).to(BF16).float().cpu().contiguous()
    b = (_rand(cout, seed=seed + 3, dtype=torch.float32) * 0.3).to(BF16).float().cpu().contiguous()
    y = ops.frame_conv_small(x, wt, b, frames, cin)
    xs = x[..., :cin].float().reshape(clips, frames, h, w, cin).permute(0, 4, 1, 2, 3)
    ref = F.conv3d(xs, wt.to(DEVICE)[:, :, :, None, None], b.to(DEVICE), padding=(1, 0, 0))
    ref = ref.permute(0, 2, 1, 3, 4).reshape(clips * frames, cout, h, w).to(BF16).float()
    _sync()
    return _report(f"frame_conv_small {clips}x{frames} frames {h}x{w} {cin}->{cout}", y, ref, 2 ** -7, 2e-3)


def check_timestep_embedding(seed=0):
    ops = _ops()
    t = torch.tensor([999.0, 981.0, 501.0, 1.0, 0.0, 13.0], device=DEVICE)
    recs = []
    for dim, round_t in ((320, False), (320, True), (1280, True), (256, False)):
        tt = t.to(BF16).float() if round_t else t
        half = dim // 2
        freq = torch.exp(-math.log(10000.0) * torch.arange(half, device=DEVICE, dtype=torch.float32) / half)
        arg = tt[:, None] * freq[None, :]
        ref = torch.cat([torch.cos(arg), torch.sin(arg)], dim=-1).to(BF16).float()
        out = ops.timestep_embedding(t, dim, flip_sin_to_cos=True, freq_shift=0.0, round_t_bf16=round_t)
        _sync()
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
    _sync()


def check_router(seed=0):
    ops = _ops()
    logits = _rand(13, 7, seed=seed + 1, dtype=torch.float32)
    mask = torch.tensor([1, 1, 0, 1, 0, 0, 0], dtype=torch.uint8, device=DEVICE)
    masked = logits.clone()
    masked[:, mask == 0] -= 1e6
    ref = torch.softmax(masked, dim=-1)
    out = ops.router_weights(logits, mask)
    _report("router_weights", out, ref, 1e-5, 1e-7)
    xs = [_rand(4, 8, 8, 64, seed=seed + 10 + i) for i in range(3)]
    w = torch.tensor([0.5, 0.3, 0.2], device=DEVICE)
    acc = None
    for x, wk in zip(xs, w.to(BF16)):
        term = (x * wk)
        acc = term if acc is None else acc + term
    out = ops.router_merge(xs, w)
    _sync()
    _report("router_merge", out, acc, 0.0, 0.0)


def check_cfg(seed=0):
    ops = _ops()
    eu, et = _rand(2, 4, 16, 16, seed=seed + 1), _rand(2, 4, 16, 16, seed=seed + 2)
    lat = _rand(2, 4, 16, 16, seed=seed + 3, dtype=torch.float32).to(BF16).float()
    g, sigma, sigma_next = 5.0, 3.2, 2.7
    div = math.sqrt(sigma_next ** 2 + 1)
    row = torch.tensor([981.0, sigma, sigma_next, div], device=DEVICE)
    eps = (eu + (g * (et - eu)).to(BF16)).to(BF16)
    x0 = lat - (torch.tensor(sigma, device=DEVICE) * eps).float()  # 0-dim fp32 * bf16 tensor -> bf16
    ref = (lat + (lat - x0) / sigma * (sigma_next - sigma)).to(BF16)
    nxt = torch.empty_like(eu)
    out = ops.cfg_euler(eu, et, lat, g, row, model_in_next=nxt)
    _sync()
    _report("cfg_euler (bf16 latents)", out, ref, 2 ** -7, 1e-3)
    _report("cfg_euler next_in", nxt, (ref / torch.tensor(div, device=DEVICE)).to(BF16), 2 ** -7, 1e-3)
    a_t, a_prev = 0.3, 0.45
    row = torch.tensor([500.0, a_t, a_prev, 1.0], device=DEVICE)
    epsf = eps.float()
    x0 = (lat - math.sqrt(1 - a_t) * epsf) / math.sqrt(a_t)
    ref = math.sqrt(a_prev) * x0 + math.sqrt(1 - a_prev) * epsf
    out = ops.cfg_ddim(eu, et, lat, g, row, round_latents_bf16=False)
    _sync()
    _report("cfg_ddim (fp32 latents)", out, ref, 1e-5, 1e-5)


# ------------------------------------------------------------------------------------------------
# layouts and variants the pipelines call the kernels with: float64 references on the same bf16 inputs, bf16 rounding
# applied at the kernels' rounding points (the ones tests/ops_emulator.py lists per op), tolerances of the header
# ------------------------------------------------------------------------------------------------
def _r64(t):
    """round to bf16, keep computing in float64"""
    return t.to(BF16).to(F64)


def _exact(name, ok, extra=None):
    rec = {"check": name, "ok": bool(ok)}
    if extra:
        rec.update(extra)
    RESULTS.append(rec)
    return rec


def _attn_ref64(q, k, v, kv_idx, scale, chunk=256):
    """q [B, Lq, H, d], k / v [Bk, Lk, H, d]; query batch b attends to K/V batch kv_idx[b].  float64, query axis in chunks
    so that the score matrix stays small."""
    qd = q.to(F64).permute(0, 2, 1, 3)
    kd = k.to(F64).permute(0, 2, 1, 3)[kv_idx]
    vd = v.to(F64).permute(0, 2, 1, 3)[kv_idx]
    out = torch.empty(qd.shape[:3] + (vd.shape[3],), dtype=F64, device=q.device)
    for i in range(0, qd.shape[2], chunk):
        p = torch.softmax(qd[:, :, i:i + chunk] @ kd.transpose(-1, -2) * scale, dim=-1)
        out[:, :, i:i + chunk] = p @ vd
    return out.permute(0, 2, 1, 3)


def _attn_verdict(name, q, k, v, kv_idx, scale, out, rows=None):
    """check_attention's criteria (rtol 2e-2 / atol 2e-3, and at most 2x the error of torch's bf16 SDPA on the same
    inputs), the SDPA bound applied to every (batch, head) on its own so that one wrong head cannot hide in the totals.
    rows: the launch's batch indices of q / out when they hold a sample of its batch entries."""
    ref = _attn_ref64(q, k, v, kv_idx, scale)
    sd = F.scaled_dot_product_attention(*(t.permute(0, 2, 1, 3) for t in (q, k[kv_idx], v[kv_idx])), scale=scale)
    err_bh = (out.to(F64) - ref).abs().amax(dim=(1, 3))              # [B, H]
    sd_bh = (sd.permute(0, 2, 1, 3).to(F64) - ref).abs().amax(dim=(1, 3))
    ratio = err_bh / (2.0 * sd_bh + 1e-3)
    wb, wh = divmod(int(err_bh.argmax()), err_bh.shape[1])
    rb, rh = divmod(int(ratio.argmax()), ratio.shape[1])
    lb = (lambda i: i) if rows is None else (lambda i: int(rows[i]))
    # gain per (batch, head) about the mean of V over the keys: a wrong softmax temperature moves every output of a row
    # toward or away from it; torch's bf16 SDPA is the yardstick of the gain and of the RMS error per (batch, head)
    vmean = v.to(F64)[kv_idx].mean(dim=1, keepdim=True)
    sd = sd.permute(0, 2, 1, 3)
    rec = _report(name, out, ref, 2e-2, 2e-3, dims=("b", "q", "h", "d"), rows=rows, units=(0, 1, 2),
                  gain=((0, 2), vmean, None), eager=sd, stats_ref=_r64(ref), extra={
        "sdpa_bf16_max_err": float(sd_bh.max()), "worst_bh": f"b{lb(wb)}h{wh}", "worst_bh_err": float(err_bh[wb, wh]),
        "worst_bh_sdpa_err": float(sd_bh[wb, wh]), "max_bh_err_over_2x_sdpa": float(ratio[rb, rh]),
        "max_ratio_bh": f"b{lb(rb)}h{rh}"})
    if float(ratio.max()) > 1.0:
        rec["ok"] = False
        rec["why"] = "; ".join(w for w in (f"(batch, head) b{lb(rb)}h{rh}: error larger than 2x torch bf16 SDPA",
                                            rec.get("why")) if w)
    return rec


def _pad_heads(t, dp):
    """[B, L, H, d] -> [B, L, H, dp]: the zero-padded head layout the packed projection weights produce"""
    return F.pad(t, (0, dp - t.shape[-1]))


def check_attention_fused_qkv(b, heads, l, d, seed=0):
    """Self-attention on Q / K / V column views of ONE [B, L, 3 * H * Dp] projection (row stride 3 * H * Dp), as
    layers.Attention.forward slices them."""
    ops = _ops()
    dp = (d + 63) // 64 * 64
    inner = heads * dp
    q, k, v = (_rand(b, l, heads, d, seed=seed + i) for i in (1, 2, 3))
    qkv = torch.stack([_pad_heads(t, dp) for t in (q, k, v)], dim=2).reshape(b, l, 3 * inner)
    out = ops.attention(qkv[:, :, :inner], qkv[:, :, inner:2 * inner], qkv[:, :, 2 * inner:], heads, dp, d ** -0.5)
    _sync()
    out = out.reshape(b, l, heads, dp)[..., :d]
    return _attn_verdict(f"attention fused-qkv b{b} h{heads} l{l} d{d}", q, k, v, torch.arange(b, device=q.device),
                         d ** -0.5, out)


def check_attention_cross_kv(b, heads, lq, lk, d, kv_batch_div=1, seed=0):
    """Cross-attention with K / V as the two halves of one [B / kv_batch_div, Lk, 2 * H * Dp] projection of the context.
    kv_batch_div > 1: the frames of a clip share their clip's context, and every clip's context is different."""
    ops = _ops()
    dp = (d + 63) // 64 * 64
    inner = heads * dp
    bk = b // kv_batch_div
    q = _rand(b, lq, heads, d, seed=seed + 1)
    k, v = _rand(bk, lk, heads, d, seed=seed + 2), _rand(bk, lk, heads, d, seed=seed + 3)
    kv = torch.stack([_pad_heads(t, dp) for t in (k, v)], dim=2).reshape(bk, lk, 2 * inner)
    out = ops.attention(_pad_heads(q, dp).reshape(b, lq, inner), kv[:, :, :inner], kv[:, :, inner:], heads, dp,
                        d ** -0.5, kv_batch_div=kv_batch_div)
    _sync()
    out = out.reshape(b, lq, heads, dp)[..., :d]
    kv_idx = torch.arange(b, device=q.device) // kv_batch_div
    return _attn_verdict(f"attention cross-kv b{b} h{heads} lq{lq} lk{lk} d{d} kv_div{kv_batch_div}", q, k, v, kv_idx,
                         d ** -0.5, out)


def check_temporal_attention_fused(clips, frames, hw, heads, seed=0):
    """Frame-axis attention on Q / K / V column views of one [rows, 3 * inner] projection (row_stride 3 * inner), as the
    temporal transformers of the UNets and the video adapter call it.  Tolerance of check_temporal_attention."""
    ops = _ops()
    inner = heads * 64
    qkv = _rand(clips * frames * hw, 3 * inner, seed=seed + 1)
    q, k, v = qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:]
    out = ops.temporal_attention(q, k, v, clips, frames, hw, heads, 0.125, row_stride=3 * inner)
    _sync()
    return temporal_attention_verdict(f"temporal_attention fused-qkv b{clips} f{frames} hw{hw} h{heads}", q, k, v,
                                      clips, frames, hw, heads, 0.125, out)


def temporal_attention_verdict(name, q, k, v, clips, frames, hw, heads, scale, out):
    """ops.temporal_attention vs float64 at check_temporal_attention's tolerance, worst frame reported"""
    def seq(t):  # rows (clip, frame, pixel) -> [clip, pixel, head, frame, 64]
        return t.to(F64).reshape(clips, frames, hw, heads, 64).permute(0, 2, 3, 1, 4)
    p = torch.softmax(seq(q) @ seq(k).transpose(-1, -2) * scale, dim=-1)
    ref = (p @ seq(v)).permute(0, 3, 1, 2, 4).reshape(clips, frames, hw, heads * 64)
    out = out.reshape(ref.shape)
    err_f = (out.to(F64) - ref).abs().amax(dim=(0, 2, 3))  # worst error per frame
    wf = int(err_f.argmax())
    # units: the (clip, pixel, head) sequences; gain about each sequence's mean of V over the frames; yardstick: torch's
    # bf16 SDPA on the same sequences
    vmean = seq(v).mean(dim=3, keepdim=True).permute(0, 3, 1, 2, 4)

    def seq16(t):
        return t.reshape(clips, frames, hw, heads, 64).permute(0, 2, 3, 1, 4)
    sd = F.scaled_dot_product_attention(seq16(q), seq16(k), seq16(v), scale=scale).permute(0, 3, 1, 2, 4)
    return _report(name, out, ref, 2e-2, 6e-3, {"worst_frame": wf, "worst_frame_err": float(err_f[wf])},
                   dims=("clip", "frame", "pixel", "ch"), units=(0, 2, 3), gain=((), vmean, None), eager=sd,
                   unit_shape=(clips, frames, hw, heads, 64), stats_ref=_r64(ref))


EPILOGUES = ("bias", "bias_silu", "bias_scale", "bias_scale_res", "rowvec", "bias_res", "rowvec_res", "bias_res_blend",
             "rowvec_res_blend", "geglu")


def check_gemm_epilogue(kind, m, k, n, rows_per_vec=0, seed=0):
    """One bf16 GEMM epilogue combination (`kind`: parts of EPILOGUES joined by '_'), run twice.  The first run writes a
    fresh aligned output and is checked against the float64 reference.  The second writes channels [4, 4 + n) of a
    wider buffer, with the residual / blend source / row vector at the same offset in buffers of that width: the 8-byte
    base offset sends the storers down the element-wise drain, which must reproduce the first run bit for bit and leave
    the bytes around the slice alone."""
    ops = _ops()
    parts = kind.split("_")
    geglu = kind == "geglu"
    x = _rand(m, k, seed=seed + 1)
    w_rows = 2 * n if geglu else n
    w = _rand(w_rows, k, scale=k ** -0.5, seed=seed + 2)
    b = _rand(w_rows, seed=seed + 3) if ("bias" in parts or geglu) else None
    scale = 0.7 if "scale" in parts else 1.0
    rv = _rand(m // rows_per_vec, n, seed=seed + 4) if "rowvec" in parts else None
    res = _rand(m, n, seed=seed + 5) if "res" in parts else None
    xs = _rand(m, n, seed=seed + 6) if "blend" in parts else None
    alpha = torch.sigmoid(torch.tensor([0.3], device=DEVICE)).to(BF16).float() if xs is not None else None
    act = ops.ACT_GEGLU if geglu else ops.ACT_SILU if "silu" in parts else ops.ACT_NONE
    wk, bk = ops.pack_geglu_weight(w, b, 256) if geglu else (w, b)
    bias = ops.bias_f32(bk)
    kw = dict(act=act, out_scale=scale, rows_per_vec=rows_per_vec, blend_alpha=alpha)
    call = dict(x=x, w=wk, bias=bias, rowvec=rv, residual=res, blend_src=xs, out=None, out_fp32=False, bn=0, **kw)
    out = ops.linear(**call)

    def slot(t):  # the same values in columns [4, 4 + n) of an [rows, n + 16] buffer
        if t is None:
            return None
        buf = _rand(t.shape[0], n + 16, seed=seed + 9)
        buf[:, 4:4 + n] = t
        return buf[:, 4:4 + n]
    obuf = torch.full((m, n + 16), 7.0, device=DEVICE, dtype=BF16)
    ops.linear(x, wk, bias, rowvec=slot(rv), residual=slot(res), blend_src=slot(xs), out=obuf[:, 4:4 + n], **kw)
    _sync()
    name = f"gemm epilogue {kind} m{m} k{k} n{n} bn{gemm_bn(w_rows, geglu)}"
    linear_verdict(name, call, out, lambda **changes: ops.linear(**{**call, **changes}))
    same = torch.equal(obuf[:, 4:4 + n].view(torch.int16), out.view(torch.int16))
    n_diff = int((obuf[:, 4:4 + n].view(torch.int16) != out.view(torch.int16)).sum())
    untouched = bool((obuf[:, :4] == 7.0).all()) and bool((obuf[:, 4 + n:] == 7.0).all())
    return _exact(f"{name} element-wise drain == aligned, bytes around the slice kept", same and untouched,
                  {"n_diff": n_diff, "n": out.numel(), "untouched": untouched})


def check_temporal_conv_epilogue(b, f, h, w, c, cout, seed=0):
    """Conv3d (3,1,1) over the frames with row vector + residual + AlphaBlender in one epilogue (the temporal ResNet's
    convs in the video adapter).  f = 1: both frame taps fall on the zero padding."""
    ops = _ops()
    x = _rand(b * f, h, w, c, seed=seed + 1)
    wt = _rand(cout, c, 3, 1, 1, scale=(3 * c) ** -0.5, seed=seed + 2)
    bias = ops.bias_f32(_rand(cout, seed=seed + 3))
    rv = _rand(b * f, cout, seed=seed + 4)
    res = _rand(b * f, h, w, cout, seed=seed + 5)
    xs = _rand(b * f, h, w, cout, seed=seed + 6)
    alpha = torch.sigmoid(torch.tensor([-0.4], device=DEVICE)).to(BF16).float()
    call = dict(x=x, w_packed=ops.pack_conv_weight(wt), bias=bias, frames=f, rowvec=rv, residual=res, blend_src=xs,
                blend_alpha=alpha)
    out = ops.temporal_conv(**call)
    _sync()
    return temporal_conv_verdict(f"temporal_conv rowvec+res+blend b{b} f{f} {h}x{w} c{c}->{cout}", call, out)


# ---- per-launch verdicts of the GEMM family: the reference and tolerance of one call, given its arguments `a` (the op's
# parameter names) and what it wrote; shared with tests/launch_checks.py ----
def _epilogue_chain64(v, *, act=0, scale=1.0, rv=None, res=None, xs=None, alpha=None, multi=False):
    """The bf16 epilogue of the GEMM kernels applied in float64 to the pre-activation v (bias included): round, SiLU,
    scale, + row vector, + residual, AlphaBlender, rounding after each step.  -> (ref, rtol, mag).
    Tolerance: one rounding: 1 ulp; bias + rounding + blend: 1 ulp of the largest intermediate; a row vector and / or
    residual before it (or `multi`): 2 ulps of the largest intermediate, since two boundary flips can stack."""
    v = _r64(v)
    if act == 1:
        v = _r64(F.silu(v))
    if scale != 1.0:
        v = _r64(v * scale)
    mag = v.abs()
    if rv is not None:
        v = _r64(v + rv)
        mag = torch.maximum(mag, v.abs())
    if res is not None:
        v = _r64(v + res)
        mag = torch.maximum(torch.maximum(mag, res.abs()), v.abs())
    if xs is not None:
        a = alpha.to(F64).reshape(())
        v = _r64(_r64(a * xs) + _r64(_r64(1.0 - a) * v))
        mag = torch.maximum(torch.maximum(mag, xs.abs()), v.abs())
    multi = multi or rv is not None or (res is not None and xs is None)
    return v, 2 ** -6 if multi else 2 ** -7, mag if (multi or xs is not None) else None


def _f32_epilogue_verdict(name, pre, out, a, rv, dims, rows=None):
    """the fp32-output epilogue applied in float64 to the kernel's own fp32 pre-activation (bias included): SiLU rounded
    to bf16, x out_scale, + row vector rounded to bf16, + residual NOT rounded (include/ctrl_adapter_b200.h).  A rounding
    step may flip one bf16 ulp of its intermediate (rtol 2^-7 of the largest one); without one the tolerance is a few
    fp32 ulps of the largest intermediate, so a rounded residual sum (half a bf16 ulp) fails."""
    v = pre.to(F64)
    rounded = a["act"] == 1 or rv is not None
    if a["act"] == 1:
        v = _r64(F.silu(v))
    if a["out_scale"] != 1.0:
        v = v * a["out_scale"]
    mag = v.abs()
    if rv is not None:
        v = _r64(v + rv)
        mag = torch.maximum(mag, v.abs())
    if a["residual"] is not None:
        v = v + a["residual"].to(F64)
        mag = torch.maximum(mag, v.abs())
    return _report(name, out, v, 2 ** -7 if rounded else 2 ** -20, 1e-6, mag=mag, dims=dims, rows=rows,
                   units=tuple(range(out.dim() - 1)))


def _sum_floor(abs_sum):
    """absolute floor of the fp32-accumulation checks: atol 1e-4, raised to 2^-16 of sum |x_k w_k| where that is larger.
    Where the products cancel, an fp32 sum over K terms is off by a multiple of 2^-24 of sum |x_k w_k| that grows with
    K.  Measured on an H100 80GB HBM3 (400 W power limit): the GEMM kernel's fp32 output of the 3x3 convolutions over
    1280 channels (K = 11520) of the video UNets is off by up to 1.6e-4 near zero outputs, about 2^-18 of their sum
    |x_k w_k|, where torch's own fp32 convolution (TF32 off) on the same values is off by 1.2e-5: the tensor-core
    accumulation over the whole K is about 10x less precise than cuDNN's, yet far below a bf16 ulp of the outputs the
    pipelines consume.  A wrong tap, channel or row is off by O(|x_k w_k|), far above 2^-16 of the sum."""
    return torch.clamp(abs_sum * 2.0 ** -16, min=1e-4)


_PRE_ONLY = dict(act=0, out_scale=1.0, rowvec=None, residual=None, blend_src=None, blend_alpha=None, out=None,
                 out_fp32=True)


def linear_verdict(name, a, out, rerun, rows=None):
    """ops.linear.  fp32 output: the float64 product (x out_scale) at rtol 1e-3 / atol 1e-4; with SiLU, a row vector or
    a residual, the pre-activation at that tolerance and then _f32_epilogue_verdict on it.  bf16 output:
    rerun(**changes) -- the same call with fp32 output and only the bias (same kernel, tiles and summation order) -- vs
    float64 at that tolerance, then the epilogue's rounding chain applied in float64 to that pre-activation.  A
    pre-activation within an fp32 ulp or two of a bf16 rounding tie rounds either way depending on the summation order
    (cuBLAS's own fp32 result rounds ~3300 of the 25.6 M pre-activations of a 5000-row GEGLU away from the exact value),
    and SiLU, GELU x value or a scale carry that one-ulp flip past the output tolerance, so the epilogue is checked
    against the input it was given.  rows: evaluate the reference on these rows only (an index tensor; the kernel still
    runs on the whole launch)."""
    if rows is not None:  # the row-indexed operands and outputs, restricted to `rows`
        pick = lambda t: None if t is None else t[rows]  # noqa: E731
        full_rerun, x_rows = rerun, pick(a["x"]).contiguous()
        # the re-run on those rows alone: a row's K summation does not depend on the other rows of the launch
        rerun = lambda **changes: full_rerun(**dict(changes, x=x_rows))  # noqa: E731
        rv_rows = None if a["rowvec"] is None else rows // a["rows_per_vec"]
        a = dict(a, x=pick(a["x"]), residual=pick(a["residual"]), blend_src=pick(a["blend_src"]), rows_per_vec=1,
                 rowvec=None if rv_rows is None else a["rowvec"][rv_rows])
        out = pick(out)
    x, w, bias, act = a["x"], a["w"], a["bias"], a["act"]
    exact = x.to(F64) @ w.to(F64).t()
    atol = _sum_floor(x.to(F64).abs() @ w.to(F64).abs().t())
    if bias is not None:
        exact = exact + bias.to(F64)
    dims = ("row", "col")
    rv = a["rowvec"]
    if rv is not None:
        rv = rv.to(F64).repeat_interleave(a["rows_per_vec"], dim=0)
    if a["out_fp32"]:
        if act == 2 or a["blend_src"] is not None:
            raise NotImplementedError("linear: fp32 output with GEGLU or blend")
        if act == 0 and rv is None and a["residual"] is None:
            ref = exact * a["out_scale"] if a["out_scale"] != 1.0 else exact
            return [_report(name, out, ref, 1e-3, atol * abs(a["out_scale"]), dims=dims, units=(0,))]
        pre = rerun(**_PRE_ONLY)
        _sync()
        return [_report(f"{name} pre-activation", pre, exact, 1e-3, atol, dims=dims, units=(0,)),
                _f32_epilogue_verdict(name, pre, out, a, rv, dims)]
    pre = rerun(**_PRE_ONLY)
    _sync()
    recs = [_report(f"{name} pre-activation", pre, exact, 1e-3, atol, dims=dims, units=(0,))]
    if act == 2:  # GEGLU: value / gate columns interleaved per 256-wide tile (ops.pack_geglu_weight)
        if a["out_scale"] != 1.0 or any(a[k] is not None for k in ("rowvec", "residual", "blend_src")):
            raise NotImplementedError("linear: GEGLU with a further epilogue")
        m, n = pre.shape[0], w.shape[0] // 2
        p4 = pre.to(F64).reshape(m, n // 128, 2, 128)
        h = _r64(torch.cat([p4[:, :, 0].reshape(m, n), p4[:, :, 1].reshape(m, n)], dim=1))
        recs.append(_report(name, out, _r64(h[:, :n] * _r64(F.gelu(h[:, n:]))), 2 ** -6, 2e-3, dims=dims, units=(0,)))
        return recs
    f64 = (lambda t: None if t is None else t.to(F64))
    ref, rtol, mag = _epilogue_chain64(
        pre.to(F64), act=act, scale=a["out_scale"], res=f64(a["residual"]), xs=f64(a["blend_src"]),
        alpha=a["blend_alpha"], rv=rv)
    recs.append(_report(name, out, ref, rtol, 1e-3, mag=mag, dims=dims, units=(0,)))
    return recs


def conv2d_ref(a, rows=None, dtype=F64):
    """The convolution of an ops.conv2d call (arguments `a`) in `dtype`: F.conv2d on the concatenated sources with the
    call's padding (pad (0, 1): one zero row / column at the bottom / right), plus the bias when the call has one.
    -> (out, sum |x_k w_k|), both channels-last [N, Ho, Wo, Cout].  rows: these images only."""
    x, x2, w, bias = a["x"], a.get("x2"), a["w_packed"], a.get("bias")
    k, stride = a["ksize"], a["stride"]
    ii = slice(None) if rows is None else torch.tensor(rows, device=x.device)
    xin = x[ii] if x2 is None else torch.cat([x[ii], x2[ii]], dim=3)
    ct, cout = xin.shape[3], w.shape[0]
    kpt = a["k_per_tap"] if a.get("k_per_tap") is not None else w.shape[1] // (k * k)
    wt = w.to(dtype).reshape(cout, k * k, kpt)[:, :, :ct].permute(0, 2, 1).reshape(cout, ct, k, k)
    xd = xin.to(dtype).permute(0, 3, 1, 2)
    pad = (k // 2, k // 2) if a.get("pad") is None else tuple(a["pad"])
    if pad == (0, 1):
        xd, padding = F.pad(xd, (0, 1, 0, 1)), 0
    else:
        padding = pad[0]

    def conv(x_, w_, b_=None):
        return F.conv2d(x_, w_, b_, stride=stride, padding=padding).permute(0, 2, 3, 1)
    return conv(xd, wt, None if bias is None else bias.to(dtype)), conv(xd.abs(), wt.abs())


def conv2d_verdict(name, a, out, rerun, rows=None):
    """ops.conv2d: the checks of linear_verdict on the channels-last output [N, Ho, Wo, Cout] against conv2d_ref.
    rows: evaluate the reference on these images only (the kernel still runs on the whole launch)."""
    if a["act"] == 2:
        raise NotImplementedError("conv2d: GEGLU")
    exact, abs_sum = conv2d_ref(a, rows)
    atol = _sum_floor(abs_sum)
    del abs_sum
    # torch's own fp32 convolution on the same values: how far an fp32 accumulation of this launch lands from float64
    fp32_err = float((conv2d_ref(a, rows, torch.float32)[0] - exact).abs().max())
    ii = slice(None) if rows is None else torch.tensor(rows, device=out.device)
    dims = ("img", "y", "x", "ch")
    f64 = (lambda t: None if t is None else t[ii].to(F64))
    if a["out_fp32"] and (a["act"] != 0 or a["rowvec"] is not None or a["residual"] is not None):
        if a["blend_src"] is not None:
            raise NotImplementedError("conv2d: fp32 output with a blend")
        pre = rerun(**_PRE_ONLY)[ii]
        _sync()
        rv = a["rowvec"]
        if rv is not None:
            rv = (rv[ii] if rv.shape[0] > 1 else rv).to(F64)[:, None, None, :]
        return [_report(f"{name} pre-activation", pre, exact, 1e-3, atol, dims=dims, rows=rows, units=(0, 1, 2)),
                _f32_epilogue_verdict(name, pre, out[ii], {**a, "residual": f64(a["residual"])}, rv, dims, rows)]
    if a["out_fp32"]:
        if a["blend_src"] is not None:
            raise NotImplementedError("conv2d: fp32 output with a blend")
        ref = exact * a["out_scale"] if a["out_scale"] != 1.0 else exact
        if a["residual"] is not None:
            ref = ref + f64(a["residual"])
        return [_report(name, out[ii], ref, 1e-3, atol * abs(a["out_scale"]), {"torch_fp32_max_err": fp32_err},
                        dims=dims, rows=rows, units=(0, 1, 2))]
    pre = rerun(**_PRE_ONLY)[ii]
    _sync()
    recs = [_report(f"{name} pre-activation", pre, exact, 1e-3, atol, {"torch_fp32_max_err": fp32_err}, dims=dims,
                    rows=rows, units=(0, 1, 2))]
    del exact
    rv = a["rowvec"]
    if rv is not None:
        rv = (rv[ii] if rv.shape[0] > 1 else rv).to(F64)[:, None, None, :]
    ref, rtol, mag = _epilogue_chain64(pre.to(F64), act=a["act"], scale=a["out_scale"], rv=rv, res=f64(a["residual"]),
                                       xs=f64(a["blend_src"]), alpha=a["blend_alpha"])
    recs.append(_report(name, out[ii], ref, rtol, 1e-3, mag=mag, dims=dims, rows=rows, units=(0, 1, 2)))
    return recs


def temporal_conv_ref(a, frames=None):
    """The float64 Conv3d (3, 1, 1) of an ops.temporal_conv call (arguments `a`) over the frames, zero frames at both
    ends of every clip, plus the bias when the call has one.  -> (out, sum |x_k w_k|), both [clip, frame, pixel,
    Cout].  frames: these output frames (of every clip) only."""
    x, w, bias, f = a["x"], a["w_packed"], a.get("bias"), a["frames"]
    bf, h, w_, c = x.shape
    b, cout = bf // f, w.shape[0]
    fi = list(range(f)) if frames is None else list(frames)
    x4 = x.reshape(b, f, h * w_, c)
    wd = w.to(F64).reshape(cout, 3, w.shape[1] // 3)[:, :, :c]
    acc = torch.zeros(b, len(fi), h * w_, cout, dtype=F64, device=x.device)
    abs_sum = torch.zeros_like(acc)
    for j, fr in enumerate(fi):
        for t in range(3):
            if 0 <= fr + t - 1 < f:
                xt = x4[:, fr + t - 1].to(F64)
                acc[:, j] += xt @ wd[:, t].t()
                abs_sum[:, j] += xt.abs() @ wd[:, t].abs().t()
    if bias is not None:
        acc += bias.to(F64)
    return acc, abs_sum


def temporal_conv_verdict(name, a, out, frames=None):
    """ops.temporal_conv (Conv3d (3, 1, 1) over the frames, zero frames at both ends of every clip): the float64 chain
    with check_temporal_conv_epilogue's tolerance, 2 ulps of the largest intermediate (the op has no fp32 output).
    frames: evaluate these output frames (of every clip) only."""
    f = a["frames"]
    bf, h, w_, _ = a["x"].shape
    b, cout = bf // f, a["w_packed"].shape[0]
    fi = list(range(f)) if frames is None else list(frames)
    acc = temporal_conv_ref(a, fi)[0]
    rv = a["rowvec"]
    if rv is not None:
        rv = rv.to(F64).reshape(b, f, 1, cout)[:, fi] if rv.shape[0] > 1 else rv.to(F64).reshape(1, 1, 1, cout)
    f64 = (lambda t: None if t is None else t.reshape(b, f, h * w_, cout)[:, fi].to(F64))
    ref, rtol, mag = _epilogue_chain64(acc, rv=rv, res=f64(a["residual"]), xs=f64(a["blend_src"]),
                                       alpha=a["blend_alpha"], multi=True)
    return _report(name, out.reshape(b, f, h * w_, cout)[:, fi], ref, rtol, 1e-3, mag=mag,
                   dims=("clip", "frame", "pixel", "ch"), rows=None, units=(0, 1, 2))


def check_linear_f32_scale(m, n, k, seed=0):
    """fp32 output with out_scale: the attention scores q k^T * C^-0.5 of the VAE mid block."""
    ops = _ops()
    q, kk = _rand(m, k, seed=seed + 1), _rand(n, k, seed=seed + 2)
    call = dict(x=q, w=kk, bias=None, act=0, residual=None, rowvec=None, rows_per_vec=0, blend_src=None,
                blend_alpha=None, out_scale=k ** -0.5, out=None, out_fp32=True, bn=0)
    out = ops.linear(**call)
    _sync()
    return linear_verdict(f"linear f32 out_scale m{m} n{n} k{k}", call, out, None)[0]


def _bf16_ulp(a):
    e = torch.frexp(a.abs().clamp_min(2.0 ** -126))[1]
    return torch.ldexp(torch.ones_like(a), e - 8)


def _chain_verdict(name, out, ref, tol, extra=None):
    """out vs a float64 chain at an element-wise tolerance `tol` (the scheduler steps), and the direction statistics of
    tests/error_stats.py over blocks of 4096 elements (elements with |ref| <= tol left out of the bias)"""
    err = (out.to(F64) - ref).abs()
    ratio = torch.where(torch.isfinite(out), err / tol, math.inf)
    bad = int((ratio > 1.0).sum())
    rec = {"max_abs_err": float(err.max()), "max_err_over_tol": float(ratio.max()), "n_bad": bad, "n": out.numel()}
    rec.update(extra or {})
    del err, ratio
    stats = es.direction(out, ref, None, tol=tol)
    rec = _exact(name, bad == 0 and rec.get("model_in_next_ok", True), rec)
    _add_direction(rec, stats)
    return rec


def _next_input_ok(nxt, out, div):
    """the next model input: bf16(latents' / div) within one bf16 ulp of the latents the kernel wrote, over div"""
    if nxt is None:
        return True
    want = out.to(F64) / div
    return bool(((nxt.to(F64) - want).abs() <= _bf16_ulp(want)).all())


def check_cfg_ddim_layout(v_prediction, bf16_latents, shape=(2, 4, 16, 32, 32), seed=0):
    """Classifier-free guidance + DDIM step as the I2VGen-XL loop runs it (tolerance: cfg_ddim_verdict)."""
    ops = _ops()
    eu, et = _rand(*shape, seed=seed + 1), _rand(*shape, seed=seed + 2)
    lat = _rand(*shape, seed=seed + 3, dtype=torch.float32)
    if bf16_latents:
        lat = lat.to(BF16).float()
    call = dict(eps_uncond=eu, eps_text=et, latents=lat, guidance=9.0,
                step_row=torch.tensor([500.0, 0.3, 0.45, 0.0], device=DEVICE), latents_out=None,
                model_in_next=torch.empty(shape, device=DEVICE, dtype=BF16), round_latents_bf16=bf16_latents,
                v_prediction=v_prediction)
    out = ops.cfg_ddim(**call)
    _sync()
    return cfg_ddim_verdict(f"cfg_ddim {'v' if v_prediction else 'epsilon'} {'bf16' if bf16_latents else 'fp32'} latents",
                            call, out, call["model_in_next"])


def cfg_ddim_verdict(name, a, out, nxt):
    """ops.cfg_ddim.  bf16 latents: within 1 bf16 ulp of the float64 chain with the kernel's rounding points (ulp of the
    largest intermediate of the chain, so that a quotient rounded to one side of a tie in fp32 cannot fail it); fp32
    latents: rtol 1e-6 of the chain's term magnitudes.  The next model input is the written latents in bf16, exactly."""
    bf16_latents, g, row = a["round_latents_bf16"], a["guidance"], a["step_row"]
    rr = _r64 if bf16_latents else (lambda t: t)
    at32, ap32 = row[1:2].cpu(), row[2:3].cpu()  # the fp32 values the kernel reads; 1 - a is an fp32 subtraction
    sa, sb, sap, sbp = (rr(t.to(F64).sqrt().to(out.device)) for t in (at32, 1.0 - at32, ap32, 1.0 - ap32))
    u, c, x = a["eps_uncond"].to(F64), a["eps_text"].to(F64), a["latents"].to(F64)
    mo = _r64(u + _r64(g * _r64(c - u)))
    if a["v_prediction"]:
        x0 = rr(rr(sa * x) - rr(sb * mo))
        eps = rr(rr(sa * mo) + rr(sb * x))
        terms = [sap * (sa * x.abs() + sb * mo.abs()), sbp * (sa * mo.abs() + sb * x.abs())]
    else:
        x0 = rr(rr(x - rr(sb * mo)) / sa)
        eps = mo
        terms = [sap * (x.abs() + sb * mo.abs()) / sa, sbp * mo.abs()]
    t1, t2 = rr(sap * x0), rr(sbp * eps)
    ref = rr(t1 + t2)
    if bf16_latents:
        tol = _bf16_ulp(torch.stack([ref.abs(), x0.abs(), eps.abs(), t1.abs(), t2.abs()]).amax(dim=0))
    else:
        tol = 1e-6 * torch.maximum(ref.abs(), terms[0] + terms[1])
    nxt_ok = nxt is None or torch.equal(nxt, out.to(BF16))
    return _chain_verdict(name, out, ref, tol, {"model_in_next_ok": nxt_ok})


def cfg_euler_verdict(name, a, out, nxt, v_prediction=False):
    """ops.cfg_euler (epsilon) / ops.cfg_euler_v (v-prediction, guidance per frame of [clips, frames, ...] latents) vs the
    float64 chain with the kernel's rounding points.  bf16 latents: within 1 bf16 ulp of the largest intermediate; fp32
    latents: rtol 1e-6 of the chain's term magnitudes.  The next model input: within 1 bf16 ulp of the written latents
    over bf16(sqrt(sigma_next^2 + 1))."""
    row = a["step_row"].cpu()
    s32, sn32 = row[1:2], row[2:3]  # fp32 scalars as the kernel reads them
    sigma, sigma_next = float(s32), float(sn32)
    div = float(row[3:4].to(BF16))
    u, c, x = a["eps_uncond"].to(F64), a["eps_text"].to(F64), a["latents"].to(F64)
    if v_prediction:
        f = a["frames"]
        g = a["guidance_per_frame"].to(F64).reshape(1, f, *([1] * (x.dim() - 2)))
        mo = _r64(u + _r64(g * _r64(c - u)))
        c_out = float((-s32 / torch.sqrt(s32 * s32 + 1.0)).to(BF16))  # fp32 arithmetic, one bf16 rounding
        t1 = _r64(mo * c_out)
        x0 = t1 + x / float(s32 * s32 + 1.0)
    else:
        mo = _r64(u + _r64(float(torch.tensor(a["guidance"], dtype=torch.float32)) * _r64(c - u)))
        t1 = _r64(float(s32.to(BF16)) * mo)
        x0 = x - t1
    d = (x - x0) / sigma * (sigma_next - sigma)
    ref = x + d
    # the fp32 evaluation of the chain: a few fp32 ulps of its largest term.  Where the step cancels the latents (sigma
    # 700 -> 0 in one or two Karras steps: x' = x0 of O(1) from x of O(700)) this exceeds a bf16 ulp of the result
    tol32 = 1e-6 * torch.stack([ref.abs(), x.abs(), (x.abs() + t1.abs()) * abs((sigma_next - sigma) / sigma)]).amax(dim=0)
    if a["round_latents_bf16"]:
        ref = _r64(ref)
        tol = _bf16_ulp(torch.stack([ref.abs(), mo.abs(), t1.abs(), x0.abs()]).amax(dim=0)) + tol32
    else:
        tol = tol32
    return _chain_verdict(name, out, ref, tol, {"model_in_next_ok": _next_input_ok(nxt, out, div)})


def check_cfg_euler_layout(v_prediction, bf16_latents, shape=(2, 14, 4, 36, 64), seed=0):
    """Classifier-free guidance + Euler step as the SDXL loop (epsilon) and the SVD loop (v-prediction, guidance per
    frame of [clips, frames, 4, h, w] latents) run it, against the float64 chain of cfg_euler_verdict."""
    ops = _ops()
    eu, et = _rand(*shape, seed=seed + 1), _rand(*shape, seed=seed + 2)
    lat = _rand(*shape, seed=seed + 3, dtype=torch.float32) * 8.0
    if bf16_latents:
        lat = lat.to(BF16).float()
    sigma, sigma_next = 11.3, 9.7
    row = torch.tensor([900.0, sigma, sigma_next, math.sqrt(sigma_next ** 2 + 1.0)], device=DEVICE)
    nxt = torch.empty(shape, device=DEVICE, dtype=BF16)
    call = dict(eps_uncond=eu, eps_text=et, latents=lat, step_row=row, latents_out=None, model_in_next=nxt,
                round_latents_bf16=bf16_latents)
    if v_prediction:
        f = shape[1]
        call.update(frames=f, guidance_per_frame=torch.linspace(1.0, 3.0, f, device=DEVICE).to(BF16).float())
        out = ops.cfg_euler_v(**call)
    else:
        call.update(guidance=5.0)
        out = ops.cfg_euler(**call)
    _sync()
    return cfg_euler_verdict(f"cfg_euler{'_v' if v_prediction else ''} {'bf16' if bf16_latents else 'fp32'} latents "
                             f"{tuple(shape)}", call, out, nxt, v_prediction)


def _latent_encoder_ref64(x, clips, frames, params):
    """float64 restatement of the I2VGen-XL image-latent encoder with the kernel's bf16 rounding points (ops_emulator
    lists them).  Returns y [clips, pixel, frame, 4] and, per output row, the largest magnitude of its intermediates."""
    n, h, w_, _ = x.shape
    p = params.to(F64)
    sizes = [("ln_w", 4), ("ln_b", 4), ("wq", 32), ("wk", 32), ("wv", 32), ("wo", 32), ("bo", 4), ("w1", 64), ("b1", 16),
             ("w2", 64), ("b2", 4)]
    o, prm = 0, {}
    for key, sz in sizes:
        prm[key] = p[o:o + sz]
        o += sz
    wq, wk, wv = (prm[key].reshape(8, 4) for key in ("wq", "wk", "wv"))
    wo, w1, w2 = prm["wo"].reshape(4, 8), prm["w1"].reshape(16, 4), prm["w2"].reshape(4, 16)
    xs = x[..., :4].to(F64).reshape(clips, frames, h * w_, 4).permute(0, 2, 1, 3)  # [clip, pixel, frame, 4]
    xn = _r64(F.layer_norm(xs, (4,), prm["ln_w"], prm["ln_b"], 1e-5))
    q, k, v = (_r64(xn @ m.t()) for m in (wq, wk, wv))

    def heads(t):
        return t.reshape(*t.shape[:-1], 2, 4).transpose(-2, -3)  # [clip, pixel, head, frame, 4]
    a = _r64(torch.softmax(heads(q) @ heads(k).transpose(-1, -2) * 0.5, dim=-1) @ heads(v))
    a = a.transpose(-2, -3).reshape(q.shape)
    hcur = _r64(_r64(a @ wo.t() + prm["bo"]) + xs)
    u = _r64(_r64(F.gelu(_r64(hcur @ w1.t() + prm["b1"]))))
    ff = _r64(u @ w2.t() + prm["b2"])
    y = _r64(ff + hcur)
    mag = torch.cat([t.abs() for t in (xs, xn, q, k, v, a, hcur, u, ff, y)], dim=-1).amax(dim=-1, keepdim=True)
    return y, mag


def latent_encoder_verdict(name, x, clips, frames, params, out):
    """ops.i2vgen_latent_encoder: channels 4.. of the output exactly zero, channels 0..3 within 2 ulps of the largest
    intermediate of the float64 restatement"""
    h, w = x.shape[1:3]
    y, mag = _latent_encoder_ref64(x, clips, frames, params)
    o4 = out[..., :4].reshape(clips, frames, h * w, 4).permute(0, 2, 1, 3)
    return [_exact(f"{name} channels 4..{x.shape[3] - 1} zero", bool((out[..., 4:] == 0).all())),
            _report(name, o4, y, 2 ** -6, 1e-3, mag=mag.expand_as(y), dims=("clip", "pixel", "frame", "ch"),
                    units=(0, 1))]


def check_latent_encoder(clips, frames, h=10, w=10, c_stride=8, seed=0):
    """The I2VGen-XL image-latent encoder (one thread per (clip, pixel); hw = 100 is not a multiple of the 64-thread
    block).  Channels 4..7 of the input are nonzero; those of the output must be exactly zero."""
    ops = _ops()
    x = _rand(clips * frames, h, w, c_stride, seed=seed + 1)
    scales = [1.0, 1.0, 0.5, 0.5, 0.5, 0.35, 1.0, 0.5, 1.0, 0.25, 1.0]
    counts = [4, 4, 32, 32, 32, 32, 4, 64, 16, 64, 4]
    params = torch.cat([_rand(cnt, seed=seed + 10 + i, dtype=torch.float32) * s
                        for i, (cnt, s) in enumerate(zip(counts, scales))])
    params[:4] += 1.0  # LayerNorm weight around 1
    params = params.to(BF16).float().contiguous()
    out = ops.i2vgen_latent_encoder(x, clips, frames, params)
    _sync()
    return latent_encoder_verdict(f"i2vgen_latent_encoder b{clips} f{frames} hw{h * w} c_stride{c_stride}", x, clips,
                                  frames, params, out)[-1]


def groupnorm_verdict(name, a, out, samples=None):
    """ops.group_norm vs float64 over the concatenated sources (statistics over imgs_per_sample consecutive images when
    > 1), SiLU and nearest 2x up-sampling as requested, rounded to bf16: rtol 2^-7 / atol 2e-3 (check_groupnorm).
    samples: evaluate on these samples (groups of imgs_per_sample images) only."""
    x, x2, ips, groups = a["x"], a["x2"], a["imgs_per_sample"], a["groups"]
    n, h, w, _ = x.shape
    imgs = None if samples is None else [s * ips + j for s in samples for j in range(ips)]
    ii = slice(None) if imgs is None else torch.tensor(imgs, device=x.device)
    xin = (x[ii] if x2 is None else torch.cat([x[ii], x2[ii]], dim=3)).to(F64)
    nn, ct = xin.shape[0], xin.shape[3]
    eager = _groupnorm_eager(xin, a, ips, groups) if xin.numel() <= es.THIN else None  # bounded memory
    t = xin.reshape(nn // ips, ips * h * w, groups, ct // groups)  # in place from here: a 14-frame 576x1024 sample
    t.sub_(t.mean(dim=(1, 3), keepdim=True))                       # is 8.5 GB in float64
    t.mul_(torch.rsqrt(t.square().mean(dim=(1, 3), keepdim=True) + a["eps"]))
    y = t.reshape(nn, h, w, ct).mul_(a["gamma"].to(F64)).add_(a["beta"].to(F64))
    if a["silu"]:
        y = F.silu(y, inplace=True)
    if a["up2x"]:
        y = y.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    # direction: bias over the (sample, group) units, gain per (sample, group) about each channel's beta (SiLU of it),
    # its se clustered by the (sample, pixel, group) units inside
    center = a["beta"].to(F64)
    center = (F.silu(center) if a["silu"] else center).reshape(1, 1, groups, ct // groups)
    return _report(name, out[ii], _r64(y), 2 ** -7, 2e-3, dims=("img", "y", "x", "ch"), rows=imgs, units=(0, 2),
                   gain=((0, 2), center, (0, 1, 2)), eager=eager, unit_shape=(nn // ips, -1, groups, ct // groups))


def _groupnorm_eager(xin, a, ips, groups):
    """torch's eager GroupNorm (+ SiLU, + up-sampling) on the same bf16 inputs, fp32 arithmetic, one rounding to bf16:
    the gain's yardstick"""
    nn, h, w, ct = xin.shape
    x3 = xin.float().reshape(nn // ips, ips * h * w, ct).transpose(1, 2)
    y = F.group_norm(x3, groups, a["gamma"].float(), a["beta"].float(), a["eps"]).transpose(1, 2).reshape(nn, h, w, ct)
    if a["silu"]:
        y = F.silu(y)
    if a["up2x"]:
        y = y.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    return y.to(BF16)


def layernorm_verdict(name, a, out):
    """ops.layer_norm vs float64, rounded to bf16: rtol 2^-7 / atol 2e-3 (check_layernorm); with add_rowvec the input is
    bf16(x + row vector[row // rows_per_vec]), and the returned sum must be exactly that"""
    x, rv = a["x"], a["add_rowvec"]
    c = x.shape[-1]
    xf = x.reshape(-1, c).to(F64)
    y, ysum = out if a["return_sum"] else (out, None)
    recs = []
    if rv is not None:
        xf = _r64(xf + rv.to(F64).repeat_interleave(a["rows_per_vec"], dim=0))
        if ysum is not None:
            recs.append(_report(f"{name} sum", ysum.reshape(-1, c), xf, 0.0, 0.0, dims=("row", "ch")))
    ref = _r64(F.layer_norm(xf, (c,), a["gamma"].to(F64), a["beta"].to(F64), a["eps"]))
    # direction: units the rows, gain about beta; yardstick: torch's LayerNorm on the same bf16 input, fp32 arithmetic
    eager = F.layer_norm(xf.float(), (c,), a["gamma"].float(), a["beta"].float(), a["eps"]).to(BF16)
    recs.append(_report(name, y.reshape(-1, c), ref, 2 ** -7, 2e-3, dims=("row", "ch"), units=(0,),
                        gain=((), a["beta"].to(F64), None), eager=eager))
    return recs


def vae_latents_verdict(name, a, out):
    """ops.vae_latents vs a float64 statement of the posterior and the three layouts: zeros, position planes and the
    mode (no noise) bit-exact, a sample (with noise) within one bf16 ulp.  Layout I2VGEN: rows r -> image r % n,
    frame 0 = sample x scale, frame k = k / (F - 1); SVD: [zeros, latent] repeated num_videos times, on every frame."""
    m = a["moments"].to(F64).permute(0, 3, 1, 2)
    noise, layout, frames, nv = a["noise"], a["layout"], a["frames"], a["num_videos"]
    n = m.shape[0]
    v = m[:, :4]
    if noise is not None:
        v = v + torch.exp(0.5 * m[:, 4:].clamp(-30.0, 20.0)) * noise.to(F64)
    tol = _bf16_ulp(v) if noise is not None else torch.zeros_like(v)
    if layout == 0:
        ref, tol_all = v, tol
    elif layout == 1:
        pos = torch.arange(frames, dtype=F64, device=v.device) / max(frames - 1, 1)
        ref = pos.to(BF16).to(F64)[None, None, :, None, None].expand(n, 4, frames, *v.shape[2:]).clone()
        tol_all = torch.zeros_like(ref)
        ref[:, :, 0] = v * a["scale"]
        tol_all[:, :, 0] = _bf16_ulp(v * a["scale"]) if noise is not None else 0.0
        ref, tol_all = ref.repeat(2 * nv, 1, 1, 1, 1), tol_all.repeat(2 * nv, 1, 1, 1, 1)
    else:
        ref = torch.cat([torch.zeros_like(v), v]).repeat(nv, 1, 1, 1)[:, None].expand(-1, frames, -1, -1, -1)
        tol_all = torch.cat([torch.zeros_like(tol), tol]).repeat(nv, 1, 1, 1)[:, None].expand(-1, frames, -1, -1, -1)
    exact = tol_all == 0
    ref = torch.where(exact, ref.to(BF16).to(F64), ref)
    return _chain_verdict(name, out, ref, torch.where(exact, 2.0 ** -1074, tol_all), {"shape": tuple(out.shape)})


def check_groupnorm_offset(n, h, w, c, seed=0):
    """GroupNorm statistics are one-pass fp32 sums of x and x^2 with no shift: half of the groups sit at mean 40 with
    std 0.5, where E[x^2] - E[x]^2 cancels (mean / std)^2 = 6400-fold.  Tolerance of check_groupnorm."""
    ops = _ops()
    grp = torch.arange(c, device=DEVICE) // (c // 32)
    off = (grp % 2 == 0)
    mean = torch.where(off, 40.0, 0.0)[None, :, None, None]
    std = torch.where(off, 0.5, 1.0)[None, :, None, None]
    x = (_rand(n, c, h, w, seed=seed + 1, dtype=torch.float32) * std + mean).to(BF16)
    gamma = _rand(c, seed=seed + 2, dtype=torch.float32) * 0.2 + 1.0
    beta = _rand(c, seed=seed + 3, dtype=torch.float32) * 0.2
    call = dict(x=_nhwc(x), gamma=gamma, beta=beta, eps=1e-6, groups=32, silu=False, up2x=False, x2=None,
                imgs_per_sample=1, out=None)
    out = ops.group_norm(**call)
    _sync()
    return groupnorm_verdict(f"groupnorm mean40/std0.5 groups n{n} {h}x{w} c{c}", call, out)


def layout_cases(small=False):
    """[(name, check)] of the layout checks; small=True: reduced sizes for the CPU run over the emulator (same layouts,
    same edges: partial tiles, padded head dims, frame counts either side of 16, shared contexts)."""
    s = small
    cases = [
        ("attn_fused_qkv_d64", lambda: check_attention_fused_qkv(2, 3 if s else 10, 200 if s else 1000, 64)),
        ("attn_fused_qkv_d40", lambda: check_attention_fused_qkv(2, 2 if s else 10, 150 if s else 300, 40)),
        ("attn_fused_qkv_d160", lambda: check_attention_fused_qkv(2, 2 if s else 10, 150 if s else 300, 160)),
        ("attn_cross_kv", lambda: check_attention_cross_kv(2, 2 if s else 10, 130 if s else 1000, 77, 64)),
        ("attn_cross_kv_batch_div", lambda: check_attention_cross_kv(8 if s else 32, 2 if s else 5, 64 if s else 256, 77,
                                                                     64, kv_batch_div=4 if s else 16)),
    ]
    hw = 11 if s else 99  # not a multiple of the pixels per tile (8 for F <= 16, 4 above)
    for f in (1, 2, 3, 16, 17, 25, 32):
        cases.append((f"tattn_fused_f{f}", lambda f=f: check_temporal_attention_fused(2, f, hw, 2 if s else 5)))
    cases.append(("tattn_fused_svd_xt", lambda: check_temporal_attention_fused(1 if s else 2, 25, 36 if s else 576,
                                                                               2 if s else 5)))
    gemm = [  # (kind, m, k, n, rows_per_vec): n_out picks BN 160 / 256 / 64 / 128 / 128 / 160 / 256 / 128 / 64 / 256
        ("bias", 1000, 320, 320, 0), ("bias_silu", 1000, 320, 1280, 0), ("bias_scale", 1000, 256, 64, 0),
        ("bias_scale_res", 1000, 320, 384, 0), ("rowvec", 1024, 320, 384, 256), ("bias_res", 9000, 640, 640, 0),
        ("rowvec_res", 8192, 320, 1280, 64), ("bias_res_blend", 1000, 320, 128, 0),
        ("rowvec_res_blend", 1024, 320, 64, 256), ("geglu", 1000, 320, 1280, 0)]
    for kind, m, k, n, rpv in gemm:
        if s:
            m, k = (256 if rpv else 200), 64
            rpv = 64 if rpv else 0
        cases.append((f"gemm_{kind}", lambda a=(kind, m, k, n, rpv): check_gemm_epilogue(*a[:4], rows_per_vec=a[4])))
    cases += [
        ("temporal_conv_epilogue_f16", lambda: check_temporal_conv_epilogue(2, 4 if s else 16, 4 if s else 8,
                                                                            4 if s else 8, 64 if s else 320,
                                                                            64 if s else 320)),
        ("temporal_conv_epilogue_f1", lambda: check_temporal_conv_epilogue(2, 1, 4 if s else 8, 4 if s else 8,
                                                                           64 if s else 320, 64 if s else 320)),
        ("linear_f32_out_scale", lambda: check_linear_f32_scale(256 if s else 4096, 256 if s else 4096, 512)),
    ]
    for vpred in (False, True):
        for bf in (True, False):
            cases.append((f"cfg_ddim_{'v' if vpred else 'eps'}_{'bf16' if bf else 'fp32'}",
                          lambda v=vpred, b=bf: check_cfg_ddim_layout(v, b, (2, 4, 4, 8, 8) if s else (2, 4, 16, 32, 32))))
            cases.append((f"cfg_euler_{'v' if vpred else 'eps'}_{'bf16' if bf else 'fp32'}",
                          lambda v=vpred, b=bf: check_cfg_euler_layout(v, b, (2, 3, 4, 6, 8) if s else (2, 14, 4, 36, 64))))
    for f in (1, 16, 32):
        cases.append((f"latent_encoder_f{f}", lambda f=f: check_latent_encoder(2, f)))
    cases += [
        ("groupnorm_offset", lambda: check_groupnorm_offset(1 if s else 2, 16 if s else 64, 16 if s else 64,
                                                            64 if s else 320)),
        ("groupnorm_offset_vae_plane", lambda: check_groupnorm_offset(1, 32 if s else 512, 32 if s else 512, 128)),
    ]
    return cases


LAYOUT_CHECKS = layout_cases()


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
    groups = {"attn": [
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
        # a single, partial KV tile (Lk = 77 / 80 / 33 / 1 of 128: the key-tail mask decides every row's softmax, and at
        # Lk = 1 127 of the 128 keys are masked), grids of up to 2560 CTAs, a partial last query tile, padded head dim
        lambda: check_attention(16, 20, 1024, 77, 64),
        lambda: check_attention(8, 16, 700, 80, 64),
        lambda: check_attention(6, 10, 1280, 33, 40),
        lambda: check_attention(4, 8, 640, 1, 64),
        lambda: check_temporal_attention(2, 16, 64, 5),
        lambda: check_temporal_attention(1, 14, 100, 10),
    ], "misc": [
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
    ], "layouts": [fn for _, fn in LAYOUT_CHECKS]}
    plan = groups[group] if group else [fn for fns in groups.values() for fn in fns]
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
