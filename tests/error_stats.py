"""Which way a kernel's error points: statistics of one (out, ref) pair beyond the element-wise allowance of
tests/kernel_checks.py, and their verdict.

The element-wise allowance |out - ref| <= atol + rtol * |ref| bounds how large each error is.  It cannot tell unbiased
rounding noise from a systematic error of the same size: an epilogue that rounds its bf16 output toward zero stays
within 1 ulp everywhere, yet shifts every output by about a quarter of an ulp; a softmax scale off by 0.3 % or a
GroupNorm whose rstd is off by 2^-11 moves every output of a row or group the same way.  Across the hundreds of launches
of a denoising step and the 25-50 steps of a run, zero-mean noise mostly averages out while such errors add up.

Statistics of one record (`direction`), from the kernel output `out` and the float64 reference `ref` the verdict
already builds (for bf16 outputs, rounded at the kernel's rounding points):
  * bias: the signed error in bf16 ulps of the reference, u = (out - ref) / ulp_bf16(ref), as mean(u) (a floor /
    ceiling bias) and mean(sign(ref) * u) (a bias toward zero, negative, or away from it).  Elements whose |ref| is
    within the check's atol, zero or subnormal are left out.
  * gain: the least-squares slope delta = sum (out - ref) * r / sum r^2 of the error on r = ref - center, per gain
    group: the whole record by default; per (sample, group) about beta for GroupNorm; per (batch, head) about the mean
    of V over the keys for attention.
  * relative RMS error ||out - ref|| / ||ref|| per gain group, and the same of an eager torch op on the same inputs where
    the verdict has one (torch's bf16 SDPA for attention), with their ratio (the largest over the gain groups).

Errors are not independent element by element (an attention row shares its max and sum, a GroupNorm group its rstd), so
each verdict names its independent units: axes of `out` (GEMM / conv output rows or pixels; attention (b, q-row, h);
temporal attention (clip, pixel, head); norm rows or (sample, group)) or, without them, blocks of 4096 consecutive
elements.  Means are taken over units and their standard error se is the spread across units, measured (a cluster
estimate): records with fewer than MIN_UNITS units get se = inf, so their direction bound is loose on its own.
Records of more than THIN elements (the largest census launches) are evaluated on every k-th index of their longest
axis, which keeps the float64 temporaries bounded.  The gain's se clusters its residual the same way, by the units
inside each gain group.

Verdict: a record fails when
  * |mean u| or |mean sign(ref) * u| > max(BIAS_FLOOR, Z * se): 1/32 ulp;
  * |delta| of any gain group > max(GAIN_FLOOR, 2 |delta_eager|, Z * se): 2^-12, 1/32 of a bf16 ulp in relative terms,
    delta_eager being the same statistic of the eager bf16 torch op where the verdict passes one.
The reference is the one at the kernel's rounding points, the bf16 output rounding included.  Attention's element-wise
verdicts compare with the unrounded float64 output; their statistics use it rounded to bf16 (kernel_checks passes
`stats_ref`).  Against the unrounded output, correct round-to-nearest alone has a gain about the mean of V: where a row's
softmax is nearly one-hot the exact output lies within an ulp of the dominant bf16 V value and rounding snaps it back
there, away from the mean.  Over the correct emulation with 4 frames and logits of std 6 that gain is 1.1e-4, all of it
the rounding (the rounded exact output has the same); on the activations of one SVD launch (4 frames, 144 pixels, 20
heads) it reached 3.1e-3 at 8.6 se.  Against the rounded reference the emulation's gain is below 1e-7.
The GEMM and convolution verdicts pass no eager yardstick: their bf16 references are the epilogue chain applied to the
kernel's own fp32 pre-activation, so the gain bound is max(GAIN_FLOOR, Z * se), stricter than with cuBLAS's (which
rounds to nearest as well, so 2 |delta_eager| would add nothing above the floor).
The relative RMS error and its ratio to the eager op's are reported, not bounded.  Measured on an H100 80GB HBM3, the
ratio of attention's RMS error per (batch, head) to torch's bf16 SDPA's, worst per census row and per direction case
(256 records): min 1.000, median 1.000, 90th percentile 1.010, max 1.030.  An attention whose softmax scale is 0.3 %
high reaches 0.985 and one whose exp2 is a degree-2 polynomial 0.998 (the gain catches both), so no RMS bound
separates them from the real kernel; P truncated to bf16 reaches 5.2.

Z = 7: with at least MIN_UNITS = 32 units the standardised mean is t-distributed with >= 31 degrees of freedom, whose
two-sided tail beyond 7 is below 1e-7, so a false alarm over the few thousand records of every tier together stays
below one in a thousand.
"""
from __future__ import annotations

import math

import torch

F64 = torch.float64
Z = 7.0
MIN_UNITS = 32
BIAS_FLOOR = 1.0 / 32
GAIN_FLOOR = 2.0 ** -12
BLOCK = 4096
THIN = 1 << 26  # records with more elements are evaluated on every k-th index of their longest axis
BLOCKS = "blocks"  # units= of a record whose independent units are blocks of BLOCK consecutive elements


def bf16_ulp(a):
    """the bf16 ulp of |a| (normal range), as a float64 tensor"""
    e = torch.frexp(a.abs().to(F64).clamp_min(2.0 ** -126))[1]
    return torch.ldexp(torch.ones_like(a, dtype=F64), e - 8)


def _keep(t, axes):
    """sum t over every axis not in `axes`, keeping dims"""
    other = [d for d in range(t.dim()) if d not in axes]
    return t.sum(dim=other, keepdim=True) if other else t


def _blocks(t):
    """[n] -> [ceil(n / BLOCK), BLOCK], zero-padded"""
    t = t.reshape(-1)
    pad = -t.numel() % BLOCK
    if pad:
        t = torch.cat([t, t.new_zeros(pad)])
    return t.reshape(-1, BLOCK)


def _cluster_mean(x, w, axes):
    """mean of x (per element, 0 where w is 0) over the elements with w = 1, and its cluster standard error over the
    units `axes` -> (mean, se, units)"""
    sx, sw = _keep(x, axes).reshape(-1), _keep(w, axes).reshape(-1)
    live = sw > 0
    n_units = int(live.sum())
    tot = float(sw.sum())
    if tot == 0:
        return 0.0, math.inf, 0
    mean = float(sx.sum()) / tot
    if n_units < MIN_UNITS:
        return mean, math.inf, n_units
    resid = (sx - mean * sw)[live]
    se = math.sqrt(float(resid.square().sum()) * n_units / (n_units - 1)) / tot
    return mean, se, n_units


def _gain(e, r, groups, units):
    """per gain group (axes `groups`, a subset of `units`): slope of e on r, its cluster se over `units`, and the number
    of units per group -> (delta, se) as tensors over the groups"""
    nc, dc = _keep(e * r, units), _keep(r * r, units)
    ng, dg = _keep(nc, groups), _keep(dc, groups)
    delta = ng / dg.clamp_min(1e-300)
    k = nc.numel() // max(ng.numel(), 1)
    if k < MIN_UNITS:
        se = torch.full_like(delta, math.inf)
    else:
        se = torch.sqrt(_keep((nc - delta * dc).square(), groups) * k / (k - 1)) / dg.clamp_min(1e-300)
    return delta.reshape(-1), se.reshape(-1)


def direction(out, ref, atol, *, units=BLOCKS, gain_groups=(), gain_units=None, center=None, eager=None, tol=None):
    """statistics and verdict of one record (module docstring) -> dict of new record fields, "ok" and "why".
    out, ref: the same shape; atol: scalar or tensor broadcastable to ref (elements with |ref| <= atol are left out of
    the bias); tol: instead of atol, an element-wise tolerance with the same role; units: axes of out naming independent
    units (BLOCKS: blocks of 4096 elements); gain_groups: axes of the gain groups, () the whole record; gain_units: the
    units the gain's se clusters by, a superset of gain_groups (default: units); center: broadcastable to ref, the
    gain's origin; eager: an eager torch op's output on the same inputs."""
    if ref.numel() > THIN:  # a strided subset of the longest axis: the same units' structure, bounded temporaries
        ax = max(range(ref.dim()), key=lambda d: ref.shape[d])
        step = -(-ref.numel() // THIN)
        pick = (slice(None),) * ax + (slice(None, None, step),)
        thin = (lambda t: t if not torch.is_tensor(t) or t.dim() != ref.dim() or t.shape[ax] != ref.shape[ax]
                else t[pick])
        out, eager, center, atol, tol, ref = (thin(t) for t in (out, eager, center, atol, tol, ref))
    out = out.to(F64)
    ref = ref.to(F64)
    eager = None if eager is None else eager.to(F64)
    floor = tol if tol is not None else atol
    if torch.is_tensor(floor):
        floor = floor.to(F64)
    fin = torch.isfinite(out)
    if isinstance(units, str):
        shape = ref.shape
        if center is not None:
            center = _blocks(torch.as_tensor(center, dtype=F64, device=ref.device).expand(shape))
        if torch.is_tensor(floor):
            floor = _blocks(floor.expand(shape))
        if eager is not None:
            eager = _blocks(eager.to(F64))
        out, ref, fin = _blocks(out), _blocks(ref), _blocks(fin)
        units, gain_groups, gain_units = (0,), (), None
        pad = torch.zeros_like(fin)
        pad.reshape(-1)[:math.prod(shape)] = True
        fin = fin & pad
    units = tuple(units)
    err = torch.where(fin, out - ref, 0.0)
    ulp = bf16_ulp(ref)
    w = (fin & (ref.abs() > floor) & (ref.abs() >= 2.0 ** -126)).to(F64)
    u = err / ulp * w
    rec = {"units": int(_keep(w, units).numel())}
    b, b_se, nu = _cluster_mean(u, w, units)
    b0, b0_se, _ = _cluster_mean(torch.sign(ref) * u, w, units)
    del u
    bound, bound0 = max(BIAS_FLOOR, Z * b_se), max(BIAS_FLOOR, Z * b0_se)
    rec.update(bias_ulp=b, bias_bound=bound, bias0_ulp=b0, bias0_bound=bound0, bias_units=nu)
    why = []
    if abs(b) > bound:
        why.append(f"bias: mean u = {b:.4g} ulp > bound {bound:.3g}")
    if abs(b0) > bound0:
        why.append(f"bias toward zero: mean sign*u = {b0:.4g} ulp > bound {bound0:.3g}")

    r = ref if center is None else ref - center
    r = torch.where(fin, r, 0.0)
    gu = units if gain_units is None else tuple(gain_units)
    delta, se = _gain(err, r, tuple(gain_groups), gu)
    gbound = torch.clamp(Z * se, min=GAIN_FLOOR)
    if eager is not None:
        ee = torch.where(fin, eager.to(F64) - ref, 0.0)
        d_eager, _ = _gain(ee, r, tuple(gain_groups), gu)
        gbound = torch.maximum(gbound, 2.0 * d_eager.abs())
    ratio = delta.abs() / gbound
    wg = int(ratio.argmax())
    rec.update(gain=float(delta[wg]), gain_bound=float(gbound[wg]), gain_over_bound=float(ratio[wg]),
               gain_max=float(delta.abs().max()), gain_group=wg)
    if eager is not None:
        rec["gain_eager"] = float(d_eager[wg])
    if float(ratio[wg]) > 1.0:
        why.append(f"gain: delta = {float(delta[wg]):.4g} (group {wg}) > bound {float(gbound[wg]):.3g}")
    del r
    if eager is not None:
        groups = tuple(gain_groups)
        ref2 = _keep(torch.where(fin, ref, 0.0).square(), groups).clamp_min(1e-300)
        rms_g = torch.sqrt(_keep(err.square(), groups) / ref2).reshape(-1)
        rms_e = torch.sqrt(_keep(ee.square(), groups) / ref2).reshape(-1)
        rr = rms_g / rms_e.clamp_min(1e-300)
        wr = int(rr.argmax())
        rec.update(rms=float(rms_g[wr]), rms_eager=float(rms_e[wr]), rms_ratio=float(rr[wr]), rms_group=wr)
    rec["ok"] = not why
    rec["why"] = "; ".join(why)
    return rec
