"""The GEMM epilogue restated bit for bit, and the accumulators it starts from.

Every step of the bf16 epilogue of gemm_conv_kernel is an IEEE fp32 add or multiply followed by one bf16
round-to-nearest-even, except the two activations, which are functions of a bf16 input (the epilogue rounds acc + bias
before applying them) and so are fully described by a table of 65,536 entries:

    v = r(acc + bias)                                  (r(acc) without a bias)
    v = T_silu[v]                  SiLU                 (T_silu[x]: the kernel's bf16 SiLU of x)
    v = r(r(a + bias_a) * G[r(g + bias_g)])           GEGLU (G[x]: the kernel's bf16 GELU of x)
    v = r(v * scale)                                   scale != 1
    v = r(v + rowvec);  v = r(v + residual)
    v = r(r(alpha * src) + r(r(1 - alpha) * v))        AlphaBlender

The fp32-output instantiation keeps fp32 throughout, rounding only after the row vector:
    v = acc + bias;  v = v * scale;  v = r(v + rowvec);  v = v + residual
(its SiLU acts on the unrounded acc + bias, which no table describes, so it is not restated).

accumulators(): the fp32 accumulators of a call -- the same op, operands, geometry and N tile with fp32 output and an
empty epilogue (no bias, no activation, scale 1, no row vector / residual / blend), which shares the main loop and so
the summation order of the bf16 instantiations at that N tile.  accumulator_verdict(): those accumulators against the
float64 contraction of the same operands, so that a main-loop error every instantiation shares (a wrong tap, a dropped
K block) cannot hide in them.  expected(): the chain above in torch fp32 on the accumulators' device.  compare(): bits
against bits, with a diagnosis of a mismatch.  slot() / guard_intact(): an output view inside a buffer of sentinel
bits, and whether a call left those bits alone.  Used by tests/test_gemm_epilogue_exact_gpu.py on the kernels and by
tests/test_gemm_epilogue_exact_cpu.py on tests/ops_emulator.py.
"""
from __future__ import annotations

import inspect

import torch

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
ACT_NONE, ACT_SILU, ACT_GEGLU = 0, 1, 2
STEPS = ("bias", "act", "scale", "rowvec", "residual", "blend")


def r(t):
    """round to bf16, keep computing in fp32"""
    return t.to(BF16).float()


def bf16_index(t):
    """bf16 bit patterns of t (rounded to bf16 first) as indices 0..65535"""
    return t.to(BF16).view(torch.int16).long() & 0xFFFF


def all_bf16(device):
    """the 65,536 bf16 values in bit-pattern order, as fp32"""
    return torch.arange(65536, dtype=torch.int32, device=device).to(torch.int16).view(BF16).float()


def resolved_bn(op, call):
    """ca_gemm's N tile for the call (csrc/gemm_conv.cu, restated in tests/abi_domain.gemm_bn)"""
    from tests.abi_domain import gemm_bn
    w = call["w"] if op == "linear" else call["w_packed"]
    return gemm_bn(w.shape[0], call.get("act", ACT_NONE) == ACT_GEGLU, call.get("bn", 0))


def geglu_halves(t, bn):
    """[..., n tiles * bn] in ops.pack_geglu_weight's order -> (value [..., n], gate [..., n]), n = half the columns"""
    lead, cols = t.shape[:-1], t.shape[-1]
    q = t.reshape(*lead, cols // bn, 2, bn // 2)
    return q[..., 0, :].reshape(*lead, cols // 2), q[..., 1, :].reshape(*lead, cols // 2)


_EMPTY = dict(bias=None, act=ACT_NONE, out_scale=1.0, rowvec=None, residual=None, blend_src=None, blend_alpha=None,
              out=None, out_fp32=True)


def accumulators(op, call, ops):
    """-> the call's fp32 accumulators in its output's shape; for GEGLU those of the packed weight run as a plain GEMM
    at the same N tile, value and gate columns interleaved per tile (geglu_halves splits them)"""
    if op == "temporal_conv":
        return _temporal_conv_fp32(call, ops)
    fn = getattr(ops, op)
    params = inspect.signature(fn).parameters
    kw = dict(call)
    kw.update({k: v for k, v in _EMPTY.items() if k in params})
    if "bn" in params:
        kw["bn"] = resolved_bn(op, call)
    return fn(**kw)


def accumulator_verdict(label, op, call, acc, atol_cap=1e-3):
    """acc (accumulators()) against the float64 contraction of the call's operands, without the bias: the census's
    pre-activation bound, rtol 1e-3 and atol max(1e-4, 2^-16 sum |x_k w_k|) (kernel_checks._sum_floor), the atol capped
    at atol_cap; with the direction statistics of kernel_checks._report.  A convolution over more than 4 images is
    evaluated on the first, middle and last.  -> the record"""
    from tests import kernel_checks as kc
    rows = None
    if op == "linear":
        x, w = call["x"].to(F64), call["w"].to(F64)
        exact, abs_sum = x @ w.t(), x.abs() @ w.abs().t()
        dims, units = ("row", "col"), (0,)
    elif op == "conv2d":
        n = call["x"].shape[0]
        rows = [0, n // 2, n - 1] if n > 4 else None
        exact, abs_sum = kc.conv2d_ref({**call, "bias": None}, rows)
        acc = acc if rows is None else acc[rows]
        dims, units = ("img", "y", "x", "ch"), (0, 1, 2)
    else:
        exact, abs_sum = kc.temporal_conv_ref({**call, "bias": None})
        acc = acc.reshape(exact.shape)
        dims, units = ("clip", "frame", "pixel", "ch"), (0, 1, 2)
    atol = kc._sum_floor(abs_sum).clamp_(max=atol_cap)
    del abs_sum
    return kc._report(f"{label} accumulators", acc, exact, 1e-3, atol, dims=dims, rows=rows, units=units)


def _temporal_conv_fp32(call, ops):
    """ops.temporal_conv has no fp32 output: the call is made with an empty epilogue and an fp32 `out`, and its GEMM
    descriptor gets out_fp32 at launch, so that the box, taps and strides are those of the call under test"""
    if not hasattr(ops, "_launch"):
        raise ValueError("temporal_conv accumulators need the CUDA op layer")
    x, w = call["x"], call["w_packed"]
    out = torch.empty(*x.shape[:3], w.shape[0], device=x.device, dtype=F32)
    launch = ops._launch

    def fp32_launch(fam, flops, nbytes, name, desc, *rest):
        desc._obj.out_fp32 = 1  # desc: ctypes.byref of the GemmDesc
        return launch(fam, flops, nbytes, name, desc, *rest)
    ops._launch = fp32_launch
    try:
        ops.temporal_conv(x, w, None, call["frames"], out=out)
    finally:
        ops._launch = launch
    return out


def _lookup(table, v):
    return table[bf16_index(v)]


def expected(acc, *, gate=None, bias=None, act=ACT_NONE, scale=1.0, rowvec=None, residual=None, blend_src=None,
             blend_alpha=None, out_fp32=False, tables=None, drop=None, swap=None, unrounded=None):
    """The epilogue chain on the accumulators.  bias: [n] fp32 (GEGLU: (value bias, gate bias)); rowvec / residual /
    blend_src: broadcastable to acc; tables: {"silu": T_silu, "gelu": G}, fp32 [65536] indexed by bf16 bits.
    Diagnostic variants of the chain (compare() tries them on a mismatch): drop = a step left out, swap = a step done
    after the next one, unrounded = a step without its bf16 rounding."""
    rr = lambda t, step: t if step == unrounded else r(t)  # noqa: E731
    if out_fp32:
        if act != ACT_NONE or blend_src is not None:
            raise ValueError("the fp32-output chain is restated without activation and blend")
        v = acc if bias is None or drop == "bias" else acc + bias
        if scale != 1.0 and drop != "scale":
            v = v * scale
        if rowvec is not None and drop != "rowvec":
            v = rr(v + rowvec.float(), "rowvec")
        if residual is not None and drop != "residual":
            v = v + residual.float()
        return v
    bias_a, bias_g = bias if act == ACT_GEGLU and bias is not None else (bias, None)
    steps = []
    steps.append(("bias", lambda v: rr(v if bias_a is None else v + bias_a, "bias")))
    if act == ACT_SILU:
        steps.append(("act", lambda v: _lookup(tables["silu"], v)))
    elif act == ACT_GEGLU:
        g = r(gate if bias_g is None else gate + bias_g)
        steps.append(("act", lambda v: rr(v * _lookup(tables["gelu"], g), "act")))
    if scale != 1.0:
        steps.append(("scale", lambda v: rr(v * scale, "scale")))
    if rowvec is not None:
        steps.append(("rowvec", lambda v: rr(v + rowvec.float(), "rowvec")))
    if residual is not None:
        steps.append(("residual", lambda v: rr(v + residual.float(), "residual")))
    if blend_src is not None:
        a = blend_alpha.float().reshape(())
        steps.append(("blend", lambda v: r(r(a * blend_src.float()) + r(rr(1.0 - a, "blend") * v))))
    names = [s[0] for s in steps]
    if swap is not None and swap in names[:-1]:
        i = names.index(swap)
        steps[i], steps[i + 1] = steps[i + 1], steps[i]
    v = acc.float()
    for name, fn in steps:
        if name != drop:
            v = fn(v)
    return v


def present_steps(kw):
    """the steps of expected()'s chain a call has"""
    s = ["bias"]
    if kw.get("act", ACT_NONE) != ACT_NONE:
        s.append("act")
    if kw.get("scale", 1.0) != 1.0:
        s.append("scale")
    s += [k for k, a in (("rowvec", "rowvec"), ("residual", "residual"), ("blend", "blend_src")) if kw.get(a) is not None]
    return s


def _int_view(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32)


SENTINEL = -1  # the bits around a slot: all ones, a NaN in bf16 and in fp32


def slot(t, left=4, right=12, flat=False):
    """t's values in columns [left, left + n) of a [rows, left + n + right] buffer whose other elements hold SENTINEL;
    flat=True: in a contiguous view at element `left` of a flat buffer (a convolution's channels-last output).
    left = 4 bf16 puts the view 8 bytes off 16-byte alignment"""
    if flat:
        return slot(t.reshape(1, -1), left, right).view(t.shape)
    buf = torch.empty(*t.shape[:-1], left + t.shape[-1] + right, device=t.device, dtype=t.dtype)
    _int_view(buf).fill_(SENTINEL)
    view = buf[..., left:left + t.shape[-1]]
    view.copy_(t)
    return view


def guard_intact(view):
    """every element of the buffer of a slot() view outside the view still holds SENTINEL"""
    buf = view._base
    outside = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    outside.as_strided(view.shape, view.stride(), view.storage_offset()).fill_(False)
    return bool((_int_view(buf)[outside] == SENTINEL).all())


def compare(label, out, acc, chain, *, n_tile_cols):
    """out (the kernel's bf16 / fp32 output, shape [..., n]) vs expected(acc, **chain), bit for bit (a NaN matches only
    the same NaN bits: the kernel writes one canonical NaN and so does torch).  -> (ok, message).  On a mismatch the
    message gives the number of differing elements, the first one as (row, col) of the output flattened to
    [rows, n] with its N tile (n_tile_cols output columns per tile), the kernel's bits against the expected bits, and the
    first variant of the chain -- a step dropped, done after the next one, or left unrounded -- that would match."""
    fp32 = bool(chain.get("out_fp32"))
    exp = expected(acc, **chain)
    exp = exp if fp32 else exp.to(BF16)
    a, b = _int_view(out.contiguous()), _int_view(exp.contiguous())
    if torch.equal(a, b):
        return True, f"{label}: {out.numel()} elements bit-identical"
    n = out.shape[-1]
    diff = (a != b).reshape(-1)
    first = int(diff.nonzero()[0])
    row, col = divmod(first, n)
    width = 8 if fp32 else 4
    mask = (1 << (4 * width)) - 1
    kb, eb = int(a.reshape(-1)[first]) & mask, int(b.reshape(-1)[first]) & mask
    msg = (f"{label}: {int(diff.sum())} of {out.numel()} elements differ; first at (row {row}, col {col}), N tile "
           f"{col // n_tile_cols}: kernel 0x{kb:0{width}x} ({float(out.reshape(-1)[first]):.6g}), expected "
           f"0x{eb:0{width}x} ({float(exp.reshape(-1)[first]):.6g})")
    msg += "; " + diagnose(out, acc, chain)
    return False, msg


def diagnose(got, acc, chain):
    """the first chain variant (in chain order: drop, swap with the next step, no rounding) whose bits equal got"""
    steps = present_steps(chain)
    dt = F32 if chain.get("out_fp32") else BF16
    for step in steps:
        for kind in ("drop", "swap", "unrounded"):
            try:
                v = expected(acc, **chain, **{kind: step}).to(dt)
            except (TypeError, ValueError, KeyError):
                continue
            if torch.equal(_int_view(v.contiguous()), _int_view(got.contiguous())):
                return f"matches the chain with step '{step}' {_KIND[kind]}"
    return "no single dropped, swapped or unrounded step explains it"


_KIND = {"drop": "dropped", "swap": "done after the next step", "unrounded": "left unrounded"}


# ---- activation tables through a GEMM's own epilogue ----
def silu_table(ops, bn, device):
    """T_silu[bits] of the bf16 epilogue at N tile bn: one GEMM with zero operands and one column per bf16 input, the
    input as that column's bias, so acc + bias is the input exactly (+0 + x = x, -0 giving +0), whatever the tensor
    cores do with subnormal or non-finite operands.  65,536 columns: more N tiles than SMs, so every CTA takes several
    tiles and their biases through the double-buffered bias row."""
    x = all_bf16(device)
    k = 64
    a = torch.zeros(2, k, device=device, dtype=BF16)
    w = torch.zeros(65536, k, device=device, dtype=BF16)
    y = ops.linear(a, w, x.contiguous(), act=ACT_SILU, bn=bn)
    return y[0].float()


def gelu_table(ops, bn, device):
    """G[bits] of the GEGLU epilogue at N tile bn: zero operands, value bias 1 and gate bias x per output column, so
    the output r(r(1) * G[x]) is G[x].  The column count is padded to a multiple of bn / 2 (the packing's unit)."""
    x = all_bf16(device)
    half = bn // 2
    n = (65536 + half - 1) // half * half
    gate = torch.zeros(n, device=device)
    gate[:65536] = x
    b = torch.cat([torch.ones(n, device=device), gate])
    w = torch.zeros(2 * n, 64, device=device, dtype=BF16)
    from ctrl_adapter_b200.ops import pack_geglu_weight
    wk, bk = pack_geglu_weight(w, b, bn)
    a = torch.zeros(2, 64, device=device, dtype=BF16)
    y = ops.linear(a, wk, bk.contiguous(), act=ACT_GEGLU, bn=bn)
    return y[0, :65536].float()


def ulps(got, ref64):
    """distance in bf16 steps between got (bf16-valued) and float64 ref rounded to bf16 (sign-magnitude bit patterns
    mapped to ordered integers, so -0 and +0 are one point); NaN / inf positions are the caller's"""
    def ordered(t):
        i = t.to(BF16).view(torch.int16).long()
        return torch.where(i < 0, -(i & 0x7FFF), i)
    return (ordered(got.float()) - ordered(ref64.float())).abs()
