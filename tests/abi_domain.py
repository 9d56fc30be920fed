"""The argument domain of every C entry point of include/ctrl_adapter_b200.h, and a seeded sampler over it.

DOMAIN: per entry point, the valid placeholder arguments and the header's constraints, each as (argument, last value
inside, first value outside).  tests/test_abi_domain_cpu.py calls the library with each value and no GPU: inside must
pass validation (it then fails with CA_ERR_CUDA), outside must return CA_ERR_INVALID with a message naming the
argument.  Faulting regions -- misaligned vectors, grid dimensions past 65535, channel counts past their stride -- are
closed by those validations and never launched.

cases(small): the `ops` calls of the GPU sweep, each tagged with the host dispatch branches it takes, predicted by
restating the dispatch rules of csrc/ in Python (gemm_bn, layernorm_variant, ...): every boundary value of a size
argument, every branch, and a few seeded interior points.  Calls that `ops` cannot express (LayerNorm in place) go to
the C entry point through `_lib` with the header's argument names.  small=True: reduced sizes for the CPU run over
tests/ops_emulator.py, as in kernel_checks.layout_cases(small=True).

On the GPU the predictions are checked against what ran: KernelTrace records the kernels of each case's first launch,
kernel_labels parses their template arguments into the name-visible labels, visible_parts gives the labels a predicted
branch implies, and observed_dispatch requires the two to agree case by case.
"""
from __future__ import annotations

import ctypes as C
import random
import re
import time
from dataclasses import dataclass, field
from typing import Callable, Tuple

import torch

BF16, F32 = torch.bfloat16, torch.float32

# ----------------------------------------------------------------------------------------------------------------------
# host dispatch rules restated (csrc/gemm_conv.cu, norm.cu, attention.cu, temporal_attention.cu, elementwise.cu)
# ----------------------------------------------------------------------------------------------------------------------


def gemm_bn(w_rows, geglu=False, bn=0):
    if bn:
        return bn
    if geglu or w_rows % 256 == 0:
        return 256
    if w_rows % 160 == 0:
        return 160
    if w_rows % 128 == 0:
        return 128
    return 64 if w_rows <= 64 else 128 if w_rows <= 128 else 256


def gemm_operand_path(*, vec, out_fp32=False, geglu=False, residual=False, blend=False, res_strides=(8, 0, 0, 0),
                      out_dims=(1, 1, 1, 1)):
    """True: residual / blend source come by TMA (gemm_conv_kernel<BN, bf16, kOps = true>).  The bf16 non-GEGLU
    epilogue on the aligned path with either source present, unless a row dim of the output has a negative residual
    stride, or stride 0 with more than one point (a broadcast, which a tensor map cannot express)"""
    if not (vec and not out_fp32 and not geglu and (residual or blend)):
        return False
    return all(s >= 0 and not (s == 0 and d > 1) for s, d in zip(res_strides, out_dims))


def gemm_branches(w_rows, *, act=0, out_fp32=False, bn=0, vec=True, rowvec=False, residual=False, blend=False,
                  res_strides=(8, 0, 0, 0), out_dims=(1, 1, 1, 1)):
    """res_strides / out_dims: ca_gemm's res_strides and out_dims (the defaults: a plain row-major source)"""
    n_tile = gemm_bn(w_rows, act == 2, bn)
    b = [f"gemm bn{n_tile}" + (" forced" if bn else " auto")]
    if out_fp32:
        b.append("gemm epilogue f32")
    elif act == 2:
        b.append("gemm epilogue geglu")
    else:
        b.append("gemm epilogue bf16")
        kind = int(rowvec) | 2 * int(residual) | 4 * int(blend)
        if gemm_operand_path(vec=vec, residual=residual, blend=blend, res_strides=res_strides, out_dims=out_dims):
            b += [f"gemm operands tma bn{n_tile}", f"gemm operands tma kind{kind}"]
        else:
            b.append(f"gemm storer kind{kind} {'vec' if vec else 'elementwise'}")
            if vec and kind >= 2:
                b.append(f"gemm operands global kind{kind} vec")
    return b


def attention_nwg(head_dim_pad, lq, lk):
    """consumer warpgroups of attention_kernel (use_wg3): 3 (192-row query tiles) for head dim 64 with more than one KV
    tile, unless their padding exceeds the 128-row tiles' by more than lq / 25"""
    if head_dim_pad != 64 or lk <= 128:
        return 2
    pad192 = -lq % 192
    pad128 = -lq % 128
    return 3 if 25 * (pad192 - pad128) <= lq else 2


def attention_branches(head_dim_pad, lq, lk, kv_div):
    dq, nwg, div = head_dim_pad // 64, attention_nwg(head_dim_pad, lq, lk), "1" if kv_div == 1 else ">1"
    b = [f"attention DQ{dq} kv_div{div}"]
    if nwg == 3:
        b.append(f"attention DQ{dq} NWG3 kv_div{div}")
    else:
        b.append(f"attention DQ{dq} NWG2 {'multi-tile' if lk > 128 else 'single-tile'}")
    return b


def layernorm_variant(c, rv):
    nvec = c // 8
    lanes = 8 if (nvec + 7) // 8 <= 5 else 16 if (nvec + 15) // 16 <= 5 else 32
    return f"layernorm NV{(nvec + lanes - 1) // lanes} L{lanes} RV{int(rv)}"


LAYERNORM_VARIANTS = [f"layernorm NV{nv} L{ln} RV{rv}" for ln, nvs in ((8, range(1, 6)), (16, range(3, 6)),
                                                                       (32, range(3, 9))) for nv in nvs for rv in (0, 1)]


def expected_branches():
    """every branch the sampler must reach"""
    b = {f"gemm bn{n} {m}" for n in (64, 128, 160, 256) for m in ("auto", "forced")}
    b |= {f"gemm storer kind{k} {d}" for k in range(8) for d in ("vec", "elementwise")}
    b |= {"gemm epilogue f32", "gemm epilogue geglu", "gemm epilogue bf16"}
    b |= {f"gemm operands tma bn{n}" for n in (64, 128, 160, 256)} | {f"gemm operands tma kind{k}" for k in range(2, 8)}
    b |= {f"gemm operands global kind{k} vec" for k in range(2, 8)}
    b |= set(LAYERNORM_VARIANTS) | {"layernorm in place"}
    b |= {f"attention DQ{d} kv_div{k}" for d in (1, 2, 3) for k in ("1", ">1")}
    b |= {"attention DQ1 NWG3 kv_div1", "attention DQ1 NWG3 kv_div>1"}
    b |= {f"attention DQ{d} NWG2 {t}" for d in (1, 2, 3) for t in ("multi-tile", "single-tile")}
    b |= {"temporal_attention SEQ16", "temporal_attention SEQ32"}
    b |= {f"gn_apply silu{s} up{u}" for s in (0, 1) for u in (0, 1)}
    b |= {"nchw_to_nhwc src bf16", "nchw_to_nhwc src fp32", "nhwc_to_nchw dst bf16", "nhwc_to_nchw dst fp32"}
    return b


# ----------------------------------------------------------------------------------------------------------------------
# the dispatch as launched: every choice above that is a template argument shows in the kernel's name
# ----------------------------------------------------------------------------------------------------------------------
_KERNELS = ("attention_kernel", "gemm_conv_kernel", "layernorm_kernel", "temporal_attention_tc_kernel",
            "gn_apply_kernel", "nchw_to_nhwc_kernel", "nhwc_to_nchw_kernel")
_DEMANGLED = re.compile(r"\b(" + "|".join(_KERNELS) + r")<([^<>()]*)>")
_MANGLED = re.compile(r"\d+(" + "|".join(_KERNELS) + r")I((?:L[ib]\d+E|f|14__nv_bfloat16)+)E")
_MANGLED_ARG = re.compile(r"L[ib](\d+)E|(f)|(14__nv_bfloat16)")
_EPILOGUES = {0: "bf16", 1: "geglu", 2: "f32"}  # GemmEpilogue


def kernel_instantiation(name):
    """kernel name as the profiler reports it (demangled, or an Itanium-mangled symbol) -> (kernel, template arguments
    as ints / 'bf16' / 'fp32'), or None for a kernel without dispatch in its name"""
    m = _DEMANGLED.search(name)
    if m:
        args = []
        for a in (x.strip() for x in m.group(2).split(",")):
            a = re.sub(r"^\((?:int|bool)\)", "", a)
            args.append({"true": 1, "false": 0, "float": "fp32", "__nv_bfloat16": "bf16"}.get(a) if not a.isdigit()
                        else int(a))
        return m.group(1), tuple(args)
    m = _MANGLED.search(name)
    if m:
        args = tuple(int(i) if i else "fp32" if f else "bf16" for i, f, _ in _MANGLED_ARG.findall(m.group(2)))
        return m.group(1), args
    return None


def kernel_labels(name):
    """the branch labels one launched kernel shows (the name-visible part of the labels the cases predict)"""
    inst = kernel_instantiation(name)
    if inst is None:
        return set()
    k, a = inst
    if k == "attention_kernel":
        return {f"attention DQ{a[0]}", f"attention DQ{a[0]} NWG{a[1]}"}
    if k == "gemm_conv_kernel":
        b = {f"gemm bn{a[0]}", f"gemm epilogue {_EPILOGUES[a[1]]}"}
        return b | {f"gemm kOps{a[2]}"} if a[1] == 0 else b  # kOps exists for the plain bf16 epilogue only
    if k == "layernorm_kernel":
        return {f"layernorm NV{a[0]} L{a[1]} RV{a[2]}"}
    if k == "temporal_attention_tc_kernel":
        return {f"temporal_attention SEQ{a[0]}"}
    if k == "gn_apply_kernel":
        return {f"gn_apply silu{a[0]} up{a[1]}"}
    return {f"nchw_to_nhwc src {a[0]}" if k == "nchw_to_nhwc_kernel" else f"nhwc_to_nchw dst {a[0]}"}


def visible_parts(branch):
    """the kernel_labels a predicted branch implies; empty for one decided at run time inside one instantiation (the
    storer kind, vectorised vs element-wise draining, kv_batch_div, the KV tile count, LayerNorm in place)"""
    m = re.fullmatch(r"gemm bn(\d+) (auto|forced)", branch)
    if m:
        return {f"gemm bn{m.group(1)}"}
    if branch.startswith("gemm epilogue "):
        return {branch}
    if branch.startswith("gemm storer ") or branch.startswith("gemm operands global "):
        return {"gemm kOps0"}
    m = re.fullmatch(r"gemm operands tma (bn(\d+)|kind\d)", branch)
    if m:
        return {"gemm kOps1"} | ({f"gemm bn{m.group(2)}"} if m.group(2) else set())
    m = re.fullmatch(r"attention DQ(\d)( NWG(\d))?.*", branch)
    if m:
        return {f"attention DQ{m.group(1)}"} | ({f"attention DQ{m.group(1)} NWG{m.group(3)}"} if m.group(2) else set())
    if re.fullmatch(r"layernorm NV\d+ L\d+ RV\d|temporal_attention SEQ\d+|gn_apply silu\d up\d|"
                    r"nchw_to_nhwc src \w+|nhwc_to_nchw dst \w+", branch):
        return {branch}
    return set()


# ----------------------------------------------------------------------------------------------------------------------
# the sampler
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    op: str                      # ops function, or "lib:<entry point>" for a direct C call
    label: str
    branches: Tuple[str, ...]
    make: Callable = field(repr=False)  # (device, generator) -> kwargs of the call


def _rn(g, shape, dev, scale=1.0, dtype=BF16):
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(dev)


def _inner(t, pad=64):
    """t as a view inside a larger allocation with finite neighbours on both sides (as the caching allocator leaves
    them), so that a read past its end picks up a plausible value in the step and NaN in the guarded replay"""
    flat = torch.randn(t.numel() + 2 * pad).to(t.dtype).to(t.device)
    flat[pad:pad + t.numel()] = t.reshape(-1)
    return flat[pad:pad + t.numel()].view(t.shape)


def _slot(t, left=4, right=12):
    """t's values in columns [left, left + n) of a [rows, left + n + right] buffer: a strided view, not 16-byte
    aligned for left = 4 bf16, with stride gaps holding finite values"""
    rows, n = t.shape
    buf = torch.randn(rows, left + n + right).to(t.dtype).to(t.device)
    buf[:, left:left + n] = t
    return buf[:, left:left + n]


def _gemm_cases(s):
    out = []
    m, k = (192, 64) if s else (640, 128)
    sizes = {64: 40, 128: 96, 160: 320, 256: 512}  # w_rows whose automatic N tile is the key
    for bn_auto, n in sizes.items():
        for kind in range(8):
            for vec in (True, False):
                rv, res, bl = bool(kind & 1), bool(kind & 2), bool(kind & 4)

                def make(dev, g, n=n, rv=rv, res=res, bl=bl, vec=vec):
                    kw = dict(x=_rn(g, (m, k), dev), w=_rn(g, (n, k), dev, k ** -0.5), bias=_rn(g, (n,), dev, 0.5, F32))
                    kw["bias"] = kw["bias"].to(BF16).float()
                    if rv:
                        kw["rowvec"], kw["rows_per_vec"] = _rn(g, (m // 64, n), dev), 64
                    if res:
                        kw["residual"] = _rn(g, (m, n), dev)
                    if bl:
                        kw["blend_src"] = _rn(g, (m, n), dev)
                        kw["blend_alpha"] = torch.tensor([0.3], device=dev).to(BF16).float()
                    if not vec:  # the element-wise drain: output, residual and blend source not 16-byte aligned
                        kw["out"] = _slot(torch.zeros(m, n, dtype=BF16, device=dev))
                        for a in ("residual", "blend_src"):
                            if a in kw:
                                kw[a] = _slot(kw[a])
                    return kw
                out.append(Case("linear", f"linear m{m} k{k} n{n} kind{kind} {'vec' if vec else 'elem'}",
                                tuple(gemm_branches(n, vec=vec, rowvec=rv, residual=res, blend=bl)), make))
    for bn in (64, 128, 160, 256):  # forced N tile on a width none of them divides evenly
        n = 200
        out.append(Case("linear", f"linear n{n} bn{bn}", tuple(gemm_branches(n, bn=bn)),
                        lambda dev, g, n=n, bn=bn: dict(x=_rn(g, (m, k), dev), w=_rn(g, (n, k), dev, k ** -0.5),
                                                        bn=bn)))
    # fp32 epilogue: SiLU, scale, row vector and residual, with n_out not a multiple of 8
    for act, rv, res, scale in ((1, False, False, 1.0), (0, True, False, 1.0), (0, False, True, 1.0),
                                (0, False, True, 0.7), (1, True, True, 0.5)):
        n = 36

        def make(dev, g, n=n, act=act, rv=rv, res=res, scale=scale):
            kw = dict(x=_rn(g, (m, k), dev), w=_rn(g, (n, k), dev, k ** -0.5), out_fp32=True, act=act,
                      out_scale=scale, bias=_rn(g, (n,), dev, 0.5).float())
            if rv:
                kw["rowvec"], kw["rows_per_vec"] = _rn(g, (m // 64, n), dev), 64
            if res:
                kw["residual"] = _rn(g, (m, n), dev)
            return kw
        out.append(Case("linear", f"linear f32 n{n} act{act} rv{int(rv)} res{int(res)} scale{scale}",
                        tuple(gemm_branches(n, act=act, out_fp32=True)), make))
    from ctrl_adapter_b200.ops import pack_geglu_weight

    def geglu(dev, g):
        w, b = _rn(g, (512, k), dev, k ** -0.5), _rn(g, (512,), dev, 0.5)
        wi, bi = pack_geglu_weight(w, b)
        return dict(x=_rn(g, (m, k), dev), w=wi, bias=bi.float(), act=2)
    out.append(Case("linear", "linear geglu n256", tuple(gemm_branches(512, act=2)), geglu))
    # convolution with the fp32 epilogue's SiLU and per-sample row vector
    def conv(dev, g):
        from ctrl_adapter_b200.ops import pack_conv_weight
        x = _rn(g, (2, 6, 10, 64), dev)
        return dict(x=x, w_packed=pack_conv_weight(_rn(g, (40, 64, 3, 3), dev, 64 ** -0.5 / 3)), bias=None,
                    act=1, rowvec=_rn(g, (2, 40), dev), out_fp32=True)
    out.append(Case("conv2d", "conv3x3 f32 silu rowvec", tuple(gemm_branches(40, act=1, out_fp32=True)), conv))
    return out


def _epilogue_linear(label, m, k, n, kind, *, bn=0, rpv=40, res_pad=0, broadcast=False, out_over_res=False):
    """a bf16 linear with storer kind `kind` (1 row vector, 2 residual, 4 blend source).  res_pad: residual and blend
    source as 16-byte-aligned views with row stride n + res_pad (ops.linear reads both with the residual's stride);
    broadcast: both are one row expanded along M (stride 0); out_over_res: the output written over the residual"""
    rv, res, bl = bool(kind & 1), bool(kind & 2), bool(kind & 4)

    def make(dev, g):
        kw = dict(x=_rn(g, (m, k), dev), w=_rn(g, (n, k), dev, k ** -0.5), bias=_rn(g, (n,), dev, 0.5).float(), bn=bn)
        if rv:
            kw["rowvec"], kw["rows_per_vec"] = _rn(g, (m // rpv, n), dev), rpv

        def source():
            if broadcast:
                return _rn(g, (1, n), dev).expand(m, n)
            t = _rn(g, (m, n), dev)
            return _slot(t, 0, res_pad) if res_pad else t
        if res:
            kw["residual"] = source()
        if bl:
            kw["blend_src"] = source()
            kw["blend_alpha"] = torch.tensor([0.3], device=dev).to(BF16).float()
        if out_over_res:
            kw["out"] = kw["residual"]
        return kw
    stride = 0 if broadcast else n + res_pad  # ops.linear's res_strides and out_dims
    rs, dims = ((stride, rpv * stride, 0, 0), (rpv, m // rpv, 1, 1)) if rv else ((stride, 0, 0, 0), (m, 1, 1, 1))
    return Case("linear", label, tuple(gemm_branches(n, bn=bn, rowvec=rv, residual=res, blend=bl, res_strides=rs,
                                                     out_dims=dims)), make)


def _gemm_operand_cases():
    """the bf16 epilogue's residual / blend source by TMA (kOps): every N tile automatic and forced, partial 32-column
    slabs (n_out 8, 24, 40, 168, 200), M not a multiple of 128 with more tiles than SMs, strided sources, row vectors
    over fewer than 128 rows (the 2-D box), the output written over the residual, convolutions with boxes reaching past
    the image; and the broadcast sources (stride 0 along M) that keep the per-chunk global loads"""
    out = []
    for i, n in enumerate((8, 24, 40, 96, 168, 320)):  # automatic N tile 64, 64, 64, 128, 256, 160
        kind = 2 + i
        out.append(_epilogue_linear(f"linear ops n{n} kind{kind}", 200, 64, n, kind))
    for bn in (64, 128, 160, 256):
        for kind in range(2, 8):
            out.append(_epilogue_linear(f"linear ops n200 bn{bn} kind{kind}", 200, 64, 200, kind, bn=bn))
    out.append(_epilogue_linear("linear ops m4500 n200 bn64 kind6", 4500, 64, 200, 6, bn=64))  # 144 tiles
    out.append(_epilogue_linear("linear ops m4500 n320 bn64 kind7 rpv180", 4500, 64, 320, 7, bn=64, rpv=180))
    out.append(_epilogue_linear("linear ops m9000 n512 kind2", 9000, 64, 512, 2))  # BN 256: 142 tiles
    for n, bn, kind in ((96, 0, 2), (96, 0, 4), (96, 0, 6), (200, 160, 7)):
        out.append(_epilogue_linear(f"linear ops n{n} bn{bn} kind{kind} source stride n+8", 200, 64, n, kind, bn=bn,
                                    res_pad=8))
    for kind in (3, 7):
        out.append(_epilogue_linear(f"linear ops m192 n96 kind{kind} rpv48", 192, 64, 96, kind, rpv=48))
    for bn, kind in ((64, 2), (128, 2), (160, 6), (256, 3)):
        out.append(_epilogue_linear(f"linear ops n200 bn{bn} kind{kind} out over residual", 200, 64, 200, kind, bn=bn,
                                    out_over_res=True))
    for kind, n in zip(range(2, 8), (40, 96, 320, 512, 40, 320)):  # automatic N tile 64, 128, 160, 256, 64, 160
        out.append(_epilogue_linear(f"linear broadcast sources m192 n{n} kind{kind}", 192, 64, n, kind, rpv=64,
                                    broadcast=True))
    from ctrl_adapter_b200.ops import pack_conv_weight

    def conv(n, h, w, c0, c1, cout, kind):
        def make(dev, g):
            kw = dict(x=_rn(g, (n, h, w, c0), dev), bias=_rn(g, (cout,), dev, 0.5).float(),
                      w_packed=pack_conv_weight(_rn(g, (cout, c0 + c1, 3, 3), dev, (c0 + c1) ** -0.5 / 3)))
            if c1:
                kw["x2"] = _rn(g, (n, h, w, c1), dev)
            if kind & 1:
                kw["rowvec"] = _rn(g, (n, cout), dev)
            if kind & 2:
                kw["residual"] = _rn(g, (n, h, w, cout), dev)
            if kind & 4:
                kw["blend_src"] = _rn(g, (n, h, w, cout), dev)
                kw["blend_alpha"] = torch.tensor([0.7], device=dev).to(BF16).float()
            return kw
        out.append(Case("conv2d", f"conv3x3 n{n} {h}x{w} c{c0}+{c1} cout{cout} kind{kind}",
                        tuple(gemm_branches(cout, rowvec=bool(kind & 1), residual=bool(kind & 2),
                                            blend=bool(kind & 4))), make))
    conv(2, 6, 10, 64, 0, 40, 2)
    conv(2, 6, 10, 64, 0, 40, 7)
    conv(2, 5, 7, 64, 32, 96, 6)
    conv(1, 6, 10, 64, 0, 40, 3)
    conv(1, 5, 7, 64, 32, 168, 6)
    for frames, kind in ((5, 6), (3, 7)):
        def make_t(dev, g, frames=frames, kind=kind):
            c, cout = 64, 96
            kw = dict(x=_rn(g, (2 * frames, 3, 5, c), dev), bias=_rn(g, (cout,), dev, 0.5).float(), frames=frames,
                      w_packed=pack_conv_weight(_rn(g, (cout, c, 3, 1, 1), dev, (3 * c) ** -0.5)),
                      residual=_rn(g, (2 * frames, 3, 5, cout), dev), blend_src=_rn(g, (2 * frames, 3, 5, cout), dev),
                      blend_alpha=torch.tensor([0.4], device=dev).to(BF16).float())
            if kind & 1:
                kw["rowvec"] = _rn(g, (2 * frames, cout), dev)
            return kw
        out.append(Case("temporal_conv", f"temporal_conv frames{frames} kind{kind}",
                        tuple(gemm_branches(96, rowvec=bool(kind & 1), residual=True, blend=True)), make_t))
    return out


def _norm_cases(s):
    out = []
    # LayerNorm: one width per (NV, L) instantiation, 8 <= c <= 2048, with and without the row vector
    widths = {"layernorm NV1 L8 RV0": 8}
    for c in range(8, 2049, 8):
        widths.setdefault(layernorm_variant(c, False), c)
    widths["layernorm NV1 L8 RV0"] = 8
    for variant, c in sorted(widths.items(), key=lambda kv: kv[1]):
        for rv in (False, True):
            rows = 40 if rv else 37  # 37: a short last step of every lane group

            def make(dev, g, c=c, rv=rv, rows=rows):
                kw = dict(x=_rn(g, (rows, c), dev), gamma=_rn(g, (c,), dev, 0.2, F32) + 1.0,
                          beta=_rn(g, (c,), dev, 0.2, F32), eps=1e-5)
                if rv:
                    kw.update(add_rowvec=_rn(g, (5, c), dev), rows_per_vec=8, return_sum=True)
                return kw
            out.append(Case("layer_norm", f"layernorm rows{rows} c{c} rv{int(rv)}", (layernorm_variant(c, rv),), make))
    for c, rv in ((320, False), (640, True), (2048, False)):  # in place: y (or y_sum) aliases x
        def make(dev, g, c=c, rv=rv):
            return dict(x=_rn(g, (37 if not rv else 40, c), dev), gamma=_rn(g, (c,), dev, 0.2, F32) + 1.0,
                        beta=_rn(g, (c,), dev, 0.2, F32), eps=1e-5,
                        add_rowvec=_rn(g, (5, c), dev) if rv else None, rows_per_vec=8 if rv else 0)
        out.append(Case("lib:ca_layernorm", f"layernorm in place c{c} rv{int(rv)}",
                        ("layernorm in place", layernorm_variant(c, rv)), make))
    # GroupNorm: group counts other than 32 (groups of 4 channels split an 8-channel vector), both channel extremes,
    # concatenated sources, samples of several images, the four apply variants
    gn = [(8, 0, 1), (24, 0, 6), (40, 0, 5), (48, 0, 3), (72, 0, 9), (64, 0, 64), (128, 64, 16), (4096, 0, 64),
          (320, 0, 32), (96, 32, 2)]
    for i, (c0, c1, groups) in enumerate(gn):
        silu, up = bool(i & 1), bool(i & 2)
        ips = 2 if i % 3 == 0 else 1
        h, w = (3, 5) if c0 + c1 >= 2048 else (6, 7)

        def make(dev, g, c0=c0, c1=c1, groups=groups, silu=silu, up=up, ips=ips, h=h, w=w):
            return dict(x=_rn(g, (2 * ips, h, w, c0), dev) + 0.5, gamma=_rn(g, (c0 + c1,), dev, 0.2, F32) + 1.0,
                        beta=_rn(g, (c0 + c1,), dev, 0.2, F32), eps=1e-6, groups=groups, silu=silu, up2x=up,
                        x2=_rn(g, (2 * ips, h, w, c1), dev) if c1 else None, imgs_per_sample=ips)
        out.append(Case("group_norm", f"groupnorm c{c0}+{c1} groups{groups} silu{int(silu)} up{int(up)} ips{ips}",
                        (f"gn_apply silu{int(silu)} up{int(up)}",), make))
    return out


def _attention_tile_cases():
    """KV rings of more than one tile and the 192-row query tiles (attention_nwg) under guard bands: head dim 64 on
    both sides of every flip of the tile rule, lk 129 (a 1-key last tile) to 1300 (11 tiles through the 4-slot ring),
    shared contexts, fused-QKV views (row stride 3 C), an output view with gap columns, head dims 128 and 192.  peaks:
    (query row, key) pairs whose query is 3x that key, so the row's logits peak there ~20 above the rest: in the
    ragged last KV tile (every earlier tile's running max and sum must be rescaled) or in the first"""
    out = []

    def case(dp, lq, lk, *, b=1, heads=2, div=1, fused=False, out_gap=0, peaks=()):
        def make(dev, g):
            d, c = dp - 16, heads * dp  # zero-padded head dim, as the modules pack it

            def padded(bb, ll):
                t = torch.zeros(bb, ll, heads, dp)
                t[..., :d] = torch.randn(bb, ll, heads, d, generator=g)
                return t
            q, k, v = padded(b, lq), padded(b // div, lk), padded(b // div, lk)
            for row, key in peaks:
                q[:, row] = 3.0 * k[torch.arange(b) // div, key]
            if fused:  # Q, K, V as column views of one [b, l, 3 C] projection
                qkv = torch.cat([t.reshape(b, lq, c) for t in (q, k, v)], dim=2).to(BF16).to(dev)
                kw = dict(q=qkv[..., :c], k=qkv[..., c:2 * c], v=qkv[..., 2 * c:])
            else:
                kw = {n: t.reshape(t.shape[0], t.shape[1], c).to(BF16).to(dev) for n, t in zip("qkv", (q, k, v))}
            if out_gap:
                kw["out"] = torch.zeros(b, lq, c + out_gap, dtype=BF16, device=dev)[..., :c]
            return dict(kw, heads=heads, head_dim_pad=dp, scale=d ** -0.5, kv_batch_div=div)
        tags = " fused-qkv" * fused + f" out gap{out_gap}" * bool(out_gap) + f" peaks{list(peaks)}" * bool(peaks)
        out.append(Case("attention", f"attention dp{dp} b{b} lq{lq} lk{lk} kv_div{div}{tags}",
                        tuple(attention_branches(dp, lq, lk, div)), make))
    for lq, lk in ((1, 128), (1, 129), (128, 257), (129, 257), (144, 1300), (191, 129), (192, 128), (192, 129),
                   (193, 257), (576, 1300), (577, 257), (1599, 129), (1600, 257)):
        case(64, lq, lk)
    case(64, 192, 300, b=4, div=2, peaks=((0, 299), (191, 0)))
    case(64, 300, 300, fused=True, peaks=((5, 299), (77, 3)))
    case(64, 577, 577, fused=True)
    case(64, 384, 300, out_gap=16)
    case(64, 193, 1300, peaks=((0, 1299), (192, 0)))
    case(128, 300, 257, out_gap=16, peaks=((1, 256), (299, 2)))
    case(192, 200, 300, b=4, div=2, peaks=((3, 299), (150, 0)))
    return out


def _attention_cases(s):
    out = []
    for dp in (64, 128, 192):
        for div in (1, 2):
            b, heads, lq, lk = 4, 2, (130 if s else 300), 77

            def make(dev, g, dp=dp, div=div, b=b, heads=heads, lq=lq, lk=lk):
                d = dp - 16  # zero-padded head dim, as the modules pack it
                def padded(bb, ll):
                    t = torch.zeros(bb, ll, heads, dp)
                    t[..., :d] = torch.randn(bb, ll, heads, d, generator=g)
                    return t.reshape(bb, ll, heads * dp).to(BF16).to(dev)
                return dict(q=padded(b, lq), k=padded(b // div, lk), v=padded(b // div, lk), heads=heads,
                            head_dim_pad=dp, scale=d ** -0.5, kv_batch_div=div)
            out.append(Case("attention", f"attention dp{dp} kv_div{div}", tuple(attention_branches(dp, lq, lk, div)),
                            make))
    out += _attention_tile_cases()
    hw = 11 if s else 37
    for frames in range(1, 33):  # every frame count either SEQ instantiation takes
        def make(dev, g, frames=frames):
            heads, clips = 1, 2
            qkv = _rn(g, (clips * frames * hw, 3 * heads * 64), dev)
            return dict(q=qkv[:, :64], k=qkv[:, 64:128], v=qkv[:, 128:], clips=clips, frames=frames, hw=hw, heads=heads,
                        scale=0.125, row_stride=3 * heads * 64)
        out.append(Case("temporal_attention", f"temporal_attention frames{frames}",
                        (f"temporal_attention SEQ{16 if frames <= 16 else 32}",), make))
    return out


def _small_op_cases(s, rng):
    out = []
    for n in (8, 8 * 37, 8 * rng.randint(40, 400)):
        out.append(Case("silu", f"silu n{n}", (), lambda dev, g, n=n: dict(x=_inner(_rn(g, (n,), dev, 3.0)))))
        out.append(Case("add", f"add n{n}", (), lambda dev, g, n=n: dict(a=_inner(_rn(g, (n,), dev)),
                                                                       b=_inner(_rn(g, (n,), dev)))))
    for fp32 in (False, True):
        for c, cp in ((1, 1), (3, 8), (4, 4), (33, 40)):
            out.append(Case("nchw_to_nhwc", f"nchw_to_nhwc {'fp32' if fp32 else 'bf16'} c{c} c_pad{cp}",
                            (f"nchw_to_nhwc src {'fp32' if fp32 else 'bf16'}",),
                            lambda dev, g, c=c, cp=cp, fp32=fp32: dict(x=_rn(g, (2, c, 5, 7), dev, dtype=F32 if fp32
                                                                              else BF16), c_pad=cp)))
            out.append(Case("nhwc_to_nchw", f"nhwc_to_nchw {'fp32' if fp32 else 'bf16'} c{c} c_stride{cp}",
                            (f"nhwc_to_nchw dst {'fp32' if fp32 else 'bf16'}",),
                            lambda dev, g, c=c, cp=cp, fp32=fp32: dict(x=_rn(g, (2, 5, 7, cp), dev), c=c, fp32=fp32)))
    for (ry, rx) in ((1, 1), (2, 2), (4, 1), (1, 3), (2, 5)):
        out.append(Case("avgpool", f"avgpool ratio {ry}x{rx}", (),
                        lambda dev, g, ry=ry, rx=rx: dict(x=_rn(g, (2, 3 * ry, 4 * rx, 8), dev), oh=3, ow=4)))
    for c in (8, 24):
        out.append(Case("upsample2x", f"upsample2x c{c}", (), lambda dev, g, c=c: dict(x=_rn(g, (2, 3, 5, c), dev))))
    for cols in (4, 8, 12, 300, 1028):  # cols % 8 == 4 leaves a half vector pair per row
        out.append(Case("softmax_rows", f"softmax_rows cols{cols}", (),
                        lambda dev, g, cols=cols: dict(x=_rn(g, (5, cols), dev, 4.0, F32))))
    for e in (1, 7, 8, 9, 16, 31, 32):
        def make(dev, g, e=e):
            mask = torch.tensor([0 if i % 3 == 2 else 1 for i in range(e)], dtype=torch.uint8, device=dev)
            return dict(logits=_rn(g, (3, e), dev, 2.0, F32), mask=mask)
        out.append(Case("router_weights", f"router_weights experts{e}", (), make))
    for k in range(1, 9):
        out.append(Case("router_merge", f"router_merge nactive{k}", (),
                        lambda dev, g, k=k: dict(xs=[_rn(g, (2, 3, 4, 16), dev) for _ in range(k)],
                                                 w=_rn(g, (k,), dev, 0.5, F32))))
    for dim, flip, shift, rnd in ((2, True, 0.0, False), (7, True, 0.0, False), (7, False, 1.0, True),
                                  (320, True, 0.0, True), (321, False, 1.0, False)):
        out.append(Case("timestep_embedding", f"timestep_embedding dim{dim} flip{int(flip)} shift{shift}", (),
                        lambda dev, g, dim=dim, flip=flip, shift=shift, rnd=rnd: dict(
                            t=torch.tensor([0.0, 1.0, 17.5, 999.0], device=dev), dim=dim, flip_sin_to_cos=flip,
                            freq_shift=shift, round_t_bf16=rnd)))
    for cin, cout, frames in ((1, 1, 1), (3, 3, 3), (4, 4, 2), (2, 4, 5)):
        out.append(Case("frame_conv_small", f"frame_conv_small cin{cin} cout{cout} frames{frames}", (),
                        lambda dev, g, cin=cin, cout=cout, frames=frames: dict(
                            x=_rn(g, (2 * frames, 5, 7, 8), dev), w_host=torch.randn(cout, cin, 3, generator=g) * 0.5,
                            bias_host=torch.randn(cout, generator=g), frames=frames, cin=cin)))
    for frames, cs in ((1, 4), (2, 8), (17, 4), (32, 8)):
        def make(dev, g, frames=frames, cs=cs):
            params = (torch.randn(288, generator=g) * 0.5).to(BF16).float()
            params[:4] += 1.0
            return dict(x=_rn(g, (2 * frames, 3, 5, cs), dev), clips=2, frames=frames, params=params.to(dev))
        out.append(Case("i2vgen_latent_encoder", f"i2vgen_latent_encoder frames{frames} c_stride{cs}", (), make))
    for layout, frames, nv in ((0, 1, 1), (1, 2, 1), (1, 5, 2), (2, 1, 1), (2, 3, 2)):
        out.append(Case("vae_latents", f"vae_latents layout{layout} frames{frames} nv{nv}", (),
                        lambda dev, g, layout=layout, frames=frames, nv=nv: dict(
                            moments=_rn(g, (2, 3, 5, 8), dev), layout=layout,
                            noise=_rn(g, (2, 4, 3, 5), dev, dtype=F32) if layout != 2 else None, frames=frames,
                            num_videos=nv, scale=0.18215)))
    return out


def _scheduler_cases(s):
    """CFG + scheduler updates: rounded and fp32 latents, with and without the next model input, written to a new
    tensor or over the latents; Euler at 1 and 3 frames per clip, DDIM epsilon and v prediction"""
    out = []
    shape = (2, 3, 4, 6, 8)
    euler_row = [900.0, 11.3, 9.7, (9.7 ** 2 + 1) ** 0.5]
    for rnd, nxt, in_place in ((True, True, False), (False, False, True), (True, False, True), (False, True, False)):
        def make(dev, g, rnd=rnd, nxt=nxt, in_place=in_place, shape=shape):
            lat = _rn(g, shape, dev, 8.0, F32)
            kw = dict(eps_uncond=_rn(g, shape, dev), eps_text=_rn(g, shape, dev), latents=lat, guidance=5.0,
                      step_row=torch.tensor(euler_row, device=dev), round_latents_bf16=rnd,
                      latents_out=lat if in_place else None,
                      model_in_next=torch.empty(shape, dtype=BF16, device=dev) if nxt else None)
            return kw
        tag = f"round{int(rnd)} next{int(nxt)} in_place{int(in_place)}"
        out.append(Case("cfg_euler", f"cfg_euler {tag}", (), make))
        for frames in (1, 3):
            def make_v(dev, g, rnd=rnd, nxt=nxt, in_place=in_place, frames=frames):
                shp = (2, frames, 4, 6, 8)
                lat = _rn(g, shp, dev, 8.0, F32)
                return dict(eps_uncond=_rn(g, shp, dev), eps_text=_rn(g, shp, dev), latents=lat,
                            guidance_per_frame=torch.linspace(1.0, 3.0, frames).to(BF16).float().to(dev), frames=frames,
                            step_row=torch.tensor(euler_row, device=dev), round_latents_bf16=rnd,
                            latents_out=lat if in_place else None,
                            model_in_next=torch.empty(shp, dtype=BF16, device=dev) if nxt else None)
            out.append(Case("cfg_euler_v", f"cfg_euler_v frames{frames} {tag}", (), make_v))
        for vpred in (False, True):
            def make_d(dev, g, rnd=rnd, nxt=nxt, in_place=in_place, vpred=vpred, shape=shape):
                lat = _rn(g, shape, dev, 1.0, F32)
                return dict(eps_uncond=_rn(g, shape, dev), eps_text=_rn(g, shape, dev), latents=lat, guidance=9.0,
                            step_row=torch.tensor([500.0, 0.3, 0.45, 0.0], device=dev), round_latents_bf16=rnd,
                            v_prediction=vpred, latents_out=lat if in_place else None,
                            model_in_next=torch.empty(shape, dtype=BF16, device=dev) if nxt else None)
            out.append(Case("cfg_ddim", f"cfg_ddim vpred{int(vpred)} {tag}", (), make_d))
    # Conv3d (3, 1, 1) over the frames through the GEMM: one frame, and several with a per-frame row vector + residual
    from ctrl_adapter_b200.ops import pack_conv_weight
    for frames, epi in ((1, False), (5, True)):
        def make_t(dev, g, frames=frames, epi=epi):
            c, cout = 64, 96
            kw = dict(x=_rn(g, (2 * frames, 3, 5, c), dev),
                      w_packed=pack_conv_weight(_rn(g, (cout, c, 3, 1, 1), dev, (3 * c) ** -0.5)),
                      bias=_rn(g, (cout,), dev, 0.5).float(), frames=frames)
            if epi:
                kw.update(rowvec=_rn(g, (2 * frames, cout), dev), residual=_rn(g, (2 * frames, 3, 5, cout), dev))
            return kw
        out.append(Case("temporal_conv", f"temporal_conv frames{frames} rowvec+residual{int(epi)}",
                        tuple(gemm_branches(96, rowvec=epi, residual=epi)), make_t))
    return out


def cases(small=False, seed=0):
    rng = random.Random(seed)
    return (_gemm_cases(small) + _gemm_operand_cases() + _norm_cases(small) + _attention_cases(small) +
            _small_op_cases(small, rng) + _scheduler_cases(small))


# ----------------------------------------------------------------------------------------------------------------------
# the C domain: valid placeholder arguments and (argument, last inside, first outside) per entry point
# ----------------------------------------------------------------------------------------------------------------------
P = 1 << 20  # placeholder pointer, 256-byte aligned: validation fails (or passes) before anything is dereferenced


@dataclass
class Entry:
    args: dict                  # argument name -> valid value, in the C order (desc fields for the struct entries)
    constraints: list           # (argument, last value inside, first value outside[, status outside]); a value that is
                                # a dict sets several arguments at once, the constraint is still named by `argument`
    desc: str = None            # ctypes struct the arguments fill, passed by pointer with a NULL stream


def _attn_args():
    return dict(q=P, k=P, v=P, out=P, batch=4, heads=2, lq=128, lk=77, head_dim_pad=64, scale=0.125,
                q_row_stride=128, q_batch_stride=128 * 128, k_row_stride=128, k_batch_stride=128 * 77,
                v_row_stride=128, v_batch_stride=128 * 77, out_row_stride=128, out_batch_stride=128 * 128,
                kv_batch_div=2)


def _gemm_args():
    """a 256 x 64 -> 64 linear (ops.linear's descriptor)"""
    z4 = [0, 0, 0, 0]
    return dict(nsrc=1, a=[P, None], a_channels=[64, 0], a_c_off=[0, 0], a_c_len=[64, 0], a_dims=[256, 1, 1, 1],
                a_strides=[[64, 16384, 16384, 16384], z4], box=[128, 1, 1, 1], ntaps=1, tap_off=[z4] * 9,
                tap_c_off=[0] * 9, w=P, w_rows=64, w_k_per_tap=64, bias=None, out=P, out_fp32=0, n_out=64,
                out_dims=[256, 1, 1, 1], out_strides=[64, 0, 0, 0], act=0, out_scale=1.0, rowvec=None,
                rowvec_strides=z4, residual=None, blend_src=None, res_strides=z4, blend_alpha=None, bn=0)


_GEGLU = dict(act=2, w_rows=512, n_out=256, bn=256)
_CFG = dict(eps_uncond=P, eps_text=P, latents_in=P, n=64)
_INVALID, _UNSUPPORTED = 1, 3

DOMAIN = {
    "ca_gemm": Entry(_gemm_args(), [
        ("nsrc", dict(nsrc=2, a=[P, P], a_channels=[64, 64], a_c_len=[64, 64], w_k_per_tap=128,
                      a_strides=[[64, 16384, 16384, 16384], [64, 16384, 16384, 16384]]), 3),
        ("ntaps", 9, 10), ("box", [128, 1, 1, 1], [64, 1, 1, 1]), ("bn", 256, 96),
        ("n_out", dict(w_rows=56, n_out=56), dict(w_rows=60, n_out=60)),
        ("w_rows", _GEGLU, dict(_GEGLU, w_rows=384, n_out=192)),
        ("out_fp32", _GEGLU, dict(_GEGLU, out_fp32=1), _UNSUPPORTED),
        ("out_fp32", dict(blend_src=P, blend_alpha=P), dict(blend_src=P, blend_alpha=P, out_fp32=1), _UNSUPPORTED),
        ("a_channels", [64, 0], [56, 0]), ("a_c_off", dict(a_c_off=[8, 0], a_channels=[72, 0]), dict(a_c_off=[4, 0], a_channels=[72, 0])), ("w_k_per_tap", 64, 56)], desc="GemmDesc"),
    "ca_attention": Entry(_attn_args(), [
        ("batch", 65534, 65536), ("heads", 65535, 65536), ("out", P + 4, P + 2), ("out_row_stride", 130, 129),
        ("out_batch_stride", 128 * 128 + 2, 128 * 128 + 1), ("kv_batch_div", 4, 3)], desc="AttentionDesc"),
    "ca_temporal_attention": Entry(dict(q=P, k=P, v=P, clips=1, frames=16, hw=16, heads=1, scale=0.125,
                                        in_row_stride=192, out=P, stream=None), [
        ("frames", 32, 33), ("in_row_stride", 200, 196), ("out", P + 4, P + 2), ("clips", 1, 0), ("heads", 1, 0)]),
    "ca_groupnorm_stats": Entry(dict(x0=P, c0=320, x1=None, c1=0, n=2, rows=64, groups=32, sums=P, stream=None), [
        ("groups", 64, 65), ("n", 65535, 65536), ("x0", P + 16, P + 8), ("rows", 1, 0), ("c0", 4096, 4128),
        ("x1", dict(x1=P + 16, c1=64), dict(x1=P + 8, c1=64))]),
    "ca_groupnorm_apply": Entry(dict(x0=P, c0=320, x1=P, c1=64, n=4, h=8, w=8, imgs_per_sample=2, groups=32,
                                     eps=1e-6, sums=P, gamma=P, beta=P, silu=1, up2x=1, y=P, stream=None), [
        ("n", 65534, 65536), ("x0", P + 16, P + 8), ("x1", P + 16, P + 8), ("y", P + 16, P + 8),
        ("imgs_per_sample", 4, 3), ("h", 1, 0), ("w", 1, 0), ("groups", 64, 65)]),
    "ca_layernorm": Entry(dict(x=P, rows=37, c=320, eps=1e-5, gamma=P, beta=P, add_rowvec=P, rows_per_vec=8,
                               y_sum=P, y=P, stream=None), [
        ("c", 2048, 2056), ("gamma", P + 16, P + 4), ("beta", P + 16, P + 8), ("add_rowvec", P + 16, P + 8),
        ("y", P + 16, P + 8), ("y_sum", P + 16, P + 8), ("x", P + 16, P + 8), ("rows", 2 ** 31 - 65, 2 ** 31 - 64)]),
    "ca_timestep_embedding": Entry(dict(t=P, n=2, dim=320, flip_sin_to_cos=1, freq_shift=0.0, round_t_bf16=0,
                                        out=P, stream=None), [("dim", 2, 1), ("n", 1, 0)]),
    "ca_silu": Entry(dict(x=P, n=64, y=P, stream=None), [("n", 64, 60), ("x", P + 16, P + 8), ("y", P + 16, P + 2)]),
    "ca_add": Entry(dict(a=P, b=P, n=64, y=P, stream=None), [
        ("n", 64, 60), ("a", P + 16, P + 8), ("b", P + 16, P + 8), ("y", P + 16, P + 8)]),
    "ca_nchw_to_nhwc": Entry(dict(x=P, src_fp32=1, n=2, c=3, hw=35, c_pad=8, y=P, stream=None), [
        ("c_pad", 3, 2), ("n", 65535, 65536), ("c", 1, 0), ("hw", 1, 0), ("hw", 2 ** 32 - 1, 2 ** 32),
        ("c_pad", 65535 * 32, 65535 * 32 + 1)]),
    "ca_nhwc_to_nchw": Entry(dict(x=P, n=2, c=3, c_stride=8, hw=35, y=P, dst_fp32=1, stream=None), [
        ("c_stride", 3, 2), ("n", 65535, 65536), ("c", 1, 0), ("hw", 1, 0), ("hw", 2 ** 32 - 1, 2 ** 32),
        ("c", dict(c=65535 * 32, c_stride=65535 * 32), dict(c=65535 * 32 + 1, c_stride=65535 * 32 + 1))]),
    "ca_avgpool": Entry(dict(x=P, n=1, h=12, w=10, c=8, oh=3, ow=5, y=P, stream=None), [
        ("oh", 12, 5), ("ow", 10, 4)]),
    "ca_upsample2x": Entry(dict(x=P, n=1, h=4, w=4, c=16, y=P, stream=None), [
        ("c", 16, 12), ("x", P + 16, P + 8), ("y", P + 16, P + 8)]),
    "ca_router_weights": Entry(dict(logits=P, mask=P, nrouters=3, nexperts=8, weights=P, stream=None), [
        ("nexperts", 32, 33), ("nrouters", 1, 0)]),
    "ca_router_merge": Entry(dict(xs=[P] * 8, w=P, nactive=8, n=64, y=P, stream=None), [
        ("nactive", 8, 9), ("n", 64, 60), ("xs", [P] * 8, None), ("xs[7]", P + 16, P + 8), ("y", P + 16, P + 8)]),
    "ca_softmax_rows": Entry(dict(x=P, rows=5, cols=12, y=P, stream=None), [
        ("cols", 4, 2), ("rows", 1, 0), ("x", P + 16, P + 8), ("y", P + 8, P + 4)]),
    "ca_frame_conv_small": Entry(dict(x=P, clips=1, frames=4, hw=16, c_stride=8, cin=3, cout=3, w_host=P,
                                      bias_host=None, y=P, stream=None), [
        ("cin", 4, 5), ("cout", 4, 5), ("c_stride", 4, 6), ("frames", 65535, 65536), ("x", P + 8, P + 4),
        ("y", P + 4, P + 2)]),
    "ca_cfg_euler": Entry(dict(_CFG, guidance=7.5, step_row=P, round_latents_bf16=1, latents_out=P,
                               model_in_next=None, stream=None), [
        ("n", 0, -1), ("step_row", P, None), ("latents_out", P, None), ("latents_in", P, None)]),
    "ca_cfg_euler_v": Entry(dict(_CFG, guidance=P, frames=2, frame_elems=16, step_row=P, round_latents_bf16=0,
                                 latents_out=P, model_in_next=P, stream=None), [
        ("frames", 4, 0), ("frame_elems", 32, 0), ("n", 128, 80), ("guidance", P, None), ("step_row", P, None)]),
    "ca_cfg_ddim": Entry(dict(_CFG, guidance=7.5, step_row=P, round_latents_bf16=1, v_prediction=1, latents_out=P,
                              model_in_next=P, stream=None), [
        ("n", 0, -1), ("eps_text", P, None), ("latents_out", P, None)]),
    "ca_i2vgen_latent_encoder": Entry(dict(x=P, clips=1, frames=16, hw=16, c_stride=8, params=P, y=P, stream=None), [
        ("frames", 32, 33), ("c_stride", 4, 3), ("clips", 1, 0), ("hw", 1, 0)]),
    "ca_vae_latents": Entry(dict(moments=P, noise=None, n=1, hw=64, latent_channels=4, layout=1, frames=4,
                                 num_videos=1, scale=0.18, out=P, stream=None), [
        ("moments", P + 16, P + 8), ("layout", 2, 3), ("latent_channels", 4, 5), ("frames", 1, 0),
        ("num_videos", 1, 0), ("out", P, None)]),
}


def boundaries():
    """[(entry point, argument, inside, outside, status outside)] over the whole table"""
    return [(name, c[0], c[1], c[2], c[3] if len(c) > 3 else _INVALID)
            for name, e in DOMAIN.items() for c in e.constraints]


def _set_field(d, k, v):
    cur = getattr(d, k)
    if not isinstance(v, (list, tuple)):
        setattr(d, k, v)
        return
    for i, x in enumerate(v):  # array fields element by element (rows of 2-D arrays likewise)
        if isinstance(x, (list, tuple)):
            for j, y in enumerate(x):
                cur[i][j] = y
        else:
            cur[i] = x


def c_call(lib, name, args):
    """call entry point `name` with the argument dict (desc entries fill their struct) -> status"""
    from ctrl_adapter_b200 import _lib
    entry = DOMAIN[name]
    if entry.desc is not None:
        d = getattr(_lib, entry.desc)()
        for k, v in args.items():
            _set_field(d, k, v)
        return getattr(lib, name)(C.byref(d), None)
    vals = []
    for k, v in args.items():
        if isinstance(v, list):  # a host array of device pointers
            v = (C.c_void_p * len(v))(*v)
        elif k == "w_host":  # a host array the entry point reads before it launches
            v = (C.c_float * 48)()
        vals.append(v)
    return getattr(lib, name)(*vals)


def with_value(name, arg, value):
    args = dict(DOMAIN[name].args)
    if isinstance(value, dict):
        args.update(value)
    elif "[" in arg:
        base, i = arg[:-1].split("[")
        args[base] = list(args[base])
        args[base][int(i)] = value
    else:
        args[arg] = value
    return args


# ----------------------------------------------------------------------------------------------------------------------
# running the sweep
# ----------------------------------------------------------------------------------------------------------------------
def layernorm_in_place(a, device):
    """ca_layernorm with y (no row vector) or y_sum (row vector) aliasing x; -> (y, y_sum).  On the CPU the same
    aliasing is emulated: the emulated results are written over x."""
    x = a["x"]
    rows, c = x.shape
    if torch.device(device).type != "cuda":
        from tests import ops_emulator as emu
        y, ys = emu.layer_norm(x, a["gamma"], a["beta"], a["eps"], add_rowvec=a["add_rowvec"],
                               rows_per_vec=a["rows_per_vec"], return_sum=True)
        if ys is None:
            x.copy_(y)
            return x, None
        x.copy_(ys)
        return y, x
    from ctrl_adapter_b200 import _lib, ops
    rv = a["add_rowvec"]
    y = x if rv is None else torch.empty_like(x)
    y_sum = x if rv is not None else None
    _lib.check(_lib.load().ca_layernorm(x.data_ptr(), rows, c, float(a["eps"]), a["gamma"].data_ptr(),
                                        a["beta"].data_ptr(), None if rv is None else rv.data_ptr(), a["rows_per_vec"],
                                        None if y_sum is None else y_sum.data_ptr(), y.data_ptr(),
                                        ops._stream()), "ca_layernorm")
    return y, y_sum


class KernelTrace:
    """with KernelTrace() as tr, Recorder() as rec: -- wraps the `ops` entry points before the recorder wraps them, so
    that the first launch after arm() (the recorder's in-step launch, not its re-runs or replay) runs under
    torch.profiler, kernel trace only (ProfilerActivity.CUDA: no hardware counters).  tr.names: the CUDA events of that
    launch (None: nothing ran under the trace)."""

    def __init__(self):
        self.armed, self.names, self._saved = False, None, {}

    def __enter__(self):
        from ctrl_adapter_b200 import ops
        from tests import launch_checks as lc
        for name in lc.OPS:
            fn = self._saved[name] = getattr(ops, name)
            setattr(ops, name, self._wrap(fn))
        return self

    def __exit__(self, *exc):
        from ctrl_adapter_b200 import ops
        for name, fn in self._saved.items():
            setattr(ops, name, fn)
        self._saved = {}
        return False

    def arm(self):
        self.armed, self.names = True, None

    def _wrap(self, fn):
        def traced(*args, **kw):
            if not self.armed:
                return fn(*args, **kw)
            return self.run(lambda: fn(*args, **kw))
        return traced

    def run(self, call):
        from torch.autograd import DeviceType
        from torch.profiler import ProfilerActivity, profile
        self.armed = False
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            # margins on both sides of the launch: a trace now and then comes back without the launch's device events
            # (3 of 319 traces in one sweep without them, 1 of 319 with them; run_cases then traces the case again)
            time.sleep(0.005)
            ret = call()
            torch.cuda.synchronize()
            time.sleep(0.005)
        self.names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
        return ret


def run_cases(cs, device, recorder, trace=None):
    """every case: `ops` calls through the (entered) recorder, direct C calls checked here.  trace: an entered
    KernelTrace; the names of the kernels each case's first launch ran go to trace.seen[case label].
    -> {case label: (op, rows checked, worst err/tol, ok, why)}"""
    from ctrl_adapter_b200 import ops
    from tests import kernel_checks as kc
    from tests import launch_checks as lc
    out = {}
    if trace is not None:
        trace.seen = {}
    for i, case in enumerate(cs):
        g = torch.Generator().manual_seed(1000 + i)
        kw = case.make(device, g)
        if trace is not None:
            trace.arm()
        if case.op.startswith("lib:"):
            pre = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in kw.items()}
            if trace is None:
                y, ys = layernorm_in_place(kw, device)
            else:
                y, ys = trace.run(lambda: layernorm_in_place(kw, device))
                _retrace(trace, case, i, device)
            kc._sync()
            row = lc.Row(case.op, ())
            try:
                row.add(kc.layernorm_verdict(case.label, {**pre, "return_sum": ys is not None},
                                             (y, ys) if ys is not None else y))
            except Exception as e:  # noqa: BLE001 -- a case the verdict cannot handle fails
                row.fail(f"{type(e).__name__}: {e}"[:300])
            out[case.label] = (case.op, [row])
            continue
        before = set(recorder.rows)
        getattr(ops, case.op)(**kw)
        kc._sync()
        if trace is not None:
            _retrace(trace, case, i, device)
        new = [recorder.rows[k] for k in recorder.rows if k not in before]
        if not new:  # the same configuration as an earlier case: that row stands for it
            new = [recorder.rows[lc.config_key(case.op, _bound(case.op, kw))]]
        out[case.label] = (case.op, new)
    return out


def _retrace(trace, case, i, device):
    """trace.seen[case label] = the trace's CUDA events.  A trace that came back without any: the case launched again
    on fresh inputs (the same configuration, its first launch already checked) under a new trace, at most twice"""
    from ctrl_adapter_b200 import ops
    for _ in range(2):
        if trace.names:
            break
        kw = case.make(device, torch.Generator().manual_seed(1000 + i))
        trace.arm()
        if case.op.startswith("lib:"):
            trace.run(lambda: layernorm_in_place(kw, device))
        else:
            getattr(ops, case.op)(**kw)
        torch.cuda.synchronize()
    trace.seen[case.label] = trace.names


def _bound(op, kw):
    from tests import launch_checks as lc
    b = lc._SIGS[op].bind(**kw)
    b.apply_defaults()
    return dict(b.arguments)


def summary(cs, results):
    """one line per case, then per entry point: cases, branches, worst err/tol"""
    lines = [f"{'case':<58} {'err/tol':>8}  result"]
    fam = {}
    for case in cs:
        op, rows = results[case.label]
        worst = max(r.worst for r in rows)
        ok = all(r.ok for r in rows)
        lines.append(f"{case.label:<58} {worst:>8.3f}  {'ok' if ok else 'FAIL ' + '; '.join(sum((r.why for r in rows), []))}")
        n, br, w = fam.get(op, (0, set(), 0.0))
        fam[op] = (n + 1, br | set(case.branches), max(w, worst))
    lines.append(f"\n{'entry point':<24} {'cases':>6} {'branches':>9} {'worst err/tol':>14}")
    for op, (n, br, w) in sorted(fam.items()):
        lines.append(f"{op:<24} {n:>6} {len(br):>9} {w:>14.3f}")
    return "\n".join(lines)


def failures(results):
    return [(label, r) for label, (_, rows) in results.items() for r in rows if not r.ok]


def observed_dispatch(cs, seen):
    """cases vs the kernels their first launch ran (seen: {case label: CUDA event names}).
    -> (problems, reached, instantiations): a problem per case whose trace holds no CUDA event, or whose predicted
    name-visible labels are not exactly those of its kernels; the branches reached, each counted only where its
    name-visible part was observed; {kernel<template arguments>: number of cases}"""
    problems, reached, inst = [], set(), {}
    for case in cs:
        names = seen.get(case.label)
        if not names:
            problems.append(f"{case.label}: torch.profiler recorded no CUDA kernel event for its first launch")
            continue
        observed = set().union(*(kernel_labels(n) for n in names))
        predicted = set().union(*(visible_parts(b) for b in case.branches))
        if predicted != observed:
            problems.append(f"{case.label}: predicted {sorted(predicted - observed)}, observed {sorted(observed - predicted)}")
        reached |= {b for b in case.branches if visible_parts(b) <= observed}
        for k in {kernel_instantiation(n) for n in names} - {None}:
            key = f"{k[0]}<{', '.join(map(str, k[1]))}>"
            inst[key] = inst.get(key, 0) + 1
    return problems, reached, inst


def dispatch_summary(reached, inst):
    """the kernel instantiations observed, and the expected branches that are run-time switches (predicted only)"""
    lines = [f"\n{'observed instantiation':<44} {'cases':>6}"]
    lines += [f"{k:<44} {n:>6}" for k, n in sorted(inst.items())]
    predicted = sorted(b for b in expected_branches() & reached if not visible_parts(b))
    partly = sorted(b for b in expected_branches() & reached if visible_parts(b) and visible_parts(b) != {b})
    lines.append(f"\nbranches observed in kernel names: {len(expected_branches() & reached) - len(predicted) - len(partly)}")
    lines.append(f"observed in part (the instantiation; the rest a run-time switch): {', '.join(partly)}")
    lines.append(f"predicted only (run-time switches): {', '.join(predicted)}")
    return "\n".join(lines)
