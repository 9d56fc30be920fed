"""pytest -m gpu: the GEMM kernel -- every instantiation and storer path -- bit for bit (tests/gemm_exact.py).

Each case runs one `ops` call and the same call's fp32 accumulators (the fp32-output instantiation at the same N tile
with an empty epilogue), and requires the accumulators to be within the census's pre-activation bound of the float64
contraction of the same operands (gx.accumulator_verdict), the call's output bits to equal the epilogue chain restated
in torch fp32 on those accumulators, and every byte around an output slot to keep its sentinel.  Cases that come from
fp32-output parity checks (torch_ref) also keep their bound against the torch fp32 op.  SiLU and GELU, the two inexact
steps, enter as tables of the kernel's own results over all 65,536 bf16 inputs; the tables are checked against float64
here, over the ranges where a bound holds.

The cases form a covering set: every N tile (64, 128, 160, 256) x {plain, SiLU, GEGLU} x {no bias, bias} x {scale 1,
0.7}, with fp32 biases that are not bf16-valued and differ per column, and N tile counts that divide the 132-CTA grid
(each CTA keeps one N tile) or are coprime to it (each CTA walks the N tiles), partial last M and N tiles and more than
2 x 132 tiles; every storer kind 0-7 on the vectorised and element-wise drains and kinds 2-7 with TMA operands
(`kOps`), broadcast sources, the output written over its own residual, row vectors over fewer than 128 rows; both
bias-buffer counts (one at BN 256 GEGLU and BN 256 kOps, two elsewhere); 1x1, 3x3 stride 1 and 2, two-source and
temporal convolutions, production shapes among them; fp32-output chains; and, labelled `(was ...)`, the shapes of the
GEMM tests they replace (_migrated_cases).  Each call runs under torch.profiler once: the gemm_conv_kernel<BN, EPI,
kOps> it launched must be the predicted one, and every instantiation of launch_bn must be reached.  `-s` prints the
tables' worst ulp per range, the instantiations, the worst accumulator error over tolerance per case group, the time
and the peak device memory."""
from __future__ import annotations

import math
import re
import time
import zlib
from dataclasses import dataclass
from typing import Callable

import pytest
import torch

from tests import gemm_exact as gx
from tests import kernel_checks as kc
from tests.abi_domain import gemm_operand_path, kernel_instantiation

pytestmark = pytest.mark.gpu
BF16, F64 = torch.bfloat16, torch.float64
DEV = "cuda"
OBSERVED: dict = {}


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device is visible (there is no CPU fallback to test)")
    from ctrl_adapter_b200 import _lib
    _lib.check(_lib.load().ca_device_ok(), "ca_device_ok")
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\ntest_gemm_epilogue_exact_gpu: {time.perf_counter() - t0:.1f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def _ops():
    from ctrl_adapter_b200 import ops
    return ops


@pytest.fixture(scope="module")
def tables():
    ops = _ops()
    return {bn: {"silu": gx.silu_table(ops, bn, DEV), "gelu": gx.gelu_table(ops, bn, DEV)} for bn in (64, 128, 160, 256)}


# ---------------------------------------------------------------------------------------------------------------------
# activation tables
# ---------------------------------------------------------------------------------------------------------------------
def _ranges_report(name, got, ref, ranges, failures):
    """got (bf16-valued fp32 [65536]) vs float64 ref over named ranges of the inputs: (label, mask, bound, kind) with
    kind 'ulp' (bf16 steps from ref rounded to bf16) or 'abs' (|got - ref|)."""
    u = gx.ulps(got, ref)
    lines = []
    for label, mask, bound, kind in ranges:
        if kind == "ulp":
            worst = int(u[mask].max())
        else:
            worst = float((got[mask].double() - ref[mask]).abs().max())
        lines.append(f"  {name} {label}: worst {worst:.3g} {'ulp' if kind == 'ulp' else 'abs'} (bound {bound:.3g})")
        if worst > bound:
            i = int(torch.nonzero(mask & ((u > bound) if kind == "ulp" else ((got.double() - ref).abs() > bound)))[0])
            failures.append(f"{name} {label}: worst {worst:.3g} > {bound:.3g}, first at input "
                            f"{float(gx.all_bf16(DEV)[i]):.6g}: got {float(got[i]):.6g}, float64 {float(ref[i]):.6g}")
    print("\n".join(lines))


def _special(name, got, ref64, x, failures):
    """+-inf and NaN inputs give what the float64 formula gives (NaN matching NaN)"""
    for v in (math.inf, -math.inf, math.nan):
        i = int(torch.nonzero((x == v) if not math.isnan(v) else torch.isnan(x))[0])
        g, e = float(got[i]), float(ref64[i])
        same = (math.isnan(g) and math.isnan(e)) or g == e
        if not same:
            failures.append(f"{name} at {v}: got {g}, float64 formula {e}")


def _silu_ranges(x):
    """below -87 the GEMM's __fdividef returns 0 once 1 + e^-x passes 2^126; |SiLU| there is at most 87 e^-87 < 2^-119"""
    fin = torch.isfinite(x)
    return [("x >= -87", fin & (x >= -87), 1, "ulp"), ("x < -87", fin & (x < -87), 2.0 ** -119, "abs")]


def test_activation_tables(tables):
    """T_silu and G through the GEMM's epilogue at every N tile: one device function, so one table; against float64
    SiLU x / (1 + e^-x) and GELU x Phi(x) = x / 2 erfc(-x / sqrt 2)"""
    x = gx.all_bf16(DEV)
    x64 = x.double()
    failures = []
    for name in ("silu", "gelu"):
        for bn in (64, 128, 160):
            a, b = tables[bn][name], tables[256][name]
            same = torch.equal(a.view(torch.int32), b.view(torch.int32)) or torch.equal(
                torch.nan_to_num(a, nan=7.0), torch.nan_to_num(b, nan=7.0))
            if not same:
                failures.append(f"{name} table at BN {bn} differs from BN 256 at {int((a != b).sum())} inputs")
    silu64 = x64 / (1 + torch.exp(-x64))
    gelu64 = x64 * 0.5 * torch.special.erfc(-x64 / math.sqrt(2.0))
    fin = torch.isfinite(x)
    print("\nGEMM epilogue activation tables vs float64 (worst per range over all bf16 inputs):")
    _ranges_report("GEMM SiLU", tables[256]["silu"], silu64, _silu_ranges(x), failures)
    _ranges_report("GEMM GELU", tables[256]["gelu"], gelu64,
                   [("x >= -6", fin & (x >= -6), 1, "ulp"), ("x < -6", fin & (x < -6), 2.0 ** -30, "abs")], failures)
    _special("GEMM SiLU", tables[256]["silu"], silu64, x, failures)
    _special("GEMM GELU", tables[256]["gelu"], gelu64, x, failures)
    assert not failures, "\n".join(failures)


def test_standalone_silu_table():
    """ops.silu over all bf16 inputs (a true division, unlike the GEMM's __fdividef): the same bounds"""
    x = gx.all_bf16(DEV)
    got = _ops().silu(x.to(BF16)).float()
    x64 = x.double()
    silu64 = x64 / (1 + torch.exp(-x64))
    failures = []
    print("\nops.silu vs float64:")
    _ranges_report("ops.silu", got, silu64, _silu_ranges(x), failures)
    _special("ops.silu", got, silu64, x, failures)
    assert not failures, "\n".join(failures)


# ---------------------------------------------------------------------------------------------------------------------
# the epilogue cases
# ---------------------------------------------------------------------------------------------------------------------
def _gen(seed):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    return g


def _rn(g, shape, scale=1.0):
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(BF16)


def _bias(g, n, scale=1.0):
    """fp32, not bf16-valued, a different value per column"""
    return torch.randn(n, generator=g, device=DEV) * scale


def _alpha(v=0.3027):
    """a bf16 alpha whose 1 - alpha is not bf16-valued (155 / 512), so the rounding of 1 - alpha shows"""
    return torch.tensor([v], device=DEV).to(BF16).float()


@dataclass
class Case:
    label: str
    op: str
    make: Callable  # (generator) -> the op's keyword arguments
    drain: str  # "vec", "elementwise", "tma" or "f32"
    torch_ref: bool = False  # also the output vs the torch fp32 op (TF32 off) at rtol 1e-3 / atol 1e-4
    acc_atol: float = 1e-3  # cap of the accumulator verdict's atol


def _linear(label, m, k, n, *, act=0, bias=True, scale=1.0, kind=0, bn=0, rpv=0, broadcast=False, out_slot=False,
            src_slot=None, out_over_res=False, out_fp32=False, bias_scale=1.0, torch_ref=False, acc_atol=1e-3):
    """a linear; kind: 1 row vector, 2 residual, 4 blend source (storer kinds 0-7).  broadcast: residual and blend
    source one row expanded along M; src_slot (left, right): row vector, residual and blend source at column `left` of
    rows left + n + right wide (gx.slot); out_slot: the output 8 bytes off 16-byte alignment"""
    ops = _ops()
    rv, res, bl = bool(kind & 1), bool(kind & 2), bool(kind & 4)
    left, right = src_slot or (0, 0)
    place = (lambda t: t) if src_slot is None else (lambda t: gx.slot(t, left, right))

    def make(g):
        w_rows = 2 * n if act == 2 else n
        kw = dict(x=_rn(g, (m, k)), w=_rn(g, (w_rows, k), k ** -0.5), act=act, out_scale=scale, bn=bn,
                  out_fp32=out_fp32)
        b = _bias(g, w_rows, bias_scale) if bias else None
        if act == 2:
            kw["w"], b = ops.pack_geglu_weight(kw["w"], b, bn or 256)
        kw["bias"] = b
        if rv:
            r_ = rpv or m
            kw["rowvec"], kw["rows_per_vec"] = place(_rn(g, (m // r_, n))), r_
        src = (lambda: _rn(g, (1, n)).expand(m, n)) if broadcast else (lambda: place(_rn(g, (m, n))))
        if res:
            kw["residual"] = src()
        if bl:
            kw["blend_src"], kw["blend_alpha"] = src(), _alpha()
        if out_slot:
            kw["out"] = gx.slot(torch.full((m, n), math.nan, device=DEV, dtype=BF16))
        if out_over_res:
            kw["out"] = kw["residual"]
        return kw
    stride = n + left + right
    vec = not out_slot and left % 8 == 0 and stride % 8 == 0
    tma = gemm_operand_path(vec=vec, out_fp32=out_fp32, geglu=act == 2, residual=res, blend=bl,
                            res_strides=(0 if broadcast else stride, 0, 0, 0), out_dims=(m, 1, 1, 1))
    drain = "f32" if out_fp32 else "tma" if tma else "vec" if vec else "elementwise"
    return Case(label, "linear", make, drain, torch_ref, acc_atol)


def _conv(label, n, h, w, c, cout, *, ksize=3, stride=1, c2=0, act=0, scale=1.0, kind=0, bn=0, rv_rows=None,
          out_slot=False, out_fp32=False, torch_ref=False):
    """a 3x3 or 1x1 convolution with bias; kind as for _linear; out_slot: the output a contiguous view 8 bytes off
    16-byte alignment"""
    ops = _ops()
    ho, wo = (h, w) if stride == 1 else (h // 2, w // 2)

    def make(g):
        wt = _rn(g, (cout, c + c2, ksize, ksize), (ksize * ksize * (c + c2)) ** -0.5)
        kw = dict(x=_rn(g, (n, h, w, c)), w_packed=ops.pack_conv_weight(wt, 64 if stride == 2 else 8),
                  bias=_bias(g, cout), ksize=ksize, stride=stride, act=act, out_scale=scale, bn=bn, out_fp32=out_fp32)
        if c2:
            kw["x2"] = _rn(g, (n, h, w, c2))
        if kind & 1:
            kw["rowvec"] = _rn(g, (rv_rows or n, cout))
        if kind & 2:
            kw["residual"] = _rn(g, (n, ho, wo, cout))
        if kind & 4:
            kw["blend_src"], kw["blend_alpha"] = _rn(g, (n, ho, wo, cout)), _alpha(0.4)
        if out_slot:
            kw["out"] = gx.slot(torch.full((n, ho, wo, cout), math.nan, device=DEV, dtype=BF16), flat=True)
        return kw
    tma = gemm_operand_path(vec=not out_slot, out_fp32=out_fp32, residual=bool(kind & 2), blend=bool(kind & 4))
    drain = "f32" if out_fp32 else "tma" if tma else "elementwise" if out_slot else "vec"
    return Case(label, "conv2d", make, drain, torch_ref)


def _temporal(label, b, f, h, w, c, cout, kind, rv_rows=None):
    """a Conv3d (3, 1, 1) over the frames with bias; kind as for _linear"""
    ops = _ops()

    def make(g):
        x = _rn(g, (b * f, h, w, c))
        wt = _rn(g, (cout, c, 3, 1, 1), (3 * c) ** -0.5)
        kw = dict(x=x, w_packed=ops.pack_conv_weight(wt), bias=_bias(g, cout), frames=f)
        if kind & 1:
            kw["rowvec"] = _rn(g, (rv_rows or b * f, cout))
        if kind & 2:
            kw["residual"] = _rn(g, (b * f, h, w, cout))
        if kind & 4:
            kw["blend_src"], kw["blend_alpha"] = _rn(g, (b * f, h, w, cout)), _alpha(0.4)
        return kw
    return Case(label, "temporal_conv", make, "tma" if kind & 6 else "vec")


def _matrix_cases():
    """BN x {plain, SiLU, GEGLU} x {no bias, bias} x {scale 1, 0.7}; N tile counts 5 (coprime to the 132-CTA grid, a
    partial last N tile except for GEGLU) and 2 (dividing it), 140 M tiles (the last partial): 280 or 700 tiles"""
    out = []
    m, k = 128 * 140 - 45, 128
    for bn in (64, 128, 160, 256):
        for act, an in ((0, "plain"), (1, "silu"), (2, "geglu")):
            for bias in (False, True):
                for scale in (1.0, 0.7):
                    coprime = bias == (scale == 1.0)
                    nt = 5 if coprime else 2
                    n = nt * bn // 2 if act == 2 else nt * bn - 24
                    label = (f"linear bn{bn} {an} {'bias' if bias else 'nobias'} scale{scale:g} m{m} n{n} "
                             f"ntiles_n{nt}")
                    out.append(_linear(label, m, k, n, act=act, bias=bias, scale=scale, bn=bn))
    return out


def _storer_cases():
    out = []
    m, k = 1000, 64
    for kind in range(8):
        # vectorised drain: kinds 0 / 1 plain; 2-7 with broadcast sources (stride 0 along M: no tensor map), and GEGLU
        if kind < 2:
            out.append(_linear(f"linear vec kind{kind} rpv40", m, k, 200, kind=kind, rpv=40))
        else:
            out.append(_linear(f"linear vec broadcast kind{kind} rpv40", m, k, 200, kind=kind, rpv=40,
                               broadcast=True))
        out.append(_linear(f"linear geglu vec kind{kind} bn128 scale0.7", m, k, 192, act=2, bn=128, kind=kind,
                           rpv=200, scale=0.7))
        # element-wise drain: the output 8 bytes off 16-byte alignment
        out.append(_linear(f"linear elementwise kind{kind} silu", m, k, 200, act=1, kind=kind, rpv=40, out_slot=True))
        if kind >= 2:  # TMA operands (kOps): N tiles 64, 128, 160, 256, 64, 160, partial slabs
            bn = (64, 128, 160, 256, 64, 160)[kind - 2]
            out.append(_linear(f"linear tma kind{kind} bn{bn} scale0.7", m, k, 200, kind=kind, bn=bn, rpv=40,
                               scale=0.7))
    out.append(_linear("linear geglu elementwise kind7 bn256", m, k, 256, act=2, kind=7, rpv=40, out_slot=True))
    # BN 256 with TMA operands: one bias buffer; 5 N tiles (coprime), 700 tiles
    out.append(_linear("linear tma kind2 bn256 bias m17875 n1128", 128 * 140 - 45, 128, 1128, kind=2, bn=256))
    out.append(_linear("linear tma kind6 bn160 silu out over residual", m, k, 320, act=1, kind=6, bn=160,
                       out_over_res=True))
    out.append(_linear("linear tma kind3 bn64 out over residual rpv40", m, k, 200, kind=3, bn=64, rpv=40,
                       out_over_res=True))
    out.append(_linear("linear geglu vec kind2 out over residual", m, k, 256, act=2, kind=2, out_over_res=True))
    return out


def _conv_cases():
    out = [
        _conv("conv 3x3 n16 128x128 c320->320 residual (production)", 16, 128, 128, 320, 320, kind=2),
        _conv("conv 1x1 n2 24x40 c320->640 rowvec+residual", 2, 24, 40, 320, 640, ksize=1, kind=3),
        _conv("conv 1x1 n2 24x40 c640->320 silu scale0.7 rowvec[1]", 2, 24, 40, 640, 320, ksize=1, act=1, scale=0.7,
              kind=1, rv_rows=1),
        _conv("conv 3x3 s2 n2 48x80 c128->256 silu", 2, 48, 80, 128, 256, stride=2, act=1),
        _conv("conv 3x3 s2 n2 48x80 c320->320 rowvec+residual+blend", 2, 48, 80, 320, 320, stride=2, kind=7),
        _conv("conv 3x3 x2 n2 32x48 c128+64->192 residual+blend", 2, 32, 48, 128, 192, c2=64, kind=6),
        _conv("conv 3x3 n3 20x36 c64->200 bn64 scale0.7", 3, 20, 36, 64, 200, bn=64, scale=0.7),
        _temporal("temporal b2 f14 24x40 c320->320 rowvec+residual+blend (production)", 2, 14, 24, 40, 320, 320, 7),
        _temporal("temporal b1 f5 12x20 c640->640 rowvec[1]", 1, 5, 12, 20, 640, 640, 1, rv_rows=1),
        _temporal("temporal b2 f3 8x8 c320->320 residual", 2, 3, 8, 8, 320, 320, 2),
    ]
    # production linears: a 1280-wide projection with residual, the 10240-row GEGLU
    out.append(_linear("linear m8192 k1280 n1280 residual (production)", 8192, 1280, 1280, kind=2))
    out.append(_linear("linear geglu m8192 k1280 n5120 (production)", 8192, 1280, 5120, act=2))
    return out


def _f32_cases():
    out = []
    m, k = 3000, 128
    for kind, scale, bn in ((0, 0.7, 64), (1, 1.0, 128), (2, 1.0, 160), (3, 0.7, 256), (2, 0.7, 0)):
        out.append(_linear(f"linear f32 kind{kind} scale{scale:g} bn{bn}", m, k, 328, kind=kind, scale=scale, bn=bn,
                           rpv=40, out_fp32=True))
    return out


def _migrated_cases():
    """the shapes of the GEMM tests these cases replace, labelled by origin: `was staging` -- many tiles per CTA, conv
    boxes past the output, an output slice; `was stmatrix` -- the plain epilogue at every BN, m50001; `was tma` -- TMA
    operands at many tiles and the same calls on the element-wise drain, output over its residual, a residual row stride
    of n + 4; `was gemm` / `was conv` -- the fp32-reference parity checks (fp32 outputs keep their torch fp32 bound; GEGLU
    keeps the 1e-4 accumulator atol its pre-activation had); `was shapes` -- the SVD latent levels"""
    out = [
        _linear("linear m50001 k640 n1280 residual (was staging)", 50001, 640, 1280, kind=2),
        _linear("linear m40000 k320 n640 residual (was staging)", 40000, 320, 640, kind=2),
        _conv("conv 3x3 n3 13x11 c320->320 rowvec+residual (was staging)", 3, 13, 11, 320, 320, kind=3),
        _conv("conv 3x3 n2 9x23 c640->640 residual scale0.5 (was staging)", 2, 9, 23, 640, 640, kind=2, scale=0.5),
        _linear("linear m9000 k640 n640 nobias residual+blend (was staging)", 9000, 640, 640, kind=6, bias=False),
        _linear("linear geglu m8192 k640 n2560 (was staging)", 8192, 640, 2560, act=2, acc_atol=1e-4),
        _linear("linear m2000 k320 n320 residual output slice (was staging)", 2000, 320, 320, kind=2, out_slot=True),
    ]
    for bn, n in ((64, 104), (128, 200), (160, 400), (256, 640)):
        for bias in (True, False):
            out.append(_linear(f"linear m50001 k320 n{n} bn{bn} plain {'bias' if bias else 'nobias'} (was stmatrix)",
                               50001, 320, n, bias=bias, bn=bn))
    for name, m, k, n, rpv in (("res_blend", 50001, 640, 1280, 0), ("bias_res_blend", 40000, 320, 640, 0),
                               ("res_blend", 9000, 256, 384, 0), ("res", 20000, 128, 64, 0),
                               ("blend", 30000, 320, 1280, 0), ("rowvec_res", 8192, 320, 640, 64),
                               ("rowvec_res_blend", 8192, 320, 1280, 32), ("silu_scale_rowvec_res", 6144, 640, 1280, 2048)):
        parts = name.split("_")
        kind = int("rowvec" in parts) | 2 * int("res" in parts) | 4 * int("blend" in parts)
        for slot in (False, True):
            out.append(_linear(f"linear {name} m{m} k{k} n{n} rpv{rpv} {'elementwise' if slot else 'aligned'} (was tma)",
                               m, k, n, kind=kind, rpv=rpv, bias="bias" in parts, act=int("silu" in parts),
                               scale=0.7 if "scale" in parts else 1.0, out_slot=slot, src_slot=(4, 12) if slot else None))
    for n, h, w, c, cout, blend in ((3, 13, 11, 320, 320, True), (2, 9, 23, 640, 1280, False),
                                    (4, 7, 5, 256, 640, True)):
        for slot in (False, True):
            out.append(_conv(f"conv 3x3 n{n} {h}x{w} c{c}->{cout} residual{'+blend' if blend else ''} "
                             f"{'elementwise' if slot else 'aligned'} (was tma)", n, h, w, c, cout,
                             kind=6 if blend else 2, out_slot=slot))
    for n in (1280, 640):
        out.append(_linear(f"linear m30000 k640 n{n} out over residual (was tma)", 30000, 640, n, kind=2,
                           out_over_res=True))
    out.append(_linear("linear m9000 k320 n640 residual stride n+4 (was tma)", 9000, 320, 640, kind=2, src_slot=(0, 4)))
    out += [
        _linear("linear f32 m256 k64 n64 (was gemm)", 256, 64, 64, out_fp32=True, torch_ref=True),
        _linear("linear f32 m128 k128 n128 nobias (was gemm)", 128, 128, 128, bias=False, out_fp32=True, torch_ref=True),
        _linear("linear f32 m1000 k512 n320 (was gemm)", 1000, 512, 320, out_fp32=True, torch_ref=True),
        _linear("linear m4096 k320 n512 (was gemm)", 4096, 320, 512),
        _linear("linear m300 k2048 n1280 residual (was gemm)", 300, 2048, 1280, kind=2),
        _linear("linear f32 m154 k768 n320 bn64 (was gemm)", 154, 768, 320, bn=64, out_fp32=True, torch_ref=True),
        _linear("linear m16 k320 n1280 silu (was gemm)", 16, 320, 1280, act=1),
        _linear("linear m50000 k512 n640 bn128 (was gemm)", 50000, 512, 640, bn=128),
        _linear("linear geglu m1024 k512 n2048 (was gemm)", 1024, 512, 2048, act=2, acc_atol=1e-4),
        _linear("linear m1024 k512 n512 nobias rowvec rpv256 (was gemm)", 1024, 512, 512, kind=1, rpv=256, bias=False),
        _linear("linear m192 k320 n320 nobias rowvec rpv64 (was gemm)", 192, 320, 320, kind=1, rpv=64, bias=False),
        _linear("linear m512 k2048 n512 nobias residual+blend (was gemm)", 512, 2048, 512, kind=6, bias=False),
        _linear("linear m3000 k640 n640 residual (was gemm)", 3000, 640, 640, kind=2),
        _linear("linear m1100 k320 n1920 (was gemm)", 1100, 320, 1920),
        _linear("linear m2048 k1280 n1280 residual (was gemm)", 2048, 1280, 1280, kind=2),
        _linear("linear m700 k256 n328 residual (was gemm)", 700, 256, 328, kind=2),
        _linear("linear m520 k192 n40 nobias (was gemm)", 520, 192, 40, bias=False),
        _linear("linear geglu m5000 k640 n2560 (was gemm)", 5000, 640, 2560, act=2, acc_atol=1e-4),
        _conv("conv 3x3 f32 n2 16x16 c64->64 (was conv)", 2, 16, 16, 64, 64, out_fp32=True, torch_ref=True),
        _conv("conv 3x3 f32 n2 32x32 c320->320 (was conv)", 2, 32, 32, 320, 320, out_fp32=True, torch_ref=True),
        _conv("conv 3x3 n3 8x8 c1280->1280 rowvec+residual (was conv)", 3, 8, 8, 1280, 1280, kind=3),
        _conv("conv 3x3 n2 64x64 c320->320 rowvec (was conv)", 2, 64, 64, 320, 320, kind=1),
        _conv("conv 1x1 n2 16x16 c640->320 residual (was conv)", 2, 16, 16, 640, 320, ksize=1, kind=2),
        _conv("conv 3x3 x2 n2 16x16 c640+320->640 (was conv)", 2, 16, 16, 640, 640, c2=320),
        _conv("conv 3x3 s2 f32 n2 32x32 c320->320 (was conv)", 2, 32, 32, 320, 320, stride=2, out_fp32=True,
              torch_ref=True),
        _conv("conv 3x3 s2 f32 n2 64x64 c16->32 (was conv)", 2, 64, 64, 16, 32, stride=2, out_fp32=True, torch_ref=True),
        _conv("conv 3x3 f32 n2 64x64 c8->16 (was conv)", 2, 64, 64, 8, 16, out_fp32=True, torch_ref=True),
        _conv("conv 3x3 s2 n2 24x40 c96->256 (was conv)", 2, 24, 40, 96, 256, stride=2),
        _conv("conv 3x3 f32 n2 18x32 c128->64 (was conv)", 2, 18, 32, 128, 64, out_fp32=True, torch_ref=True),
        _conv("conv 1x1 n2 16x16 c320->320 scale0.7 (was conv)", 2, 16, 16, 320, 320, ksize=1, scale=0.7),
        _temporal("temporal b2 f16 8x8 c128->128 rowvec (was conv)", 2, 16, 8, 8, 128, 128, 1),
        _temporal("temporal b1 f14 16x16 c320->320 rowvec (was conv)", 1, 14, 16, 16, 320, 320, 1),
        _conv("conv 3x3 n2 36x64 c320->320 residual (was shapes)", 2, 36, 64, 320, 320, kind=2),
        _conv("conv 3x3 n2 18x32 c640->640 rowvec (was shapes)", 2, 18, 32, 640, 640, kind=1),
        _conv("conv 3x3 n2 64x16 c64->128 (was shapes)", 2, 64, 16, 64, 128),
        _conv("conv 3x3 n1 64x32 c64->64 (was shapes)", 1, 64, 32, 64, 64),
        _linear("linear m1232 k2048 n2560 (was shapes)", 1232, 2048, 2560),
        _linear("linear m4608 k320 n960 (was shapes)", 4608, 320, 960),
    ]
    return out


CASES = _matrix_cases() + _storer_cases() + _conv_cases() + _f32_cases() + _migrated_cases()
ACC_WORST: dict = {}  # case group -> (worst accumulator error / tolerance, case label)


def _profile(call):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(0.005)
            ret = call()
            torch.cuda.synchronize()
            time.sleep(0.005)
        names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
        if names:
            return ret, names
    return ret, []


def _expand_rowvec(op, kw):
    rv = kw.get("rowvec")
    if rv is None:
        return None
    if op == "linear":
        return rv.repeat_interleave(kw["rows_per_vec"], dim=0)
    return rv.reshape(rv.shape[0], 1, 1, -1)


def _torch_fp32(op, kw):
    """the call's bias-only op in torch fp32 with TF32 off"""
    flags = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        if op == "conv2d":
            return kc.conv2d_ref(kw, dtype=torch.float32)[0]
        ref = kw["x"].float() @ kw["w"].float().t()
        return ref if kw["bias"] is None else ref + kw["bias"]
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = flags


def _group(label):
    m = re.search(r"\((was \w+)\)", label)
    return m.group(1) if m else label.split()[0]


@pytest.mark.parametrize("case", CASES, ids=[c.label for c in CASES])
def test_epilogue_exact(case, tables):
    ops = _ops()
    kw = case.make(_gen(zlib.crc32(case.label.encode())))
    bn = gx.resolved_bn(case.op, kw)
    act = kw.get("act", 0)
    raw = gx.accumulators(case.op, kw, ops)
    failures = []
    rec = gx.accumulator_verdict(case.label, case.op, kw, raw, atol_cap=case.acc_atol)
    if not rec["ok"]:
        failures.append(f"{rec['check']}: {rec.get('why') or rec}")
    group = _group(case.label)
    if rec["max_err_over_tol"] > ACC_WORST.get(group, (-1.0,))[0]:
        ACC_WORST[group] = (rec["max_err_over_tol"], case.label)
    acc, gate = gx.geglu_halves(raw, bn) if act == 2 else (raw, None)
    residual = kw.get("residual")
    if residual is not None and kw.get("out") is residual:
        residual = residual.clone()
    out, names = _profile(lambda: getattr(ops, case.op)(**kw))
    torch.cuda.synchronize()
    insts = {kernel_instantiation(n) for n in names} - {None}
    gemm = [a for k_, a in insts if k_ == "gemm_conv_kernel"]
    epi = 2 if case.drain == "f32" else 1 if act == 2 else 0
    predicted = (bn, epi, int(case.drain == "tma")) if epi == 0 else (bn, epi)
    assert gemm, f"{case.label}: torch.profiler recorded no gemm_conv_kernel launch ({names})"
    got = tuple(gemm[0][:3]) if epi == 0 else tuple(gemm[0][:2])
    assert len(gemm) == 1 and got == predicted, f"{case.label}: launched {gemm}, predicted {predicted}"
    OBSERVED[gemm[0][:3]] = OBSERVED.get(gemm[0][:3], 0) + 1
    bias = kw.get("bias")
    if act == 2 and bias is not None:
        bias = gx.geglu_halves(bias, bn)
    chain = dict(gate=gate, bias=bias, act=act, scale=kw.get("out_scale", 1.0), rowvec=_expand_rowvec(case.op, kw),
                 residual=residual, blend_src=kw.get("blend_src"), blend_alpha=kw.get("blend_alpha"),
                 out_fp32=kw.get("out_fp32", False), tables=tables[bn])
    ok, msg = gx.compare(f"{case.label} [{case.drain}]", out, acc, chain, n_tile_cols=bn // 2 if act == 2 else bn)
    if not ok:
        failures.append(msg)
    if kw.get("out") is not None and kw["out"]._base is not None and not gx.guard_intact(kw["out"]):
        failures.append(f"{case.label}: bytes around the output slot changed")
    if case.torch_ref:
        rec = kc._report(f"{case.label} vs torch fp32", out, _torch_fp32(case.op, kw), 1e-3, 1e-4)
        if not rec["ok"]:
            failures.append(f"{rec['check']}: {rec}")
    assert not failures, "\n".join(failures)


def test_every_instantiation_reached():
    """gemm_conv_kernel<BN, EPI, kOps>: per BN the fp32, GEGLU, plain and plain-with-TMA-operands instantiations that
    launch_bn dispatches to, each seen by the profiler in some case above.  `-s` also prints the worst accumulator error
    over its tolerance per case group."""
    want = {(bn, e, o) for bn in (64, 128, 160, 256) for e, o in ((0, 0), (0, 1), (1, 0), (2, 0))}
    print("\nobserved gemm_conv_kernel<BN, EPI, kOps> (cases):")
    for key in sorted(OBSERVED):
        print(f"  gemm_conv_kernel<{', '.join(map(str, key))}>: {OBSERVED[key]}")
    print("worst accumulator error / tolerance per case group:")
    for group, (ratio, label) in sorted(ACC_WORST.items()):
        print(f"  {group}: {ratio:.3g} ({label})")
    missing = want - set(OBSERVED)
    assert not missing, f"instantiations never launched: {sorted(missing)}"
