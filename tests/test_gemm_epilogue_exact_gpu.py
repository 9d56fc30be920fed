"""pytest -m gpu: every bf16 instantiation and storer path of the GEMM epilogue, bit for bit (tests/gemm_exact.py).

Each case runs one `ops` call and the same call's fp32 accumulators (the fp32-output instantiation at the same N tile
with an empty epilogue), and requires the call's output bits to equal the epilogue chain restated in torch fp32 on those
accumulators.  SiLU and GELU, the two inexact steps, enter as tables of the kernel's own results over all 65,536 bf16
inputs; the tables are checked against float64 here, over the ranges where a bound holds.

The cases form a covering set: every N tile (64, 128, 160, 256) x {plain, SiLU, GEGLU} x {no bias, bias} x {scale 1,
0.7}, with fp32 biases that are not bf16-valued and differ per column, and N tile counts that divide the 132-CTA grid
(each CTA keeps one N tile) or are coprime to it (each CTA walks the N tiles), partial last M and N tiles and more than
2 x 132 tiles; every storer kind 0-7 on the vectorised and element-wise drains and kinds 2-7 with TMA operands
(`kOps`), broadcast sources, the output written over its own residual, row vectors over fewer than 128 rows; both
bias-buffer counts (one at BN 256 GEGLU and BN 256 kOps, two elsewhere); 1x1, 3x3 stride 1 and 2, two-source and
temporal convolutions, production shapes among them; and fp32-output chains.  Each call runs under torch.profiler
once: the gemm_conv_kernel<BN, EPI, kOps> it launched must be the predicted one, and every instantiation of
launch_bn must be reached.  `-s` prints the tables' worst ulp per range, the instantiations, the time and the peak
device memory."""
from __future__ import annotations

import math
import time
import zlib
from dataclasses import dataclass
from typing import Callable

import pytest
import torch

from tests import gemm_exact as gx
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


def _slot(t, off=4):
    """t's values in columns [off, off + n) of a wider buffer: a view 8 bytes off 16-byte alignment"""
    buf = torch.zeros(*t.shape[:-1], t.shape[-1] + 16, device=DEV, dtype=t.dtype)
    buf[..., off:off + t.shape[-1]] = t
    return buf[..., off:off + t.shape[-1]]


@dataclass
class Case:
    label: str
    op: str
    make: Callable  # (generator) -> the op's keyword arguments
    drain: str  # "vec", "elementwise", "tma" or "f32"
    broadcast: bool = False


def _linear(label, m, k, n, *, act=0, bias=True, scale=1.0, kind=0, bn=0, rpv=0, drain=None, broadcast=False,
            out_slot=False, out_over_res=False, out_fp32=False, bias_scale=1.0):
    """a linear; kind: 1 row vector, 2 residual, 4 blend source (storer kinds 0-7)"""
    ops = _ops()
    rv, res, bl = bool(kind & 1), bool(kind & 2), bool(kind & 4)

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
            kw["rowvec"], kw["rows_per_vec"] = _rn(g, (m // r_, n)), r_
        src = (lambda: _rn(g, (1, n)).expand(m, n)) if broadcast else (lambda: _rn(g, (m, n)))
        if res:
            kw["residual"] = src()
        if bl:
            kw["blend_src"], kw["blend_alpha"] = src(), _alpha()
        if out_slot:
            kw["out"] = _slot(torch.zeros(m, n, device=DEV, dtype=BF16))
        if out_over_res:
            kw["out"] = kw["residual"]
        return kw
    if drain is None:
        vec = not out_slot
        tma = gemm_operand_path(vec=vec, out_fp32=out_fp32, geglu=act == 2, residual=res, blend=bl,
                                res_strides=(0 if broadcast else n, 0, 0, 0), out_dims=(m, 1, 1, 1))
        drain = "f32" if out_fp32 else "tma" if tma else "vec" if vec else "elementwise"
    return Case(label, "linear", make, drain, broadcast)


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
    ops = _ops()
    out = []

    def conv(label, n, h, w, c, cout, *, ksize=3, stride=1, c2=0, act=0, scale=1.0, kind=0, bn=0, rv_rows=None):
        def make(g):
            x = _rn(g, (n, h, w, c))
            wt = _rn(g, (cout, c + c2, ksize, ksize), (ksize * ksize * (c + c2)) ** -0.5)
            ho, wo = (h, w) if stride == 1 else (h // 2, w // 2)
            kw = dict(x=x, w_packed=ops.pack_conv_weight(wt), bias=_bias(g, cout), ksize=ksize, stride=stride,
                      act=act, out_scale=scale, bn=bn)
            if c2:
                kw["x2"] = _rn(g, (n, h, w, c2))
            if kind & 1:
                kw["rowvec"] = _rn(g, (rv_rows or n, cout))
            if kind & 2:
                kw["residual"] = _rn(g, (n, ho, wo, cout))
            if kind & 4:
                kw["blend_src"], kw["blend_alpha"] = _rn(g, (n, ho, wo, cout)), _alpha(0.4)
            return kw
        return Case(label, "conv2d", make, "tma" if kind & 6 else "vec")
    out.append(conv("conv 3x3 n16 128x128 c320->320 residual (production)", 16, 128, 128, 320, 320, kind=2))
    out.append(conv("conv 1x1 n2 24x40 c320->640 rowvec+residual", 2, 24, 40, 320, 640, ksize=1, kind=3))
    out.append(conv("conv 1x1 n2 24x40 c640->320 silu scale0.7 rowvec[1]", 2, 24, 40, 640, 320, ksize=1, act=1,
                    scale=0.7, kind=1, rv_rows=1))
    out.append(conv("conv 3x3 s2 n2 48x80 c128->256 silu", 2, 48, 80, 128, 256, stride=2, act=1))
    out.append(conv("conv 3x3 s2 n2 48x80 c320->320 rowvec+residual+blend", 2, 48, 80, 320, 320, stride=2, kind=7))
    out.append(conv("conv 3x3 x2 n2 32x48 c128+64->192 residual+blend", 2, 32, 48, 128, 192, c2=64, kind=6))
    out.append(conv("conv 3x3 n3 20x36 c64->200 bn64 scale0.7", 3, 20, 36, 64, 200, bn=64, scale=0.7))

    def temporal(label, b, f, h, w, c, cout, kind, rv_rows=None):
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
    out.append(temporal("temporal b2 f14 24x40 c320->320 rowvec+residual+blend (production)", 2, 14, 24, 40, 320, 320,
                        7))
    out.append(temporal("temporal b1 f5 12x20 c640->640 rowvec[1]", 1, 5, 12, 20, 640, 640, 1, rv_rows=1))
    out.append(temporal("temporal b2 f3 8x8 c320->320 residual", 2, 3, 8, 8, 320, 320, 2))
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


CASES = _matrix_cases() + _storer_cases() + _conv_cases() + _f32_cases()


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


@pytest.mark.parametrize("case", CASES, ids=[c.label for c in CASES])
def test_epilogue_exact(case, tables):
    ops = _ops()
    kw = case.make(_gen(zlib.crc32(case.label.encode())))
    bn = gx.resolved_bn(case.op, kw)
    act = kw.get("act", 0)
    acc, gate = gx.accumulators(case.op, kw, ops)
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
    assert ok, msg


def test_every_instantiation_reached():
    """gemm_conv_kernel<BN, EPI, kOps>: per BN the fp32, GEGLU, plain and plain-with-TMA-operands instantiations that
    launch_bn dispatches to, each seen by the profiler in some case above"""
    want = {(bn, e, o) for bn in (64, 128, 160, 256) for e, o in ((0, 0), (0, 1), (1, 0), (2, 0))}
    print("\nobserved gemm_conv_kernel<BN, EPI, kOps> (cases):")
    for key in sorted(OBSERVED):
        print(f"  gemm_conv_kernel<{', '.join(map(str, key))}>: {OBSERVED[key]}")
    missing = want - set(OBSERVED)
    assert not missing, f"instantiations never launched: {sorted(missing)}"
