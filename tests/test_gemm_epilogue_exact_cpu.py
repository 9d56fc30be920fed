"""CPU: the power of the bit-exact epilogue check of tests/gemm_exact.py, over the emulated op layer.

The correct emulation (tests/ops_emulator.py, whose GEGLU honours the N tile, the output scale and the storer operands
as the kernel does) passes the exact check on every case below.  Each wrong variant of the epilogue chain -- the kind
of change an epilogue rewrite makes by accident -- passes the float64 verdict that the layout checks and the launch
census apply to the same call (kernel_checks.linear_verdict, launch_checks.VERIFIERS["linear"]) -- or, for GEGLU with
a scale, gets no float64 verdict at all -- and fails the exact check.  An unrounded 1 - alpha is flagged by both.  `-s` prints `old verdicts: pass; exact: n differing at (r, c)` per variant.

Two wrong variants that every instantiation shares -- a main loop that drops the last 64-wide K block, and an
element-wise drain that also writes one column past its output slot -- pass the exact check, whose accumulators come
from the same op layer, and fail the accumulator verdict against float64 or the guard bytes around the slot.  `-s`
prints `current exact check: pass; new: <accumulator verdict | guard bytes> fails` for each, after the correct
emulation passing all three on the same call."""
import functools
import types

import pytest
import torch
import torch.nn.functional as F

from tests import gemm_exact as gx
from tests import kernel_checks as kc
from tests import launch_checks as lc
from tests import ops_emulator as emu

BF16 = torch.bfloat16
r = gx.r


@pytest.fixture(scope="module", autouse=True)
def _cpu_device():
    saved = kc.DEVICE
    kc.DEVICE = "cpu"
    yield
    kc.DEVICE = saved


@pytest.fixture(scope="module")
def tables():
    return {bn: {"silu": gx.silu_table(emu, bn, "cpu"), "gelu": gx.gelu_table(emu, bn, "cpu")} for bn in (128, 256)}


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _call(*, m=512, k=128, n=256, act=0, bias=True, bias_scale=1.0, wscale=1.0, scale=1.0, kind=0, rpv=32, bn=0,
          alpha=0.3027, out_slot=False, seed=0):
    """a linear's arguments (ops.linear's parameter names); kind: 1 row vector, 2 residual, 4 blend source; out_slot:
    the output a gx.slot view"""
    g = _g(seed)
    rn = lambda *s, sc=1.0: (torch.randn(*s, generator=g) * sc).to(BF16)  # noqa: E731
    w_rows = 2 * n if act == 2 else n
    w = rn(w_rows, k, sc=wscale * k ** -0.5)
    b = torch.randn(w_rows, generator=g) * bias_scale if bias else None
    if act == 2:
        from ctrl_adapter_b200.ops import pack_geglu_weight
        w, b = pack_geglu_weight(w, b, bn or 256)
    return dict(x=rn(m, k), w=w, bias=b, act=act, residual=rn(m, n) if kind & 2 else None,
                rowvec=rn(m // rpv, n) if kind & 1 else None, rows_per_vec=rpv if kind & 1 else 0,
                blend_src=rn(m, n) if kind & 4 else None,
                blend_alpha=torch.tensor([alpha]).to(BF16).float() if kind & 4 else None,
                out_scale=scale, out=gx.slot(torch.full((m, n), float("nan")).to(BF16)) if out_slot else None,
                out_fp32=False, bn=bn)


def _exact(call, out, tables, ops=emu):
    """the exact check of the call's output, the accumulators taken from ops.linear"""
    bn = gx.resolved_bn("linear", call)
    raw = gx.accumulators("linear", call, ops)
    acc, gate = gx.geglu_halves(raw, bn) if call["act"] == 2 else (raw, None)
    bias = call["bias"]
    if call["act"] == 2 and bias is not None:
        bias = gx.geglu_halves(bias, bn)
    rv = call["rowvec"]
    chain = dict(gate=gate, bias=bias, act=call["act"], scale=call["out_scale"],
                 rowvec=None if rv is None else rv.repeat_interleave(call["rows_per_vec"], 0),
                 residual=call["residual"], blend_src=call["blend_src"], blend_alpha=call["blend_alpha"],
                 tables=tables[bn])
    return gx.compare("linear", out, acc, chain, n_tile_cols=bn // 2 if call["act"] == 2 else bn)


CORRECT = {
    "plain bias scale0.7": dict(scale=0.7),
    "silu bias rowvec+residual": dict(act=1, kind=3),
    "bias residual+blend": dict(kind=6),
    "silu scale0.7 rowvec+residual+blend bn128": dict(act=1, scale=0.7, kind=7, bn=128),
    "geglu bn256 nobias": dict(act=2, bias=False),
    "geglu bn128 scale0.7 rowvec+residual+blend": dict(act=2, bn=128, scale=0.7, kind=7),
}


@pytest.mark.parametrize("name", list(CORRECT))
def test_exact_check_passes_emulator(name, tables):
    call = _call(**CORRECT[name])
    ok, msg = _exact(call, emu.linear(**call), tables)
    assert ok, msg


# ---- wrong variants of the bf16 chain (the fp32-output path, which gives the accumulators, stays correct) ----
def _variant(which):
    def linear(x, w, bias=None, *, act=0, residual=None, rowvec=None, rows_per_vec=0, blend_src=None,
               blend_alpha=None, out_scale=1.0, out=None, out_fp32=False, bn=0):
        if out_fp32:
            return emu.linear(x, w, bias, act=act, residual=residual, rowvec=rowvec, rows_per_vec=rows_per_vec,
                              out_scale=out_scale, out=out, out_fp32=True, bn=bn)
        xf, wf = x.float(), w.float()
        rv = None if rowvec is None else rowvec.float().repeat_interleave(rows_per_vec, 0)
        tile = gx.resolved_bn("linear", dict(w=w, act=act, bn=bn))
        scaled = False
        if act == 2:
            a, g = gx.geglu_halves(xf @ wf.t(), tile)
            if bias is not None:
                ba, bg = gx.geglu_halves(bias.float(), tile)
                a, g = a + ba, g + bg
            v = r(a) * r(F.gelu(r(g)))
            if not (which == "geglu product unrounded before the scale" and out_scale != 1.0):
                v = r(v)
        else:
            v = xf @ wf.t()
            if bias is not None:
                b = bias.float()
                if which == "bias of the previous N tile":
                    b = torch.roll(b, tile)  # column j takes the bias of column j - BN
                v = v + b
            if which == "scale applied before the rounding" and out_scale != 1.0:
                v, scaled = r(v * out_scale), True
            elif which == "SiLU of the unrounded acc + bias" and act == 1:
                pass
            else:
                v = r(v)
            if act == 1:
                v = r(F.silu(v))
        if out_scale != 1.0 and not scaled:
            v = r(v * out_scale)
        if which == "residual added before the row vector" and rv is not None and residual is not None:
            v = r(r(v + residual.float()) + rv)
        elif which == "row vector and residual summed in fp32, one rounding" and rv is not None and residual is not None:
            v = r(v + rv + residual.float())
        else:
            if rv is not None:
                v = r(v + rv)
            if residual is not None:
                v = r(v + residual.float())
        if blend_src is not None:
            al = blend_alpha.float().reshape(())
            one_minus = 1.0 - al if which == "1 - alpha left unrounded" else r(1.0 - al)
            v = r(r(al * blend_src.float()) + r(one_minus * v))
        y = v.to(BF16)
        if out is not None:
            out.copy_(y)
            return out
        return y
    return linear


# each variant on a call that exercises it, at magnitudes where the old verdicts' allowances (one bf16 ulp plus an
# atol of 1e-3, and the direction statistics) cannot see it: the pre-activation of SiLU at 0.05 of the usual scale;
# biases 2^-14 of the products.  An unrounded 1 - alpha is the exception: where it moves any output bits it is a gain
# error of the blended term of 2^-15 or more, which the direction statistics (alpha 0.3027: gain shift 0.0025 against a
# bound of 0.00024) or the one-ulp allowance (alpha 2^-8 - 2^-15) already flag; it stays here to show the exact check
# catches it too
VARIANTS = {
    "residual added before the row vector": dict(kind=3),
    "row vector and residual summed in fp32, one rounding": dict(kind=3),
    "SiLU of the unrounded acc + bias": dict(act=1, wscale=0.05, bias_scale=0.05),
    "scale applied before the rounding": dict(scale=0.7),
    "1 - alpha left unrounded": dict(kind=4),
    "bias of the previous N tile": dict(n=640, bn=128, bias_scale=2.0 ** -14),
    "geglu product unrounded before the scale": dict(act=2, scale=0.7),
}
OLD_VERDICTS_CATCH = {"1 - alpha left unrounded"}


def _old_verdicts(call, fn):
    """the float64 verdicts of kernel_checks / launch_checks on the call: (all pass, note)"""
    out = fn(**call)
    rerun = lambda **changes: fn(**{**call, **changes})  # noqa: E731
    try:
        recs = kc.linear_verdict("linear", call, out, rerun)
        recs += lc.VERIFIERS["linear"](call, out, rerun)[0]
    except NotImplementedError as e:
        return None, f"no float64 verdict for this call ({e})"
    bad = [rec for rec in recs if not rec["ok"]]
    return not bad, "pass" if not bad else f"FAIL ({bad[0]['check']}: {bad[0].get('why') or bad[0]['max_err_over_tol']})"


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_exact_check_catches_wrong_variant(variant, tables):
    call = _call(**VARIANTS[variant])
    fn = _variant(variant)
    # the correct emulation passes both on this very call
    ok_ref, note_ref = _old_verdicts(call, emu.linear)
    exact_ref, msg_ref = _exact(call, emu.linear(**call), tables)
    assert exact_ref and ok_ref in (True, None), f"correct emulation: old verdicts {note_ref}; {msg_ref}"
    old_ok, note = _old_verdicts(call, fn)
    exact_ok, msg = _exact(call, fn(**call), tables)
    detail = msg.split(": ", 1)[1].split("; first at ")
    where = detail[1].split(", N tile")[0] if len(detail) > 1 else ""
    print(f"{variant}: old verdicts: {note}; exact: {detail[0].split(' of ')[0]} differing at {where}")
    if variant in OLD_VERDICTS_CATCH:
        assert old_ok is False, f"{variant}: expected the old verdicts to flag it ({note})"
    else:
        assert old_ok in (True, None), f"{variant}: the old verdicts already fail it ({note})"
    assert not exact_ok, f"{variant}: the exact check passes it"


# ---- wrong main loops and drains that every instantiation shares, so the exact check, which takes its accumulators
# from the same op layer, cannot see them: the accumulator verdict against float64 and the guard bytes around an
# output slot do ----
@functools.wraps(emu.linear, assigned=())  # gx.accumulators reads ops.linear's signature
def _k_block_dropped(x, w, *args, **kw):
    """the main loop stops one 64-wide K block short, in the fp32 and the bf16 output alike"""
    x = x.clone()
    x[:, -64:] = 0
    return emu.linear(x, w, *args, **kw)


@functools.wraps(emu.linear, assigned=())
def _past_the_slot(*args, out=None, **kw):
    """the element-wise drain (an output off 16-byte alignment) also writes the column after the output's last"""
    y = emu.linear(*args, out=out, **kw)
    if out is not None and out.data_ptr() % 16:
        torch.as_strided(out, (out.shape[0], 1), out.stride(), out.storage_offset() + out.shape[1]).copy_(out[:, -1:])
    return y


SHARED = {
    "main loop drops the last 64-wide K block": (_k_block_dropped, dict(kind=2)),
    "element-wise drain writes one column past the slot": (_past_the_slot, dict(kind=2, out_slot=True)),
}


def _checks(fn, tables, **kw):
    """(exact check ok, accumulator verdict ok, guard bytes ok) of fn on _call(**kw), the accumulators from fn"""
    call = _call(**kw)
    ops = types.SimpleNamespace(linear=fn)
    out = ops.linear(**call)
    exact_ok = _exact(call, out, tables, ops)[0]
    acc_ok = gx.accumulator_verdict("linear", "linear", call, gx.accumulators("linear", call, ops))["ok"]
    guard_ok = call["out"] is None or gx.guard_intact(call["out"])
    return exact_ok, acc_ok, guard_ok


@pytest.mark.parametrize("variant", list(SHARED))
def test_new_checks_catch_shared_error(variant, tables):
    fn, kw = SHARED[variant]
    word = lambda ok: "pass" if ok else "FAIL"  # noqa: E731
    ref = _checks(emu.linear, tables, **kw)
    print(f"correct emulation ({variant} call): current exact check: {word(ref[0])}; "
          f"accumulator verdict: {word(ref[1])}; guard bytes: {word(ref[2])}")
    assert all(ref), f"correct emulation: {ref}"
    exact_ok, acc_ok, guard_ok = _checks(fn, tables, **kw)
    caught = [name for name, ok in (("accumulator verdict", acc_ok), ("guard bytes", guard_ok)) if not ok]
    print(f"{variant}: current exact check: {word(exact_ok)}; new: {' and '.join(caught) or 'nothing'} fails")
    assert exact_ok, f"{variant}: the current exact check already fails it"
    assert caught, f"{variant}: neither the accumulator verdict nor the guard bytes fail it"
