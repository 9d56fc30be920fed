"""CPU: the ABI domain sweep (tests/abi_domain.py) can pass and can fail, and the library rejects every argument just
outside the header's domain.
(a) every sampled case at reduced size passes over the emulated op layer (tests/ops_emulator.py), under the guarded
    recorder of tests/launch_checks.py, and the cases reach every predicted dispatch branch;
(b) each deliberately wrong variant of an emulated op below fails at least one case (printed with -s);
(c) for every constraint of abi_domain.DOMAIN, the real library (ctypes, no GPU) lets the last value inside through
    validation and rejects the first value outside with CA_ERR_INVALID and a message naming the argument."""
import pytest
import torch

from tests import abi_domain as ad
from tests import kernel_checks as kc
from tests import launch_checks as lc
from tests import ops_emulator as emu

BF16 = torch.bfloat16


@pytest.fixture(scope="module", autouse=True)
def _cpu_device():
    saved = kc.DEVICE
    kc.DEVICE = "cpu"
    torch.set_grad_enabled(False)
    yield
    kc.DEVICE = saved
    torch.set_grad_enabled(True)


CASES = ad.cases(small=True)


def _sweep(wrong=None):
    with emu.patched_ops() as ops:
        for name, fn in (wrong or {}).items():
            setattr(ops, name, fn)
        with lc.Recorder() as rec:
            return ad.run_cases(CASES, "cpu", rec)


def test_sweep_passes_on_emulator():
    res = _sweep()
    print("\n" + ad.summary(CASES, res))
    bad = ad.failures(res)
    assert not bad, "\n".join(f"{label}: {r.why}" for label, r in bad[:5])


def test_sweep_reaches_every_branch():
    reached = set().union(*(c.branches for c in CASES))
    assert ad.expected_branches() <= reached, sorted(ad.expected_branches() - reached)
    assert {c.op for c in CASES if not c.op.startswith("lib:")} == set(lc.OPS)
    from ctrl_adapter_b200 import _lib
    assert set(ad.DOMAIN) == set(_lib.SIGNATURES) - {"ca_abi_version", "ca_last_error", "ca_device_ok"}


# ---- wrong variants (each a small wrapper around the correct emulation) ----
def _silu_reads_past_end(x):
    """the last vector read 8 elements late: past the operand's end"""
    flat = x.reshape(-1)
    late = torch.empty(0, dtype=x.dtype).set_(x.untyped_storage(), x.storage_offset() + 8, (8,), (1,))
    return emu.silu(torch.cat([flat[:-8], late]).reshape(x.shape))


def _linear_residual_gap(x, w, bias=None, *, residual=None, **kw):
    """each row's last 8 residual columns read from the stride gap after the row"""
    if residual is not None and not residual.is_contiguous():
        m, n = residual.shape
        gap = torch.empty(0, dtype=residual.dtype).set_(residual.untyped_storage(), residual.storage_offset() + n,
                                                        (m, 8), residual.stride())
        residual = torch.cat([residual[:, :-8], gap], dim=1)
    return emu.linear(x, w, bias, residual=residual, **kw)


def _gn_ignores_groups(x, gamma, beta, eps, *, groups=32, **kw):
    """one group whatever `groups` says"""
    return emu.group_norm(x, gamma, beta, eps, groups=1, **kw)


def _linear_f32_rounds_residual(x, w, bias=None, *, residual=None, out_fp32=False, out=None, **kw):
    """fp32 epilogue: the residual sum rounded to bf16"""
    y = emu.linear(x, w, bias, residual=residual, out_fp32=out_fp32, **kw)
    if out_fp32 and residual is not None:
        y = y.to(BF16).float()
    if out is not None:
        out.copy_(y)
        return out
    return y


def _nchw_pad_unwritten(x, c_pad=None):
    """channels c..c_pad left as the allocation had them"""
    y = emu.nchw_to_nhwc(x, c_pad)
    y[..., x.shape[1]:] = float("nan")
    return y


def _embedding_no_trailing_zero(t, dim, **kw):
    """odd dim: the last column left unwritten"""
    y = emu.timestep_embedding(t, dim, **kw)
    if dim % 2:
        y[:, -1] = float("nan")
    return y


def _router_mask_first_8(logits, mask):
    """the mask ignored past expert 8"""
    if mask is not None:
        mask = mask.clone()
        mask[8:] = 1
    return emu.router_weights(logits, mask)


VARIANTS = {
    "silu: reads one vector past its end": {"silu": _silu_reads_past_end},
    "linear: residual read from the stride gap": {"linear": _linear_residual_gap},
    "group_norm: groups ignored": {"group_norm": _gn_ignores_groups},
    "linear: fp32 epilogue rounds the residual": {"linear": _linear_f32_rounds_residual},
    "nchw_to_nhwc: pad channels unwritten": {"nchw_to_nhwc": _nchw_pad_unwritten},
    "timestep_embedding: odd dim without the trailing zero": {"timestep_embedding": _embedding_no_trailing_zero},
    "router_weights: mask ignored past expert 8": {"router_weights": _router_mask_first_8},
}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_sweep_catches_wrong_variant(variant):
    bad = ad.failures(_sweep(VARIANTS[variant]))
    print(f"\n{variant}: caught by " + ("; ".join(f"{label} [{r.where}] {r.why[0][:80]}" for label, r in bad[:2])
                                       or "NOTHING"))
    assert bad, f"no case notices: {variant}"


# ---- (c) the library's validation at every boundary of the domain ----
# The calls run in a child process that sees no CUDA device (CUDA_VISIBLE_DEVICES=""), on every machine: an
# out-of-domain argument is never handed to a GPU, and a value inside the domain, once it has passed validation, fails
# at the first CUDA call with CA_ERR_CUDA instead of launching on the placeholder pointers.
BOUNDARIES = ad.boundaries()
_CHILD = """
import json, sys
from ctrl_adapter_b200 import _lib
from tests import abi_domain as ad
lib = _lib.load()
out = []
for name, arg, inside, outside, _ in ad.boundaries():
    st_out = ad.c_call(lib, name, ad.with_value(name, arg, outside))
    msg = lib.ca_last_error().decode(errors="replace")
    st_in = ad.c_call(lib, name, ad.with_value(name, arg, inside))
    out.append([st_out, msg, st_in, lib.ca_last_error().decode(errors="replace")])
json.dump(out, sys.stdout)
"""


@pytest.fixture(scope="module")
def boundary_results():
    import json
    import os
    import subprocess
    import sys
    from ctrl_adapter_b200 import build
    build.build()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", _CHILD], cwd=root, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout)


@pytest.mark.parametrize("i", range(len(BOUNDARIES)), ids=[f"{b[0]}-{b[1]}-{b[3]}" for b in BOUNDARIES])
def test_domain_boundary(boundary_results, i):
    import re
    name, arg, inside, outside, want = BOUNDARIES[i]
    st_out, msg, st_in, msg_in = boundary_results[i]
    print(f"\n{name} {arg}: outside -> status {st_out}, {msg}; inside -> status {st_in}, {msg_in}")
    assert st_out == want, f"{name}: {arg} = {outside} returned {st_out} ({msg})"
    assert re.search(rf"\b{re.escape(arg.split('[')[0])}\b", msg), msg
    assert st_in == 2, f"{name}: {arg} = {inside} returned {st_in} ({msg_in}), expected CA_ERR_CUDA"
