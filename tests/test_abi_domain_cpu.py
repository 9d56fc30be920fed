"""CPU: the ABI domain sweep (tests/abi_domain.py) can pass and can fail, and the library rejects every argument just
outside the header's domain.
(a) every sampled case at reduced size passes over the emulated op layer (tests/ops_emulator.py), under the guarded
    recorder of tests/launch_checks.py, and the cases reach every predicted dispatch branch;
(b) each deliberately wrong variant of an emulated op below fails at least one case (printed with -s);
(c) for every constraint of abi_domain.DOMAIN, the real library (ctypes, no GPU) lets the last value inside through
    validation and rejects the first value outside with CA_ERR_INVALID and a message naming the argument;
(d) the restated 192-row attention tile rule matches its boundary table, and the kernel-name parser of the GPU sweep
    reads fixed demangled and mangled names."""
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


def _attention_tiled(q, k, v, heads, head_dim_pad, scale, out=None, kv_batch_div=1, *, rescale=True,
                     ragged_tail=True):
    """online softmax over 128-key tiles.  rescale=False: the running sum and output are not rescaled when a later tile
    raises the row max; ragged_tail=False: with more than one tile, the keys of a partial last tile are dropped"""
    b, lq, _ = q.shape
    lk = k.shape[1]
    qh = q.float().reshape(b, lq, heads, head_dim_pad).permute(0, 2, 1, 3)
    kb = torch.arange(b) // kv_batch_div
    kh, vh = (t.float().reshape(t.shape[0], lk, heads, head_dim_pad).permute(0, 2, 1, 3)[kb] for t in (k, v))
    if not ragged_tail and lk > 128:
        kh, vh = kh[:, :, :lk // 128 * 128], vh[:, :, :lk // 128 * 128]
    m = torch.full((b, heads, lq, 1), -float("inf"))
    l, o = torch.zeros(b, heads, lq, 1), torch.zeros(b, heads, lq, head_dim_pad)
    for j in range(0, kh.shape[2], 128):
        s = qh @ kh[:, :, j:j + 128].transpose(-1, -2) * scale
        m_new = torch.maximum(m, s.amax(-1, keepdim=True))
        p = torch.exp(s - m_new)
        corr = torch.exp(m - m_new) if rescale else torch.ones_like(m)
        l, o, m = l * corr + p.sum(-1, keepdim=True), o * corr + p @ vh[:, :, j:j + 128], m_new
    y = (o / l).permute(0, 2, 1, 3).reshape(b, lq, heads * head_dim_pad).to(BF16)
    if out is not None:
        out.copy_(y)
        return out
    return y


def _attention_no_rescale(*args, **kw):
    return _attention_tiled(*args, **kw, rescale=False)


def _attention_drops_ragged_tail(*args, **kw):
    return _attention_tiled(*args, **kw, ragged_tail=False)


def _read_as(t, shape, stride):
    """t's storage read from t's first element with another shape / stride; elements past the storage are NaN (a guard
    band)"""
    flat = torch.empty(0, dtype=t.dtype).set_(t.untyped_storage(), t.storage_offset(),
                                                (t.untyped_storage().nbytes() // t.element_size() - t.storage_offset(),))
    idx = sum(torch.arange(n).reshape([-1 if i == d else 1 for i in range(len(shape))]) * s
              for d, (n, s) in enumerate(zip(shape, stride)))
    nan = torch.full((), float("nan"), dtype=t.dtype)
    return torch.where(idx < flat.numel(), flat[idx.clamp(max=flat.numel() - 1)], nan)


def _linear_residual_output_stride(x, w, bias=None, *, residual=None, out=None, **kw):
    """the residual (and blend source) read with the output's row stride instead of its own"""
    m, n = x.shape[0], w.shape[0]
    ostride = (n, 1) if out is None else out.stride()
    if residual is not None and residual.stride() != ostride:
        residual = _read_as(residual, (m, n), ostride)
        if kw.get("blend_src") is not None:
            kw["blend_src"] = _read_as(kw["blend_src"], (m, n), ostride)
    return emu.linear(x, w, bias, residual=residual, out=out, **kw)


def _linear_broadcast_as_contiguous(x, w, bias=None, *, residual=None, blend_src=None, **kw):
    """a residual / blend source broadcast along M (stride 0) read as if it were a contiguous [M, N]"""
    fix = lambda t: t if t is None or t.stride(0) != 0 else _read_as(t, t.shape, (t.shape[1], 1))  # noqa: E731
    return emu.linear(x, w, bias, residual=fix(residual), blend_src=fix(blend_src), **kw)


VARIANTS = {
    "attention: running sum and output not rescaled when a later KV tile raises the max":
        {"attention": _attention_no_rescale},
    "attention: the keys of a ragged last KV tile dropped": {"attention": _attention_drops_ragged_tail},
    "linear: residual read with the output's row stride": {"linear": _linear_residual_output_stride},
    "linear: broadcast residual / blend source read as contiguous": {"linear": _linear_broadcast_as_contiguous},
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


# ---- (d) the restated dispatch rules and the kernel-name parser of the GPU sweep ----
# (lq, lk, head_dim_pad, 192-row tiles?): the boundaries of ca_attention's use_wg3.  1600 is where 25 (pad192 - pad128)
# == lq: the rule's <= decides it.
NWG_TABLE = ([(lq, 257, 64, False) for lq in (1, 64, 127, 128)] +
             [(129, 257, 64, True), (192, 257, 64, True), (193, 257, 64, False), (256, 257, 64, False),
              (257, 257, 64, True), (576, 257, 64, True), (577, 257, 64, False), (1599, 257, 64, False),
              (1600, 257, 64, True), (2880, 257, 64, True), (2881, 257, 64, False), (2944, 257, 64, False),
              (2945, 257, 64, True), (192, 128, 64, False), (192, 129, 64, True)] +
             [(lq, 1300, dp, False) for dp in (128, 192) for lq in (129, 192, 576, 1600, 2945, 4096)])


def test_attention_nwg_table():
    got = [(lq, lk, dp, ad.attention_nwg(dp, lq, lk) == 3) for lq, lk, dp, _ in NWG_TABLE]
    assert got == NWG_TABLE
    assert all(ad.attention_nwg(64, lq, lk) == 3 for lq in range(2945, 20000) for lk in (129, 4096))
    assert all(ad.attention_nwg(64, lq, 128) == 2 for lq in range(1, 20000))


KERNEL_NAMES = [
    ("void ca::attention_kernel<1, 3>(CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, ca::AttnParams)",
     {"attention DQ1", "attention DQ1 NWG3"}),
    ("void ca::attention_kernel<3, 2>(CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, ca::AttnParams)",
     {"attention DQ3", "attention DQ3 NWG2"}),
    ("_ZN2ca16attention_kernelILi2ELi2EEEv14CUtensorMap_stS1_S1_NS_10AttnParamsE",
     {"attention DQ2", "attention DQ2 NWG2"}),
    ("void ca::gemm_conv_kernel<160, 0, true>(CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, "
     "CUtensorMap_st, ca::GemmParams)", {"gemm bn160", "gemm epilogue bf16", "gemm kOps1"}),
    ("void ca::gemm_conv_kernel<64, 0, false>(CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, "
     "CUtensorMap_st, ca::GemmParams)", {"gemm bn64", "gemm epilogue bf16", "gemm kOps0"}),
    ("void ca::gemm_conv_kernel<256, 1, false>(CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, "
     "CUtensorMap_st, ca::GemmParams)", {"gemm bn256", "gemm epilogue geglu"}),
    ("_ZN2ca16gemm_conv_kernelILi128ELi2ELb0EEEv14CUtensorMap_stS1_S1_S1_S1_NS_10GemmParamsE",
     {"gemm bn128", "gemm epilogue f32"}),
    ("void ca::layernorm_kernel<3, 16, true>(__nv_bfloat16 const*, long long, int, float, float const*, float const*, "
     "__nv_bfloat16 const*, int, __nv_bfloat16*, __nv_bfloat16*)", {"layernorm NV3 L16 RV1"}),
    ("void ca::temporal_attention_tc_kernel<32>(CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, ca::TaParams)",
     {"temporal_attention SEQ32"}),
    ("void ca::gn_apply_kernel<false, true>(__nv_bfloat16 const*, int, __nv_bfloat16 const*, int, int, int, int, int, "
     "float, double const*, float const*, float const*, __nv_bfloat16*)", {"gn_apply silu0 up1"}),
    ("void ca::nchw_to_nhwc_kernel<float>(float const*, int, long long, int, __nv_bfloat16*)",
     {"nchw_to_nhwc src fp32"}),
    ("_ZN2ca19nhwc_to_nchw_kernelI14__nv_bfloat16EEvPKS1_iixPT_", {"nhwc_to_nchw dst bf16"}),
    ("void ca::gn_stats_kernel(__nv_bfloat16 const*, int, __nv_bfloat16 const*, int, int, int, double*)", set()),
    ("void at::native::vectorized_elementwise_kernel<4, at::native::FillFunctor<float>, std::array<char*, 1ul> >"
     "(int, at::native::FillFunctor<float>, std::array<char*, 1ul>)", set()),
    ("Memcpy DtoD (Device -> Device)", set()),
]


@pytest.mark.parametrize("name,labels", KERNEL_NAMES, ids=[n[:48] for n, _ in KERNEL_NAMES])
def test_kernel_labels(name, labels):
    assert ad.kernel_labels(name) == labels


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
