"""pytest -m gpu: the GEMM's bf16 epilogue with residual / blend source loaded by TMA into a ring of operand slabs
(the aligned path).  Each case also runs the same call through the element-wise drain, which reads every operand
from global memory, and requires the two to agree bit for bit."""
import math

import pytest
import torch

from tests import kernel_checks as kc

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device is visible (there is no CPU fallback to test)")
    from ctrl_adapter_b200 import _lib
    _lib.check(_lib.load().ca_device_ok(), "ca_device_ok")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _bits(t):
    return t.contiguous().view(torch.int16)


@pytest.mark.parametrize("kind,m,k,n,rpv", [
    # many tiles per CTA, both sources: one 32-column group in flight at BN 256, so every slab slot's phase wraps
    ("res_blend", 50001, 640, 1280, 0),
    ("bias_res_blend", 40000, 320, 640, 0),     # BN 160: five groups, two in flight
    ("res_blend", 9000, 256, 384, 0),            # BN 128
    ("res", 20000, 128, 64, 0),                  # BN 64
    ("blend", 30000, 320, 1280, 0),              # blend source without residual
    # row vector whose rows change inside a tile (64 rows per vector: 2 samples per 128-row tile)
    ("rowvec_res", 8192, 320, 640, 64),
    ("rowvec_res_blend", 8192, 320, 1280, 32),
    ("silu_scale_rowvec_res", 6144, 640, 1280, 2048),
])
def test_tma_operands_match_element_wise(kind, m, k, n, rpv):
    kc.RESULTS.clear()
    kc.check_gemm_epilogue(kind, m, k, n, rows_per_vec=rpv)
    bad = [r for r in kc.RESULTS if not r["ok"]]
    assert not bad, bad


@pytest.mark.parametrize("n,h,w,c,cout,blend", [
    (3, 13, 11, 320, 320, True),     # BN 160: the last 32-column group, 4-D boxes past the output
    (2, 9, 23, 640, 1280, False),    # BN 256
    (4, 7, 5, 256, 640, True),       # more rows of the box outside the output than inside
])
def test_conv_boxes_past_the_output(n, h, w, c, cout, blend):
    """3x3 conv with residual (+ blend source): the TMA boxes of the operand slabs reach past the image, which the
    hardware fills with zeros and the storers skip.  The element-wise drain (an output base 8 bytes off 16-byte
    alignment) must produce the same bits."""
    from ctrl_adapter_b200 import ops
    x = kc._rand(n, h, w, c, seed=1)
    wp = ops.pack_conv_weight(kc._rand(cout, c, 3, 3, scale=1.0 / math.sqrt(9 * c), seed=2))
    b = ops.bias_f32(kc._rand(cout, seed=3))
    res = kc._rand(n, h, w, cout, seed=4)
    xs = kc._rand(n, h, w, cout, seed=5) if blend else None
    alpha = torch.sigmoid(torch.tensor([0.3], device="cuda")).to(BF16).float() if blend else None
    kw = dict(residual=res, blend_src=xs, blend_alpha=alpha)
    ref = ops.conv2d(x, wp, b, **kw)
    buf = torch.full((ref.numel() + 16,), 7.0, device="cuda", dtype=BF16)
    ops.conv2d(x, wp, b, out=buf[4:4 + ref.numel()].view(ref.shape), **kw)
    torch.cuda.synchronize()
    assert torch.equal(_bits(buf[4:4 + ref.numel()]), _bits(ref.reshape(-1)))
    assert bool((buf[:4] == 7.0).all()) and bool((buf[4 + ref.numel():] == 7.0).all())
    # and the aligned result is the epilogue of the conv: compare with the float64 verdict of the launch
    kc.RESULTS.clear()
    kc.check_conv(n, h, w, c, cout, out_fp32=False, residual=True)
    bad = [r for r in kc.RESULTS if not r["ok"]]
    assert not bad, bad


@pytest.mark.parametrize("m,k,n", [(30000, 640, 1280), (30000, 640, 640)])
def test_output_in_place_over_residual(m, k, n):
    """out is the residual's storage: each tile reads its own residual slabs before it writes them."""
    from ctrl_adapter_b200 import ops
    x = kc._rand(m, k, seed=1)
    w = kc._rand(n, k, scale=1.0 / math.sqrt(k), seed=2)
    b = ops.bias_f32(kc._rand(n, seed=3))
    res = kc._rand(m, n, seed=4)
    ref = ops.linear(x, w, b, residual=res)
    ops.linear(x, w, b, residual=res, out=res)
    torch.cuda.synchronize()
    assert torch.equal(_bits(res), _bits(ref))


def test_unaligned_residual_stride_takes_element_wise_path():
    """A residual row stride of n + 4 elements is not a multiple of 8: no tensor map, the element-wise drain, and the
    same bits as the aligned call."""
    from ctrl_adapter_b200 import ops
    m, k, n = 9000, 320, 640
    x = kc._rand(m, k, seed=1)
    w = kc._rand(n, k, scale=1.0 / math.sqrt(k), seed=2)
    b = ops.bias_f32(kc._rand(n, seed=3))
    res = kc._rand(m, n, seed=4)
    wide = kc._rand(m, n + 4, seed=5)
    wide[:, :n] = res
    ref = ops.linear(x, w, b, residual=res)
    out = ops.linear(x, w, b, residual=wide[:, :n])
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(ref))
