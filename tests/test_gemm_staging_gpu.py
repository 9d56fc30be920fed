"""pytest -m gpu: the GEMM's staged bf16 epilogue (consumers stage the tile in shared memory, the storer warps of
warpgroup 0 add row vector / residual / AlphaBlender and write it).  Cases that reuse the staging tile and its
barrier phases over many tiles per CTA, 4-D conv boxes with rows outside the output, and the element-wise drain
for an output that is not 16-byte aligned."""
import math

import pytest
import torch

from tests import kernel_checks as kc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device is visible (there is no CPU fallback to test)")
    from ctrl_adapter_b200 import _lib
    _lib.check(_lib.load().ca_device_ok(), "ca_device_ok")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


@pytest.mark.parametrize("case", [
    # more than 2 x 132 tiles, residual, partial last M tile (BN 256: 3 ring stages next to the staging tile)
    lambda: kc.check_linear(50001, 640, 1280, out_fp32=False, residual=True),
    # BN 160 (padded staging rows), residual, many tiles
    lambda: kc.check_linear(40000, 320, 640, out_fp32=False, residual=True),
    # 3x3 conv whose 4-D boxes reach past the output: row vector + residual
    lambda: kc.check_conv(3, 13, 11, 320, 320, out_fp32=False, rowvec=True, residual=True),
    lambda: kc.check_conv(2, 9, 23, 640, 640, out_fp32=False, residual=True, scale=0.5),
    # AlphaBlender over many tiles
    lambda: kc.check_linear_blend(9000, 640, 640),
    # GEGLU at BN 256 over many tiles (half-width staging tile, 4 ring stages)
    lambda: kc.check_geglu(8192, 640, 2560),
])
def test_staged_epilogue(case):
    kc.RESULTS.clear()
    rec = case()
    bad = [r for r in kc.RESULTS if not r["ok"]]
    assert not bad, bad


def test_unaligned_output_slice():
    """Output written into channels [4, 324) of a 336-wide buffer: the base is not 16-byte aligned, so the storers take
    the element-wise path.  It must produce what the aligned path produces, and leave the rest of the buffer alone."""
    from ctrl_adapter_b200 import ops
    m, k, n = 2000, 320, 320
    x = kc._rand(m, k, seed=1)
    w = kc._rand(n, k, scale=1.0 / math.sqrt(k), seed=2)
    b = ops.bias_f32(kc._rand(n, seed=3))
    res = kc._rand(m, n, seed=4)
    ref = ops.linear(x, w, b, residual=res)
    buf = torch.full((m, 336), 7.0, device="cuda", dtype=torch.bfloat16)
    ops.linear(x, w, b, residual=res, out=buf[:, 4:4 + n])
    torch.cuda.synchronize()
    assert torch.equal(buf[:, 4:4 + n].view(torch.int16), ref.view(torch.int16))
    assert bool((buf[:, :4] == 7.0).all()) and bool((buf[:, 4 + n:] == 7.0).all())
