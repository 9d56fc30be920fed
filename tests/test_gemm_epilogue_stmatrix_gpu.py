"""pytest -m gpu: the GEMM's plain bf16 epilogue (bias, no activation, scale 1, no row vector / residual / blend) is
the fp32 result rounded once to bf16.  The consumers stage it with stmatrix, add the bias only when there is one and
leave the single rounding to the pack, so its bytes must equal round-to-nearest-even of the same call's fp32-output
instantiation, which shares the main loop and hence the accumulators.  Each BN (64, 128 and 256 stage into
XOR-swizzled rows, 160 into padded rows) runs with a partial last M and N tile and more than 2 x 132 tiles, so every
CTA goes through both buffers of the double-buffered bias more than once."""
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


# (BN, output columns): the last N tile is partial in each case
_TILES = [(64, 104), (128, 200), (160, 400), (256, 640)]


@pytest.mark.parametrize("with_bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("bn,n", _TILES, ids=[f"bn{bn}" for bn, _ in _TILES])
def test_plain_bf16_is_rounded_fp32(bn, n, with_bias):
    from ctrl_adapter_b200 import ops
    m, k = 50001, 320  # 391 M tiles, the last one partial
    x = kc._rand(m, k, seed=11)
    w = kc._rand(n, k, scale=1.0 / math.sqrt(k), seed=12)
    # any fp32 bias, not only bf16-valued ones
    g = torch.Generator(device="cuda")
    g.manual_seed(13)
    b = torch.randn(n, generator=g, device="cuda") if with_bias else None
    assert m // 128 * math.ceil(n / bn) > 2 * 132
    out = ops.linear(x, w, b, bn=bn)
    ref = ops.linear(x, w, b, bn=bn, out_fp32=True)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), ref.to(torch.bfloat16).view(torch.int16))
