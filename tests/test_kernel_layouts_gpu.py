"""pytest -m gpu: the kernels called the way the pipelines call them (tests/kernel_checks.py, LAYOUT_CHECKS): attention
on views of fused Q/K/V and K/V projections and with per-clip contexts, temporal attention on fused views for 1..32
frames, every bf16 GEMM epilogue through both store paths, the temporal conv's full epilogue, the VAE's scaled fp32
scores, the DDIM step, the I2VGen-XL latent encoder and GroupNorm on groups far from zero mean, all against float64
references."""
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


@pytest.mark.parametrize("name,check", kc.LAYOUT_CHECKS, ids=[n for n, _ in kc.LAYOUT_CHECKS])
def test_layout(name, check):
    kc.RESULTS.clear()
    check()
    for r in kc.RESULTS:
        print(r)
    bad = [r for r in kc.RESULTS if not r["ok"]]
    assert not bad, bad
