"""pytest -m gpu: the attention, norm and small kernels against a PyTorch fp32 reference of the same op (see
tests/kernel_checks.py for the per-check tolerances; the GEMM kernel is checked by test_gemm_epilogue_exact_gpu.py).
All calls go through the C ABI (ctypes -> libctrl_adapter_b200.so)."""
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


@pytest.mark.parametrize("group", ["attn", "misc"])
def test_kernel_group(group):
    res = kc.run_all(group=group)
    bad = [r for r in res if not r["ok"]]
    assert not bad, f"{len(bad)} kernel parity checks failed: {bad[:3]}"
    assert len(res) >= 8
