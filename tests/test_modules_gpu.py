"""pytest -m gpu: the H100 modules (ControlNetAdapter, ControlNetRouter, ControlNetModel, SDXL UNet2DConditionModel)
against the oracle on identical name-seeded weights/inputs (tolerances: tests/module_checks.py header)."""
import pytest
import torch

from tests import module_checks as mc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device is visible (there is no CPU fallback to test)")


@pytest.mark.parametrize("group", ["adapter", "controlnet", "unet", "video", "vae", "step", "loops"])
def test_module_group(group):
    res = mc.run(group)
    bad = [r for r in res if not r["ok"]]
    assert not bad, f"module parity failed: {bad}"
