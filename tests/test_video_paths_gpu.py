"""pytest -m gpu: Stable-Video-Diffusion UNet, the SVD denoising loop (ca_cfg_euler_v), the sparse key-frame path of the
I2VGen-XL loop and the SVD-geometry kernel shapes against the oracle; the folded conditioning convolutions against their
zero-padded form.

A failure here is red like any other test (nothing is xfail-guarded)."""
import json
import os

import pytest
import torch

from tests import module_checks as mc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device is visible (there is no CPU fallback to test)")


@pytest.mark.parametrize("group", ["shapes", "svd", "sparse", "svd_loop", "fold"])
def test_video_group(group):
    res = [dict(r) for r in mc.run(group)]
    out = os.path.join(ROOT, "gpurun_out")
    if os.path.isdir(out):  # keep the records of the run (scratch directory, merged back by gpurun)
        with open(os.path.join(out, f"gpu_group_{group}.json"), "w") as f:
            json.dump(res, f, indent=1, default=str)
    bad = [r for r in res if not r["ok"]]
    assert res and not bad, f"{group}: parity failed: {json.dumps(bad, default=str)[:1500]}"
