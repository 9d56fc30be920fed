"""pytest -m gpu -s: the launch census (tests/launch_checks.py) at the geometry the product runs.  One eager step of each
benchmark workload as bench.py builds it (batch 1: SDXL 1024^2 = 128^2 latents, I2VGen-XL 16 frames at 64^2, SVD 14
frames at 72x128, I2VGen-XL with three ControlNets and the router), with the recorder installed before the modules are
built so that the step-invariant work of prepare() is covered too; and the VAE at the pipelines' resolutions: decode of
a 128^2 latent, encode of a 512^2 image (I2VGen-XL) and of a 576x1024 image (SVD temporal VAE) with the latents of both
video layouts, and the temporal decoder on one 14-frame chunk at 72x128.  Every distinct kernel launch is checked
against a float64 reference of its op; each case prints one row per distinct configuration."""
import time

import pytest
import torch

from tests import launch_checks as lc

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


def _step(workload):
    import bench
    loop, _ = bench.build_ours(workload, 1, 1024, "cuda", 0)
    loop.step(0)


def _image(n, h, w, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.tanh(torch.randn(n, 3, h, w, generator=g, device="cuda")).to(BF16)


def _vae_decode_sdxl():
    from ctrl_adapter_b200.vae import AutoencoderKL
    with torch.device("cuda"):
        m = AutoencoderKL().to(BF16).eval()
    g = torch.Generator(device="cuda").manual_seed(1)
    m.decode(torch.randn(1, 4, 128, 128, generator=g, device="cuda").to(BF16))


def _vae_encode():
    from ctrl_adapter_b200 import pipelines
    from ctrl_adapter_b200.vae import AutoencoderKL, AutoencoderKLTemporalDecoder
    with torch.device("cuda"):
        kl, tv = AutoencoderKL().to(BF16).eval(), AutoencoderKLTemporalDecoder().to(BF16).eval()
    pipelines.i2vgen_image_latents(kl, _image(1, 512, 512, 2), 16, 1)
    pipelines.svd_image_latents(tv, _image(1, 576, 1024, 3), 14, 1)


def _vae_decode_svd():
    from ctrl_adapter_b200.vae import AutoencoderKLTemporalDecoder
    with torch.device("cuda"):
        m = AutoencoderKLTemporalDecoder().to(BF16).eval()
    g = torch.Generator(device="cuda").manual_seed(4)
    m.decode(torch.randn(14, 4, 72, 128, generator=g, device="cuda").to(BF16), num_frames=14)


CASES = {"sdxl": lambda: _step("sdxl"), "i2vgen": lambda: _step("i2vgen"), "svd": lambda: _step("svd"),
         "multi": lambda: _step("multi"), "vae_decode_1024": _vae_decode_sdxl, "vae_encode_512_576x1024": _vae_encode,
         "vae_temporal_decode_14x72x128": _vae_decode_svd}


@pytest.mark.parametrize("case", list(CASES))
def test_launch_census(case):
    torch.manual_seed(0)
    t0 = time.time()
    with torch.no_grad(), lc.Recorder() as rec:
        CASES[case]()
    torch.cuda.synchronize()
    fam = rec.families()
    print(f"\n== {case}: {sum(v[0] for v in fam.values())} launches, {len(rec.rows)} distinct configurations, "
          f"{sum(v[2] for v in fam.values())} sampled, {time.time() - t0:.0f} s")
    print(rec.table())
    print("per op: " + "; ".join(f"{op} {n} launches / {d} configs / {s} sampled / worst err/tol {w:.3f}"
                                 for op, (n, d, s, w) in sorted(fam.items())))
    bad = rec.failures()
    assert not bad, "\n".join(f"{r.op} {lc.key_summary(r.key)} [{r.where}]: {r.why}" for r in bad[:10])
