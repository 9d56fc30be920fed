"""CPU tests of the VAE encoder half (AutoencoderKL / AutoencoderKLTemporalDecoder ``encode``) and of the image
preprocessing of the two video pipelines: module wiring over the emulated op layer vs the restated diffusers encoder,
key sets and parameter counts, the loading rules, ``ca_vae_latents`` argument checks, and the preprocessing
restatements (no GPU needed)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle.weights import seeded_init_, seeded_tensor
from tests import ops_emulator as emu

BF16 = torch.bfloat16
KW = dict(block_out_channels=(32, 64, 64, 64), layers_per_block=1)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_preprocess_golden.json")


def _q(t):
    return t.to(BF16).float()


def _image(n, h, w, seed_name="enc_x"):
    """seeded image in [-1, 1] whose bottom row and right column carry large values (they only reach the output through
    the bottom / right padding of the down-samplers)"""
    x = torch.tanh(seeded_tensor(seed_name, (n, 3, h, w)))
    x[:, :, -1, :] = 4.0 * torch.sign(x[:, :, -1, :]) + x[:, :, -1, :]
    x[:, :, :, -1] = -4.0 + x[:, :, :, -1]
    return _q(x)


def _pair(temporal: bool, seed: int):
    from ctrl_adapter_b200 import vae
    from oracle import vae_encoder as ov
    o = seeded_init_((ov.AutoencoderKLTemporalDecoder if temporal else ov.AutoencoderKL)(**KW), seed).eval()
    m = (vae.AutoencoderKLTemporalDecoder if temporal else vae.AutoencoderKL)(**KW)
    m.load_state_dict(o.state_dict())
    for p_ in o.parameters():
        p_.data = _q(p_.data)
    return o, m.to(BF16).eval()


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


@pytest.mark.parametrize("temporal", [False, True], ids=["kl", "temporal"])
def test_emulated_encode_matches_oracle(temporal):
    """encode -> mode() and sample(noise) on a non-square 64 x 96 image vs the restated diffusers encoder; the check sees
    the down-samplers' bottom / right padding: the symmetric-padding variant of the same module fails it."""
    o, m = _pair(temporal, 21 if temporal else 20)
    x = _image(2, 64, 96)
    noise = seeded_tensor("enc_noise", (2, 4, 8, 12))
    with torch.no_grad(), emu.patched_ops():
        post_ref = o.encode(x)[0]
        post = m.encode(x).latent_dist
        mode, smp = post.mode(), post.sample(noise=noise)
        assert mode.shape == smp.shape == (2, 4, 8, 12) and mode.dtype == BF16
        assert _rel(mode, post_ref.mode()) <= 3e-2, _rel(mode, post_ref.mode())
        assert _rel(smp, post_ref.sample(noise=noise)) <= 3e-2
        assert _rel(post.logvar, post_ref.logvar) <= 3e-2 and _rel(post.std, post_ref.std) <= 3e-2
        # the same module with symmetric (1, 1) padding in its down-samplers: measurably wrong
        for blk in m.encoder.down_blocks:
            if blk.downsamplers is not None:
                blk.downsamplers[0].conv.pad = (1, 1)
        bad = m.encode(x).latent_dist.mode()
    assert _rel(bad, post_ref.mode()) > 3e-2, _rel(bad, post_ref.mode())


def test_encode_rejects_sizes_not_multiple_of_8():
    from ctrl_adapter_b200.vae import AutoencoderKL
    m = AutoencoderKL(**KW)
    with pytest.raises(ValueError, match="divisible by 8"):
        m.encode(torch.zeros(1, 3, 64, 60))


def test_key_sets_and_parameter_counts():
    from ctrl_adapter_b200 import vae
    from oracle import vae_encoder as ov
    for ours, theirs in ((vae.AutoencoderKL, ov.AutoencoderKL),
                         (vae.AutoencoderKLTemporalDecoder, ov.AutoencoderKLTemporalDecoder)):
        with torch.device("meta"):
            a, b = ours(), theirs()
        assert set(a.state_dict()) == set(b.state_dict()), ours.__name__
        assert {k: tuple(v.shape) for k, v in a.state_dict().items()} == \
            {k: tuple(v.shape) for k, v in b.state_dict().items()}
    with torch.device("meta"):
        m, o = vae.AutoencoderKL(), ov.AutoencoderKL()
    total = sum(p.numel() for p in m.parameters())
    assert total == sum(p.numel() for p in o.parameters()) == 83_653_863  # the published SD / SDXL VAE
    dec = sum(p.numel() for k, p in m.named_parameters() if k.startswith(("decoder.", "post_quant_conv.")))
    assert dec == 49_490_199


def test_loading_rules():
    """complete encoder keys -> encodes; no encoder keys -> decode works, encode raises; one-key placeholder -> skipped,
    decode unchanged."""
    from ctrl_adapter_b200.vae import AutoencoderKL
    from oracle import vae as odec
    o, m = _pair(False, 20)
    x = _image(1, 32, 32)
    z = _q(seeded_tensor("vae_z", (1, 4, 4, 4)))
    with torch.no_grad(), emu.patched_ops():
        assert m.encoder_loaded and m.encode(x).latent_dist.mode().shape == (1, 4, 4, 4)
        ref_dec = m.decode(z).sample
    dec_only = seeded_init_(odec.AutoencoderKL(**KW), 20).state_dict()
    m2 = AutoencoderKL(**KW)
    m2.load_state_dict(dec_only)
    assert not m2.encoder_loaded
    m2 = m2.to(BF16).eval()
    with torch.no_grad(), emu.patched_ops():
        with pytest.raises(ValueError, match="encoder weights were not loaded"):
            m2.encode(x)
        assert torch.equal(m2.decode(z).sample, ref_dec)
    sd = dict(dec_only)
    sd["encoder.conv_in.weight"] = torch.zeros(1)  # placeholder: skipped like before
    m3 = AutoencoderKL(**KW)
    m3.load_state_dict(sd)
    assert not m3.encoder_loaded
    m3 = m3.to(BF16).eval()
    with torch.no_grad(), emu.patched_ops():
        assert torch.equal(m3.decode(z).sample, ref_dec)
    with pytest.raises(RuntimeError, match="missing keys"):
        AutoencoderKL(**KW).load_state_dict({k: v for k, v in dec_only.items() if k != "post_quant_conv.bias"})


@pytest.fixture(scope="module")
def lib():
    from ctrl_adapter_b200 import _lib, build
    build.build()
    return _lib.load()


_P = 256  # placeholder pointer: validation fails before anything is dereferenced
_BAD = [  # moments, noise, n, hw, latent_channels, layout, frames, num_videos, scale, out, stream
    ("frames", (_P, None, 1, 64, 4, 1, 0, 1, 0.18, _P, None), b"frames (0)"),
    ("latent_channels", (_P, None, 1, 64, 8, 1, 4, 1, 0.18, _P, None), b"latent_channels (8)"),
    ("num_videos", (_P, None, 1, 64, 4, 2, 4, 0, 1.0, _P, None), b"num_videos (0)"),
    ("moments", (None, None, 1, 64, 4, 0, 1, 1, 1.0, _P, None), b"moments"),
]


@pytest.mark.parametrize("args,names", [b[1:] for b in _BAD], ids=[b[0] for b in _BAD])
def test_vae_latents_rejects_invalid_argument(lib, args, names):
    assert lib.ca_vae_latents(*args) == 1
    assert names in lib.ca_last_error()


def test_vae_latents_emulation_layouts():
    """the emulated op (the GPU test's float64 statement has the same structure) against the reference's own tensor
    ops: prepare_image_latents (i2vgen :487-517) and _encode_vae_image + unsqueeze/repeat (svd :214-235, :580-583)."""
    from oracle.image_prep import i2vgen_prepare_image_latents, svd_image_latents
    g = torch.Generator().manual_seed(0)
    n, h, w = 2, 3, 5
    mom = torch.randn(n, h, w, 8, generator=g).to(BF16)
    noise = torch.randn(n, 4, h, w, generator=g)
    mean, logvar = mom.float().permute(0, 3, 1, 2).chunk(2, dim=1)
    smp = mean + torch.exp(0.5 * logvar.clamp(-30, 20)) * noise
    for f, nv in ((1, 1), (3, 2), (16, 1)):
        a = emu.vae_latents(mom, 1, noise, f, nv, 0.18215)
        b = i2vgen_prepare_image_latents(smp * 0.18215, f, nv).to(BF16)
        assert a.shape == (2 * n * nv, 4, f, h, w) and torch.equal(a, b)
        a = emu.vae_latents(mom, 2, None, f, nv)
        b = svd_image_latents(mean, f, nv).to(BF16)
        assert a.shape == (2 * n * nv, f, 4, h, w) and torch.equal(a, b)


def test_resize_with_antialiasing_matches_reference_golden():
    """the pipelines' restatement of the reference's utils/utils_svd.py _resize_with_antialiasing against fingerprints
    of the reference function itself (tests/golden/make_golden.py)"""
    from ctrl_adapter_b200.pipelines import _resize_with_antialiasing
    from oracle.weights import fingerprint
    gold = json.load(open(GOLDEN))
    for key, spec in gold["resize_with_antialiasing"].items():
        x = torch.rand(tuple(spec["input_shape"]), generator=torch.Generator().manual_seed(spec["seed"])) * 2 - 1
        fp = fingerprint(_resize_with_antialiasing(x, tuple(spec["size"])))
        assert fp["shape"] == spec["out"]["shape"], key
        np.testing.assert_allclose(fp["samples"], spec["out"]["samples"], rtol=0, atol=1e-5, err_msg=key)
        assert abs(fp["mean"] - spec["out"]["mean"]) <= 1e-6 and abs(fp["std"] - spec["out"]["std"]) <= 1e-6, key


@pytest.mark.parametrize("size,res", [((1500, 700), (1280, 704)), ((500, 900), (1280, 704)), ((1280, 704), (1280, 704)),
                                      ((333, 250), (224, 224))], ids=["wide", "tall", "exact", "small"])
def test_center_crop_wide(size, res):
    """_center_crop_wide: BOX resize by 1 / min(w / W, h / H) with floor-divided sizes, then the centred crop box
    (i2vgen pipeline :1180-1203)"""
    from PIL import Image
    from ctrl_adapter_b200.pipelines import _center_crop_wide
    img = Image.fromarray((np.random.default_rng(0).random((size[1], size[0], 3)) * 255).astype(np.uint8))
    scale = min(size[0] / res[0], size[1] / res[1])
    rw, rh = round(size[0] // scale), round(size[1] // scale)
    x1, y1 = (rw - res[0]) // 2, (rh - res[1]) // 2
    want = img.resize((rw, rh), resample=Image.BOX).crop((x1, y1, x1 + res[0], y1 + res[1]))
    got = _center_crop_wide(img, res)
    assert got.size == res and np.array_equal(np.asarray(got), np.asarray(want))
    got2 = _center_crop_wide([img, img], res)
    assert len(got2) == 2 and np.array_equal(np.asarray(got2[1]), np.asarray(want))
