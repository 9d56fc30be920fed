"""CPU tests of the host code at non-square latent geometry, over the emulated op layer (tests/ops_emulator.py).

1. Emulated counterparts of tests/test_geometry_gpu.py: the modules against the oracle at a geometry and its transpose
   (the full-width UNets under `slow`; the loops run on the GPU only).
2. Wrong variants: eight height / width swaps, five in the emulated ops (standing for a kernel's or descriptor's swapped
   dims) and three in the host code, each of which computes exactly the right numbers at a square size.  Each must
   pass the existing square comparisons (test_host_emulated_cpu.py's tests, run as they are) and fail a geometry case
   here; `-s` prints `square cases: pass; <case>: <statistic> = x > bound y`.
3. Geometry domain: what each loop accepts per use_size_512, checked just inside and just outside; the refusal is a
   ValueError naming height / width, raised by prepare() before any op or module is called.
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from oracle import cases
from tests import ops_emulator as emu
from tests import test_host_emulated_cpu as hec

BF16 = torch.bfloat16
torch.set_grad_enabled(False)
TOL = 3e-2


def _rel(o, p, inputs):
    """worst relative Frobenius error of the emulated module against the oracle (hec._compare without its assert)"""
    ref = hec._flat(o(**hec._map(inputs, hec._q)))
    with emu.patched_ops():
        ours = hec._flat(p(**hec._map(inputs, lambda t: t.to(BF16))))
    assert len(ours) == len(ref)
    worst = 0.0
    for a, b in zip(ours, ref):
        assert tuple(a.shape) == tuple(b.shape)
        if float(b.abs().max()) > 0.0:
            worst = max(worst, float((a.float() - b).norm() / b.norm()))
    return worst


# ---- cases (each returns its statistic; the bound is TOL) -------------------------------------------------------
def _adapter(kind, hw):
    from ctrl_adapter_b200.adapter import ControlNetAdapter
    from oracle.adapter import ControlNetAdapter as O
    if kind == "sdxl":
        kw, inputs, seed = cases.ADAPTER_SDXL_KW, cases.adapter_sdxl_inputs(2, hw=hw), 1
    else:
        kw, inputs, seed = cases.ADAPTER_VIDEO_KW, cases.adapter_video_inputs(1, 4, hw=hw), 2
    o, p = hec._pair(lambda: O(**kw), lambda: ControlNetAdapter(**kw), seed)
    return _rel(o, p, inputs)


def _controlnet(hw, skip_conv_in=False):
    from ctrl_adapter_b200.controlnet import ControlNetModel
    from oracle.controlnet import ControlNetModel as O
    o, p = hec._pair(lambda: O(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4)
    return _rel(o, p, dict(cases.controlnet_inputs(2, hw=hw), conditioning_scale=0.75, skip_conv_in=skip_conv_in))


def _i2vgen_image_tokens(hw):
    """I2VGen-XL's image-latent context tokens (first frame -> conv -> 32x32 pool -> two stride-2 convs) against the
    oracle UNet's image_latents_context_embedding: only that part of the two UNets is materialised"""
    from ctrl_adapter_b200.unet_i2vgen import I2VGenXLUNet
    from oracle.unet_i2vgen import I2VGenXLUNet as O
    from oracle.weights import seeded_init_, seeded_tensor
    with torch.device("meta"):
        o, p = O(), I2VGenXLUNet()
    oe = seeded_init_(o.image_latents_context_embedding.to_empty(device="cpu"), 7).eval()
    pe = p.image_latents_context_embedding.to_empty(device="cpu")
    pe.load_state_dict(oe.state_dict())
    pe.to(BF16)
    for prm in oe.parameters():
        prm.data = hec._q(prm.data)
    il = hec._q(seeded_tensor("geo_il", (2, 4, 3, *hw)))
    ref = oe(il[:, :, 0]).permute(0, 2, 3, 1)
    with emu.patched_ops():
        ours = p.image_latent_tokens(il[:, :, 0].to(BF16).contiguous()).float()
    return float((ours[..., :ref.shape[-1]] - ref).norm() / ref.norm())


def _image_pool(hw):
    """the loops' control-image pool to 512 x 512 against F.adaptive_avg_pool2d"""
    from ctrl_adapter_b200.loop_base import pool_control_images
    from oracle.weights import seeded_tensor
    img = hec._q(torch.sigmoid(seeded_tensor("geo_img", (2, 3, *hw))))
    with emu.patched_ops():
        ours = pool_control_images(img.to(BF16)).float()
    ref = F.adaptive_avg_pool2d(img, (512, 512))
    return float((ours - ref).norm() / ref.norm())


def _sdxl_time_ids(height, width):
    """the add_time_ids SDXLControlNetAdapterPipeline.__call__ hands its loop at height x width, against the
    reference's (height, width) + (0, 0) + (height, width) rows: max |difference| / max |reference|"""
    from ctrl_adapter_b200 import pipelines
    got = {}

    class Recorder:
        def __init__(self, *a, **k):
            pass

        def prepare(self, **kw):
            got.update(kw)
            raise StopIteration

    pipe = pipelines.SDXLControlNetAdapterPipeline(None, None, None, None, None, None, None, None, None, None)
    saved = pipelines.SDXLControlNetAdapterLoop
    pipelines.SDXLControlNetAdapterLoop = Recorder
    try:
        with pytest.raises(StopIteration):
            pipe(prompt_embeds=torch.zeros(1, 77, 2048), negative_prompt_embeds=torch.zeros(1, 77, 2048),
                 pooled_prompt_embeds=torch.zeros(1, 1280), negative_pooled_prompt_embeds=torch.zeros(1, 1280),
                 controlnet_prompt_embeds=torch.zeros(1, 77, 768), controlnet_negative_prompt_embeds=torch.zeros(1, 77, 768),
                 control_images=torch.zeros(1, 3, 512, 512), height=height, width=width)
    finally:
        pipelines.SDXLControlNetAdapterLoop = saved
    ref = torch.tensor([[height, width, 0, 0, height, width]] * 2, dtype=torch.float32)
    return float((got["add_time_ids"].float().cpu() - ref).abs().max() / ref.abs().max())


CASES = {
    "adapter[sdxl] 8x16": lambda: _adapter("sdxl", (8, 16)),
    "adapter[sdxl] 16x8": lambda: _adapter("sdxl", (16, 8)),
    "adapter[video] 8x16": lambda: _adapter("video", (8, 16)),
    "adapter[video] 16x8": lambda: _adapter("video", (16, 8)),
    "ControlNet 8x16": lambda: _controlnet((8, 16)),
    "ControlNet 16x8 skip_conv_in": lambda: _controlnet((16, 8), True),
    "I2VGen-XL image tokens 32x64": lambda: _i2vgen_image_tokens((32, 64)),
    "I2VGen-XL image tokens 96x64": lambda: _i2vgen_image_tokens((96, 64)),
    "control image pool 512x1024": lambda: _image_pool((512, 1024)),
    "SDXL time ids 768x1024": lambda: _sdxl_time_ids(768, 1024),
}


@pytest.mark.parametrize("name", list(CASES))
def test_geometry_case(name):
    """the correct host code and emulation pass every geometry case"""
    stat = CASES[name]()
    assert stat <= TOL, f"{name}: rel error {stat:.4f} > {TOL}"


# ---- wrong variants ------------------------------------------------------------------------------------------------
def _transposed(fn, x, *a, **k):
    """run fn on x's buffer read as [n, w, h, c], and read its [n, w', h', c'] result back as [n, h', w', c']"""
    n, h, w, c = x.shape
    y = fn(x.reshape(n, w, h, c), *a, **k)
    return y.reshape(n, y.shape[2], y.shape[1], y.shape[3])


_ORIG = {k: getattr(emu, k) for k in ("upsample2x", "group_norm", "conv2d", "avgpool")}


def _v_upsample(x):
    return _transposed(_ORIG["upsample2x"], x)


def _v_gn_up2x(x, *a, up2x=False, **k):
    if not up2x:
        return _ORIG["group_norm"](x, *a, **k)
    y = _ORIG["group_norm"](x, *a, up2x=False, **k)
    return _transposed(_ORIG["upsample2x"], y)


def _v_conv3x3(x, w, b, *, ksize=3, stride=1, x2=None, **k):
    if ksize != 3 or stride != 1 or x2 is not None or k.get("residual") is not None or k.get("blend_src") is not None:
        return _ORIG["conv2d"](x, w, b, ksize=ksize, stride=stride, x2=x2, **k)
    return _transposed(lambda t: _ORIG["conv2d"](t, w, b, ksize=3, stride=1, **k), x)


def _v_conv_s2(x, w, b, *, ksize=3, stride=1, **k):
    if stride != 2 or k.get("residual") is not None or k.get("blend_src") is not None:
        return _ORIG["conv2d"](x, w, b, ksize=ksize, stride=stride, **k)
    return _transposed(lambda t: _ORIG["conv2d"](t, w, b, ksize=ksize, stride=2, **k), x)


def _v_avgpool(x, oh, ow):
    n, h, w, c = x.shape
    return _ORIG["avgpool"](x.reshape(n, w, h, c), ow, oh).reshape(n, oh, ow, c)


def _host_adapter_resnet(monkeypatch):
    """channels-last activation reshaped (n, w, h, c) before the first 3x3 conv of the video adapter's spatial resnet"""
    from ctrl_adapter_b200 import adapter
    orig = adapter.AdapterSpatioTemporal.forward_nhwc

    def forward_nhwc(self, x, num_frames, t, ctx):
        if not self.add_temporal_resnet:
            return orig(self, x, num_frames, t, ctx)
        conv = self.spatial_resnets[0].conv1
        fwd = conv.forward
        conv.forward = lambda h, **k: _transposed(lambda u: fwd(u, **k), h)
        try:
            return orig(self, x, num_frames, t, ctx)
        finally:
            del conv.forward
    monkeypatch.setattr(adapter.AdapterSpatioTemporal, "forward_nhwc", forward_nhwc)


def _host_image_tokens(monkeypatch):
    """I2VGen-XL's first-frame image latent read as (b, 4, w, h) before its conv and 32x32 pool"""
    from ctrl_adapter_b200.unet_i2vgen import I2VGenXLUNet
    orig = I2VGenXLUNet.image_latent_tokens

    def image_latent_tokens(self, il_first):
        b, c, h, w = il_first.shape
        return orig(self, il_first.reshape(b, c, w, h))
    monkeypatch.setattr(I2VGenXLUNet, "image_latent_tokens", image_latent_tokens)


def _host_time_ids(monkeypatch):
    """SDXL original_size / target_size built as (width, height)"""
    from ctrl_adapter_b200 import pipelines
    orig = pipelines.sdxl_add_time_ids

    def sdxl_add_time_ids(batch, height, width, *a, **k):
        return orig(batch, width, height, *a, **k)
    monkeypatch.setattr(pipelines, "sdxl_add_time_ids", sdxl_add_time_ids)


def _emu(name, fn):
    return lambda mp: mp.setattr(emu, name, fn)


# variant -> (how to apply it, the existing square tests it must pass, the geometry case it must fail)
VARIANTS = {
    "upsample2x reading [n, w, h, c]": (_emu("upsample2x", _v_upsample), [hec.test_emulated_adapter_sdxl],
                                        "adapter[sdxl] 8x16"),
    "GroupNorm-apply up2x with (w, h)": (_emu("group_norm", _v_gn_up2x), [hec.test_emulated_adapter_sdxl],
                                         "adapter[sdxl] 16x8"),
    "3x3 conv on the transposed grid (swapped descriptor row dims)": (
        _emu("conv2d", _v_conv3x3), [hec.test_emulated_adapter_sdxl, hec.test_emulated_controlnet], "adapter[sdxl] 8x16"),
    "stride-2 parity view on the transposed grid": (
        _emu("conv2d", _v_conv_s2), [hec.test_emulated_controlnet], "ControlNet 8x16"),
    "avgpool with its per-axis ratios swapped": (
        _emu("avgpool", _v_avgpool), [lambda: _assert_ok(_image_pool((1024, 1024)))], "control image pool 512x1024"),
    "host: video adapter spatial resnet reshaped (n, w, h, c) before conv1": (
        _host_adapter_resnet, [hec.test_emulated_adapter_video], "adapter[video] 8x16"),
    "host: prepare_conditioning reading the first-frame latent as (b, 4, w, h)": (
        _host_image_tokens, [lambda: _assert_ok(_i2vgen_image_tokens((64, 64)))], "I2VGen-XL image tokens 32x64"),
    "host: SDXL original_size / target_size as (width, height)": (
        _host_time_ids, [lambda: _assert_ok(_sdxl_time_ids(1024, 1024))], "SDXL time ids 768x1024"),
}


def _assert_ok(stat):
    assert stat <= TOL, stat


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_wrong_variant(variant, monkeypatch):
    apply, square, case = VARIANTS[variant]
    apply(monkeypatch)
    for t in square:
        t()
    stat = CASES[case]()
    print(f"\n{variant}: square cases: pass; {case}: rel error = {stat:.4g} > bound {TOL:g}")
    assert stat > TOL, f"{variant} is not caught by {case} ({stat:.4g})"


# ---- geometry domain -----------------------------------------------------------------------------------------------
# (loop, use_size_512) -> latents (h, w) just inside the domain, latents just outside it
DOMAIN = {
    ("sdxl", True): ([(128, 128)], [(64, 64), (120, 128), (128, 136), (64, 128), (128, 64)]),
    ("sdxl", False): ([], [(128, 128), (64, 64), (64, 128)]),
    ("i2vgen", True): ([(64, 64)], [(32, 64), (64, 96), (96, 64)]),
    ("i2vgen", False): ([(32, 32), (32, 64), (64, 96), (96, 32)], [(24, 32), (32, 48), (40, 64), (16, 16)]),
    ("svd", True): ([(64, 64)], [(72, 128), (128, 128), (64, 72)]),
    ("svd", False): ([(8, 8), (24, 40), (72, 128), (40, 24)], [(12, 16), (24, 36), (20, 40), (4, 8)]),
}


class _Reached(Exception):
    pass


class _Module:
    """stands for a module: any use of it means prepare() got past its geometry check"""

    def __getattr__(self, name):
        if name == "nets":
            raise AttributeError(name)
        raise _Reached(name)

    def __call__(self, *a, **k):
        raise _Reached("call")


@contextlib.contextmanager
def _counted_ops():
    """the emulated ops, each counting its calls"""
    from ctrl_adapter_b200 import ops
    count = [0]

    def wrap(fn):
        def f(*a, **k):
            count[0] += 1
            return fn(*a, **k)
        return f
    with emu.patched_ops():
        saved = {n: getattr(ops, n) for n in emu._EMULATED}
        for n, fn in saved.items():
            setattr(ops, n, wrap(fn))
        try:
            yield count
        finally:
            for n, fn in saved.items():
                setattr(ops, n, fn)


def _prepare(loop_kind, use_512, h, w):
    """construct the loop around stand-in modules and call prepare() at latents h x w (control images at the size the
    pipelines make them: 8 x the latents, or 512 x 512 when use_size_512 pools)"""
    from ctrl_adapter_b200.pipeline_i2vgen import I2VGenXLControlNetAdapterLoop
    from ctrl_adapter_b200.pipeline_sdxl import SDXLControlNetAdapterLoop
    from ctrl_adapter_b200.pipeline_svd import SVDControlNetAdapterLoop
    m = _Module()
    b, f = 1, 2
    img = torch.zeros(2 * b * f, 3, 8 * h, 8 * w)
    if loop_kind == "sdxl":
        loop = SDXLControlNetAdapterLoop(m, m, m, num_inference_steps=4, use_size_512=use_512)
        loop.prepare(latents=torch.zeros(b, 4, h, w), prompt_embeds=torch.zeros(2 * b, 77, 2048),
                     add_text_embeds=torch.zeros(2 * b, 1280), add_time_ids=torch.zeros(2 * b, 6),
                     controlnet_prompt_embeds=torch.zeros(2 * b, 77, 768), control_images=img[:2 * b])
    elif loop_kind == "i2vgen":
        loop = I2VGenXLControlNetAdapterLoop(m, m, m, None, num_inference_steps=4, use_size_512=use_512)
        loop.prepare(latents=torch.zeros(b, 4, f, h, w), prompt_embeds=torch.zeros(2 * b, 77, 1024),
                     image_latents=torch.zeros(2 * b, 4, f, h, w), image_embeddings=torch.zeros(2 * b, 1, 1024),
                     fps=torch.zeros(2 * b), controlnet_prompt_embeds=torch.zeros(2 * b * f, 77, 768),
                     control_images=img)
    else:
        loop = SVDControlNetAdapterLoop(m, m, m, num_inference_steps=4, use_size_512=use_512, skip_conv_in=True)
        loop.prepare(latents=torch.zeros(b, f, 4, h, w), image_latents=torch.zeros(2 * b, f, 4, h, w),
                     image_embeddings=torch.zeros(2 * b, 1, 1024), added_time_ids=torch.zeros(2 * b, 3),
                     controlnet_prompt_embeds=torch.zeros(2 * b * f, 77, 768), control_images=img)


@pytest.mark.parametrize("loop_kind,use_512", list(DOMAIN))
def test_geometry_domain(loop_kind, use_512):
    inside, outside = DOMAIN[(loop_kind, use_512)]
    for h, w in inside:
        with _counted_ops(), pytest.raises(_Reached):
            _prepare(loop_kind, use_512, h, w)
    for h, w in outside:
        with _counted_ops() as calls:
            with pytest.raises(ValueError, match="height") as e:
                _prepare(loop_kind, use_512, h, w)
        assert calls[0] == 0, (loop_kind, use_512, h, w, calls[0])
        assert f"{h}x{w}" in str(e.value) and "width" in str(e.value), str(e.value)


def test_control_image_domain():
    """control images: multiples of 512 when use_size_512 pools them, else 8 x the latents; refused up front"""
    from ctrl_adapter_b200.loop_base import check_geometry
    check_geometry("SDXL loop", 128, 128, True, torch.zeros(2, 3, 512, 1536), multiple=4, adapter_up=2)
    with pytest.raises(ValueError, match="height 768 and width 1024"):
        check_geometry("SDXL loop", 128, 128, True, torch.zeros(2, 3, 768, 1024), multiple=4, adapter_up=2)
    check_geometry("SVD loop", 72, 128, False, torch.zeros(2, 3, 576, 1024), multiple=8, adapter_up=1)
    with pytest.raises(ValueError, match="expected height 576 and width 1024"):
        check_geometry("SVD loop", 72, 128, False, torch.zeros(2, 3, 1024, 576), multiple=8, adapter_up=1)
    with pytest.raises(ValueError, match="height 512 and width 512"):
        check_geometry("I2VGen-XL loop", 32, 64, False, [torch.zeros(2, 3, 256, 512), torch.zeros(2, 3, 512, 512)],
                       multiple=32, adapter_up=1)


def test_conv2d_stride2_odd_size_refused():
    """ops.conv2d refuses an odd height or width at stride 2 with ValueError (kept under python -O), before any call
    into the library"""
    from ctrl_adapter_b200 import ops
    x = torch.zeros(1, 6, 9, 8, dtype=BF16)
    w = torch.zeros(8, 72, dtype=BF16)
    saved = ops._req
    ops._req = lambda *a, **k: None  # the CPU tensors stand in for device tensors up to the geometry check
    try:
        with pytest.raises(ValueError, match="height 6, width 9"):
            ops.conv2d(x, w, None, stride=2)
    finally:
        ops._req = saved


# ---- emulated counterparts of the full-width GPU cases ---------------------------------------------------------------
@pytest.mark.slow
@pytest.mark.parametrize("hw", [(20, 36), (36, 20)])
def test_emulated_unet_sdxl(hw):
    from ctrl_adapter_b200.unet_sdxl import UNet2DConditionModel
    from oracle.unet_sdxl import UNet2DConditionModel as O
    o, p = hec._pair(O, UNet2DConditionModel, 6)
    hec._compare(o, p, cases.unet_sdxl_inputs(1, hw=hw))


@pytest.mark.slow
@pytest.mark.parametrize("hw", [(32, 64), (64, 32)])
def test_emulated_unet_i2vgen(hw):
    from ctrl_adapter_b200.unet_i2vgen import I2VGenXLUNet
    from oracle.unet_i2vgen import I2VGenXLUNet as O
    o, p = hec._pair(O, I2VGenXLUNet, 7)
    hec._compare(o, p, cases.unet_i2vgen_inputs(1, 2, hw=hw))


@pytest.mark.slow
@pytest.mark.parametrize("hw", [(24, 40), (40, 24)])
def test_emulated_unet_svd(hw):
    from ctrl_adapter_b200.unet_svd import UNetSpatioTemporalConditionModel
    from oracle.unet_svd import UNetSpatioTemporalConditionModel as O
    kw = dict(cases.UNET_SVD_KW, num_frames=2)
    o, p = hec._pair(lambda: O(**kw), lambda: UNetSpatioTemporalConditionModel(**kw), 8)
    hec._compare(o, p, cases.unet_svd_inputs(1, 2, hw=hw, chans=(320, 640, 1280, 1280), ctx=1024))
