"""CPU tests of the host modules' composition logic: `ctrl_adapter_b200.ops` is replaced by the plain-PyTorch emulation of
tests/ops_emulator.py (same entry points, packed-weight formats and bf16 rounding points as the CUDA kernels), and the
modules are compared with the oracle on identical name-seeded, bf16-quantised weights and inputs.

What this pins without a GPU: block wiring, skip / residual order (zip truncation), weight packing (conv taps, fused QKV,
GEGLU tile interleave, padded heads), per-image / per-clip broadcast rows, the single-token cross-attention collapse and
the reference quirks that live in host code (e.g. the (pixel, clip) ordering of `time_context`).  Kernel numerics are a
separate matter (tests/kernel_checks.py on the H100).  Tolerance: the emulation rounds to bf16 where the kernels do, the
oracle runs in fp32 -> relative Frobenius error at the bf16 level (<= 3e-2), the same bar as the GPU module checks.
"""
import pytest
import torch

from oracle import cases
from oracle.weights import seeded_init_
from tests import ops_emulator as emu

BF16 = torch.bfloat16
torch.set_grad_enabled(False)


def _q(t):
    return t.to(BF16).float()


def _map(x, fn):
    if torch.is_tensor(x):
        return fn(x) if x.is_floating_point() else x
    if isinstance(x, (list, tuple)):
        return type(x)(_map(v, fn) for v in x)
    if isinstance(x, dict):
        return {k: _map(v, fn) for k, v in x.items()}
    return x


def _flat(x):
    if torch.is_tensor(x):
        return [x]
    if isinstance(x, (list, tuple)):
        return [t for v in x for t in _flat(v)]
    return []


def _pair(make_oracle, make_ours, seed):
    o = seeded_init_(make_oracle(), seed).eval()
    sd = o.state_dict()
    with torch.device("meta"):
        p = make_ours()
    p = p.to_empty(device="cpu")
    p.load_state_dict(sd)
    p = p.to(BF16).eval()
    for prm in o.parameters():
        prm.data = _q(prm.data)
    return o, p


def _compare(o, p, inputs, tol=3e-2):
    ref = _flat(o(**_map(inputs, _q)))
    with emu.patched_ops():
        ours = _flat(p(**_map(inputs, lambda t: t.to(BF16))))
    assert len(ours) == len(ref)
    worst = 0.0
    for a, b in zip(ours, ref):
        assert tuple(a.shape) == tuple(b.shape)
        if float(b.abs().max()) == 0.0:
            assert float(a.float().abs().max()) == 0.0
            continue
        worst = max(worst, float((a.float() - b).norm() / b.norm()))
    assert worst <= tol, f"relative Frobenius error {worst:.4f}"
    return worst


def test_emulated_adapter_sdxl():
    from ctrl_adapter_b200.adapter import ControlNetAdapter
    from oracle.adapter import ControlNetAdapter as O
    o, p = _pair(lambda: O(**cases.ADAPTER_SDXL_KW), lambda: ControlNetAdapter(**cases.ADAPTER_SDXL_KW), 1)
    _compare(o, p, cases.adapter_sdxl_inputs(2, 8))


def test_emulated_adapter_video():
    from ctrl_adapter_b200.adapter import ControlNetAdapter
    from oracle.adapter import ControlNetAdapter as O
    o, p = _pair(lambda: O(**cases.ADAPTER_VIDEO_KW), lambda: ControlNetAdapter(**cases.ADAPTER_VIDEO_KW), 2)
    _compare(o, p, cases.adapter_video_inputs(1, 4, 8))


def test_emulated_controlnet():
    from ctrl_adapter_b200.controlnet import ControlNetModel
    from oracle.controlnet import ControlNetModel as O
    o, p = _pair(lambda: O(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4)
    _compare(o, p, dict(cases.controlnet_inputs(2, 8), conditioning_scale=0.75))


def test_emulated_controlnet_folded_small_convs(monkeypatch):
    """The 8 / 16 / 32-channel stride-1 convolutions of the conditioning embedding run with adjacent pixels folded into
    the channel axis (block-banded weights); the ControlNet output must not change."""
    from ctrl_adapter_b200.controlnet import ControlNetModel
    from ctrl_adapter_b200.layers import Conv2d
    from oracle.controlnet import ControlNetModel as O
    o, p = _pair(lambda: O(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4)
    inputs = dict(cases.controlnet_inputs(2, 8), conditioning_scale=1.0)
    calls = []
    orig = Conv2d.forward_folded

    def spy(self, x, **kw):
        calls.append((self.cin, self.cout, self.fold_factor(x)))
        return orig(self, x, **kw)
    monkeypatch.setattr(Conv2d, "forward_folded", spy)
    _compare(o, p, inputs)
    assert (3, 16, 8) in calls and (16, 16, 4) in calls and (32, 32, 2) in calls, calls
    # and layer-level: folded == unfolded to bf16 rounding on a ragged-free random case
    torch.manual_seed(0)
    c = Conv2d(16, 16, 3).to(BF16)
    x = torch.randn(2, 12, 16, 16).to(BF16)
    with emu.patched_ops():
        a = c(x, act=1).float()
        b = c.forward_folded(x, act=1).float()
    assert float((a - b).abs().max()) <= 2.0 ** -7 * float(a.abs().max())


def test_emulated_vae_decoder():
    """AutoencoderKL.decode (the VAE after the loop, sdxl pipeline :1414) through the emulated op layer vs the restated
    diffusers decoder: block wiring, the 512-wide single-head attention as GEMM -> softmax -> GEMM, 4 -> 8 channel
    padding of the latent / post_quant_conv / conv_out, state-dict keys (encoder.* keys of a checkpoint are skipped)."""
    from ctrl_adapter_b200.vae import AutoencoderKL, decode_latents, postprocess, tensor2vid
    from oracle.vae import AutoencoderKL as OV
    from oracle.weights import seeded_tensor
    kw = dict(block_out_channels=(32, 64, 64, 64), layers_per_block=1)
    o = seeded_init_(OV(**kw), 11).eval()
    m = AutoencoderKL(**kw)
    sd = dict(o.state_dict())
    sd["encoder.conv_in.weight"] = torch.zeros(1)  # a published checkpoint also carries the encoder half
    m.load_state_dict(sd)
    for p_ in o.parameters():
        p_.data = _q(p_.data)
    m = m.to(BF16).eval()
    z = _q(seeded_tensor("vae_z", (2, 4, 8, 8)))
    with torch.no_grad(), emu.patched_ops():
        ref = o.decode(z)[0]
        out = m.decode(z).sample
        vid = decode_latents(m, z.reshape(1, 2, 4, 8, 8).permute(0, 2, 1, 3, 4) * m.config.scaling_factor)
    assert out.shape == ref.shape == (2, 3, 64, 64)
    rel = float((out.float() - ref).norm() / ref.norm())
    assert rel <= 3e-2, rel
    assert vid.shape == (1, 3, 2, 64, 64) and float((vid[0].permute(1, 0, 2, 3) - out.float()).abs().max()) == 0.0
    assert postprocess(out, "np").shape == (2, 64, 64, 3) and len(postprocess(out, "pil")) == 2
    assert tensor2vid(vid, "pt").shape == (1, 2, 3, 64, 64)


def test_emulated_vae_temporal_decoder():
    """AutoencoderKLTemporalDecoder.decode (the SVD VAE, svd pipeline :265-292) through the emulated op layer vs the
    restated diffusers decoder: SpatioTemporalResBlocks with the switched learned alpha (mix factors moved off 0 so the
    switch matters), temporal eps 1e-5 vs spatial 1e-6, time_conv_out over the frames of the chunk, chunked
    decode_latents (a chunk is one temporal unit, also across clips)."""
    from ctrl_adapter_b200.vae import AutoencoderKLTemporalDecoder, svd_decode_latents
    from oracle.vae import AutoencoderKLTemporalDecoder as OV
    from oracle.weights import seeded_tensor
    kw = dict(block_out_channels=(32, 64, 64), layers_per_block=1)
    o = seeded_init_(OV(**kw), 12).eval()
    with torch.no_grad():
        for i, (n_, p_) in enumerate(o.named_parameters()):
            if n_.endswith("mix_factor"):
                p_.fill_(0.8 - 0.35 * i % 1.7)
    m = AutoencoderKLTemporalDecoder(**kw)
    sd = dict(o.state_dict())
    sd["encoder.conv_in.weight"] = torch.zeros(1)
    sd["quant_conv.weight"] = torch.zeros(1)
    m.load_state_dict(sd)
    for p_ in o.parameters():
        p_.data = _q(p_.data)
    m = m.to(BF16).eval()
    z = _q(seeded_tensor("vae_t_z", (6, 4, 8, 8)))
    with torch.no_grad(), emu.patched_ops():
        ref = o.decode(z, num_frames=3)[0]
        out = m.decode(z, num_frames=3).sample
        # two clips of 3 frames decoded 4 frames at a time: chunks [0:4] and [4:6] are the temporal units
        vid = svd_decode_latents(m, z.reshape(2, 3, 4, 8, 8) * m.config.scaling_factor, 3, decode_chunk_size=4)
        ref_chunks = torch.cat([o.decode(z[:4], num_frames=4)[0], o.decode(z[4:], num_frames=2)[0]])
    assert out.shape == ref.shape == (6, 3, 32, 32)
    rel = float((out.float() - ref).norm() / ref.norm())
    assert rel <= 3e-2, rel
    # the temporal path is live: decoding the same frames as single-frame units gives a different answer
    with torch.no_grad(), emu.patched_ops():
        single = m.decode(z, num_frames=1).sample
    assert float((single.float() - out.float()).abs().max()) > 1e-2
    assert vid.shape == (2, 3, 3, 32, 32) and vid.dtype == torch.float32
    v = vid.permute(0, 2, 1, 3, 4).reshape(6, 3, 32, 32)
    assert float((v - ref_chunks).norm() / ref_chunks.norm()) <= 3e-2
    with pytest.raises(ValueError):
        m.decode(z[:5], num_frames=3)
    # the pipeline class decodes through the same function and post-processes like the reference (:787-792)
    from ctrl_adapter_b200.pipelines import SVDControlNetAdapterPipeline
    from ctrl_adapter_b200.vae import tensor2vid
    pipe = SVDControlNetAdapterPipeline(vae=m, image_encoder=None, unet=None, scheduler=None, feature_extractor=None,
                                        adapter=None, helper=None, controlnet=None)
    with torch.no_grad(), emu.patched_ops():
        v2 = pipe.decode_latents(z.reshape(2, 3, 4, 8, 8) * m.config.scaling_factor, 3, 4)
    assert float((v2 - vid).abs().max()) == 0.0
    assert tensor2vid(v2, "np").shape == (2, 3, 32, 32, 3) and len(tensor2vid(v2, "pil")[0]) == 3


@pytest.mark.slow
def test_emulated_unet_svd():
    """Two clips with DIFFERENT image tokens + 5-D residuals with surplus entries: covers the per-clip broadcast rows and
    the (pixel, clip) `time_context` ordering quirk of the temporal blocks."""
    from ctrl_adapter_b200.unet_svd import UNetSpatioTemporalConditionModel
    from oracle.unet_svd import UNetSpatioTemporalConditionModel as O
    o, p = _pair(lambda: O(**cases.UNET_SVD_KW), lambda: UNetSpatioTemporalConditionModel(**cases.UNET_SVD_KW), 8)
    _compare(o, p, cases.unet_svd_inputs(2, 3, 16, with_residuals=True, chans=(320, 640, 1280, 1280), ctx=1024))
    _compare(o, p, cases.unet_svd_inputs(1, 2, 16, with_residuals=False, chans=(320, 640, 1280, 1280), ctx=1024))
    # non-square latents (the 576 x 1024 configuration is 72 x 128): 16 x 24 here
    inp = cases.unet_svd_inputs(1, 2, 16, with_residuals=True, chans=(320, 640, 1280, 1280), ctx=1024)
    inp["sample"] = torch.cat([inp["sample"], inp["sample"][..., :8]], dim=-1)
    inp["down_block_additional_residuals"] = [torch.cat([t, t[..., : t.shape[-1] // 2]], dim=-1)
                                              for t in inp["down_block_additional_residuals"]]
    m = inp["mid_block_additional_residual"]
    inp["mid_block_additional_residual"] = torch.cat([m, m[..., : m.shape[-1] // 2]], dim=-1)
    _compare(o, p, inp)


@pytest.mark.slow
def test_emulated_unet_i2vgen():
    from ctrl_adapter_b200.unet_i2vgen import I2VGenXLUNet
    from oracle.unet_i2vgen import I2VGenXLUNet as O
    o, p = _pair(lambda: O(), lambda: I2VGenXLUNet(), 7)
    _compare(o, p, cases.unet_i2vgen_inputs(2, 2, 16, with_residuals=True))


@pytest.mark.slow
def test_emulated_unet_sdxl():
    from ctrl_adapter_b200.unet_sdxl import UNet2DConditionModel
    from oracle.unet_sdxl import UNet2DConditionModel as O
    o, p = _pair(lambda: O(), lambda: UNet2DConditionModel(), 6)
    _compare(o, p, cases.unet_sdxl_inputs(2, 16, with_residuals=True))


@pytest.mark.slow
def test_emulated_i2vgen_loop_multi_controlnet_router():
    """One I2VGen-XL iteration with TWO ControlNets run through MultiControlNetModel, the router's masked softmax and
    the weighted merge (incl. the w[e // F] indexing quirk) vs the restated reference loop."""
    from ctrl_adapter_b200.adapter import ControlNetAdapter, ControlNetRouter
    from ctrl_adapter_b200.controlnet import ControlNetModel, MultiControlNetModel
    from ctrl_adapter_b200.pipeline_i2vgen import I2VGenXLControlNetAdapterLoop
    from ctrl_adapter_b200.unet_i2vgen import I2VGenXLUNet
    from oracle.adapter import ControlNetAdapter as OA, ControlNetRouter as OR
    from oracle.controlnet import ControlNetModel as OC, MultiControlNetModel as OM
    from oracle.pipeline_i2vgen import DDIMScheduler, i2vgen_step
    from oracle.unet_i2vgen import I2VGenXLUNet as OU
    from oracle.weights import seeded_tensor
    b, f, r = 1, 4, 32  # the 32x32 image-latent pool needs latents that are multiples of 32
    n = 2 * b * f
    kw = dict(cases.ADAPTER_VIDEO_KW, num_frames=f)
    oad, ad = _pair(lambda: OA(**kw), lambda: ControlNetAdapter(**kw), 2)
    oun, un = _pair(lambda: OU(), lambda: I2VGenXLUNet(), 7)
    nets = [_pair(lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 40 + k) for k in range(2)]
    ocn, cn = OM([p_[0] for p_ in nets]), MultiControlNetModel([p_[1] for p_ in nets])
    rk = dict(cases.ROUTER_KW, num_experts=3)
    orouter = seeded_init_(OR(**rk), 3).eval()
    router = ControlNetRouter(**rk)
    router.load_state_dict(orouter.state_dict())
    masks = [1, 1, 0]
    images = [_q(torch.sigmoid(seeded_tensor(f"v_img{k}", (n, 3, 8 * r, 8 * r)))) for k in range(2)]
    inp = dict(latents=seeded_tensor("v_lat", (b, 4, f, r, r)), prompt_embeds=seeded_tensor("v_pe", (2 * b, 77, 1024)),
               image_latents=seeded_tensor("v_il", (2 * b, 4, f, r, r)),
               image_embeddings=seeded_tensor("v_ie", (2 * b, 1, 1024)), fps=torch.tensor([16.0] * (2 * b)),
               controlnet_prompt_embeds=seeded_tensor("v_cpe", (n, 77, 768)))
    inp = {k: _q(v) for k, v in inp.items()}
    sch = DDIMScheduler()
    sch.set_timesteps(50)
    with emu.patched_ops():
        loop = I2VGenXLControlNetAdapterLoop(cn, ad, un, router, num_inference_steps=50, guidance_scale=9.0, use_size_512=False,
                                             inference_expert_masks=masks)
        loop.prepare(control_images=images, **inp)
        lat = i2vgen_step(ocn, oad, oun, sch, 0, inp["latents"], inp["prompt_embeds"], inp["image_latents"],
                          inp["image_embeddings"], inp["fps"], inp["controlnet_prompt_embeds"], images, router=orouter,
                          masks=masks, use_size_512=False)
        loop.step(0)
    ours = loop.latents_bcfhw().float()
    rel = float((ours - lat).norm() / lat.norm())
    assert rel <= 2e-2, rel


@pytest.mark.slow
@pytest.mark.parametrize("sparse", [None, [0, 2]])
def test_emulated_i2vgen_loop(sparse):
    """Two whole I2VGen-XL iterations (ControlNet -> adapter -> UNet with injection -> CFG -> DDIM) through the emulated
    op layer vs the restated reference loop, dense and with sparse key frames (gather -> adapter on 2 frames -> scatter
    into zero residuals, i2vgen_xl pipeline :1024-1033, :1053-1073)."""
    from ctrl_adapter_b200.adapter import ControlNetAdapter
    from ctrl_adapter_b200.controlnet import ControlNetModel
    from ctrl_adapter_b200.pipeline_i2vgen import I2VGenXLControlNetAdapterLoop
    from ctrl_adapter_b200.unet_i2vgen import I2VGenXLUNet
    from oracle.adapter import ControlNetAdapter as OA
    from oracle.controlnet import ControlNetModel as OC
    from oracle.pipeline_i2vgen import DDIMScheduler, i2vgen_step
    from oracle.unet_i2vgen import I2VGenXLUNet as OU
    from oracle.weights import seeded_tensor
    b, f, r = 1, 4, 32  # the 32x32 image-latent pool needs latents that are multiples of 32
    n = 2 * b * f
    kw = dict(cases.ADAPTER_VIDEO_KW, num_frames=f)
    oad, ad = _pair(lambda: OA(**kw), lambda: ControlNetAdapter(**kw), 2)
    oun, un = _pair(lambda: OU(), lambda: I2VGenXLUNet(), 7)
    ocn, cn = _pair(lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4)
    images = _q(torch.sigmoid(seeded_tensor("v_img", (n, 3, 8 * r, 8 * r))))
    inp = dict(latents=seeded_tensor("v_lat", (b, 4, f, r, r)), prompt_embeds=seeded_tensor("v_pe", (2 * b, 77, 1024)),
               image_latents=seeded_tensor("v_il", (2 * b, 4, f, r, r)),
               image_embeddings=seeded_tensor("v_ie", (2 * b, 1, 1024)), fps=torch.tensor([16.0] * (2 * b)),
               controlnet_prompt_embeds=seeded_tensor("v_cpe", (n, 77, 768)))
    inp = {k: _q(v) for k, v in inp.items()}
    sch = DDIMScheduler()
    sch.set_timesteps(50)
    lat = inp["latents"]
    with emu.patched_ops():
        loop = I2VGenXLControlNetAdapterLoop(cn, ad, un, None, num_inference_steps=50, guidance_scale=9.0, use_size_512=False,
                                             sparse_frames=sparse)
        loop.prepare(control_images=images, **inp)
        for i in range(2):
            lat = i2vgen_step(ocn, oad, oun, sch, i, lat, inp["prompt_embeds"], inp["image_latents"],
                              inp["image_embeddings"], inp["fps"], inp["controlnet_prompt_embeds"], images,
                              sparse_frames=sparse, use_size_512=False)
            loop.step(i)
    ours = loop.latents_bcfhw().float()
    rel = float((ours - lat).norm() / lat.norm())
    assert rel <= 2e-2, rel


@pytest.mark.slow
@pytest.mark.parametrize("sparse", [None, [0, 2]])
def test_emulated_svd_loop(sparse):
    """Two whole SVD iterations (ControlNet -> adapter -> SVD UNet with 5-D-equivalent injection -> per-frame CFG ->
    Euler v-prediction) through the emulated op layer vs the restated reference loop (oracle/pipeline_svd.py)."""
    from ctrl_adapter_b200.adapter import ControlNetAdapter
    from ctrl_adapter_b200.controlnet import ControlNetModel
    from ctrl_adapter_b200.pipeline_svd import SVDControlNetAdapterLoop
    from ctrl_adapter_b200.unet_svd import UNetSpatioTemporalConditionModel
    from oracle.adapter import ControlNetAdapter as OA
    from oracle.controlnet import ControlNetModel as OC
    from oracle.pipeline_svd import EulerDiscreteSchedulerSVD, svd_step
    from oracle.unet_svd import UNetSpatioTemporalConditionModel as OU
    from oracle.weights import seeded_tensor
    b, f, r, steps = 1, 3, 16, 25
    n = 2 * b * f
    kw = dict(cases.ADAPTER_VIDEO_KW, backbone_model_name="svd", num_frames=f)
    oad, ad = _pair(lambda: OA(**kw), lambda: ControlNetAdapter(**kw), 2)
    oun, un = _pair(lambda: OU(**cases.UNET_SVD_KW), lambda: UNetSpatioTemporalConditionModel(**cases.UNET_SVD_KW), 8)
    ocn, cn = _pair(lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4)
    images = _q(torch.sigmoid(seeded_tensor("s_img", (n, 3, 8 * r, 8 * r))))
    il = seeded_tensor("s_il", (b, f, 4, r, r))
    inp = dict(latents=seeded_tensor("s_lat", (b, f, 4, r, r)),
               image_latents=torch.cat([torch.zeros_like(il), il]),
               image_embeddings=torch.cat([torch.zeros(b, 1, 1024), seeded_tensor("s_ie", (b, 1, 1024))]),
               added_time_ids=torch.tensor([[6.0, 127.0, 0.02]] * (2 * b)),
               controlnet_prompt_embeds=seeded_tensor("s_cpe", (n, 77, 768)))
    inp = {k: _q(v) for k, v in inp.items()}
    sch = EulerDiscreteSchedulerSVD()
    sch.set_timesteps(steps)
    lat = (inp["latents"] * sch.init_noise_sigma).to(BF16)  # prepare_latents: the latent dtype is the model dtype
    flags = dict(use_size_512=False, skip_conv_in=True, skip_time_emb=False)
    with emu.patched_ops():
        loop = SVDControlNetAdapterLoop(cn, ad, un, num_inference_steps=steps, sparse_frames=sparse, **flags)
        loop.prepare(control_images=images, **inp)
        assert float((loop.latents - lat.float()).abs().max()) == 0.0
        for i in range(2):
            # oracle in fp32 modules but bf16 latents / model outputs, as the reference runs them under autocast
            lat = svd_step(ocn, oad, oun, sch, i, lat.float(), inp["image_latents"], inp["image_embeddings"],
                           inp["added_time_ids"], inp["controlnet_prompt_embeds"], images, sparse_frames=sparse,
                           **flags).to(BF16)
            loop.step(i)
    ours = loop.latents
    rel = float((ours - lat.float()).norm() / lat.float().norm())
    assert rel <= 2e-2, rel
