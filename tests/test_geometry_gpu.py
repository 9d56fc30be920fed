"""pytest -m gpu: the modules and denoising loops against the oracle at non-square, non-power-of-two latent geometry.

At a square size a swap of height and width anywhere in the host code (a conv descriptor's row dims, the parity view of
a stride-2 conv, an up-sampler, a channels-last reshape, a pool's per-axis ratio, SDXL's size micro-conditioning) gives
exactly the right numbers, so the square module checks of module_checks.py cannot see it.  Every case here runs at a
geometry and at its transpose, with ragged TMA boxes and odd bottom levels (20 x 36 -> 5 x 9), and at the benchmark's
own SVD geometry (72 x 128 latents, use_size_512=False, skip_conv_in=True).

Comparison as in module_checks._compare: the truth is the oracle in fp32 (TF32 off) on the same bf16-quantised weights
and inputs; rel_fro and max bounds, and no worse than 1.5 x the eager bf16-autocast error + 2e-3 wherever eager runs.
`-s` prints one row per case: rel_fro, max_rel, the eager error and the bound.
"""
import pytest
import torch

from tests import module_checks as mc

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device is visible (there is no CPU fallback to test)")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.cuda.reset_peak_memory_stats()
    yield
    print(f"\npeak device memory of tests/test_geometry_gpu.py: {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


def _report(rec, tol_rel):
    bound = f"rel_fro <= {tol_rel:g}" + (f", <= 1.5 x eager + 2e-3 = {1.5 * rec['eager_rel_fro'] + 2e-3:.4f}"
                                         if rec["eager_rel_fro"] else "")
    print(f"\n[{'ok  ' if rec['ok'] else 'FAIL'}] {rec['check']}: rel_fro={rec['rel_fro']:.4f} "
          f"max_rel={rec['max_rel']:.4f} eager_rel_fro={rec['eager_rel_fro']:.4f} ({bound})")
    assert rec["ok"], rec
    torch.cuda.empty_cache()


def _loop(name, ours, ref, eager):
    """a few-step trajectory: judged like module_checks' `loops` group, no worse than 1.5 x the error the reference's
    own eager bf16-autocast trajectory accumulates against the fp32 truth"""
    torch.cuda.synchronize()
    _report(mc._compare(name, ours, ref, eager, tol_rel=6e-2, tol_max=0.2), 6e-2)


def _module(name, make_oracle, make_ours, seed, inputs, tol_rel=2e-2, tol_max=6e-2):
    call = lambda m, i: m(**i)  # noqa: E731
    sd, ref, eager, inp16 = mc._oracle_runs(make_oracle, seed, inputs, call)
    with torch.device("cuda"):
        ours_m = make_ours()
    ours_m.load_state_dict(sd)
    ours_m = ours_m.to(BF16).cuda().eval()
    ours = ours_m(**inp16)
    torch.cuda.synchronize()
    del ours_m
    _report(mc._compare(name, ours, ref, eager, tol_rel=tol_rel, tol_max=tol_max), tol_rel)


@pytest.mark.parametrize("hw", [(24, 40), (40, 24), (20, 36), (36, 20)])
def test_unet_sdxl(hw):
    from ctrl_adapter_b200.unet_sdxl import UNet2DConditionModel
    from oracle import cases
    from oracle.unet_sdxl import UNet2DConditionModel as OU
    _module(f"SDXL UNet n=1 latents {hw[0]}x{hw[1]}", OU, UNet2DConditionModel, 6,
            cases.unet_sdxl_inputs(1, hw=hw), tol_rel=3e-2, tol_max=8e-2)


@pytest.mark.parametrize("skip_conv_in", [False, True])
@pytest.mark.parametrize("hw", [(24, 40), (40, 24)])
def test_controlnet(hw, skip_conv_in):
    from ctrl_adapter_b200.controlnet import ControlNetModel
    from oracle import cases
    from oracle.controlnet import ControlNetModel as OC
    inputs = dict(cases.controlnet_inputs(2, hw=hw), skip_conv_in=skip_conv_in, conditioning_scale=0.75)
    _module(f"ControlNet n=2 latents {hw[0]}x{hw[1]} (cond {8 * hw[0]}x{8 * hw[1]}) skip_conv_in={int(skip_conv_in)} "
            f"scale 0.75", lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4, inputs)


@pytest.mark.parametrize("kind", ["sdxl", "video"])
@pytest.mark.parametrize("hw", [(24, 40), (40, 24)])
def test_adapter(hw, kind):
    from ctrl_adapter_b200.adapter import ControlNetAdapter
    from oracle import cases
    from oracle.adapter import ControlNetAdapter as OA
    if kind == "sdxl":
        kw, inputs, seed = cases.ADAPTER_SDXL_KW, cases.adapter_sdxl_inputs(2, hw=hw), 1
    else:
        kw, inputs, seed = dict(cases.ADAPTER_VIDEO_KW, num_frames=4), cases.adapter_video_inputs(1, 4, hw=hw), 2
    _module(f"adapter[{kind}] residual grid {hw[0]}x{hw[1]}", lambda: OA(**kw), lambda: ControlNetAdapter(**kw), seed,
            inputs)


@pytest.mark.parametrize("hw", [(32, 64), (64, 32), (64, 96), (96, 64)])
def test_unet_i2vgen(hw):
    """image-latent pool to 32 x 32 at ratios (1, 2), (2, 1), (2, 3), (3, 2)"""
    from ctrl_adapter_b200.unet_i2vgen import I2VGenXLUNet
    from oracle import cases
    from oracle.unet_i2vgen import I2VGenXLUNet as OU
    _module(f"I2VGen-XL UNet b=1 F=4 latents {hw[0]}x{hw[1]}", OU, I2VGenXLUNet, 7,
            cases.unet_i2vgen_inputs(1, 4, hw=hw), tol_rel=3e-2, tol_max=8e-2)


@pytest.mark.parametrize("hw,f", [((24, 40), 2), ((40, 24), 2), ((72, 128), 2)])
def test_unet_svd(hw, f):
    """released width (the reduced-width configuration has head dims the product refuses); 72 x 128 is the
    benchmark's spatial geometry"""
    from ctrl_adapter_b200.unet_svd import UNetSpatioTemporalConditionModel
    from oracle import cases
    from oracle.unet_svd import UNetSpatioTemporalConditionModel as OU
    kw = dict(cases.UNET_SVD_KW, num_frames=f)
    _module(f"SVD UNet b=1 F={f} latents {hw[0]}x{hw[1]}", lambda: OU(**kw),
            lambda: UNetSpatioTemporalConditionModel(**kw), 8,
            cases.unet_svd_inputs(1, f, hw=hw, chans=(320, 640, 1280, 1280), ctx=1024), tol_rel=3e-2, tol_max=8e-2)


@pytest.mark.parametrize("hw", [(24, 40), (40, 24)])
def test_svd_loop(hw):
    """the two iterations of a 2-step SVD schedule vs svd_step in the benchmark's loop configuration (use_size_512=False,
    skip_conv_in=True).  Two steps take sigma from 700 to 0.002, so the latents are the model's denoised prediction: at
    the start of a long schedule they are the initial noise to within bf16 rounding, which hides the model output"""
    from ctrl_adapter_b200.adapter import ControlNetAdapter
    from ctrl_adapter_b200.controlnet import ControlNetModel
    from ctrl_adapter_b200.pipeline_svd import SVDControlNetAdapterLoop
    from ctrl_adapter_b200.unet_svd import UNetSpatioTemporalConditionModel
    from oracle import cases
    from oracle.adapter import ControlNetAdapter as OA
    from oracle.controlnet import ControlNetModel as OC
    from oracle.pipeline_svd import EulerDiscreteSchedulerSVD, svd_step
    from oracle.unet_svd import UNetSpatioTemporalConditionModel as OU
    from oracle.weights import seeded_tensor
    b, f, nsteps = 1, 4, 2
    h, w = hw
    n = 2 * b * f
    kw = dict(cases.ADAPTER_VIDEO_KW, backbone_model_name="svd", num_frames=f)
    ukw = dict(cases.UNET_SVD_KW, num_frames=f)
    oad, ad = mc._build_pair(lambda: OA(**kw), lambda: ControlNetAdapter(**kw), 2)
    oun, un = mc._build_pair(lambda: OU(**ukw), lambda: UNetSpatioTemporalConditionModel(**ukw), 8)
    ocn, cn = mc._build_pair(lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4)
    images = mc._q(torch.sigmoid(seeded_tensor("g_img", (n, 3, 8 * h, 8 * w)))).cuda()
    il = seeded_tensor("g_il", (b, f, 4, h, w))
    inp = dict(latents=seeded_tensor("g_lat", (b, f, 4, h, w)), image_latents=torch.cat([torch.zeros_like(il), il]),
               image_embeddings=torch.cat([torch.zeros(b, 1, 1024), seeded_tensor("g_ie", (b, 1, 1024))]),
               added_time_ids=torch.tensor([[6.0, 127.0, 0.02]] * (2 * b)),
               controlnet_prompt_embeds=seeded_tensor("g_cpe", (n, 77, 768)))
    inp = {k: mc._q(v).cuda() for k, v in inp.items()}
    sch = EulerDiscreteSchedulerSVD()
    sch.set_timesteps(nsteps, device="cuda")
    flags = dict(use_size_512=False, skip_conv_in=True, skip_time_emb=False)
    loop = SVDControlNetAdapterLoop(cn, ad, un, num_inference_steps=nsteps, **flags)
    loop.prepare(control_images=images, **inp)
    args = (inp["image_latents"], inp["image_embeddings"], inp["added_time_ids"], inp["controlnet_prompt_embeds"], images)
    lat = (inp["latents"] * sch.init_noise_sigma).to(BF16)
    with torch.no_grad():
        for i in range(nsteps):
            lat = svd_step(ocn, oad, oun, sch, i, lat.float(), *args, **flags).to(BF16)
            loop.step(i)
        e = [m.to(BF16) for m in (ocn, oad, oun)]
        el = (inp["latents"] * sch.init_noise_sigma).to(BF16)
        a16 = [t.to(BF16) for t in args]
        with torch.autocast("cuda", dtype=BF16):
            for i in range(nsteps):
                el = svd_step(*e, sch, i, el, *a16, **flags).to(BF16)
    _loop(f"SVD loop {nsteps} of {nsteps} steps B=1 F={f} latents {h}x{w} use_size_512=0 skip_conv_in=1",
          loop.latents, lat.float(), el.float())


@pytest.mark.parametrize("hw", [(32, 64), (64, 32)])
def test_i2vgen_loop(hw):
    """the first iteration of a 2-step I2VGen-XL schedule (t 501 -> 1: the latents become the model's prediction) vs
    i2vgen_step, ControlNet at the latent resolution (use_size_512=False)"""
    from ctrl_adapter_b200.adapter import ControlNetAdapter
    from ctrl_adapter_b200.controlnet import ControlNetModel
    from ctrl_adapter_b200.pipeline_i2vgen import I2VGenXLControlNetAdapterLoop
    from ctrl_adapter_b200.unet_i2vgen import I2VGenXLUNet
    from oracle import cases
    from oracle.adapter import ControlNetAdapter as OA
    from oracle.controlnet import ControlNetModel as OC
    from oracle.pipeline_i2vgen import DDIMScheduler, i2vgen_step
    from oracle.unet_i2vgen import I2VGenXLUNet as OU
    from oracle.weights import seeded_tensor
    b, f, nsteps = 1, 4, 2
    h, w = hw
    n = 2 * b * f
    kw = dict(cases.ADAPTER_VIDEO_KW, num_frames=f)
    oad, ad = mc._build_pair(lambda: OA(**kw), lambda: ControlNetAdapter(**kw), 2)
    oun, un = mc._build_pair(OU, I2VGenXLUNet, 7)
    ocn, cn = mc._build_pair(lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4)
    images = mc._q(torch.sigmoid(seeded_tensor("g_vimg", (n, 3, 8 * h, 8 * w)))).cuda()
    inp = dict(latents=seeded_tensor("g_vlat", (b, 4, f, h, w)), prompt_embeds=seeded_tensor("g_vpe", (2 * b, 77, 1024)),
               image_latents=seeded_tensor("g_vil", (2 * b, 4, f, h, w)),
               image_embeddings=seeded_tensor("g_vie", (2 * b, 1, 1024)), fps=torch.tensor([16.0] * (2 * b)),
               controlnet_prompt_embeds=seeded_tensor("g_vcpe", (n, 77, 768)))
    inp = {k: mc._q(v).cuda() for k, v in inp.items()}
    sch = DDIMScheduler()
    sch.set_timesteps(nsteps, device="cuda")
    loop = I2VGenXLControlNetAdapterLoop(cn, ad, un, None, num_inference_steps=nsteps, guidance_scale=9.0,
                                         use_size_512=False)
    loop.prepare(control_images=images, **inp)
    args = (inp["prompt_embeds"], inp["image_latents"], inp["image_embeddings"], inp["fps"], inp["controlnet_prompt_embeds"])
    with torch.no_grad():
        lat = i2vgen_step(ocn, oad, oun, sch, 0, inp["latents"], *args, images, use_size_512=False)
        loop.step(0)
        e = [m.to(BF16) for m in (ocn, oad, oun)]
        a16 = [t.to(BF16) if t.is_floating_point() else t for t in args]
        with torch.autocast("cuda", dtype=BF16):
            el = i2vgen_step(*e, sch, 0, inp["latents"].to(BF16), *a16, images.to(BF16), use_size_512=False)
    _loop(f"I2VGen-XL loop 1 of {nsteps} steps B=1 F={f} latents {h}x{w} use_size_512=0", loop.latents_bcfhw(), lat,
          el.float())


@pytest.mark.parametrize("img_hw", [(512, 1024), (1024, 512)])
def test_sdxl_loop(img_hw):
    """the two iterations of a 2-step SDXL schedule through CUDA-graph replay.  The SDXL loop runs 128 x 128 latents only (its 2x adapter turns
    the ControlNet's pooled 64 x 64 into the UNet's 128 x 128), so the off-square geometry here is the control image's:
    pooled to 512 x 512 at ratios (1, 2) and (2, 1)"""
    from ctrl_adapter_b200.adapter import ControlNetAdapter
    from ctrl_adapter_b200.controlnet import ControlNetModel
    from ctrl_adapter_b200.pipeline_sdxl import SDXLControlNetAdapterLoop
    from ctrl_adapter_b200.pipelines import sdxl_add_time_ids
    from ctrl_adapter_b200.unet_sdxl import UNet2DConditionModel
    from oracle import cases
    from oracle.adapter import ControlNetAdapter as OA
    from oracle.controlnet import ControlNetModel as OC
    from oracle.pipeline_sdxl import EulerDiscreteScheduler, sdxl_step
    from oracle.unet_sdxl import UNet2DConditionModel as OU
    from oracle.weights import seeded_tensor
    b, nsteps = 1, 2
    ocn, cn = mc._build_pair(lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4)
    oad, ad = mc._build_pair(lambda: OA(**cases.ADAPTER_SDXL_KW), lambda: ControlNetAdapter(**cases.ADAPTER_SDXL_KW), 1)
    oun, un = mc._build_pair(OU, UNet2DConditionModel, 6)
    inp = dict(latents=seeded_tensor("g_slat", (b, 4, 128, 128)), prompt_embeds=seeded_tensor("g_spe", (2 * b, 77, 2048)),
               add_text_embeds=seeded_tensor("g_ste", (2 * b, 1280)),
               add_time_ids=sdxl_add_time_ids(b, 1024, 1024, original_size=img_hw),
               controlnet_prompt_embeds=seeded_tensor("g_scpe", (2 * b, 77, 768)),
               control_images=torch.sigmoid(seeded_tensor("g_simg", (2 * b, 3, *img_hw))))
    inp = {k: mc._q(v).cuda() for k, v in inp.items()}
    sch = EulerDiscreteScheduler()
    sch.set_timesteps(nsteps, device="cuda")
    loop = SDXLControlNetAdapterLoop(cn, ad, un, num_inference_steps=nsteps, guidance_scale=5.0, use_size_512=True)
    loop.prepare(**inp)
    lat = mc._q(inp["latents"] * sch.init_noise_sigma)
    args = (inp["prompt_embeds"], inp["add_text_embeds"], inp["add_time_ids"], inp["controlnet_prompt_embeds"],
            inp["control_images"])
    with torch.no_grad():
        for i in range(nsteps):
            lat = sdxl_step(ocn, oad, oun, sch, i, lat, *args, cond_scale=1.0, use_size_512=True)
            loop.step_graph(i)
        e = [m.to(BF16) for m in (ocn, oad, oun)]
        el = mc._q(inp["latents"] * sch.init_noise_sigma).to(BF16)
        a16 = [t.to(BF16) for t in args]
        with torch.autocast("cuda", dtype=BF16):
            for i in range(nsteps):
                el = sdxl_step(*e, sch, i, el, *a16, cond_scale=1.0, use_size_512=True).to(BF16)
    _loop(f"SDXL loop {nsteps} of {nsteps} steps graph replay, latents 128x128, control images {img_hw[0]}x{img_hw[1]}",
          loop.latents, lat, el.float())
