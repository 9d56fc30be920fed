"""GPU parity checks at module level: the H100 modules (ctrl_adapter_b200.*) against the oracle on identical
name-seeded weights and inputs.

Comparison point (SURVEY.md "hard parts"): the ground truth is the oracle in fp32 (TF32 off) evaluated with the SAME
bf16-quantised weights and inputs, so only activation rounding differs.  bf16 activations cannot meet rtol 1e-3
element-wise through a deep chain (bf16 eps = 3.9e-3), so the stated bound per module is
    rel_fro = ||out - ref|| / ||ref||  <=  tol_rel          (default 2e-2)
    max|out - ref| / max|ref|          <=  tol_max          (default 6e-2)
and, where the oracle is also run as the reference's own eager bf16-autocast path on the GPU, our error against the
fp32 truth must not exceed 1.5x the eager path's error (+ small slack) -- i.e. we are as close to the truth as the
reference implementation is.

Stand-alone report:  python -m tests.module_checks [--group adapter|controlnet|unet|step] [--json out.json]
"""
from __future__ import annotations

import json
import sys
import time

import torch

BF16 = torch.bfloat16
RESULTS = []


def _q(t):
    """quantise a float tensor to bf16-representable values (kept in fp32)"""
    return t.to(BF16).float() if torch.is_tensor(t) and t.is_floating_point() else t


def _map(obj, fn):
    if torch.is_tensor(obj):
        return fn(obj)
    if isinstance(obj, dict):
        return {k: _map(v, fn) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_map(v, fn) for v in obj)
    return obj


def _flat(out):
    ts = []

    def rec(o):
        if torch.is_tensor(o):
            ts.append(o)
        elif isinstance(o, (list, tuple)):
            for v in o:
                rec(v)
    rec(out)
    return ts


def _compare(name, ours, ref, eager=None, tol_rel=2e-2, tol_max=6e-2, extra=None):
    ours_f, ref_f = _flat(ours), _flat(ref)
    assert len(ours_f) == len(ref_f), f"{name}: {len(ours_f)} vs {len(ref_f)} tensors"
    eager_f = _flat(eager) if eager is not None else [None] * len(ref_f)
    worst = {"check": name, "rel_fro": 0.0, "max_rel": 0.0, "eager_rel_fro": 0.0, "ok": True, "n_tensors": len(ref_f)}
    for i, (o, r, e) in enumerate(zip(ours_f, ref_f, eager_f)):
        assert tuple(o.shape) == tuple(r.shape), f"{name}[{i}]: shape {tuple(o.shape)} vs {tuple(r.shape)}"
        o, r = o.float().cpu(), r.float().cpu()
        if float(r.abs().max()) == 0.0:
            ok = float(o.abs().max()) == 0.0
            worst["ok"] &= ok
            continue
        rel = float((o - r).norm() / r.norm())
        mx = float((o - r).abs().max() / r.abs().max())
        ok = rel <= tol_rel and mx <= tol_max and bool(torch.isfinite(o).all())
        if e is not None:
            erel = float((e.float().cpu() - r).norm() / r.norm())
            worst["eager_rel_fro"] = max(worst["eager_rel_fro"], erel)
            ok = ok and rel <= 1.5 * erel + 2e-3
        worst["rel_fro"] = max(worst["rel_fro"], rel)
        worst["max_rel"] = max(worst["max_rel"], mx)
        if not ok:
            worst["ok"] = False
            worst.setdefault("bad", []).append(i)
    if extra:
        worst.update(extra)
    RESULTS.append(worst)
    return worst


def _oracle_runs(make_oracle, seed, inputs, call):
    """fp32 truth (bf16-quantised weights/inputs) and eager bf16-autocast runs of the oracle on the GPU."""
    from oracle.weights import seeded_init_
    with torch.device("cuda"):
        m = make_oracle()
    m = seeded_init_(m.cuda(), seed).eval()  # .cuda(): legacy torch.Tensor([..]) parameters ignore the device context
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    for p in m.parameters():
        p.data = _q(p.data)
    inp32 = _map(inputs, lambda t: _q(t).cuda() if t.is_floating_point() else t.cuda())
    with torch.no_grad():
        ref = call(m, inp32)
        m16 = m.to(BF16)
        inp16 = _map(inputs, lambda t: t.to(BF16).cuda() if t.is_floating_point() else t.cuda())
        with torch.autocast("cuda", dtype=BF16):
            eager = call(m16, inp16)
    ref = _map(ref, lambda t: t.float().cpu())
    eager = _map(eager, lambda t: t.float().cpu())
    del m, m16
    torch.cuda.empty_cache()
    return sd, ref, eager, inp16


def check_adapter(kind="sdxl", n=2, r=8, frames=4):
    from ctrl_adapter_b200.adapter import ControlNetAdapter
    from oracle import cases
    from oracle.adapter import ControlNetAdapter as OAdapter
    if kind == "sdxl":
        kw, inputs, seed = cases.ADAPTER_SDXL_KW, cases.adapter_sdxl_inputs(n, r), 1
    else:
        kw, inputs, seed = dict(cases.ADAPTER_VIDEO_KW, num_frames=frames), cases.adapter_video_inputs(n, frames, r), 2
    call = lambda m, i: m(**i)  # noqa: E731
    sd, ref, eager, inp16 = _oracle_runs(lambda: OAdapter(**kw), seed, inputs, call)
    with torch.device("cuda"):
        ours_m = ControlNetAdapter(**kw)
    ours_m.load_state_dict(sd)
    ours_m = ours_m.to(BF16).cuda().eval()
    ours = ours_m(**inp16)
    torch.cuda.synchronize()
    # unselected blocks must come back as zero tensors of the input's shape, mid None for SDXL
    return _compare(f"ControlNetAdapter[{kind}] n={n} r={r}", ours, ref, eager)


def check_controlnet(n=2, r=8, skip_conv_in=False, scale=1.0):
    from ctrl_adapter_b200.controlnet import ControlNetModel
    from oracle import cases
    from oracle.controlnet import ControlNetModel as OCN
    inputs = dict(cases.controlnet_inputs(n, r), skip_conv_in=skip_conv_in, conditioning_scale=scale)
    call = lambda m, i: m(**i)  # noqa: E731
    sd, ref, eager, inp16 = _oracle_runs(lambda: OCN(**cases.CONTROLNET_KW), 4, inputs, call)
    with torch.device("cuda"):
        ours_m = ControlNetModel(**cases.CONTROLNET_KW)
    ours_m.load_state_dict(sd)
    ours_m = ours_m.to(BF16).cuda().eval()
    ours = ours_m(**inp16)
    torch.cuda.synchronize()
    return _compare(f"ControlNetModel n={n} r={r} skip_conv_in={int(skip_conv_in)} scale={scale}", ours, ref, eager)


def check_unet_sdxl(n=2, r=16, with_residuals=True):
    from ctrl_adapter_b200.unet_sdxl import UNet2DConditionModel
    from oracle import cases
    from oracle.unet_sdxl import UNet2DConditionModel as OUNet
    inputs = cases.unet_sdxl_inputs(n, r, with_residuals=with_residuals)
    call = lambda m, i: m(**i)  # noqa: E731
    sd, ref, eager, inp16 = _oracle_runs(lambda: OUNet(), 6, inputs, call)
    with torch.device("cuda"):
        ours_m = UNet2DConditionModel()
    ours_m.load_state_dict(sd)
    ours_m = ours_m.to(BF16).cuda().eval()
    ours = ours_m(**inp16)
    torch.cuda.synchronize()
    return _compare(f"UNet2DConditionModel[sdxl] n={n} r={r} residuals={int(with_residuals)}", ours, ref, eager,
                    tol_rel=3e-2, tol_max=8e-2)


def check_router():
    from ctrl_adapter_b200.adapter import ControlNetRouter
    from oracle import cases
    from oracle.adapter import ControlNetRouter as ORouter
    from oracle.weights import seeded_init_
    o = seeded_init_(ORouter(**cases.ROUTER_KW), 3)
    m = ControlNetRouter(**cases.ROUTER_KW)
    m.load_state_dict(o.state_dict())
    m = m.cuda()
    with torch.no_grad():
        ref = o(sparse_mask=cases.ROUTER_MASK)
        ours = m(sparse_mask=cases.ROUTER_MASK)
    torch.cuda.synchronize()
    return _compare("ControlNetRouter masked softmax", ours, ref, None, tol_rel=1e-5, tol_max=1e-5)


def check_unet_i2vgen(b=1, f=4, r=32, with_residuals=True):
    from ctrl_adapter_b200.unet_i2vgen import I2VGenXLUNet
    from oracle import cases
    from oracle.unet_i2vgen import I2VGenXLUNet as OUNet
    inputs = cases.unet_i2vgen_inputs(b, f, r, with_residuals=with_residuals)
    call = lambda m, i: m(**i)  # noqa: E731
    sd, ref, eager, inp16 = _oracle_runs(lambda: OUNet(), 7, inputs, call)
    with torch.device("cuda"):
        ours_m = I2VGenXLUNet()
    ours_m.load_state_dict(sd)
    ours_m = ours_m.to(BF16).cuda().eval()
    ours = ours_m(**inp16)
    torch.cuda.synchronize()
    return _compare(f"I2VGenXLUNet b={b} f={f} r={r} residuals={int(with_residuals)}", ours, ref, eager,
                    tol_rel=3e-2, tol_max=8e-2)


def check_unet_svd(b=2, f=4, r=32, with_residuals=True):
    """SVD UNet at the released width (config.json heads 5/10/20/20), two clips with different image tokens (exercises the
    per-clip broadcast form of the single-token cross attention), 5-D residuals with three surplus entries + mid."""
    from ctrl_adapter_b200.unet_svd import UNetSpatioTemporalConditionModel
    from oracle import cases
    from oracle.unet_svd import UNetSpatioTemporalConditionModel as OUNet
    inputs = cases.unet_svd_inputs(b, f, r, with_residuals=with_residuals, chans=(320, 640, 1280, 1280), ctx=1024)
    call = lambda m, i: m(**i)  # noqa: E731
    sd, ref, eager, inp16 = _oracle_runs(lambda: OUNet(**cases.UNET_SVD_KW), 8, inputs, call)
    with torch.device("cuda"):
        ours_m = UNetSpatioTemporalConditionModel(**cases.UNET_SVD_KW)
    ours_m.load_state_dict(sd)
    ours_m = ours_m.to(BF16).cuda().eval()
    ours = ours_m(**inp16)
    torch.cuda.synchronize()
    return _compare(f"UNetSpatioTemporalConditionModel[svd] b={b} f={f} r={r} residuals={int(with_residuals)}", ours, ref,
                    eager, tol_rel=3e-2, tol_max=8e-2)


def check_vae(n=2, r=32):
    """AutoencoderKL.decode at the published SDXL width (latents r x r -> images 8r x 8r) vs the restated diffusers
    decoder: fp32 truth and its eager bf16-autocast run."""
    from ctrl_adapter_b200.vae import AutoencoderKL
    from oracle.vae import AutoencoderKL as OV
    from oracle.weights import seeded_tensor
    inputs = dict(z=seeded_tensor("vae_z", (n, 4, r, r)))
    call = lambda m, i: m.decode(i["z"])[0]  # noqa: E731
    sd, ref, eager, inp16 = _oracle_runs(lambda: OV(), 11, inputs, call)
    with torch.device("cuda"):
        ours_m = AutoencoderKL()
    ours_m.load_state_dict(sd)
    ours_m = ours_m.to(BF16).cuda().eval()
    ours = ours_m.decode(inp16["z"]).sample
    torch.cuda.synchronize()
    return _compare(f"AutoencoderKL.decode n={n} latents {r}x{r}", ours, ref, eager, tol_rel=3e-2, tol_max=8e-2)


def check_vae_temporal(clips=1, frames=4, h=32, w=32):
    """AutoencoderKLTemporalDecoder.decode (the SVD VAE) at the published width vs the restated diffusers decoder: fp32
    truth and its eager bf16-autocast run.  clips * frames latents, `frames` per temporal unit."""
    from ctrl_adapter_b200.vae import AutoencoderKLTemporalDecoder
    from oracle.vae import AutoencoderKLTemporalDecoder as OV
    from oracle.weights import seeded_tensor
    inputs = dict(z=seeded_tensor("vae_t_z", (clips * frames, 4, h, w)))
    call = lambda m, i: m.decode(i["z"], num_frames=frames)[0]  # noqa: E731
    sd, ref, eager, inp16 = _oracle_runs(lambda: OV(), 12, inputs, call)
    with torch.device("cuda"):
        ours_m = AutoencoderKLTemporalDecoder()
    ours_m.load_state_dict(sd)
    ours_m = ours_m.to(BF16).cuda().eval()
    ours = ours_m.decode(inp16["z"], num_frames=frames).sample
    torch.cuda.synchronize()
    return _compare(f"AutoencoderKLTemporalDecoder.decode {clips}x{frames} frames, latents {h}x{w}", ours, ref, eager,
                    tol_rel=3e-2, tol_max=8e-2)


def _build_pair(make_oracle, make_ours, seed):
    """oracle (fp32, bf16-quantised weights, on GPU) and our module with identical weights."""
    from oracle.weights import seeded_init_
    with torch.device("cuda"):
        o = make_oracle()
        m = make_ours()
    o = seeded_init_(o.cuda(), seed).eval()
    m = m.cuda()
    m.load_state_dict(o.state_dict())
    for p_ in o.parameters():
        p_.data = _q(p_.data)
    return o, m.to(BF16).eval()


def check_step_sdxl(steps=2, nsteps=50, b=1, end=1.0, graph=False, eager_ref=False):
    """Whole SDXL denoising iterations (ControlNet -> adapter -> UNet -> CFG -> Euler) vs the restated reference loop
    (oracle/pipeline_sdxl.py) in fp32, at the real 1024x1024 geometry (the 2x adapter only fits 128^2 latents).
    `end` = control_guidance_end (the steps past it run with cond_scale 0, sdxl pipeline :1207-1211, :1346);
    `graph` steps through CUDA-graph replay (one captured graph per conditioning scale) instead of eager launches."""
    from ctrl_adapter_b200.loop_base import controlnet_keep
    from ctrl_adapter_b200.adapter import ControlNetAdapter
    from ctrl_adapter_b200.controlnet import ControlNetModel
    from ctrl_adapter_b200.pipeline_sdxl import SDXLControlNetAdapterLoop
    from ctrl_adapter_b200.unet_sdxl import UNet2DConditionModel
    from oracle import cases
    from oracle.adapter import ControlNetAdapter as OA
    from oracle.controlnet import ControlNetModel as OC
    from oracle.pipeline_sdxl import EulerDiscreteScheduler, sdxl_step
    from oracle.unet_sdxl import UNet2DConditionModel as OU
    from oracle.weights import seeded_tensor
    ocn, cn = _build_pair(lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4)
    oad, ad = _build_pair(lambda: OA(**cases.ADAPTER_SDXL_KW), lambda: ControlNetAdapter(**cases.ADAPTER_SDXL_KW), 1)
    oun, un = _build_pair(lambda: OU(), lambda: UNet2DConditionModel(), 6)
    inp = dict(latents=seeded_tensor("s_lat", (b, 4, 128, 128)), prompt_embeds=seeded_tensor("s_pe", (2 * b, 77, 2048)),
               add_text_embeds=seeded_tensor("s_te", (2 * b, 1280)),
               add_time_ids=torch.tensor([[1024.0, 1024, 0, 0, 1024, 1024]] * (2 * b)),
               controlnet_prompt_embeds=seeded_tensor("s_cpe", (2 * b, 77, 768)),
               control_images=torch.sigmoid(seeded_tensor("s_img", (2 * b, 3, 512, 512))))
    inp = {k: _q(v).cuda() for k, v in inp.items()}
    sch = EulerDiscreteScheduler()
    sch.set_timesteps(nsteps, device="cuda")
    loop = SDXLControlNetAdapterLoop(cn, ad, un, num_inference_steps=nsteps, guidance_scale=5.0, control_guidance_end=end)
    loop.prepare(**inp)
    keep = controlnet_keep(nsteps, [0.0], [end])
    lat = _q(inp["latents"] * sch.init_noise_sigma)
    args = (inp["prompt_embeds"], inp["add_text_embeds"], inp["add_time_ids"], inp["controlnet_prompt_embeds"],
            inp["control_images"])
    with torch.no_grad():
        for i in range(steps):
            lat = sdxl_step(ocn, oad, oun, sch, i, lat, *args, cond_scale=1.0 * keep[i][0])
            (loop.step_graph if graph else loop.step)(i)
    torch.cuda.synchronize()
    # the same trajectory as the reference runs it: bf16 modules under autocast, bf16 latents (the error budget of a
    # multi-step trajectory is whatever that path accumulates against the fp32 truth)
    eager = None
    if eager_ref:
        e = [m.to(BF16) for m in (ocn, oad, oun)]
        el = _q(inp["latents"] * sch.init_noise_sigma).to(BF16)
        a16 = [t.to(BF16) if t.is_floating_point() else t for t in args]
        with torch.no_grad(), torch.autocast("cuda", dtype=BF16):
            for i in range(steps):
                el = sdxl_step(*e, sch, i, el, *a16, cond_scale=1.0 * keep[i][0]).to(BF16)
        eager = el.float()
    return _compare(f"SDXL denoise loop, {steps} of {nsteps} steps, B={b} 1024x1024, guidance_end={end} graph={int(graph)}",
                    loop.latents, lat, eager, tol_rel=2e-2 if eager is None else 6e-2, tol_max=8e-2 if eager is None else 0.2)


def check_step_i2vgen(steps=2, multi=False, sparse=None, f=4, r=32, nsteps=50, end=1.0, graph=False, eager_ref=False):
    """Whole I2VGen-XL iterations (ControlNet[s] -> [router merge] -> adapter -> UNet -> CFG -> DDIM), B=1; default F=4,
    32^2 latents (use_size_512 off), r=64 / f=16 is BASELINE config 3's per-clip geometry with use_size_512 on as the
    reference has it (the reference's pooling to 64^2 at any other size yields residuals the video UNet cannot add)."""
    from ctrl_adapter_b200.loop_base import controlnet_keep
    from ctrl_adapter_b200.adapter import ControlNetAdapter, ControlNetRouter
    from ctrl_adapter_b200.controlnet import ControlNetModel, MultiControlNetModel
    from ctrl_adapter_b200.pipeline_i2vgen import I2VGenXLControlNetAdapterLoop
    from ctrl_adapter_b200.unet_i2vgen import I2VGenXLUNet
    from oracle import cases
    from oracle.adapter import ControlNetAdapter as OA, ControlNetRouter as OR
    from oracle.controlnet import ControlNetModel as OC, MultiControlNetModel as OM
    from oracle.pipeline_i2vgen import DDIMScheduler, i2vgen_step
    from oracle.unet_i2vgen import I2VGenXLUNet as OU
    from oracle.weights import seeded_tensor
    b = 1
    pool = r == 64  # use_size_512 as the reference has it by default (an identity at 64^2)
    kw = dict(cases.ADAPTER_VIDEO_KW, num_frames=f)
    oad, ad = _build_pair(lambda: OA(**kw), lambda: ControlNetAdapter(**kw), 2)
    oun, un = _build_pair(lambda: OU(), lambda: I2VGenXLUNet(), 7)
    router = orouter = masks = None
    n = 2 * b * f
    if multi:
        nets = [_build_pair(lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 40 + k)
                for k in range(2)]
        ocn, cn = OM([p_[0] for p_ in nets]), MultiControlNetModel([p_[1] for p_ in nets])
        rk = dict(cases.ROUTER_KW, num_experts=3)
        orouter, router = _build_pair(lambda: OR(**rk), lambda: ControlNetRouter(**rk), 3)
        masks = [1, 1, 0]
        images = [torch.sigmoid(seeded_tensor(f"v_img{k}", (n, 3, 8 * r, 8 * r))) for k in range(2)]
    else:
        ocn, cn = _build_pair(lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4)
        images = torch.sigmoid(seeded_tensor("v_img", (n, 3, 8 * r, 8 * r)))
    inp = dict(latents=seeded_tensor("v_lat", (b, 4, f, r, r)), prompt_embeds=seeded_tensor("v_pe", (2 * b, 77, 1024)),
               image_latents=seeded_tensor("v_il", (2 * b, 4, f, r, r)),
               image_embeddings=seeded_tensor("v_ie", (2 * b, 1, 1024)), fps=torch.tensor([16.0] * (2 * b)),
               controlnet_prompt_embeds=seeded_tensor("v_cpe", (n, 77, 768)))
    inp = {k: _q(v).cuda() for k, v in inp.items()}
    images = [_q(i).cuda() for i in images] if multi else _q(images).cuda()
    sch = DDIMScheduler()
    sch.set_timesteps(nsteps, device="cuda")
    loop = I2VGenXLControlNetAdapterLoop(cn, ad, un, router, num_inference_steps=nsteps, guidance_scale=9.0,
                                         use_size_512=pool, inference_expert_masks=masks, sparse_frames=sparse,
                                         control_guidance_end=end)
    loop.prepare(control_images=images, **inp)
    keep = controlnet_keep(nsteps, [0.0] * (2 if multi else 1), [end] * (2 if multi else 1))
    lat = inp["latents"]
    args = (inp["prompt_embeds"], inp["image_latents"], inp["image_embeddings"], inp["fps"], inp["controlnet_prompt_embeds"])
    scale_of = lambda i: [1.0 * k for k in keep[i]] if multi else 1.0 * keep[i][0]  # noqa: E731
    with torch.no_grad():
        for i in range(steps):
            lat = i2vgen_step(ocn, oad, oun, sch, i, lat, *args, images, router=orouter, masks=masks,
                              sparse_frames=sparse, use_size_512=pool, cond_scale=scale_of(i))
            (loop.step_graph if graph else loop.step)(i)
    torch.cuda.synchronize()
    eager = None
    if eager_ref and not multi:
        e = [m.to(BF16) for m in (ocn, oad, oun)]
        el = inp["latents"].to(BF16)
        a16 = [t.to(BF16) if t.is_floating_point() else t for t in args]
        with torch.no_grad(), torch.autocast("cuda", dtype=BF16):
            for i in range(steps):
                el = i2vgen_step(*e, sch, i, el, *a16, images.to(BF16), sparse_frames=sparse, use_size_512=pool,
                                 cond_scale=scale_of(i)).to(BF16)
        eager = el.float()
    return _compare(f"I2VGen-XL denoise loop multi={int(multi)} sparse={sparse}, {steps} of {nsteps} steps, B=1 F={f} "
                    f"{r}x{r} guidance_end={end} graph={int(graph)}", loop.latents_bcfhw(), lat, eager,
                    tol_rel=2e-2 if eager is None else 6e-2, tol_max=8e-2 if eager is None else 0.2)


def check_cfg_euler_v():
    """ca_cfg_euler_v against the same arithmetic in PyTorch (bf16 rounding points of the reference's tensor ops)."""
    from ctrl_adapter_b200 import ops
    from tests import ops_emulator as emu
    g = torch.Generator(device="cpu").manual_seed(5)
    b, f, c, h, w = 2, 5, 4, 16, 24
    eu = torch.randn(b, f, c, h, w, generator=g).to(BF16).cuda()
    et = torch.randn(b, f, c, h, w, generator=g).to(BF16).cuda()
    lat = (torch.randn(b, f, c, h, w, generator=g) * 30).to(BF16).float().cuda()
    guid = torch.linspace(1.0, 3.0, f).to(BF16).float().cuda()
    row = torch.tensor([1.2, 12.5, 7.25, (7.25 ** 2 + 1) ** 0.5], dtype=torch.float32).cuda()
    nxt = torch.empty_like(eu)
    out = ops.cfg_euler_v(eu, et, lat, guid, f, row, model_in_next=nxt)
    torch.cuda.synchronize()
    nxt_ref = torch.empty_like(eu)
    ref = emu.cfg_euler_v(eu, et, lat, guid, f, row.cpu(), model_in_next=nxt_ref)
    r1 = _compare("cfg_euler_v latents", out, ref, None, tol_rel=2e-3, tol_max=1e-2)
    r2 = _compare("cfg_euler_v next model input", nxt, nxt_ref, None, tol_rel=2e-3, tol_max=1e-2)
    return r1, r2


def check_step_svd(steps=2, sparse=None):
    """Whole SVD iterations (ControlNet -> adapter -> SVD UNet -> per-frame CFG -> Euler v-prediction), B=1, F=4, 32^2."""
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
    b, f, r, nsteps = 1, 4, 32, 25
    n = 2 * b * f
    kw = dict(cases.ADAPTER_VIDEO_KW, backbone_model_name="svd", num_frames=f)
    oad, ad = _build_pair(lambda: OA(**kw), lambda: ControlNetAdapter(**kw), 2)
    oun, un = _build_pair(lambda: OU(**cases.UNET_SVD_KW), lambda: UNetSpatioTemporalConditionModel(**cases.UNET_SVD_KW), 8)
    ocn, cn = _build_pair(lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4)
    images = _q(torch.sigmoid(seeded_tensor("s_img", (n, 3, 8 * r, 8 * r)))).cuda()
    il = seeded_tensor("s_il", (b, f, 4, r, r))
    inp = dict(latents=seeded_tensor("s_lat", (b, f, 4, r, r)), image_latents=torch.cat([torch.zeros_like(il), il]),
               image_embeddings=torch.cat([torch.zeros(b, 1, 1024), seeded_tensor("s_ie", (b, 1, 1024))]),
               added_time_ids=torch.tensor([[6.0, 127.0, 0.02]] * (2 * b)),
               controlnet_prompt_embeds=seeded_tensor("s_cpe", (n, 77, 768)))
    inp = {k: _q(v).cuda() for k, v in inp.items()}
    sch = EulerDiscreteSchedulerSVD()
    sch.set_timesteps(nsteps, device="cuda")
    flags = dict(use_size_512=False, skip_conv_in=True, skip_time_emb=False)
    loop = SVDControlNetAdapterLoop(cn, ad, un, num_inference_steps=nsteps, sparse_frames=sparse, **flags)
    loop.prepare(control_images=images, **inp)
    lat = (inp["latents"] * sch.init_noise_sigma).to(BF16)
    with torch.no_grad():
        for i in range(steps):
            lat = svd_step(ocn, oad, oun, sch, i, lat.float(), inp["image_latents"], inp["image_embeddings"],
                           inp["added_time_ids"], inp["controlnet_prompt_embeds"], images, sparse_frames=sparse,
                           **flags).to(BF16)
            loop.step(i)
    torch.cuda.synchronize()
    return _compare(f"SVD denoise loop sparse={sparse}, {steps} steps, B=1 F=4 32x32", loop.latents, lat.float(), None,
                    tol_rel=2e-2, tol_max=8e-2)


def check_extra_shapes():
    """Kernel-level checks at shapes that first appear with the SVD / folded-conv / wide-tile work (576 x 1024 video ->
    72 x 128 latents and its 36 x 64, 18 x 32 levels; K/V projection shape; folded conditioning convolutions)."""
    from tests import kernel_checks as kc
    kc.RESULTS.clear()
    recs = [kc.check_attention(1, 5, 16384, 16384, 64),  # the dominant SDXL adapter-A shape (128^2 tokens), per sample
            kc.check_attention(1, 5, 2304, 2304, 64), kc.check_attention(2, 10, 576, 576, 64),
            kc.check_attention(2, 20, 144, 144, 64), kc.check_temporal_attention(2, 14, 144, 10),
            kc.check_conv(2, 36, 64, 320, 320, out_fp32=False, residual=True),
            kc.check_conv(2, 18, 32, 640, 640, out_fp32=False, rowvec=True),
            kc.check_conv(2, 64, 16, 64, 128, out_fp32=False), kc.check_conv(1, 64, 32, 64, 64, out_fp32=False),
            kc.check_linear(1232, 2048, 2560, out_fp32=False), kc.check_linear(4608, 320, 960, out_fp32=False)]
    for r in recs:
        RESULTS.append(r)
    return recs


def check_controlnet_folded():
    """The three convolutions ControlNetConditioningEmbedding folds (adjacent pixels in the channel axis,
    Conv2d.forward_folded) against their zero-padded form (Conv2d.forward), both on the GPU kernels, at the resolutions
    of a 512 x 512 control image: conv_in 3 -> 16 on the 8-channel padded image, 16 -> 16 at 512^2, 32 -> 32 at 256^2.
    Same arithmetic with zeros added, so the two differ by bf16 rounding only (the bound of the CPU test)."""
    from ctrl_adapter_b200.layers import Conv2d
    from ctrl_adapter_b200.ops import ACT_SILU
    torch.manual_seed(0)
    recs = []
    for cin, cout, cs, r in ((3, 16, 8, 512), (16, 16, 16, 512), (32, 32, 32, 256)):
        with torch.device("cuda"), torch.no_grad():
            conv = Conv2d(cin, cout, 3)
            conv.bias.normal_(0.0, 0.1)
            x = torch.zeros(2, r, r, cs)
            x[..., :cin] = torch.randn(2, r, r, cin)
        conv = conv.to(BF16).eval()
        x = x.to(BF16)
        padded = conv(x, act=ACT_SILU).float()
        folded = conv.forward_folded(x, act=ACT_SILU).float()
        torch.cuda.synchronize()
        err = float((folded - padded).abs().max())
        bound = 2.0 ** -7 * float(padded.abs().max())
        fold = conv.fold_factor(x)
        rec = {"check": f"Conv2d {cin}->{cout} Cs={cs} {r}x{r} SiLU: folded x{fold} vs padded", "max_abs": err,
               "bound": bound, "ok": fold == 64 // cs and err <= bound}
        RESULTS.append(rec)
        recs.append(rec)
    return recs


GROUPS = {
    "adapter": [lambda: check_adapter("sdxl", 2, 8), lambda: check_adapter("video", 1, 8, 4), check_router],
    "controlnet": [lambda: check_controlnet(2, 8), lambda: check_controlnet(2, 16, True, 0.75)],
    "unet": [lambda: check_unet_sdxl(2, 16, True), lambda: check_unet_sdxl(1, 32, False)],
    "video": [lambda: check_unet_i2vgen(1, 4, 32, True), lambda: check_unet_i2vgen(2, 2, 32, False)],
    "vae": [lambda: check_vae(2, 32), lambda: check_vae(1, 64), lambda: check_vae_temporal(1, 4, 32, 32),
            lambda: check_vae_temporal(2, 3, 16, 24)],
    "svd": [lambda: check_unet_svd(2, 4, 32, True), lambda: check_unet_svd(1, 3, 16, False)],
    "sparse": [lambda: check_step_i2vgen(2, False, sparse=[0, 2])],
    "fold": [check_controlnet_folded],
    "shapes": [check_extra_shapes],
    "svd_loop": [check_cfg_euler_v, check_step_svd],  # sparse SVD variant: CPU-emulated only (keeps the GPU suite short)
    "step": [check_step_sdxl, lambda: check_step_i2vgen(2, False), lambda: check_step_i2vgen(1, True)],
    # round 2: config-1-style 4-step SDXL run crossing control_guidance_end through CUDA-graph replay, a B=2 step at the
    # config-2 geometry, the router path under graph capture, config 3's F=16 / 64^2 clip and a video step on either
    # side of control_guidance_end
    # (whole few-step trajectories are judged like the modules: no worse than 1.5x the error the reference's own eager
    # bf16-autocast trajectory accumulates against the fp32 truth, since a 2- or 4-step schedule amplifies rounding)
    "loops": [lambda: check_step_sdxl(4, nsteps=4, end=0.5, graph=True, eager_ref=True), lambda: check_step_sdxl(1, b=2),
              lambda: check_step_i2vgen(1, True, graph=True), lambda: check_step_i2vgen(1, f=16, r=64),
              lambda: check_step_i2vgen(2, nsteps=2, end=0.5, graph=True, eager_ref=True)],
}


def run(group=None):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    RESULTS.clear()
    names = [group] if group else list(GROUPS)
    for g in names:
        for fn in GROUPS[g]:
            n0 = len(RESULTS)
            t0 = time.time()
            try:
                fn()
            except Exception as e:
                import traceback
                RESULTS.append({"check": f"EXC in {g}", "ok": False, "why": traceback.format_exc()[-1500:]})
            for r in RESULTS[n0:]:
                flag = "ok  " if r["ok"] else "FAIL"
                print(f"[{flag}] {r['check']} ({time.time() - t0:.1f}s): " + ", ".join(
                    f"{k}={v:.3g}" if isinstance(v, float) else f"{k}={v}" for k, v in r.items() if k not in ("check", "ok")),
                    flush=True)
    return RESULTS


if __name__ == "__main__":
    if "--groups" in sys.argv:  # several groups in one process; per-group verdicts in the JSON (tests/test_zz_svd_gpu.py)
        names = sys.argv[sys.argv.index("--groups") + 1].split(",")
        verdict = {}
        for gname in names:
            res = [dict(r) for r in run(gname)]
            verdict[gname] = {"ok": all(r["ok"] for r in res), "results": res}
        if "--json" in sys.argv:
            json.dump(verdict, open(sys.argv[sys.argv.index("--json") + 1], "w"), indent=1, default=str)
        sys.exit(0 if all(v["ok"] for v in verdict.values()) else 1)
    grp = sys.argv[sys.argv.index("--group") + 1] if "--group" in sys.argv else None
    res = run(grp)
    if "--json" in sys.argv:
        json.dump(res, open(sys.argv[sys.argv.index("--json") + 1], "w"), indent=1)
    nbad = sum(1 for r in res if not r["ok"])
    print(f"{len(res) - nbad}/{len(res)} module checks ok")
    sys.exit(1 if nbad else 0)
