"""Trajectory drift report (GPU): the whole denoising schedule run three ways from the same initial noise and weights --
our loop (bf16 kernels, CUDA-graph replay), the oracle as the reference runs it (eager bf16 autocast) and the oracle in
fp32 (the truth) -- with the relative Frobenius distance to the truth after every step.

  python scripts/drift_report.py sdxl|i2vgen|svd [--steps N] [--guidance-end E] --out drift_<w>.json

sdxl: B=1 at 1024x1024 (50 steps);  i2vgen: B=1, F=16, 64x64 latents (config 3's clip geometry, 50 steps);
svd: B=1, F=14, 32x32 latents, use_size_512=False (25 steps).  Oracle = test infrastructure (tests/module_checks.py builds
the module pairs with identical name-seeded weights)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import module_checks as mc  # noqa: E402

BF16 = torch.bfloat16


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", choices=["sdxl", "i2vgen", "svd"])
    ap.add_argument("--steps", type=int, default=0)
    ap.add_argument("--guidance-end", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from ctrl_adapter_b200.loop_base import controlnet_keep
    from oracle import cases
    from oracle.weights import seeded_tensor
    q = mc._q
    w = a.workload
    if w == "sdxl":
        from ctrl_adapter_b200.adapter import ControlNetAdapter
        from ctrl_adapter_b200.controlnet import ControlNetModel
        from ctrl_adapter_b200.pipeline_sdxl import SDXLControlNetAdapterLoop
        from ctrl_adapter_b200.unet_sdxl import UNet2DConditionModel
        from oracle.adapter import ControlNetAdapter as OA
        from oracle.controlnet import ControlNetModel as OC
        from oracle.pipeline_sdxl import EulerDiscreteScheduler, sdxl_step
        from oracle.unet_sdxl import UNet2DConditionModel as OU
        n = a.steps or 50
        ocn, cn = mc._build_pair(lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4)
        oad, ad = mc._build_pair(lambda: OA(**cases.ADAPTER_SDXL_KW), lambda: ControlNetAdapter(**cases.ADAPTER_SDXL_KW), 1)
        oun, un = mc._build_pair(lambda: OU(), lambda: UNet2DConditionModel(), 6)
        inp = dict(latents=seeded_tensor("s_lat", (1, 4, 128, 128)), prompt_embeds=seeded_tensor("s_pe", (2, 77, 2048)),
                   add_text_embeds=seeded_tensor("s_te", (2, 1280)),
                   add_time_ids=torch.tensor([[1024.0, 1024, 0, 0, 1024, 1024]] * 2),
                   controlnet_prompt_embeds=seeded_tensor("s_cpe", (2, 77, 768)),
                   control_images=torch.sigmoid(seeded_tensor("s_img", (2, 3, 512, 512))))
        inp = {k: q(v).cuda() for k, v in inp.items()}
        sch = EulerDiscreteScheduler()
        sch.set_timesteps(n, device="cuda")
        loop = SDXLControlNetAdapterLoop(cn, ad, un, num_inference_steps=n, guidance_scale=5.0,
                                         control_guidance_end=a.guidance_end)
        loop.prepare(**inp)
        args = [inp[k] for k in ("prompt_embeds", "add_text_embeds", "add_time_ids", "controlnet_prompt_embeds",
                                 "control_images")]
        lat0 = q(inp["latents"] * sch.init_noise_sigma)
        ostep = lambda mods, i, lat, ar, cs: sdxl_step(*mods, sch, i, lat, *ar, cond_scale=cs)  # noqa: E731
        ours = lambda: loop.latents  # noqa: E731
        mods = (ocn, oad, oun)
    elif w == "i2vgen":
        from ctrl_adapter_b200.adapter import ControlNetAdapter
        from ctrl_adapter_b200.controlnet import ControlNetModel
        from ctrl_adapter_b200.pipeline_i2vgen import I2VGenXLControlNetAdapterLoop
        from ctrl_adapter_b200.unet_i2vgen import I2VGenXLUNet
        from oracle.adapter import ControlNetAdapter as OA
        from oracle.controlnet import ControlNetModel as OC
        from oracle.pipeline_i2vgen import DDIMScheduler, i2vgen_step
        from oracle.unet_i2vgen import I2VGenXLUNet as OU
        n, f, r = a.steps or 50, 16, 64
        kw = dict(cases.ADAPTER_VIDEO_KW, num_frames=f)
        oad, ad = mc._build_pair(lambda: OA(**kw), lambda: ControlNetAdapter(**kw), 2)
        oun, un = mc._build_pair(lambda: OU(), lambda: I2VGenXLUNet(), 7)
        ocn, cn = mc._build_pair(lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4)
        nn_ = 2 * f
        images = q(torch.sigmoid(seeded_tensor("v_img", (nn_, 3, 8 * r, 8 * r)))).cuda()
        inp = dict(latents=seeded_tensor("v_lat", (1, 4, f, r, r)), prompt_embeds=seeded_tensor("v_pe", (2, 77, 1024)),
                   image_latents=seeded_tensor("v_il", (2, 4, f, r, r)), image_embeddings=seeded_tensor("v_ie", (2, 1, 1024)),
                   fps=torch.tensor([16.0] * 2), controlnet_prompt_embeds=seeded_tensor("v_cpe", (nn_, 77, 768)))
        inp = {k: q(v).cuda() for k, v in inp.items()}
        sch = DDIMScheduler()
        sch.set_timesteps(n, device="cuda")
        loop = I2VGenXLControlNetAdapterLoop(cn, ad, un, None, num_inference_steps=n, guidance_scale=9.0,
                                             control_guidance_end=a.guidance_end)
        loop.prepare(control_images=images, **inp)
        args = [inp[k] for k in ("prompt_embeds", "image_latents", "image_embeddings", "fps", "controlnet_prompt_embeds")] + [images]
        lat0 = inp["latents"]
        ostep = lambda mods, i, lat, ar, cs: i2vgen_step(*mods, sch, i, lat, *ar, cond_scale=cs)  # noqa: E731
        ours = lambda: loop.latents_bcfhw()  # noqa: E731
        mods = (ocn, oad, oun)
    else:
        from ctrl_adapter_b200.adapter import ControlNetAdapter
        from ctrl_adapter_b200.controlnet import ControlNetModel
        from ctrl_adapter_b200.pipeline_svd import SVDControlNetAdapterLoop
        from ctrl_adapter_b200.unet_svd import UNetSpatioTemporalConditionModel
        from oracle.adapter import ControlNetAdapter as OA
        from oracle.controlnet import ControlNetModel as OC
        from oracle.pipeline_svd import EulerDiscreteSchedulerSVD, svd_step
        from oracle.unet_svd import UNetSpatioTemporalConditionModel as OU
        n, f, r = a.steps or 25, 14, 32
        nn_ = 2 * f
        kw = dict(cases.ADAPTER_VIDEO_KW, backbone_model_name="svd", num_frames=f)
        oad, ad = mc._build_pair(lambda: OA(**kw), lambda: ControlNetAdapter(**kw), 2)
        oun, un = mc._build_pair(lambda: OU(**cases.UNET_SVD_KW), lambda: UNetSpatioTemporalConditionModel(**cases.UNET_SVD_KW), 8)
        ocn, cn = mc._build_pair(lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4)
        images = q(torch.sigmoid(seeded_tensor("s_img", (nn_, 3, 8 * r, 8 * r)))).cuda()
        il = seeded_tensor("s_il", (1, f, 4, r, r))
        inp = dict(latents=seeded_tensor("s_lat", (1, f, 4, r, r)), image_latents=torch.cat([torch.zeros_like(il), il]),
                   image_embeddings=torch.cat([torch.zeros(1, 1, 1024), seeded_tensor("s_ie", (1, 1, 1024))]),
                   added_time_ids=torch.tensor([[6.0, 127.0, 0.02]] * 2),
                   controlnet_prompt_embeds=seeded_tensor("s_cpe", (nn_, 77, 768)))
        inp = {k: q(v).cuda() for k, v in inp.items()}
        sch = EulerDiscreteSchedulerSVD()
        sch.set_timesteps(n, device="cuda")
        flags = dict(use_size_512=False, skip_conv_in=True, skip_time_emb=False)
        loop = SVDControlNetAdapterLoop(cn, ad, un, num_inference_steps=n, control_guidance_end=a.guidance_end, **flags)
        loop.prepare(control_images=images, **inp)
        args = [inp[k] for k in ("image_latents", "image_embeddings", "added_time_ids", "controlnet_prompt_embeds")] + [images]
        lat0 = (inp["latents"] * sch.init_noise_sigma).to(BF16).float()
        ostep = lambda mods, i, lat, ar, cs: svd_step(*mods, sch, i, lat, *ar, cond_scale=cs, **flags)  # noqa: E731
        ours = lambda: loop.latents  # noqa: E731
        mods = (ocn, oad, oun)

    keep = controlnet_keep(n, [0.0], [a.guidance_end])
    # fp32 truth (kept per step), then the eager bf16 trajectory, then ours
    truth, lat = [], lat0
    with torch.no_grad():
        for i in range(n):
            lat = ostep(mods, i, lat, args, 1.0 * keep[i][0])
            if w == "svd":
                lat = lat.to(BF16).float()  # the reference keeps bf16 latents between steps on this path
            truth.append(lat.cpu())
    e_mods = [m.to(BF16) for m in mods]
    a16 = [t.to(BF16) if t.is_floating_point() else t for t in args]
    eager, el = [], lat0.to(BF16)
    with torch.no_grad(), torch.autocast("cuda", dtype=BF16):
        for i in range(n):
            el = ostep(e_mods, i, el, a16, 1.0 * keep[i][0]).to(BF16)
            eager.append(rel(el.cpu(), truth[i]))
    mine = []
    for i in range(n):
        loop.step_graph(i)
        mine.append(rel(ours().cpu(), truth[i]))
    rec = {"workload": w, "steps": n, "guidance_end": a.guidance_end, "ours_vs_fp32": mine, "eager_bf16_vs_fp32": eager,
           "final": {"ours": mine[-1], "eager": eager[-1]}, "max": {"ours": max(mine), "eager": max(eager)}}
    print(json.dumps({k: rec[k] for k in ("workload", "steps", "final", "max")}))
    if a.out:
        json.dump(rec, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
