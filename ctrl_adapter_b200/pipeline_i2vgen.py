"""The I2VGen-XL denoising hot loop (body of /root/reference/i2vgen_xl/pipelines/i2vgen_xl_controlnet_adapter_pipeline.py
:902-1118) on the H100 modules:

  ControlNet (or E ControlNets -> router -> weighted merge) -> Ctrl-Adapter (spatial + temporal) -> I2VGen-XL UNet with
  residual injection -> CFG -> DDIM update.

Latents are kept in (clip, frame, channel, h, w) order internally, i.e. already in the "(b f) c h w" layout the
reference permutes to around the scheduler step (:1107-1115); `latents_bcfhw()` gives the reference's view.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import ops
from .layers import as_nchw, cache_static_context, to_channels_last_bf16
from .loop_base import DenoiseLoopBase, check_geometry
from .schedulers import DDIMSchedule

BF16 = torch.bfloat16


class I2VGenXLControlNetAdapterLoop(DenoiseLoopBase):
    def __init__(self, controlnet, adapter, unet, router=None, *, num_inference_steps: int = 50,
                 guidance_scale: float = 9.0, controlnet_conditioning_scale=1.0,
                 inference_expert_masks: Optional[List[bool]] = None, skip_conv_in: bool = False,
                 skip_time_emb: bool = False, sparse_frames: Optional[List[int]] = None, use_size_512: bool = True,
                 control_guidance_start=0.0, control_guidance_end=1.0, fixed_controlnet_timestep: int = -1):
        self.controlnet, self.adapter, self.unet, self.router = controlnet, adapter, unet, router
        self.guidance_scale = float(guidance_scale)
        self.masks = inference_expert_masks
        self.skip_conv_in, self.skip_time_emb = skip_conv_in, skip_time_emb
        self.use_size_512 = use_size_512
        self.fixed_controlnet_timestep = int(fixed_controlnet_timestep)
        # sparse control (:1024-1033, :1053-1073): only these key frames of every clip go through the adapter; the other
        # frames get zero residuals
        self.sparse_frames = None if sparse_frames is None else [int(k) for k in sparse_frames]
        self.schedule = DDIMSchedule(num_inference_steps)
        self.num_inference_steps = num_inference_steps
        multi = hasattr(controlnet, "nets")
        self._init_control(controlnet_conditioning_scale, control_guidance_start, control_guidance_end,
                           len(controlnet.nets) if multi else 1)
        self._multi = multi  # a one-net MultiControlNetModel still takes list arguments

    def prepare(self, latents, prompt_embeds, image_latents, image_embeddings, fps, controlnet_prompt_embeds,
                control_images):
        """latents (B,4,F,h,w) unit noise; prompt_embeds (2B,77,1024) negative first; image_latents (2B,4,F,h,w);
        image_embeddings (2B,1,1024); fps (2B,); controlnet_prompt_embeds (2B*F,77,768); control_images: (2B*F,3,H,W)
        or a list of E such tensors (Multi-ControlNet)."""
        # use_size_512: the reference pools the ControlNet input to 64x64, but its video adapters do not up-sample, so
        # only 64x64 latents (512x512 video) fit the UNet (elsewhere it fails inside the UNet, :689); without it the
        # image latents' 32x32 pool needs multiples of 32
        check_geometry("I2VGen-XL loop", *latents.shape[-2:], self.use_size_512, control_images, multiple=32,
                       adapter_up=1)
        dev = latents.device
        b, c, f, h, w = latents.shape
        self.batch, self.frames = b, f
        lat = latents.float() * self.schedule.init_noise_sigma
        self.latents = lat.permute(0, 2, 1, 3, 4).contiguous().to(BF16).float()          # (B, F, 4, h, w) fp32 master
        self.model_in = self.latents.to(BF16).contiguous()
        self.table = torch.from_numpy(self.schedule.table()).to(dev)
        self.row = self.table[0].clone()
        self.cn_t = (torch.full((1,), float(self.fixed_controlnet_timestep), device=dev)
                     if self.fixed_controlnet_timestep >= 0 else None)                     # :951-954
        self.prompt_embeds = prompt_embeds.to(BF16).contiguous()
        self.image_latents = image_latents.to(BF16).contiguous()
        self.image_embeddings = image_embeddings.to(BF16).contiguous()
        self.fps = fps.float().contiguous()
        self.cn_embeds = controlnet_prompt_embeds.to(BF16).contiguous()
        self.images = ([i.to(BF16).contiguous() for i in control_images] if isinstance(control_images, (list, tuple))
                       else control_images.to(BF16).contiguous())
        # adapter context: the LAST sample's image embedding for every sample (reference :1048, quirk Q5)
        self.adapter_ctx = self.image_embeddings[-1].unsqueeze(0).contiguous()
        # timestep-independent UNet conditioning, computed once (exact hoist)
        self.unet._cond_cache = None
        self.unet_cond = self.unet._conditioning(self.fps, self.image_latents, self.image_embeddings, self.prompt_embeds)
        # more step-invariant work: the single-token adapter context, the ControlNets' text K/V and image embeddings,
        # the router's masked softmax (its inputs are parameters and the expert mask only)
        cache_static_context(self.adapter, self.adapter_ctx, single_token_rows=1)
        nets = list(self.controlnet.nets) if hasattr(self.controlnet, "nets") else [self.controlnet]
        imgs = self.images if isinstance(self.images, list) else [self.images]
        for net, img in zip(nets, imgs):
            cache_static_context(net, self.cn_embeds)
            net.cache_static_cond(img)
        self._router_w = None
        if self.router is not None:
            dw, mw = self.router(sparse_mask=self.masks)                                  # (12, E), (E,)
            self._active = [e for e in range(self.router.num_experts) if self.masks[e]]
            sel_idx = torch.tensor(self._active, device=dev)
            # Q6: w.repeat_interleave(F)[e] == w[e // F]
            pick = lambda wrow: wrow.repeat_interleave(f)[sel_idx].float().contiguous()  # noqa: E731
            self._router_w = ([pick(dw[k]) for k in range(self.router.num_routers)],
                              pick(mw) if mw is not None else None)
        self._init_key_frames(2 * b, f, dev)
        self._graphs = {}
        self.step_index = 0

    def _state(self):
        return [self.latents, self.model_in, self.row]

    def _load_step(self, i):
        self.row.copy_(self.table[i])

    def _controlnet_outputs(self, ctrl_in, t, scale):
        multi = isinstance(self.images, list)
        cn_scale = list(scale) if isinstance(scale, tuple) else ([scale] * len(self.images) if multi else scale)
        down, mid = self.controlnet(ctrl_in, self.cn_t if self.cn_t is not None else t,
                                    encoder_hidden_states=self.cn_embeds, controlnet_cond=self.images,
                                    conditioning_scale=cn_scale, guess_mode=False, return_dict=False,
                                    skip_conv_in=self.skip_conv_in, skip_time_emb=self.skip_time_emb)
        if self.router is not None:
            active = self._active
            dws, mw = self._router_w
            # down[i][k]: output k of the i-th ControlNet that ran; weights were picked by expert id in prepare()
            down = [as_nchw(ops.router_merge([to_channels_last_bf16(down[i][k]) for i in range(len(active))], dws[k]))
                    for k in range(self.router.num_routers)]
            mid = (as_nchw(ops.router_merge([to_channels_last_bf16(mid[i]) for i in range(len(active))], mw))
                   if mw is not None else None)
        return down, mid

    def _body(self, scale):
        b, f = self.batch, self.frames
        t = self.row[0:1]
        lat2 = torch.cat([self.model_in, self.model_in], dim=0)                  # (2B, F, 4, h, w) CFG duplication
        n = 2 * b * f
        down = mid = None
        if isinstance(scale, tuple) or scale != 0:                               # :1083 (a list never compares == 0)
            down, mid = self._controlnet_outputs(lat2.reshape(n, *lat2.shape[2:]), t, scale)  # "(b f) c h w"
        down_a, mid_a = self._video_adapter(down, mid, t, n, (lat2.shape[-2] // 8, lat2.shape[-1] // 8))
        sample = lat2.permute(0, 2, 1, 3, 4)                                     # (2B, 4, F, h, w) view
        eps = self.unet(sample, t, self.fps, self.image_latents, image_embeddings=self.image_embeddings,
                        encoder_hidden_states=self.prompt_embeds, down_block_additional_residuals=down_a,
                        mid_block_additional_residual=mid_a, return_dict=False)[0]
        eps = eps.permute(0, 2, 1, 3, 4)                                          # back to (2B, F, 4, h, w): contiguous
        ops.cfg_ddim(eps[:b].contiguous(), eps[b:].contiguous(), self.latents, self.guidance_scale, self.row,
                     latents_out=self.latents, model_in_next=self.model_in, v_prediction=self.schedule.v_prediction)

    def latents_bcfhw(self):
        return self.latents.permute(0, 2, 1, 3, 4)
