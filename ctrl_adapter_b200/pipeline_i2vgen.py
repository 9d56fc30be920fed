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
from .adapter import as_nchw, to_channels_last_bf16
from .layers import cache_static_context
from .loop_base import DenoiseLoopBase
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
        nets = len(controlnet.nets) if hasattr(controlnet, "nets") else 1
        self._init_control(controlnet_conditioning_scale, control_guidance_start, control_guidance_end,
                           nets if hasattr(controlnet, "nets") else 1)
        self._multi = hasattr(controlnet, "nets")  # a one-net MultiControlNetModel still takes list arguments

    def prepare(self, latents, prompt_embeds, image_latents, image_embeddings, fps, controlnet_prompt_embeds,
                control_images):
        """latents (B,4,F,h,w) unit noise; prompt_embeds (2B,77,1024) negative first; image_latents (2B,4,F,h,w);
        image_embeddings (2B,1,1024); fps (2B,); controlnet_prompt_embeds (2B*F,77,768); control_images: (2B*F,3,H,W)
        or a list of E such tensors (Multi-ControlNet)."""
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
        self._pool = (h, w) != (64, 64) and self.use_size_512                              # :941-947
        if self._pool:
            # the reference pools the ControlNet input to 64x64 here, but its video adapters do not up-sample, so the
            # 64x64 residuals cannot be added to a UNet running at another size (it fails inside the UNet, :689)
            raise ValueError("use_size_512=True needs 64x64 latents (512x512 video) for the I2VGen-XL backbone; pass "
                             "use_size_512=False to run the ControlNet at the latent resolution")

        def prep_image(img):
            img = img.to(BF16).contiguous()
            if self._pool and tuple(img.shape[-2:]) != (512, 512):                         # step-invariant: pooled once
                if img.shape[-2] % 512 or img.shape[-1] % 512:
                    raise NotImplementedError("control images must be 512x512 or an integer multiple of it")
                img = as_nchw(ops.avgpool(to_channels_last_bf16(img, 8), 512, 512))[:, :3].contiguous()
            return img
        self.images = ([prep_image(i) for i in control_images] if isinstance(control_images, (list, tuple))
                       else prep_image(control_images))
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
        self._sparse_rows = None
        if self.sparse_frames is not None:
            if not all(0 <= k < f for k in self.sparse_frames):
                raise ValueError("sparse_frames must index frames of the clip")
            self._sparse_rows = torch.tensor([bb * f + k for bb in range(2 * b) for k in self.sparse_frames], device=dev)
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
        rows = self._sparse_rows
        nf = f if rows is None else len(self.sparse_frames)
        mask = None if rows is None else self.sparse_frames
        control_off = (not isinstance(scale, tuple)) and scale == 0              # :1083 (a list never compares == 0)
        if not control_off:
            ctrl_in = lat2.reshape(n, *lat2.shape[2:])                           # "(b f) c h w"
            if self._pool:
                ctrl_in = as_nchw(ops.avgpool(to_channels_last_bf16(ctrl_in, 8), 64, 64))[:, :4]
            down, mid = self._controlnet_outputs(ctrl_in, t, scale)
            if rows is not None:
                # key-frame gather -> adapter on len(sparse_frames) frames per clip -> scatter into zero residuals
                # (host-side index glue over ControlNet-sized tensors; the reference's dense tensors are fp32 zeros,
                # which only changes where the skip + residual sum is rounded -- quirk Q21)
                down = [d.index_select(0, rows) for d in down]
                mid = mid.index_select(0, rows) if mid is not None else None
            down_a, mid_a = self.adapter(down, mid_block_res_sample=mid, sparsity_masking=mask, num_frames=nf,
                                         timestep=t, encoder_hidden_states=self.adapter_ctx)
        else:
            # cond_scale == 0: every ControlNet output is exactly zero and the down residuals are dropped (:1083), but
            # the mid-block adapter's output (a function of t alone) is still injected (quirk Q9)
            down_a = None
            hh, ww = (8, 8) if self._pool else (lat2.shape[-2] // 8, lat2.shape[-1] // 8)
            rows_n = n if rows is None else rows.numel()
            mid0 = torch.zeros((rows_n, hh, ww, 1280), device=lat2.device, dtype=BF16).permute(0, 3, 1, 2)
            mid_a = self.adapter.forward_mid(mid0, num_frames=nf, timestep=t, encoder_hidden_states=self.adapter_ctx)
        if rows is not None:
            def densify(x):
                full = torch.zeros((n, *x.shape[1:]), device=x.device, dtype=x.dtype).contiguous(
                    memory_format=torch.channels_last)
                full.index_copy_(0, rows, x)
                return full
            down_a = [densify(d) for d in down_a] if down_a is not None else None
            mid_a = densify(mid_a) if mid_a is not None else None
        sample = lat2.permute(0, 2, 1, 3, 4)                                     # (2B, 4, F, h, w) view
        eps = self.unet(sample, t, self.fps, self.image_latents, image_embeddings=self.image_embeddings,
                        encoder_hidden_states=self.prompt_embeds, down_block_additional_residuals=down_a,
                        mid_block_additional_residual=mid_a, return_dict=False)[0]
        eps = eps.permute(0, 2, 1, 3, 4)                                          # back to (2B, F, 4, h, w): contiguous
        ops.cfg_ddim(eps[:b].contiguous(), eps[b:].contiguous(), self.latents, self.guidance_scale, self.row,
                     latents_out=self.latents, model_in_next=self.model_in, v_prediction=self.schedule.v_prediction)

    def latents_bcfhw(self):
        return self.latents.permute(0, 2, 1, 3, 4)
