"""The Stable-Video-Diffusion denoising hot loop (body of
/root/reference/svd/pipelines/svd_controlnet_adapter_pipeline.py:640-787) on the H100 modules:

  [pool to 64x64] -> ControlNet (timestep from the step index) -> [sparse key-frame gather] -> Ctrl-Adapter (spatial +
  temporal) -> [scatter] -> SVD UNet on cat(latents, image latents) with 5-D residual injection -> per-frame CFG ->
  Euler (v-prediction) update.

Latents live in the reference's own (clip, frame, channel, h, w) order.  Per-step scalars sit in device rows so one
captured CUDA graph serves every step.

GPU parity: tests/test_video_paths_gpu.py groups `svd`, `svd_loop`; CPU: the op-layer emulation against the restated reference loop.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import ops
from .layers import cache_static_context
from .loop_base import DenoiseLoopBase, check_geometry, pool_control_images, pool_controlnet_input
from .schedulers import EulerKarrasVSchedule

BF16 = torch.bfloat16


class SVDControlNetAdapterLoop(DenoiseLoopBase):
    def __init__(self, controlnet, adapter, unet, *, num_inference_steps: int = 25, min_guidance_scale: float = 1.0,
                 max_guidance_scale: float = 3.0, controlnet_conditioning_scale: float = 1.0, use_size_512: bool = True,
                 skip_conv_in: bool = False, skip_time_emb: bool = False, sparse_frames: Optional[List[int]] = None,
                 control_guidance_start: float = 0.0, control_guidance_end: float = 1.0):
        self.controlnet, self.adapter, self.unet = controlnet, adapter, unet
        self.min_g, self.max_g = float(min_guidance_scale), float(max_guidance_scale)
        self.cond_scale = float(controlnet_conditioning_scale)
        self.use_size_512 = use_size_512
        self.skip_conv_in, self.skip_time_emb = skip_conv_in, skip_time_emb
        self.sparse_frames = None if sparse_frames is None else [int(k) for k in sparse_frames]
        self.schedule = EulerKarrasVSchedule(num_inference_steps)
        self.num_inference_steps = num_inference_steps
        self._init_control(controlnet_conditioning_scale, control_guidance_start, control_guidance_end, 1)

    def prepare(self, latents, image_latents, image_embeddings, added_time_ids, controlnet_prompt_embeds, control_images):
        """latents (B,F,4,h,w) unit noise; image_latents (2B,F,4,h,w), zeros for the unconditional half (:225-230,
        :582); image_embeddings (2B,1,1024) negative first; added_time_ids (2B,3); controlnet_prompt_embeds
        (2B*F,77,768); control_images (2B*F,3,H,W) in [0,1]."""
        check_geometry("SVD loop", *latents.shape[-2:], self.use_size_512, control_images, multiple=8, adapter_up=1)
        dev = latents.device
        b, f = latents.shape[:2]
        self.batch, self.frames = b, f
        self.latents = (latents.float() * self.schedule.init_noise_sigma).to(BF16).float().contiguous()
        self.table = torch.from_numpy(self.schedule.table()).to(dev)
        self.cn_table = torch.from_numpy(self.schedule.control_timesteps).to(dev)
        self.row = self.table[0].clone()
        self.cn_t = self.cn_table[0:1].clone()
        first_div = torch.tensor(float((self.schedule.sigmas[0] ** 2 + 1) ** 0.5), device=dev).to(BF16)
        self.model_in = (self.latents.to(BF16) / first_div).to(BF16).contiguous()
        # per-frame guidance: linspace in the latent dtype (:616-621)
        self.guidance = torch.linspace(self.min_g, self.max_g, f, device=dev).to(BF16).float().contiguous()
        self.image_latents = image_latents.to(BF16).contiguous()
        self.image_embeddings = image_embeddings.to(BF16).contiguous()
        self.added_time_ids = added_time_ids.float().contiguous()
        self.cn_embeds = controlnet_prompt_embeds.to(BF16).contiguous()
        images = control_images.to(BF16).contiguous()
        h, w = latents.shape[-2:]
        self._pool = (h, w) != (64, 64) and self.use_size_512                    # :664-670
        self.images = pool_control_images(images) if self._pool else images
        self.adapter_ctx = self.image_embeddings[-1].unsqueeze(0).contiguous()  # the LAST sample's embedding (:715)
        # step-invariant work, hoisted (exact): single-token contexts, ControlNet text K/V and image embedding
        cache_static_context(self.adapter, self.adapter_ctx, single_token_rows=1)
        cache_static_context(self.controlnet, self.cn_embeds)
        self.controlnet.cache_static_cond(self.images)
        self._init_key_frames(2 * b, f, dev)
        self._graphs = {}
        self.step_index = 0

    def _state(self):
        return [self.latents, self.model_in, self.row, self.cn_t]

    def _load_step(self, i):
        self.row.copy_(self.table[i])
        self.cn_t.copy_(self.cn_table[i:i + 1])

    def _body(self, scale):
        b, f = self.batch, self.frames
        t = self.row[0:1]
        lat2 = torch.cat([self.model_in, self.model_in], dim=0)                  # (2B, F, 4, h, w) CFG duplication
        n = 2 * b * f
        h, w = lat2.shape[-2:]
        down = mid = None
        if scale != 0:  # cond_scale == 0 (:748): ControlNet outputs are exactly zero, see _video_adapter
            ctrl_in = lat2.reshape(n, 4, h, w)                                   # "b f c h w -> (b f) c h w"
            if self._pool:
                ctrl_in = pool_controlnet_input(ctrl_in)
            down, mid = self.controlnet(ctrl_in, self.cn_t, encoder_hidden_states=self.cn_embeds,
                                        controlnet_cond=self.images, conditioning_scale=scale, guess_mode=False,
                                        return_dict=False, skip_conv_in=self.skip_conv_in,
                                        skip_time_emb=self.skip_time_emb)
        down_a, mid_a = self._video_adapter(down, mid, self.cn_t, n, (8, 8) if self._pool else (h // 8, w // 8))
        # the UNet takes "(b f) c h w" residuals as well as the reference's 5-D form; no rearrange needed
        unet_in = torch.cat([lat2, self.image_latents], dim=2)                   # (2B, F, 8, h, w) channel concat (:755)
        eps = self.unet(unet_in, t, encoder_hidden_states=self.image_embeddings, added_time_ids=self.added_time_ids,
                        down_block_additional_residuals=down_a, mid_block_additional_residual=mid_a,
                        return_dict=False)[0]                                    # (2B, F, 4, h, w)
        ops.cfg_euler_v(eps[:b].contiguous(), eps[b:].contiguous(), self.latents, self.guidance, f, self.row,
                        latents_out=self.latents, model_in_next=self.model_in)

