"""H100 host mirror of the SDXL ``UNet2DConditionModel`` (stock diffusers class in the reference: instantiated at
/root/reference/inference.py:369, called at sdxl/pipelines/sdxl_controlnet_adapter_pipeline.py:1356-1366 with the
adapter's ``down_block_additional_residuals`` and ``mid_block_additional_residual=0``).

Same state-dict keys as the diffusers model (stabilityai/stable-diffusion-xl-base-1.0 unet).  Skip connections are
consumed as a second TMA source of the up-block convolutions / GroupNorms, so ``torch.cat`` never materialises.
"""
from __future__ import annotations

import torch
from torch import nn

from . import ops
from .persistence import PretrainedMixin
from .layers import (BF16, Conv2d, DownBlock2D, MidBlock2D, Norm, ResnetBlock2D, TimestepEmbedding, Transformer2DModel,
                     UpBlock2D, _ConfigDict, add_residual, add_skip_residuals, shared_timestep, to_channels_last_bf16)


def _attentions(n, heads, c, depth, cross_dim):
    if depth == 0:
        return None
    return [Transformer2DModel(heads, c // heads, c, depth, cross_dim, True) for _ in range(n)]


def _down(cin, cout, temb, eps, heads, depth, cross_dim, add_downsample):
    return DownBlock2D([ResnetBlock2D(cin if i == 0 else cout, cout, temb, eps) for i in range(2)],
                       _attentions(2, heads, cout, depth, cross_dim),
                       Conv2d(cout, cout, 3, stride=2) if add_downsample else None)


def _up(cin, cout, prev, temb, eps, heads, depth, cross_dim, add_upsample):
    # resnet i: the previous output (prev, then cout channels) + the skip it pops (cout, cout, then cin channels)
    return UpBlock2D([ResnetBlock2D((prev if i == 0 else cout) + (cin if i == 2 else cout), cout, temb, eps)
                      for i in range(3)],
                     _attentions(3, heads, cout, depth, cross_dim),
                     Conv2d(cout, cout, 3) if add_upsample else None)


class UNet2DConditionModel(PretrainedMixin, nn.Module):
    def __init__(self, in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280),
                 transformer_layers_per_block=(1, 2, 10), attention_head_dim=(5, 10, 20), cross_attention_dim=2048,
                 addition_time_embed_dim=256, projection_class_embeddings_input_dim=2816, norm_eps=1e-5,
                 flip_sin_to_cos=True, freq_shift=0, **_ignored):
        super().__init__()
        if tuple(block_out_channels) != (320, 640, 1280):
            raise NotImplementedError("only the SDXL-base UNet topology is implemented")
        self.config = _ConfigDict(in_channels=in_channels, out_channels=out_channels, sample_size=128,
                                  block_out_channels=tuple(block_out_channels), cross_attention_dim=cross_attention_dim,
                                  addition_time_embed_dim=addition_time_embed_dim,
                                  projection_class_embeddings_input_dim=projection_class_embeddings_input_dim)
        c0, c1, c2 = block_out_channels
        temb = c0 * 4
        heads = tuple(attention_head_dim)
        depth = transformer_layers_per_block
        xd = cross_attention_dim
        self.flip_sin_to_cos, self.freq_shift = flip_sin_to_cos, freq_shift
        self.conv_in = Conv2d(in_channels, c0, 3)
        self.time_embedding = TimestepEmbedding(c0, temb)
        self.add_embedding = TimestepEmbedding(projection_class_embeddings_input_dim, temb)
        # down: DownBlock2D, CrossAttnDownBlock2D(depth 2), CrossAttnDownBlock2D(depth 10)
        self.down_blocks = nn.ModuleList([
            _down(c0, c0, temb, norm_eps, heads[0], 0, xd, True),
            _down(c0, c1, temb, norm_eps, heads[1], depth[1], xd, True),
            _down(c1, c2, temb, norm_eps, heads[2], depth[2], xd, False)])
        self.mid_block = MidBlock2D([ResnetBlock2D(c2, c2, temb, norm_eps), ResnetBlock2D(c2, c2, temb, norm_eps)],
                                    [Transformer2DModel(heads[2], c2 // heads[2], c2, depth[2], xd, True)])
        self.up_blocks = nn.ModuleList([
            _up(c1, c2, c2, temb, norm_eps, heads[2], depth[2], xd, True),
            _up(c0, c1, c2, temb, norm_eps, heads[1], depth[1], xd, True),
            _up(c0, c0, c1, temb, norm_eps, heads[0], 0, xd, False)])
        self.conv_norm_out = Norm(c0, norm_eps)
        self.conv_out = Conv2d(c0, out_channels, 3)

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, timestep_cond=None, cross_attention_kwargs=None,
                added_cond_kwargs=None, down_block_additional_residuals=None, mid_block_additional_residual=None,
                return_dict: bool = False, **_ignored):
        n = sample.shape[0]
        dev = sample.device
        if sample.shape[-1] % 4 != 0 or sample.shape[-2] % 4 != 0:
            raise NotImplementedError("latent resolution must be a multiple of 4")
        # time + SDXL micro-conditioning embedding
        t = shared_timestep(timestep, dev)
        t_emb = self.time_embedding(ops.timestep_embedding(t, 320, flip_sin_to_cos=self.flip_sin_to_cos,
                                                           freq_shift=float(self.freq_shift)))  # [1, 1280]
        text_embeds = added_cond_kwargs["text_embeds"].to(BF16)
        time_ids = added_cond_kwargs["time_ids"].to(device=dev, dtype=torch.float32).reshape(-1).contiguous()
        tid = ops.timestep_embedding(time_ids, self.config.addition_time_embed_dim,
                                     flip_sin_to_cos=self.flip_sin_to_cos, freq_shift=float(self.freq_shift))
        add_in = torch.cat([text_embeds, tid.reshape(n, -1)], dim=-1).contiguous()  # [n, 2816] (host-side glue)
        aug = self.add_embedding(add_in)
        emb = ops.add(t_emb.expand(n, -1).contiguous(), aug)
        temb_act = ops.silu(emb)
        ctx = encoder_hidden_states.to(BF16).contiguous()

        x = self.conv_in(to_channels_last_bf16(sample, 8))
        skips = [x]
        for blk in self.down_blocks:
            x, outs = blk(x, temb_act, ctx)
            skips += outs
        is_controlnet = mid_block_additional_residual is not None and down_block_additional_residuals is not None
        if is_controlnet:  # only the first 9 of the adapter's 12 tensors are consumed
            add_skip_residuals(skips, down_block_additional_residuals)
        x = self.mid_block(x, temb_act, ctx)
        if is_controlnet and isinstance(mid_block_additional_residual, torch.Tensor):
            x = add_residual(x, mid_block_additional_residual)
        for blk in self.up_blocks:
            x = blk(x, temb_act, ctx, skips=skips)
        y = self.conv_out(self.conv_norm_out.group_norm(x, silu=True))          # [n, h, w, 8]
        return (ops.nhwc_to_nchw(y, self.config.out_channels),)
