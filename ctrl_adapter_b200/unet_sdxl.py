"""H100 host mirror of the SDXL ``UNet2DConditionModel`` (stock diffusers class in the reference: instantiated at
/root/reference/inference.py:369, called at sdxl/pipelines/sdxl_controlnet_adapter_pipeline.py:1356-1366 with the
adapter's ``down_block_additional_residuals`` and ``mid_block_additional_residual=0``).

Same state-dict keys as the diffusers model (stabilityai/stable-diffusion-xl-base-1.0 unet).  Skip connections are
consumed as a second TMA source of the up-block convolutions / GroupNorms, so ``torch.cat`` never materialises.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import nn

from . import ops
from .persistence import PretrainedMixin
from .adapter import _ConfigDict, as_nchw, shared_timestep, to_channels_last_bf16
from .layers import BF16, Conv2d, Norm, ResnetBlock2D, TimestepEmbedding, Transformer2DModel


class _Down(nn.Module):
    def __init__(self, cin, cout, temb, eps, heads, depth, cross_dim, add_downsample):
        super().__init__()
        self.has_cross_attention = depth > 0
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, temb, eps) for i in range(2)])
        if depth > 0:
            self.attentions = nn.ModuleList([Transformer2DModel(heads, cout // heads, cout, depth, cross_dim, True)
                                             for _ in range(2)])
        self.downsamplers = None
        if add_downsample:
            ds = nn.Module()
            ds.conv = Conv2d(cout, cout, 3, stride=2)
            self.downsamplers = nn.ModuleList([ds])

    def forward(self, x, temb_act, ctx):
        outs = []
        for i, r in enumerate(self.resnets):
            x = r(x, temb_act)
            if self.has_cross_attention:
                x = self.attentions[i](x, ctx)
            outs.append(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0].conv(x)
            outs.append(x)
        return x, outs


class _Mid(nn.Module):
    def __init__(self, c, temb, eps, heads, depth, cross_dim):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, temb, eps), ResnetBlock2D(c, c, temb, eps)])
        self.attentions = nn.ModuleList([Transformer2DModel(heads, c // heads, c, depth, cross_dim, True)])

    def forward(self, x, temb_act, ctx):
        x = self.resnets[0](x, temb_act)
        x = self.attentions[0](x, ctx)
        return self.resnets[1](x, temb_act)


class _Up(nn.Module):
    def __init__(self, cin, cout, prev, temb, eps, heads, depth, cross_dim, add_upsample):
        super().__init__()
        self.has_cross_attention = depth > 0
        rs = []
        for i in range(3):
            skip_c = cin if i == 2 else cout
            in_c = prev if i == 0 else cout
            rs.append(ResnetBlock2D(in_c + skip_c, cout, temb, eps))
        self.resnets = nn.ModuleList(rs)
        if depth > 0:
            self.attentions = nn.ModuleList([Transformer2DModel(heads, cout // heads, cout, depth, cross_dim, True)
                                             for _ in range(3)])
        self.upsamplers = None
        if add_upsample:
            us = nn.Module()
            us.conv = Conv2d(cout, cout, 3)
            self.upsamplers = nn.ModuleList([us])

    def forward(self, x, skips, temb_act, ctx):
        for i, r in enumerate(self.resnets):
            x = r(x, temb_act, x2=skips.pop())
            if self.has_cross_attention:
                x = self.attentions[i](x, ctx)
        if self.upsamplers is not None:
            x = self.upsamplers[0].conv(ops.upsample2x(x))
        return x


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
        self.flip_sin_to_cos, self.freq_shift = flip_sin_to_cos, freq_shift
        self.conv_in = Conv2d(in_channels, c0, 3)
        self.time_embedding = TimestepEmbedding(c0, temb)
        self.add_embedding = TimestepEmbedding(projection_class_embeddings_input_dim, temb)
        # down: DownBlock2D, CrossAttnDownBlock2D(depth 2), CrossAttnDownBlock2D(depth 10)
        self.down_blocks = nn.ModuleList([
            _Down(c0, c0, temb, norm_eps, heads[0], 0, cross_attention_dim, True),
            _Down(c0, c1, temb, norm_eps, heads[1], transformer_layers_per_block[1], cross_attention_dim, True),
            _Down(c1, c2, temb, norm_eps, heads[2], transformer_layers_per_block[2], cross_attention_dim, False)])
        self.mid_block = _Mid(c2, temb, norm_eps, heads[2], transformer_layers_per_block[2], cross_attention_dim)
        self.up_blocks = nn.ModuleList([
            _Up(c1, c2, c2, temb, norm_eps, heads[2], transformer_layers_per_block[2], cross_attention_dim, True),
            _Up(c0, c1, c2, temb, norm_eps, heads[1], transformer_layers_per_block[1], cross_attention_dim, True),
            _Up(c0, c0, c1, temb, norm_eps, heads[0], 0, cross_attention_dim, False)])
        self.conv_norm_out = Norm(c0, norm_eps)
        self.conv_out = Conv2d(c0, out_channels, 3)
        self._conv_out_pad = None

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    def _conv_out_packed(self):
        """conv_out has 4 output channels; the kernel stores 16-byte vectors, so its weight rows are zero padded to 8."""
        key = self.conv_out._key()
        if self._conv_out_pad is None or self._conv_out_pad[0] != key:
            w, b = self.conv_out.packed()
            co = w.shape[0]
            cp = (co + 7) // 8 * 8
            wp = torch.zeros((cp, w.shape[1]), device=w.device, dtype=w.dtype)
            wp[:co] = w
            bp = torch.zeros(cp, device=w.device, dtype=torch.float32)
            bp[:co] = b
            self._conv_out_pad = (key, wp, bp)
        return self._conv_out_pad[1], self._conv_out_pad[2]

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
        if is_controlnet:  # zip() truncation: only the first 9 of the adapter's 12 tensors are consumed
            for i, (s, r) in enumerate(zip(skips, down_block_additional_residuals)):
                skips[i] = ops.add(s, to_channels_last_bf16(r))
        x = self.mid_block(x, temb_act, ctx)
        if is_controlnet and isinstance(mid_block_additional_residual, torch.Tensor):
            x = ops.add(x, to_channels_last_bf16(mid_block_additional_residual))
        for blk in self.up_blocks:
            x = blk(x, skips, temb_act, ctx)
        h = self.conv_norm_out.group_norm(x, silu=True)
        w, b = self._conv_out_packed()
        y = ops.conv2d(h, w, b, ksize=3)
        out = ops.nhwc_to_nchw(y, self.config.out_channels)
        return (out,)
