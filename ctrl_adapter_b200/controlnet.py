"""H100 host mirror of the frozen SD1.5 ControlNet (/root/reference/controlnet/controlnet.py:107-881) and of
``MultiControlNetModel`` (/root/reference/controlnet/multicontrolnet.py:45-99).

Same constructor kwargs (default SD1.5 topology), forward signature (including the reference's ``skip_conv_in`` /
``skip_time_emb`` additions) and state-dict keys.  Outputs are logical NCHW tensors in channels_last memory format.
"""
from __future__ import annotations

from typing import List, Optional, Tuple, Union

import torch
from torch import nn

from . import ops
from .persistence import PretrainedMixin
from .adapter import _ConfigDict, as_nchw, shared_timestep, to_channels_last_bf16
from .layers import BF16, Conv2d, ResnetBlock2D, TimestepEmbedding, Transformer2DModel
from .ops import ACT_SILU


class ControlNetConditioningEmbedding(nn.Module):
    """controlnet.py:62-104: conv_in, (conv, conv stride 2) x3, conv_out; SiLU fused into each conv's epilogue."""

    def __init__(self, out_channels: int, conditioning_channels: int = 3, block_out_channels=(16, 32, 96, 256)):
        super().__init__()
        self.conv_in = Conv2d(conditioning_channels, block_out_channels[0], 3)
        self.blocks = nn.ModuleList([])
        for i in range(len(block_out_channels) - 1):
            cin, cout = block_out_channels[i], block_out_channels[i + 1]
            self.blocks.append(Conv2d(cin, cin, 3))
            self.blocks.append(Conv2d(cin, cout, 3, stride=2))
        self.conv_out = Conv2d(block_out_channels[-1], out_channels, 3)

    # the 8- / 16- / 32-channel stride-1 convolutions at full image resolution run with 8 / 4 / 2 adjacent pixels folded
    # into the channel axis (layers.Conv2d.forward_folded) instead of padding every tap to 64 channels; the GPU test
    # group `fold` checks the folded form against the padded one
    def forward(self, cond_nhwc8):
        e = self.conv_in.forward_folded(cond_nhwc8, act=ACT_SILU)
        for blk in self.blocks:
            e = blk.forward_folded(e, act=ACT_SILU) if blk.stride == 1 else blk(e, act=ACT_SILU)
        return self.conv_out(e)


class _DownBlock(nn.Module):
    def __init__(self, cin, cout, temb, eps, heads, cross_dim, has_attn, add_downsample, layers=2):
        super().__init__()
        self.has_cross_attention = has_attn
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, temb, eps) for i in range(layers)])
        if has_attn:
            self.attentions = nn.ModuleList([Transformer2DModel(heads, cout // heads, cout, 1, cross_dim, False)
                                             for _ in range(layers)])
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


class _MidBlock(nn.Module):
    def __init__(self, c, temb, eps, heads, cross_dim):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, temb, eps), ResnetBlock2D(c, c, temb, eps)])
        self.attentions = nn.ModuleList([Transformer2DModel(heads, c // heads, c, 1, cross_dim, False)])

    def forward(self, x, temb_act, ctx):
        x = self.resnets[0](x, temb_act)
        x = self.attentions[0](x, ctx)
        return self.resnets[1](x, temb_act)


class ControlNetModel(PretrainedMixin, nn.Module):
    def __init__(self, in_channels: int = 4, conditioning_channels: int = 3, flip_sin_to_cos: bool = True,
                 freq_shift: int = 0,
                 down_block_types=("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
                 mid_block_type: Optional[str] = "UNetMidBlock2DCrossAttn", only_cross_attention=False,
                 block_out_channels=(320, 640, 1280, 1280), layers_per_block: int = 2, downsample_padding: int = 1,
                 mid_block_scale_factor: float = 1, act_fn: str = "silu", norm_num_groups: Optional[int] = 32,
                 norm_eps: float = 1e-5, cross_attention_dim: int = 1280, transformer_layers_per_block=1,
                 encoder_hid_dim=None, encoder_hid_dim_type=None, attention_head_dim=8, num_attention_heads=None,
                 use_linear_projection: bool = False, class_embed_type=None, addition_embed_type=None,
                 addition_time_embed_dim=None, num_class_embeds=None, upcast_attention: bool = False,
                 resnet_time_scale_shift: str = "default", projection_class_embeddings_input_dim=None,
                 controlnet_conditioning_channel_order: str = "rgb",
                 conditioning_embedding_out_channels=(16, 32, 96, 256), global_pool_conditions: bool = False,
                 addition_embed_type_num_heads: int = 64):
        super().__init__()
        if len(block_out_channels) != len(down_block_types):  # controlnet.py:230-233
            raise ValueError("Must provide the same number of `block_out_channels` as `down_block_types`.")
        unsupported = dict(only_cross_attention=only_cross_attention, use_linear_projection=use_linear_projection,
                           class_embed_type=class_embed_type, addition_embed_type=addition_embed_type,
                           encoder_hid_dim=encoder_hid_dim, num_class_embeds=num_class_embeds,
                           upcast_attention=upcast_attention)
        for k, v in unsupported.items():
            if v:
                raise NotImplementedError(f"{k}={v}: only the SD1.5 ControlNet topology is on the Ctrl-Adapter hot path")
        if act_fn != "silu" or norm_num_groups != 32 or resnet_time_scale_shift != "default" or layers_per_block != 2:
            raise NotImplementedError("non-default SD1.5 ControlNet hyper-parameters")
        heads = num_attention_heads or attention_head_dim
        if not isinstance(heads, int):
            raise NotImplementedError("per-block head counts")
        self.config = _ConfigDict(in_channels=in_channels, conditioning_channels=conditioning_channels,
                                  block_out_channels=tuple(block_out_channels), cross_attention_dim=cross_attention_dim,
                                  controlnet_conditioning_channel_order=controlnet_conditioning_channel_order,
                                  global_pool_conditions=global_pool_conditions, addition_embed_type=None,
                                  attention_head_dim=attention_head_dim, norm_eps=norm_eps)
        self.flip_sin_to_cos, self.freq_shift = flip_sin_to_cos, freq_shift
        c0 = block_out_channels[0]
        temb = c0 * 4
        self.conv_in = Conv2d(in_channels, c0, 3)
        self.time_embedding = TimestepEmbedding(c0, temb)
        self.controlnet_cond_embedding = ControlNetConditioningEmbedding(c0, conditioning_channels,
                                                                         conditioning_embedding_out_channels)
        self.down_blocks = nn.ModuleList([])
        self.controlnet_down_blocks = nn.ModuleList([Conv2d(c0, c0, 1)])
        out_c = c0
        for i, t in enumerate(down_block_types):
            in_c, out_c = out_c, block_out_channels[i]
            final = i == len(block_out_channels) - 1
            self.down_blocks.append(_DownBlock(in_c, out_c, temb, norm_eps, heads, cross_attention_dim,
                                               t == "CrossAttnDownBlock2D", not final))
            for _ in range(layers_per_block + (0 if final else 1)):
                self.controlnet_down_blocks.append(Conv2d(out_c, out_c, 1))
        self.controlnet_mid_block = Conv2d(block_out_channels[-1], block_out_channels[-1], 1)
        if mid_block_type != "UNetMidBlock2DCrossAttn":
            raise NotImplementedError(mid_block_type)
        self.mid_block = _MidBlock(block_out_channels[-1], temb, norm_eps, heads, cross_attention_dim)
        self._static_cond = None

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    @torch.no_grad()
    def cache_static_cond(self, controlnet_cond: torch.Tensor):
        """Computes controlnet_cond_embedding(controlnet_cond) once; forward() reuses it for this tensor object."""
        c = controlnet_cond
        if self.config.controlnet_conditioning_channel_order == "bgr":
            c = torch.flip(c, dims=[1])
        emb = self.controlnet_cond_embedding(to_channels_last_bf16(c, 8))
        self._static_cond = (controlnet_cond, controlnet_cond._version, self.conv_in._key(), emb)

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_scale: float = 1.0,
                class_labels=None, timestep_cond=None, attention_mask=None, added_cond_kwargs=None,
                cross_attention_kwargs=None, guess_mode: bool = False, return_dict: bool = True,
                skip_conv_in: bool = False, skip_time_emb: bool = False):
        order = self.config.controlnet_conditioning_channel_order
        cond_obj = controlnet_cond
        if order == "bgr":
            controlnet_cond = torch.flip(controlnet_cond, dims=[1])
        elif order != "rgb":
            raise ValueError(f"unknown `controlnet_conditioning_channel_order`: {order}")
        if attention_mask is not None or class_labels is not None or timestep_cond is not None:
            raise NotImplementedError("attention_mask / class_labels / timestep_cond are unused on the Ctrl-Adapter path")
        if self.config.global_pool_conditions:
            raise NotImplementedError("global_pool_conditions")
        n = sample.shape[0]
        dev = sample.device
        c0 = self.config.block_out_channels[0]
        # 1. time (exact t -- unlike the adapter the ControlNet does not round t to bf16; controlnet.py:751-758)
        t = shared_timestep(timestep, dev)
        emb = self.time_embedding(ops.timestep_embedding(t, c0, flip_sin_to_cos=self.flip_sin_to_cos,
                                                         freq_shift=float(self.freq_shift)))
        temb_act = ops.silu(emb)
        if skip_time_emb:
            temb_act = torch.zeros_like(temb_act)  # SiLU(0) == 0
        # 2. pre-process (controlnet.py:802-817)
        # The conditioning embedding depends only on the control image (controlnet.py:94-104, :815), not on t or the
        # latents: a loop registers the image once (cache_static_cond) and every later call with that very tensor
        # object reuses the embedding.  sample = conv_in(sample) + embedding (controlnet.py:802-817): the add is fused
        # into conv_in's epilogue (bf16 sum of two bf16 tensors, same rounding as the reference's `sample + cond`).
        st = self._static_cond
        if st is not None and st[0] is cond_obj and st[1] == cond_obj._version and st[2] == self.conv_in._key():
            cond_emb = st[3]
        else:
            cond_emb = self.controlnet_cond_embedding(to_channels_last_bf16(controlnet_cond, 8))
        x = cond_emb if skip_conv_in else self.conv_in(to_channels_last_bf16(sample, 8), residual=cond_emb)
        ctx = encoder_hidden_states.to(BF16).contiguous()
        # 3./4. down + mid
        res = [x]
        for blk in self.down_blocks:
            x, outs = blk(x, temb_act, ctx)
            res += outs
        x = self.mid_block(x, temb_act, ctx)
        # 5./6. zero convs and scaling (controlnet.py:852-868)
        if guess_mode:
            scales = (torch.logspace(-1, 0, len(res) + 1) * conditioning_scale).tolist()
        else:
            scales = [float(conditioning_scale)] * (len(res) + 1)
        down = [as_nchw(blk(r, out_scale=s)) for r, blk, s in zip(res, self.controlnet_down_blocks, scales)]
        mid = as_nchw(self.controlnet_mid_block(x, out_scale=scales[-1]))
        if not return_dict:
            return (down, mid)
        return _ConfigDict(down_block_res_samples=down, mid_block_res_sample=mid)


class MultiControlNetModel(nn.Module):
    """multicontrolnet.py:45-99: per-net outputs are returned as lists (the router weights them afterwards);
    ``zip`` truncates to the shorter of (images, scales, nets)."""

    def __init__(self, controlnets: Union[List[ControlNetModel], Tuple[ControlNetModel]]):
        super().__init__()
        self.nets = nn.ModuleList(controlnets)

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_scale, class_labels=None,
                timestep_cond=None, attention_mask=None, added_cond_kwargs=None, cross_attention_kwargs=None,
                guess_mode: bool = False, return_dict: bool = True, skip_conv_in: bool = False,
                skip_time_emb: bool = False):
        downs, mids = [], []
        for image, scale, net in zip(controlnet_cond, conditioning_scale, self.nets):
            d, m = net(sample=sample, timestep=timestep, encoder_hidden_states=encoder_hidden_states,
                       controlnet_cond=image, conditioning_scale=scale, guess_mode=guess_mode, return_dict=False,
                       skip_conv_in=skip_conv_in, skip_time_emb=skip_time_emb)
            downs.append(d)
            mids.append(m)
        return downs, mids
