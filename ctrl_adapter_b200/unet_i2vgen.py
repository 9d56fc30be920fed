"""H100 host mirror of ``I2VGenXLUNet`` (/root/reference/i2vgen_xl/models/unets/unet_i2vgen_xl.py:104-761, a diffusers
v0.27.2 copy with ``down_block_additional_residuals`` / ``mid_block_additional_residual`` added at :681-695, :709-714).

Same constructor defaults, forward signature and state-dict keys.  Video activations are ``[B*F, H, W, C]`` bf16 in
(clip, frame, pixel) order; the reference's (b f) <-> (b c f h w) <-> (b*hw f c) permutes are folded into kernel
addressing (temporal conv taps, 5-D GroupNorm statistics, frame-axis attention).

The conditioning that does not depend on the timestep -- image-latent encoder (:637-651), context tokens (:598-635) and
the fps embedding (:589-590) -- is computed by ``prepare_conditioning`` and cached (the reference recomputes it every
step; hoisting is exact).
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import nn

from . import ops
from .persistence import PretrainedMixin
from .layers import (cache_static_context, BF16, Attention, Conv2d, FeedForward, Linear, Norm, Packable, ResnetBlock2D,
                     TemporalConv, TimestepEmbedding, Transformer2DModel, _ConfigDict, add_residual, add_skip_residuals,
                     shared_timestep, to_channels_last_bf16)
from .ops import ACT_SILU


def frame_self_attention(attn: Attention, x_norm, residual, clips: int, frames: int, hw: int):
    """Self-attention over the F frames of every pixel.  x_norm/residual: [clips*frames*hw, D] rows in
    (clip, frame, pixel) order; head dim 64."""
    pk = attn.packed()
    inner = attn.heads * 64
    qkv = ops.linear(x_norm, pk["wqkv"])
    o = ops.temporal_attention(qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:], clips, frames, hw,
                               attn.heads, 0.125, row_stride=3 * inner)
    return ops.linear(o, pk["wo"], pk["bo"], residual=residual)


class _Seq(nn.Module):
    """nn.Sequential-style container whose children keep the reference's numeric names (e.g. conv1.0 / conv1.2)."""

    def __init__(self, **mods):
        super().__init__()
        for k, m in mods.items():
            self.add_module(k.lstrip("_"), m)

    def __getitem__(self, i):
        return getattr(self, str(i))


class TemporalConvLayer(nn.Module):
    """diffusers TemporalConvLayer: 4 x (GroupNorm(5-D stats) - SiLU - Conv3d(3,1,1)) + identity."""

    def __init__(self, c: int):
        super().__init__()
        self.conv1 = _Seq(_0=Norm(c, 1e-5), _2=TemporalConv(c, c))
        self.conv2 = _Seq(_0=Norm(c, 1e-5), _3=TemporalConv(c, c))
        self.conv3 = _Seq(_0=Norm(c, 1e-5), _3=TemporalConv(c, c))
        self.conv4 = _Seq(_0=Norm(c, 1e-5), _3=TemporalConv(c, c))

    def forward(self, x, frames: int):
        h = self.conv1[2](self.conv1[0].group_norm(x, silu=True, imgs_per_sample=frames), frames)
        h = self.conv2[3](self.conv2[0].group_norm(h, silu=True, imgs_per_sample=frames), frames)
        h = self.conv3[3](self.conv3[0].group_norm(h, silu=True, imgs_per_sample=frames), frames)
        return self.conv4[3](self.conv4[0].group_norm(h, silu=True, imgs_per_sample=frames), frames, residual=x)


class TransformerTemporalModel(nn.Module):
    """GroupNorm(5-D stats, eps 1e-6) - proj_in - BasicTransformerBlock with two frame-axis self-attentions
    (double_self_attention=True) - proj_out - + residual."""

    def __init__(self, heads: int, head_dim: int, in_channels: int):
        super().__init__()
        if head_dim != 64:
            raise NotImplementedError("temporal attention kernel is specialised for head dim 64")
        inner = heads * head_dim
        self.norm = Norm(in_channels, 1e-6)
        self.proj_in = Linear(in_channels, inner)
        blk = nn.Module()
        blk.norm1 = Norm(inner, 1e-5)
        blk.attn1 = Attention(inner, None, heads, head_dim)
        blk.norm2 = Norm(inner, 1e-5)
        blk.attn2 = Attention(inner, None, heads, head_dim)  # double self-attention: no cross context
        blk.norm3 = Norm(inner, 1e-5)
        blk.ff = FeedForward(inner)
        self.transformer_blocks = nn.ModuleList([blk])
        self.proj_out = Linear(inner, in_channels)

    def forward(self, x, frames: int):
        n, h, w, c = x.shape
        clips, hw = n // frames, h * w
        t = self.proj_in(self.norm.group_norm(x, silu=False, imgs_per_sample=frames).reshape(n * hw, c))
        blk = self.transformer_blocks[0]
        t = frame_self_attention(blk.attn1, blk.norm1.layer_norm(t), t, clips, frames, hw)
        t = frame_self_attention(blk.attn2, blk.norm2.layer_norm(t), t, clips, frames, hw)
        t = blk.ff(blk.norm3.layer_norm(t), residual=t)
        return self.proj_out(t, residual=x.reshape(n * hw, c)).reshape(n, h, w, c)


class _Block3D(nn.Module):
    """Down / mid / up block of unet_3d_blocks: [resnet, temp_conv, (spatial transformer, temporal transformer)] x L."""

    def __init__(self, kind: str, cin: int, cout: int, prev: int, temb: int, cross_dim: int, has_attn: bool,
                 layers: int, sampler: Optional[str]):
        super().__init__()
        self.kind, self.has_cross_attention = kind, has_attn
        heads = cout // 64
        rs, tcs, ats, tas = [], [], [], []
        for i in range(layers):
            if kind == "down":
                rin = cin if i == 0 else cout
            elif kind == "mid":
                rin = cout
            else:
                rin = (prev if i == 0 else cout) + (cin if i == layers - 1 else cout)
            rs.append(ResnetBlock2D(rin, cout, temb, 1e-5))
            tcs.append(TemporalConvLayer(cout))
        n_attn = (layers - 1) if kind == "mid" else layers
        if has_attn:
            for _ in range(n_attn):
                ats.append(Transformer2DModel(heads, 64, cout, 1, cross_dim, True))
                tas.append(TransformerTemporalModel(heads, 64, cout))
        self.resnets = nn.ModuleList(rs)
        self.temp_convs = nn.ModuleList(tcs)
        if has_attn:
            self.attentions = nn.ModuleList(ats)
            self.temp_attentions = nn.ModuleList(tas)
        self.downsamplers = self.upsamplers = None
        if sampler == "down":
            ds = nn.Module()
            ds.conv = Conv2d(cout, cout, 3, stride=2)
            self.downsamplers = nn.ModuleList([ds])
        elif sampler == "up":
            us = nn.Module()
            us.conv = Conv2d(cout, cout, 3)
            self.upsamplers = nn.ModuleList([us])

    def forward(self, x, temb_act, ctx, frames, skips=None, kv_div=1):
        outs = []
        if self.kind == "mid":
            x = self.temp_convs[0](self.resnets[0](x, temb_act), frames)
            for attn, tattn, r, tc in zip(self.attentions, self.temp_attentions, self.resnets[1:], self.temp_convs[1:]):
                x = tattn(attn(x, ctx, kv_batch_div=kv_div), frames)
                x = tc(r(x, temb_act), frames)
            return x
        for i, (r, tc) in enumerate(zip(self.resnets, self.temp_convs)):
            x = r(x, temb_act, x2=skips.pop() if self.kind == "up" else None)
            x = tc(x, frames)
            if self.has_cross_attention:
                x = self.temp_attentions[i](self.attentions[i](x, ctx, kv_batch_div=kv_div), frames)
            outs.append(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0].conv(x)
            outs.append(x)
        if self.upsamplers is not None:
            x = self.upsamplers[0].conv(ops.upsample2x(x))
        return (x, outs) if self.kind == "down" else x


class _LatentTemporalEncoder(Packable):
    """I2VGenXLTransformerTemporalEncoder (dim 4, 2 heads x 4, GELU FF 4->16->4): one tiny fused kernel."""

    def __init__(self, dim: int = 4):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=1e-5)
        attn = nn.Module()
        attn.to_q = nn.Linear(dim, 2 * dim, bias=False)
        attn.to_k = nn.Linear(dim, 2 * dim, bias=False)
        attn.to_v = nn.Linear(dim, 2 * dim, bias=False)
        attn.to_out = nn.ModuleList([nn.Linear(2 * dim, dim), nn.Dropout(0.0)])
        self.attn1 = attn
        ff = nn.Module()
        g = nn.Module()
        g.proj = nn.Linear(dim, 4 * dim)
        ff.net = nn.ModuleList([g, nn.Dropout(0.0), nn.Linear(4 * dim, dim)])
        self.ff = ff

    def pack(self):
        bf = lambda t: t.detach().to(BF16).float().reshape(-1)  # noqa: E731  (values as the bf16 model holds them)
        a, f = self.attn1, self.ff
        return torch.cat([bf(self.norm1.weight), bf(self.norm1.bias), bf(a.to_q.weight), bf(a.to_k.weight),
                          bf(a.to_v.weight), bf(a.to_out[0].weight), bf(a.to_out[0].bias), bf(f.net[0].proj.weight),
                          bf(f.net[0].proj.bias), bf(f.net[2].weight), bf(f.net[2].bias)]).contiguous()

    def forward(self, x, clips, frames):
        return ops.i2vgen_latent_encoder(x, clips, frames, self.packed())


class I2VGenXLUNet(PretrainedMixin, nn.Module):
    def __init__(self, sample_size=None, in_channels: int = 4, out_channels: int = 4,
                 down_block_types=("CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "DownBlock3D"),
                 up_block_types=("UpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D"),
                 block_out_channels=(320, 640, 1280, 1280), layers_per_block: int = 2, norm_num_groups: int = 32,
                 cross_attention_dim: int = 1024, attention_head_dim=64, num_attention_heads=None):
        super().__init__()
        if (in_channels, out_channels, layers_per_block, norm_num_groups, attention_head_dim) != (4, 4, 2, 32, 64) or \
                tuple(block_out_channels) != (320, 640, 1280, 1280):
            raise NotImplementedError("only the released I2VGen-XL UNet topology is implemented")
        self.config = _ConfigDict(sample_size=sample_size, in_channels=in_channels, out_channels=out_channels,
                                  block_out_channels=tuple(block_out_channels), cross_attention_dim=cross_attention_dim,
                                  attention_head_dim=attention_head_dim)
        c = block_out_channels
        temb = c[0] * 4
        self.conv_in = Conv2d(2 * in_channels, c[0], 3)
        self.transformer_in = TransformerTemporalModel(8, 64, c[0])
        self.image_latents_proj_in = _Seq(_0=Conv2d(4, 16, 3), _2=Conv2d(16, 16, 3), _4=Conv2d(16, 4, 3))
        self.image_latents_temporal_encoder = _LatentTemporalEncoder(4)
        self.image_latents_context_embedding = _Seq(_0=Conv2d(4, 32, 3), _3=Conv2d(32, 64, 3, stride=2),
                                                    _5=Conv2d(64, cross_attention_dim, 3, stride=2))
        self.time_embedding = TimestepEmbedding(c[0], temb)
        self.context_embedding = _Seq(_0=Linear(cross_attention_dim, temb), _2=Linear(temb, cross_attention_dim * 4))
        self.fps_embedding = _Seq(_0=Linear(c[0], temb), _2=Linear(temb, temb))
        self.down_blocks = nn.ModuleList([
            _Block3D("down", c[0], c[0], 0, temb, cross_attention_dim, True, 2, "down"),
            _Block3D("down", c[0], c[1], 0, temb, cross_attention_dim, True, 2, "down"),
            _Block3D("down", c[1], c[2], 0, temb, cross_attention_dim, True, 2, "down"),
            _Block3D("down", c[2], c[3], 0, temb, cross_attention_dim, False, 2, None)])
        self.mid_block = _Block3D("mid", c[3], c[3], 0, temb, cross_attention_dim, True, 2, None)
        self.up_blocks = nn.ModuleList([
            _Block3D("up", c[2], c[3], c[3], temb, cross_attention_dim, False, 3, "up"),
            _Block3D("up", c[1], c[2], c[3], temb, cross_attention_dim, True, 3, "up"),
            _Block3D("up", c[0], c[1], c[2], temb, cross_attention_dim, True, 3, "up"),
            _Block3D("up", c[0], c[0], c[1], temb, cross_attention_dim, True, 3, None)])
        self.conv_norm_out = Norm(c[0], 1e-5)
        self.conv_out = Conv2d(c[0], out_channels, 3)
        self._cond_cache = None

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def prepare_conditioning(self, fps, image_latents, image_embeddings, encoder_hidden_states):
        """Timestep-independent conditioning (unet_i2vgen_xl.py:589-590, :598-651).  image_latents (b,4,f,h,w)."""
        b, ch, f, h, w = image_latents.shape
        dev = image_latents.device
        fps_t = fps.to(device=dev, dtype=torch.float32).reshape(-1).contiguous()
        fe = self.fps_embedding[2](self.fps_embedding[0](ops.timestep_embedding(fps_t, 320), act=ACT_SILU))  # [b,1280]
        # context tokens: text (77) + image-latent tokens (64) + image-embedding tokens (4)
        e = self.image_latent_tokens(image_latents[:, :, 0].contiguous())      # first frame (b,4,h,w) -> [b,8,8,1024]
        ie = image_embeddings.to(BF16).reshape(-1, image_embeddings.shape[-1]).contiguous()
        ie = self.context_embedding[2](self.context_embedding[0](ie, act=ACT_SILU))
        ie = ie.reshape(-1, self.config.in_channels, self.config.cross_attention_dim)
        ctx = torch.cat([encoder_hidden_states.to(BF16), e.reshape(b, -1, e.shape[-1]), ie], dim=1).contiguous()
        # image latents of every frame -> conv stack -> per-pixel temporal encoder
        il = image_latents.permute(0, 2, 1, 3, 4).reshape(b * f, ch, h, w).contiguous()
        x = self.image_latents_proj_in[0](to_channels_last_bf16(il, 8), act=ACT_SILU)
        x = self.image_latents_proj_in[2](x, act=ACT_SILU)
        x = self.image_latents_proj_in[4](x)                                  # [b*f, h, w, 8] (4 real channels)
        il_enc = self.image_latents_temporal_encoder(x, b, f)
        return dict(fps_emb=fe, ctx=ctx, il_enc=il_enc, frames=f)

    def image_latent_tokens(self, il_first):
        """The first frame's image latents (b, 4, h, w) -> conv -> 32x32 pool -> two stride-2 convs: [b, 8, 8, 1024]
        channels-last, 64 context tokens per clip (unet_i2vgen_xl.py:210-218, :624)."""
        e = self.image_latents_context_embedding[0](to_channels_last_bf16(il_first, 8), act=ACT_SILU)
        e = ops.avgpool(e, 32, 32) if tuple(e.shape[1:3]) != (32, 32) else e  # AdaptiveAvgPool2d((32, 32))
        e = self.image_latents_context_embedding[3](e, act=ACT_SILU)
        return self.image_latents_context_embedding[5](e)

    def _conditioning(self, fps, image_latents, image_embeddings, encoder_hidden_states):
        key = tuple((t.data_ptr(), t._version, tuple(t.shape)) for t in (fps, image_latents, image_embeddings,
                                                                           encoder_hidden_states))
        if self._cond_cache is None or self._cond_cache[0] != key:
            self._cond_cache = (key, self.prepare_conditioning(fps, image_latents, image_embeddings, encoder_hidden_states))
            # the assembled context is as step-invariant as its inputs: project every cross attention's K/V once
            cache_static_context(self, self._cond_cache[1]["ctx"])
        return self._cond_cache[1]

    @torch.no_grad()
    def forward(self, sample, timestep, fps, image_latents, image_embeddings=None, encoder_hidden_states=None,
                timestep_cond=None, cross_attention_kwargs=None, return_dict: bool = False,
                down_block_additional_residuals=None, mid_block_additional_residual=None):
        b, ch, f, h, w = sample.shape
        cond = self._conditioning(fps, image_latents, image_embeddings, encoder_hidden_states)
        n = b * f
        dev = sample.device
        t = shared_timestep(timestep, dev)
        t_emb = self.time_embedding(ops.timestep_embedding(t, 320))            # [1, 1280]
        emb = ops.add(t_emb.expand(b, -1).contiguous(), cond["fps_emb"])       # [b, 1280]
        if b > 1:
            emb = emb.repeat_interleave(f, dim=0).contiguous()                 # one row per frame-sample
        temb_act = ops.silu(emb)
        ctx = cond["ctx"]
        # pre-process: cat(sample, encoded image latents) on channels -> conv_in -> temporal transformer
        s_nhwc = sample.to(BF16).permute(0, 2, 3, 4, 1).reshape(n, h, w, ch)
        x = torch.cat([s_nhwc, cond["il_enc"][..., :ch]], dim=-1).contiguous()  # [n, h, w, 8] latent-sized glue
        x = self.conv_in(x)
        x = self.transformer_in(x, f)
        skips = [x]
        for blk in self.down_blocks:
            x, outs = blk(x, temb_act, ctx, f, kv_div=f)
            skips += outs
        if down_block_additional_residuals is not None:  # 4-D or 5-D residuals (reference :681-695, :709-714)
            add_skip_residuals(skips, down_block_additional_residuals)
        x = self.mid_block(x, temb_act, ctx, f, kv_div=f)
        if mid_block_additional_residual is not None:
            x = add_residual(x, mid_block_additional_residual)
        for blk in self.up_blocks:
            x = blk(x, temb_act, ctx, f, skips=skips, kv_div=f)
        y = self.conv_out(self.conv_norm_out.group_norm(x, silu=True))         # [n, h, w, 8]
        out = ops.nhwc_to_nchw(y, ch)                                          # (b f) c h w
        return (out.reshape(b, f, ch, h, w).permute(0, 2, 1, 3, 4),)

