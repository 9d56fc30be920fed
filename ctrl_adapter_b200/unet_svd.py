"""H100 host mirror of the Stable-Video-Diffusion UNet with the reference's residual injection
(/root/reference/svd/models/unets/unet_spatio_temporal_condition.py: constructor :71-245, forward :357-526, injection
:457-471 and :485-490; instantiated at inference.py:360, called at svd/pipelines/svd_controlnet_adapter_pipeline.py).

Same state-dict keys as the reference class (stabilityai/stable-video-diffusion-img2vid[-xt] unet).  Everything runs on
the kernels the adapter's video path already uses: frames stay in (clip, frame, pixel) token order, the temporal ResNet
is a (3,1,1) multi-tap GEMM with 5-D GroupNorm statistics, the temporal transformer uses the frame-axis attention
kernel, both AlphaBlender mixes are fused into the producing GEMM epilogue, and the skip concat of the up blocks is a
second TMA source.  The conditioning of this backbone is ONE CLIP image token per clip, so every cross-attention
collapses exactly to a per-clip broadcast vector to_out(to_v(ctx)) (same identity as the adapter's quirk Q5).

Parity: GPU groups `svd`, `svd_loop` (tests/test_video_paths_gpu.py) against the restated reference class, which is
bit-exact against the reference's own class; the composition is also checked on CPU over an emulation of the op layer
(tests/test_host_emulated_cpu.py).
"""
from __future__ import annotations

import torch
from torch import nn

from . import ops
from .persistence import PretrainedMixin
from .adapter import AlphaBlender, TemporalBasicTransformerBlock, TemporalResnetBlock
from .layers import (BF16, BasicTransformerBlock, Conv2d, DownBlock2D, Linear, MidBlock2D, Norm, ResnetBlock2D,
                     TimestepEmbedding, UpBlock2D, _ConfigDict, add_residual, add_skip_residuals, shared_timestep,
                     to_channels_last_bf16)


class SpatioTemporalResBlock(nn.Module):
    """diffusers SpatioTemporalResBlock: spatial ResnetBlock2D -> TemporalResnetBlock, blended by a learned alpha."""

    def __init__(self, cin: int, cout: int, temb: int, eps: float):
        super().__init__()
        self.spatial_res_block = ResnetBlock2D(cin, cout, temb, eps)
        self.temporal_res_block = TemporalResnetBlock(cout, temb, eps)
        self.time_mixer = AlphaBlender(0.5)

    def forward(self, x, temb_act, frames: int, x2=None):
        s = self.spatial_res_block(x, temb_act, x2=x2)
        return self.temporal_res_block(s, frames, temb_act, blend_src=s, blend_alpha=self.time_mixer.alpha())


class TransformerSpatioTemporalModel(nn.Module):
    """diffusers TransformerSpatioTemporalModel for a single-token context (the only form this backbone is driven with)."""

    def __init__(self, heads: int, head_dim: int, in_channels: int, num_layers: int, cross_dim: int):
        super().__init__()
        if head_dim != 64:
            raise NotImplementedError("attention_head_dim must be 64 (released SVD UNet)")
        inner = heads * head_dim
        self.in_channels, self.inner = in_channels, inner
        self.norm = Norm(in_channels, 1e-6)
        self.proj_in = Linear(in_channels, inner)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(inner, heads, head_dim, cross_dim)
                                                 for _ in range(num_layers)])
        self.temporal_transformer_blocks = nn.ModuleList([TemporalBasicTransformerBlock(inner, heads, head_dim, cross_dim)
                                                          for _ in range(num_layers)])
        self.time_pos_embed = TimestepEmbedding(in_channels, in_channels * 4, out_dim=in_channels)
        self.time_mixer = AlphaBlender(0.5)
        self.proj_out = Linear(inner, in_channels)

    def forward(self, x, ctx_vecs, frames: int):
        """x [B*F, H, W, C]; ctx_vecs [B, Dc]: the clip's single context token (identical for all of its frames, which
        is also what the temporal blocks use: `time_context` = the first frame's context, transformer_temporal.py)."""
        n, h, w, c = x.shape
        hw = h * w
        clips = n // frames
        tok = self.norm.group_norm(x, silu=False).reshape(n * hw, c)
        hs = self.proj_in(tok)
        frames_idx = torch.arange(frames, device=x.device, dtype=torch.float32).repeat(clips)
        emb = self.time_pos_embed(ops.timestep_embedding(frames_idx, c))  # [B*F, C]; C == inner for this backbone
        alpha = self.time_mixer.alpha()
        for blk, tblk in zip(self.transformer_blocks, self.temporal_transformer_blocks):
            h3 = hs.reshape(n, hw, self.inner)
            h1 = blk.attn1(blk.norm1.layer_norm(h3), residual=h3).reshape(n * hw, self.inner)
            cv = blk.attn2.single_token_output(ctx_vecs)  # [B, inner]
            n3, hsum = blk.norm3.layer_norm(h1, add_rowvec=cv, rows_per_vec=frames * hw, return_sum=True)
            hs = blk.ff(n3, residual=hsum)
            hs = tblk(hs, emb, frames, hw, ctx_vecs, blend_src=hs, blend_alpha=alpha)
        out = self.proj_out(hs, residual=x.reshape(n * hw, c))
        return out.reshape(n, h, w, c)


def _transformers(n, heads, c, depth, cross_dim):
    return [TransformerSpatioTemporalModel(heads, c // heads, c, depth, cross_dim) for _ in range(n)]


def _down(cin, cout, temb, eps, heads, depth, cross_dim, add_downsample, cross_attn):
    return DownBlock2D([SpatioTemporalResBlock(cin if i == 0 else cout, cout, temb, eps) for i in range(2)],
                       _transformers(2, heads, cout, depth, cross_dim) if cross_attn else None,
                       Conv2d(cout, cout, 3, stride=2) if add_downsample else None)


def _up(cin, cout, prev, temb, eps, heads, depth, cross_dim, add_upsample, cross_attn):
    # resnet i: the previous output (prev, then cout channels) + the skip it pops (cout, cout, then cin channels)
    return UpBlock2D([SpatioTemporalResBlock((prev if i == 0 else cout) + (cin if i == 2 else cout), cout, temb, eps)
                      for i in range(3)],
                     _transformers(3, heads, cout, depth, cross_dim) if cross_attn else None,
                     Conv2d(cout, cout, 3) if add_upsample else None)


class UNetSpatioTemporalConditionModel(PretrainedMixin, nn.Module):
    def __init__(self, sample_size=None, in_channels: int = 8, out_channels: int = 4,
                 down_block_types=("CrossAttnDownBlockSpatioTemporal", "CrossAttnDownBlockSpatioTemporal",
                                   "CrossAttnDownBlockSpatioTemporal", "DownBlockSpatioTemporal"),
                 up_block_types=("UpBlockSpatioTemporal", "CrossAttnUpBlockSpatioTemporal",
                                 "CrossAttnUpBlockSpatioTemporal", "CrossAttnUpBlockSpatioTemporal"),
                 block_out_channels=(320, 640, 1280, 1280), addition_time_embed_dim: int = 256,
                 projection_class_embeddings_input_dim: int = 768, layers_per_block=2, cross_attention_dim=1024,
                 transformer_layers_per_block=1, num_attention_heads=(5, 10, 10, 20), num_frames: int = 25):
        super().__init__()
        if len(down_block_types) != len(up_block_types) or len(block_out_channels) != len(down_block_types):
            raise ValueError("Must provide the same number of `down_block_types`, `up_block_types` and "
                             "`block_out_channels`")  # unet_spatio_temporal_condition.py:103-112
        heads = (num_attention_heads,) * 4 if isinstance(num_attention_heads, int) else tuple(num_attention_heads)
        if (tuple(block_out_channels) != (320, 640, 1280, 1280) or layers_per_block != 2
                or transformer_layers_per_block != 1
                or tuple(down_block_types) != ("CrossAttnDownBlockSpatioTemporal",) * 3 + ("DownBlockSpatioTemporal",)):
            raise NotImplementedError("only the released SVD UNet topology is implemented")
        if any(c // h != 64 for c, h in zip(block_out_channels, heads)):
            # the checkpoints' config.json has num_attention_heads = [5, 10, 20, 20] (head dim 64 everywhere); the class
            # default (5, 10, 10, 20) would give the third stage 128-wide heads, which the frame-axis kernel does not do
            raise NotImplementedError("attention head dim must be 64: pass num_attention_heads=(5, 10, 20, 20) as the "
                                      "released stable-video-diffusion configs do")
        self.config = _ConfigDict(sample_size=sample_size, in_channels=in_channels, out_channels=out_channels,
                                  down_block_types=tuple(down_block_types), up_block_types=tuple(up_block_types),
                                  block_out_channels=tuple(block_out_channels),
                                  addition_time_embed_dim=addition_time_embed_dim,
                                  projection_class_embeddings_input_dim=projection_class_embeddings_input_dim,
                                  layers_per_block=layers_per_block, cross_attention_dim=cross_attention_dim,
                                  transformer_layers_per_block=transformer_layers_per_block,
                                  num_attention_heads=heads, num_frames=num_frames)
        c0, c1, c2, c3 = block_out_channels
        temb = c0 * 4
        xd = cross_attention_dim
        self.conv_in = Conv2d(in_channels, c0, 3)
        self.time_embedding = TimestepEmbedding(c0, temb)
        self.add_embedding = TimestepEmbedding(projection_class_embeddings_input_dim, temb)
        # class-default eps of diffusers v0.27.2 (get_down_block / get_up_block do not forward resnet_eps to these types)
        h0, h1, h2, h3 = heads
        self.down_blocks = nn.ModuleList([
            _down(c0, c0, temb, 1e-6, h0, 1, xd, True, True),
            _down(c0, c1, temb, 1e-6, h1, 1, xd, True, True),
            _down(c1, c2, temb, 1e-6, h2, 1, xd, True, True),
            _down(c2, c3, temb, 1e-5, h3, 1, xd, False, False)])
        self.mid_block = MidBlock2D([SpatioTemporalResBlock(c3, c3, temb, 1e-5) for _ in range(2)],
                                    _transformers(1, h3, c3, 1, xd))
        self.up_blocks = nn.ModuleList([
            _up(c2, c3, c3, temb, 1e-6, h3, 1, xd, True, False),
            _up(c1, c2, c3, temb, 1e-6, h2, 1, xd, True, True),
            _up(c0, c1, c2, temb, 1e-6, h1, 1, xd, True, True),
            _up(c0, c0, c1, temb, 1e-6, h0, 1, xd, False, True)])
        self.conv_norm_out = Norm(c0, 1e-5)
        self.conv_out = Conv2d(c0, out_channels, 3)

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, added_time_ids, down_block_additional_residuals=None,
                mid_block_additional_residual=None, return_dict: bool = False):
        if sample.dim() != 5:
            raise ValueError("sample must be (batch, frames, channels, height, width)")
        b, f = sample.shape[:2]
        dev = sample.device
        if sample.shape[-1] % 8 != 0 or sample.shape[-2] % 8 != 0:
            raise NotImplementedError("latent resolution must be a multiple of 8")
        if encoder_hidden_states.shape[1] != 1:
            raise NotImplementedError("the SVD backbone is driven with one image-embedding token per clip")
        # 1. time: one timestep for the whole batch (:393-406) + per-sample added_time_ids embedding (:414-418)
        t = shared_timestep(timestep, dev)
        t_emb = self.time_embedding(ops.timestep_embedding(t, 320))  # [1, 1280]
        ids = added_time_ids.to(device=dev, dtype=torch.float32).reshape(-1).contiguous()
        tid = ops.timestep_embedding(ids, self.config.addition_time_embed_dim).reshape(b, -1).contiguous()
        aug = self.add_embedding(tid)
        emb = ops.add(t_emb.expand(b, -1).contiguous(), aug)  # [B, 1280]
        temb_act = ops.silu(emb).repeat_interleave(f, dim=0).contiguous()  # one row per frame-image (:427)
        ctx_vecs = encoder_hidden_states.to(BF16).reshape(b, -1).contiguous()  # [B, Dc]; every frame shares it (:430)

        # 2. flatten frames, conv_in
        x = self.conv_in(to_channels_last_bf16(sample.flatten(0, 1), 8))
        skips = [x]
        for blk in self.down_blocks:
            x, outs = blk(x, temb_act, ctx_vecs, f)
            skips += outs
        if down_block_additional_residuals is not None:  # 4-D or 5-D residuals (:457-471, :485-490)
            add_skip_residuals(skips, down_block_additional_residuals)
        x = self.mid_block(x, temb_act, ctx_vecs, f)
        if isinstance(mid_block_additional_residual, torch.Tensor):
            x = add_residual(x, mid_block_additional_residual)
        for blk in self.up_blocks:
            x = blk(x, temb_act, ctx_vecs, f, skips=skips)
        y = self.conv_out(self.conv_norm_out.group_norm(x, silu=True))         # [B*F, H, W, 8]
        out = ops.nhwc_to_nchw(y, self.config.out_channels)  # [B*F, 4, H, W]
        out = out.reshape(b, f, *out.shape[1:])
        return (out,)
