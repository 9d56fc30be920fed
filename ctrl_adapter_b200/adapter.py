"""H100 host mirror of the reference adapter modules.

``ControlNetAdapter`` / ``AdapterSpatioTemporal`` / ``ControlNetRouter`` keep the reference's constructor kwargs,
forward signatures, return structures and state-dict keys (/root/reference/model/ctrl_adapter.py:17-44,171-224;
model/adapter_spatial_temporal.py:11-37,175-292; model/ctrl_router.py:49-58,85-112), so ``inference.py`` and the
pipelines can use them unchanged.  Tensors cross the boundary as logical NCHW; physically everything is channels-last
(``torch.channels_last`` outputs, zero-copy when the producer is another module of this package).

All arithmetic runs in the sm_90a kernels (see layers.py / ops.py); there is no PyTorch fallback.
"""
from __future__ import annotations

import json
import os
from typing import List, Optional

import torch
from torch import nn

from . import ops
from .persistence import PretrainedMixin
from .layers import (BF16, BasicTransformerBlock, FeedForward, Attention, Linear, Norm, Packable, ResnetBlock2D,
                     TemporalConv, TimestepEmbedding, _ConfigDict, as_nchw, shared_timestep, to_channels_last_bf16)
from .ops import ACT_NONE


class AlphaBlender(Packable):
    """Learned mix factor; alpha = sigmoid(mix_factor) in the parameter dtype (image_only_indicator is all zeros on
    this path, adapter_spatial_temporal.py:200).  The blend itself is fused into the producing GEMM's epilogue, which
    computes alpha * x_spatial + bf16(1 - alpha) * x_temporal.
    switch_spatial_to_temporal_mix (the temporal VAE decoder's blocks): diffusers replaces alpha by 1 - alpha first, in
    the activation dtype, so the value handed to the epilogue is bf16(1 - bf16(sigmoid(mix_factor)))."""

    def __init__(self, alpha: float = 0.5, switch_spatial_to_temporal_mix: bool = False):
        super().__init__()
        self.switch_spatial_to_temporal_mix = switch_spatial_to_temporal_mix
        self.mix_factor = nn.Parameter(torch.tensor([alpha]))

    def pack(self):
        a = torch.sigmoid(self.mix_factor.detach().to(BF16))
        if self.switch_spatial_to_temporal_mix:
            a = 1.0 - a
        return a.float().contiguous()

    def alpha(self):
        return self.packed()


class TemporalResnetBlock(nn.Module):
    """diffusers TemporalResnetBlock on [B*F, H, W, C]: 5-D GroupNorm statistics over (C/32, F, H, W), Conv3d (3,1,1).
    temb_channels None (the temporal VAE decoder): no time-embedding projection."""

    def __init__(self, c: int, temb_channels: Optional[int], eps: float):
        super().__init__()
        self.norm1 = Norm(c, eps)
        self.conv1 = TemporalConv(c, c)
        self.time_emb_proj = Linear(temb_channels, c) if temb_channels is not None else None
        self.norm2 = Norm(c, eps)
        self.conv2 = TemporalConv(c, c)

    def forward(self, x, frames: int, temb_act, blend_src=None, blend_alpha=None):
        tp = self.time_emb_proj(temb_act) if self.time_emb_proj is not None else None  # [B*F or 1, C]
        h = self.norm1.group_norm(x, silu=True, imgs_per_sample=frames)
        h = self.conv1(h, frames, rowvec=tp)
        h = self.norm2.group_norm(h, silu=True, imgs_per_sample=frames)
        return self.conv2(h, frames, residual=x, blend_src=blend_src, blend_alpha=blend_alpha)


class TemporalBasicTransformerBlock(nn.Module):
    """diffusers TemporalBasicTransformerBlock with dim == time_mix_inner_dim (is_res).  Tokens stay in
    (clip, frame, pixel) order; only the frame-axis attention kernel regroups them."""

    def __init__(self, dim: int, heads: int, head_dim: int, cross_dim: int):
        super().__init__()
        self.heads = heads
        self.norm_in = Norm(dim, 1e-5)
        self.ff_in = FeedForward(dim, dim_out=dim)
        self.norm1 = Norm(dim, 1e-5)
        self.attn1 = Attention(dim, None, heads, head_dim)
        self.norm2 = Norm(dim, 1e-5)
        self.attn2 = Attention(dim, cross_dim, heads, head_dim)
        self.norm3 = Norm(dim, 1e-5)
        self.ff = FeedForward(dim)

    def forward(self, h, emb, frames: int, hw: int, ctx_vec, blend_src=None, blend_alpha=None, ctx_src=None):
        """h [B*F*HW, D]; emb [B*F, D] frame-position embedding added first (adapter_spatial_temporal.py:279);
        ctx_vec [1, Dc] (or [B, Dc], one per clip): single-token context (cross attention over one key collapses to
        to_out(to_v(ctx)))."""
        rows, d = h.shape
        clips = rows // (frames * hw)
        n_in, x = self.norm_in.layer_norm(h, add_rowvec=emb, rows_per_vec=hw, return_sum=True)
        x = self.ff_in(n_in, residual=x)
        pk = self.attn1.packed()
        inner = self.heads * 64
        qkv = ops.linear(self.norm1.layer_norm(x), pk["wqkv"])
        o = ops.temporal_attention(qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:], clips, frames, hw,
                                   self.heads, 0.125, row_stride=3 * inner)
        x = ops.linear(o, pk["wo"], pk["bo"], residual=x)
        cv = self.attn2.single_token_output(ctx_vec, src=ctx_src)  # [1, D], or one row per clip ([B, D]: SVD backbone)
        rpv = rows
        if cv.shape[0] > 1:
            # diffusers quirk kept by the reference (transformer_temporal.py / adapter_spatial_temporal.py:247-250):
            # `time_context` is built in (pixel, clip) order but consumed by sequences in (clip, pixel) order, so the
            # frame sequence of (clip b, pixel p) attends to the context of clip (b*hw + p) % B.  Distinct contexts only
            # occur on the SVD path (CFG pair); the gather below is host-side glue over a [B, D] table.
            if cv.shape[0] != clips:
                raise ValueError("one context row per clip expected")
            idx = torch.arange(clips * hw, device=cv.device) % clips
            cv = cv[idx].reshape(clips, 1, hw, d).expand(clips, frames, hw, d).reshape(rows, d).contiguous()
            rpv = 1
        n3, x = self.norm3.layer_norm(x, add_rowvec=cv, rows_per_vec=rpv, return_sum=True)
        # NB diffusers applies norm2 before attn2 but with a single key the (normalised) query is irrelevant
        return self.ff(n3, residual=x, blend_src=blend_src, blend_alpha=blend_alpha)


class AdapterSpatioTemporal(nn.Module):
    """One Ctrl-Adapter block (adapter_spatial_temporal.py:10-292)."""

    def __init__(self, in_channels: int, out_channels: int, num_layers: int = 1, add_spatial_resnet: bool = True,
                 add_temporal_resnet: bool = True, add_spatial_transformer: bool = True,
                 add_temporal_transformer: bool = True, eps: float = 1e-6, temporal_eps: float = None,
                 merge_factor: float = 0.5, merge_strategy="learned_with_images",
                 switch_spatial_to_temporal_mix: bool = False, up_sampling_scale: float = 1.0,
                 cross_attention_dim: int = 1024, num_attention_heads: int = 8, attention_head_dim: int = 64):
        super().__init__()
        if in_channels != out_channels:
            raise ValueError("the reference only instantiates adapters with in_channels == out_channels")
        if merge_strategy != "learned_with_images" or switch_spatial_to_temporal_mix:
            raise ValueError("only the released merge configuration is supported")
        if attention_head_dim != 64:
            raise ValueError("attention_head_dim must be 64")
        c = in_channels
        self.channels = c
        self.num_attention_heads = c // attention_head_dim
        self.num_layers = num_layers
        self.up_sampling_scale = up_sampling_scale
        self.add_spatial_resnet = add_spatial_resnet
        self.add_temporal_resnet = add_temporal_resnet
        self.add_spatial_transformer = add_spatial_transformer
        self.add_temporal_transformer = add_temporal_transformer
        self.add_resnet_time_mixer = add_spatial_resnet and add_temporal_resnet
        self.add_transformer_time_mixer = add_spatial_transformer and add_temporal_transformer
        if up_sampling_scale not in (1, 1.0, 2, 2.0):
            raise ValueError("up_sampling_scale must be 1 or 2")
        if add_spatial_resnet or add_temporal_resnet:
            self.resnet_time_embedding = TimestepEmbedding(c, c)
        if add_spatial_transformer or add_temporal_transformer:
            self.norm = Norm(c, 1e-6)
            self.inner_dim = num_attention_heads * attention_head_dim  # 512 (reference quirk Q1)
            if add_temporal_transformer:
                self.transformer_time_embedding = TimestepEmbedding(c, self.inner_dim)
            self.proj_in = Linear(c, self.inner_dim)
            self.proj_out = Linear(self.inner_dim, c)
        te = temporal_eps if temporal_eps is not None else eps
        if add_spatial_resnet:
            self.spatial_resnets = nn.ModuleList([
                ResnetBlock2D(c, c, c, eps, use_in_shortcut=True, up=(i == 0 and up_sampling_scale > 1))
                for i in range(num_layers)])
        if add_temporal_resnet:
            self.temporal_resnets = nn.ModuleList([TemporalResnetBlock(c, c, te) for _ in range(num_layers)])
        if add_spatial_transformer:
            self.spatial_attentions = nn.ModuleList([
                BasicTransformerBlock(self.inner_dim, self.num_attention_heads, 64, cross_attention_dim)
                for _ in range(num_layers)])
        if add_temporal_transformer:
            self.temporal_attentions = nn.ModuleList([
                TemporalBasicTransformerBlock(self.inner_dim, self.num_attention_heads, 64, cross_attention_dim)
                for _ in range(num_layers)])
        if self.add_resnet_time_mixer:
            self.resnets_time_mixer = nn.ModuleList([AlphaBlender(merge_factor) for _ in range(num_layers)])
        if self.add_transformer_time_mixer:
            self.transformers_time_mixer = nn.ModuleList([AlphaBlender(merge_factor) for _ in range(num_layers)])

    # x: physical NHWC bf16; t: fp32 device vector; ctx: [N|1, L, Dc] bf16
    def forward_nhwc(self, x, num_frames: int, t: torch.Tensor, ctx: torch.Tensor):
        n, h, w, c = x.shape
        if not (self.add_spatial_resnet and self.add_spatial_transformer):
            raise NotImplementedError("released adapters always have the spatial resnet and transformer")
        if self.add_temporal_resnet != self.add_temporal_transformer:
            raise NotImplementedError("temporal resnet / transformer are enabled together in the released configs")
        t1 = t[:1].contiguous()  # every frame-sample shares the step's timestep (forward() refuses anything else)
        for i in range(self.num_layers):
            # resnet time embedding: Timesteps(bf16-rounded t) -> MLP -> SiLU (shared by both resnets)
            temb = self.resnet_time_embedding(ops.timestep_embedding(t1, c, round_t_bf16=True))
            temb_act = ops.silu(temb)
            x = self.spatial_resnets[i](x, temb_act)
            n, h, w, c = x.shape
            if self.add_temporal_resnet:
                x = self.temporal_resnets[i](x, num_frames, temb_act, blend_src=x,
                                             blend_alpha=self.resnets_time_mixer[i].alpha())
            hw = h * w
            tok = self.norm.group_norm(x, silu=False).reshape(n * hw, c)
            hcur = self.proj_in(tok).reshape(n, hw, self.inner_dim)
            blk = self.spatial_attentions[i]
            if ctx.shape[1] == 1:
                # single-token context (video path, i2vgen pipeline :1048): cross attention == broadcast vector.  The
                # pipelines pass ONE row ([1, 1, D]) for all samples; several distinct rows are refused, not truncated
                if ctx.shape[0] != 1:
                    raise NotImplementedError("single-token context: pass one [1, 1, D] row shared by every sample "
                                              "(image_embeddings[-1].unsqueeze(0) in the reference pipelines)")
                hcur = blk.attn1(blk.norm1.layer_norm(hcur), residual=hcur)
                cv = blk.attn2.single_token_output(ctx.reshape(-1, ctx.shape[-1])[:1].contiguous(), src=ctx)
                n3, hsum = blk.norm3.layer_norm(hcur.reshape(n * hw, -1), add_rowvec=cv, rows_per_vec=n * hw,
                                                return_sum=True)
                hs = blk.ff(n3, residual=hsum)
            else:
                cx = ctx if ctx.shape[0] == n else ctx.expand(n, -1, -1).contiguous()
                hs = blk(hcur, cx).reshape(n * hw, self.inner_dim)
            if self.add_temporal_transformer:
                frames_idx = torch.arange(num_frames, device=x.device, dtype=torch.float32).repeat(n // num_frames)
                emb = self.transformer_time_embedding(ops.timestep_embedding(frames_idx, c))  # [N, 512]
                hs = self.temporal_attentions[i](hs, emb, num_frames, hw,
                                                 ctx.reshape(-1, ctx.shape[-1])[:1].contiguous(), blend_src=hs,
                                                 blend_alpha=self.transformers_time_mixer[i].alpha(), ctx_src=ctx)
            x = self.proj_out(hs, residual=x.reshape(n * hw, c)).reshape(n, h, w, c)
        return x

    def forward(self, hidden_states, num_frames: int, timestep=None, encoder_hidden_states=None, sparsity_masking=None):
        x = to_channels_last_bf16(hidden_states)
        t = shared_timestep(timestep, x.device)
        ctx = _prep_ctx(encoder_hidden_states)
        return as_nchw(self.forward_nhwc(x, num_frames, t, ctx))


def _prep_ctx(ehs: torch.Tensor) -> torch.Tensor:
    if ehs.dim() == 2:  # adapter_spatial_temporal.py:240-241
        ehs = ehs.unsqueeze(1)
    return ehs.to(BF16).contiguous()


class ControlNetAdapter(PretrainedMixin, nn.Module):
    """ctrl_adapter.py:12-224 (num_repeats == 1)."""

    config_name = "config.json"

    def __init__(self, backbone_model_name, num_blocks=2, num_frames=8, num_adapters_per_location=3,
                 cross_attention_dim=None, adapter_type="spatial_temporal_resnet_transformer", add_spatial_resnet=True,
                 add_temporal_resnet=False, add_spatial_transformer=True, add_temporal_transformer=False,
                 add_adapter_location_A=False, add_adapter_location_B=False, add_adapter_location_C=False,
                 add_adapter_location_D=False, add_adapter_location_M=False, num_repeats=1, out_channels=None):
        super().__init__()
        if num_repeats != 1:
            raise NotImplementedError("num_repeats > 1 is experimental in the reference and unused by released configs")
        self.config = _ConfigDict(
            backbone_model_name=backbone_model_name, num_blocks=num_blocks, num_frames=num_frames,
            num_adapters_per_location=num_adapters_per_location, cross_attention_dim=cross_attention_dim,
            adapter_type=adapter_type, add_spatial_resnet=add_spatial_resnet, add_temporal_resnet=add_temporal_resnet,
            add_spatial_transformer=add_spatial_transformer, add_temporal_transformer=add_temporal_transformer,
            add_adapter_location_A=add_adapter_location_A, add_adapter_location_B=add_adapter_location_B,
            add_adapter_location_C=add_adapter_location_C, add_adapter_location_D=add_adapter_location_D,
            add_adapter_location_M=add_adapter_location_M, num_repeats=num_repeats, out_channels=out_channels)
        self.add_adapter_location_A = add_adapter_location_A
        self.add_adapter_location_B = add_adapter_location_B
        self.add_adapter_location_C = add_adapter_location_C
        self.add_adapter_location_D = add_adapter_location_D
        self.add_adapter_location_M = add_adapter_location_M
        self.num_adapters_per_location = num_adapters_per_location
        self.num_repeats = num_repeats
        self.adapter_type = adapter_type
        chans = self.get_down_block_channels()
        scale = 2 if backbone_model_name in ["sdxl"] else 1
        self.num_adapters = len(chans)
        kw = dict(cross_attention_dim=cross_attention_dim, num_layers=num_blocks, up_sampling_scale=scale,
                  add_spatial_resnet=add_spatial_resnet, add_temporal_resnet=add_temporal_resnet,
                  add_spatial_transformer=add_spatial_transformer, add_temporal_transformer=add_temporal_transformer)
        self.down_blocks_adapter = nn.ModuleList([AdapterSpatioTemporal(in_channels=c, out_channels=c, **kw) for c in chans])
        self.mid_block_adapter = AdapterSpatioTemporal(in_channels=1280, out_channels=1280, **kw) \
            if add_adapter_location_M else None

    def get_down_block_ids(self):
        ids = []
        n = self.num_adapters_per_location
        for flag, m in ((self.add_adapter_location_A, {3: [0, 1, 2], 2: [0, 2], 1: [2]}),
                        (self.add_adapter_location_B, {3: [3, 4, 5], 2: [3, 5], 1: [5]}),
                        (self.add_adapter_location_C, {3: [6, 7, 8], 2: [6, 8], 1: [8]}),
                        (self.add_adapter_location_D, {3: [9, 10, 11], 2: [9, 11], 1: [11]})):
            if flag:
                ids += m.get(n, [])
        return ids

    def get_down_block_channels(self):
        ch = []
        n = self.num_adapters_per_location
        if self.add_adapter_location_A:
            ch = [320] * n
        if self.add_adapter_location_B:
            ch += {3: [320, 640, 640], 2: [320, 640], 1: [640]}[n]
        if self.add_adapter_location_C:
            ch += {3: [640, 1280, 1280], 2: [640, 1280], 1: [1280]}[n]
        if self.add_adapter_location_D:
            ch += [1280] * n
        return ch

    @torch.no_grad()
    def forward(self, down_block_res_samples, mid_block_res_sample=None, sparsity_masking=None, num_frames=None,
                timestep=None, encoder_hidden_states=None):
        ids = self.get_down_block_ids()
        dev = down_block_res_samples[0].device
        n = down_block_res_samples[0].shape[0]
        t = shared_timestep(timestep, dev)
        ctx = _prep_ctx(encoder_hidden_states)
        out: List[torch.Tensor] = []
        cur = 0
        for i in range(12):
            if i in ids:
                x = to_channels_last_bf16(down_block_res_samples[i])
                out.append(as_nchw(self.down_blocks_adapter[cur].forward_nhwc(x, num_frames, t, ctx)))
                cur += 1
            else:
                # new zero tensor of the input's shape (ctrl_adapter.py:193); consumers in this package skip it
                out.append(torch.zeros_like(down_block_res_samples[i]))
        mid = None
        if mid_block_res_sample is not None and self.mid_block_adapter is not None:
            x = to_channels_last_bf16(mid_block_res_sample)
            mid = as_nchw(self.mid_block_adapter.forward_nhwc(x, num_frames, t, ctx))
        return out, mid


    @torch.no_grad()
    def forward_mid(self, mid_block_res_sample, num_frames=None, timestep=None, encoder_hidden_states=None):
        """Only the mid-block adapter of forward() (the loops use it on the steps whose conditioning scale is 0: the
        reference then discards the down-block outputs but still injects the mid one, i2vgen pipeline :1083)."""
        if mid_block_res_sample is None or self.mid_block_adapter is None:
            return None
        x = to_channels_last_bf16(mid_block_res_sample)
        t = shared_timestep(timestep, x.device)
        return as_nchw(self.mid_block_adapter.forward_nhwc(x, num_frames, t, _prep_ctx(encoder_hidden_states)))


class ControlNetRouter(PretrainedMixin, nn.Module):
    """model/ctrl_router.py:44-112.  The 13 routers' logits live in one [13, E] fp32 device table; masked softmax for
    all of them is one warp-shuffle kernel (one warp per router)."""

    class _Simple(nn.Module):
        def __init__(self, num_experts):
            super().__init__()
            self.num_experts = num_experts
            self.wg = nn.Linear(1, num_experts, bias=False)

    class _Equal(nn.Module):
        def __init__(self, num_experts):
            super().__init__()
            self.num_experts = num_experts

    def __init__(self, num_experts=2, backbone_model_name=None, router_type="simple_weights", embedding_dim=None,
                 num_routers=12, add_mid_block_router=True, use_sparsemax=False):
        super().__init__()
        if router_type not in ("simple_weights", "equal_weights"):
            raise ValueError(f"unknown router_type {router_type}")
        self.config = _ConfigDict(num_experts=num_experts, backbone_model_name=backbone_model_name,
                                  router_type=router_type, embedding_dim=embedding_dim, num_routers=num_routers,
                                  add_mid_block_router=add_mid_block_router, use_sparsemax=use_sparsemax)
        self.num_experts = num_experts
        self.num_routers = num_routers
        self.router_type = router_type
        self.embedding_dim = embedding_dim
        self.backbone_model_name = backbone_model_name
        self.add_mid_block_router = add_mid_block_router
        self.use_sparsemax = use_sparsemax
        cls = self._Equal if router_type == "equal_weights" else self._Simple
        self.down_blocks_router = nn.ModuleList([cls(num_experts) for _ in range(num_routers)])
        if add_mid_block_router:
            self.mid_block_router = cls(num_experts)
        self.register_buffer("_anchor", torch.zeros(1), persistent=False)

    def _logits(self) -> torch.Tensor:
        mods = list(self.down_blocks_router) + ([self.mid_block_router] if self.add_mid_block_router else [])
        if self.router_type == "equal_weights":
            dev = self._anchor.device
            return torch.zeros(len(mods), self.num_experts, device=dev, dtype=torch.float32)
        # wg(1) == wg.weight[:, 0] in the parameter dtype
        return torch.stack([m.wg.weight.detach()[:, 0] for m in mods]).float().contiguous()

    @torch.no_grad()
    def forward(self, router_input=None, sparse_mask=None, fixed_weights=None):
        logits = self._logits()
        mask = None
        if sparse_mask is not None:
            mask = torch.tensor([1 if bool(m) else 0 for m in sparse_mask], dtype=torch.uint8, device=logits.device)
        w = ops.router_weights(logits, mask)
        down = w[: self.num_routers]
        mid = w[self.num_routers] if self.add_mid_block_router else None
        return down, mid


def router_merge(res_lists, weights_row: torch.Tensor, active: List[int], num_frames: int):
    """Weighted merge of E ControlNet outputs for one block (i2vgen_xl pipeline :1001-1022).
    Reproduces the reference indexing quirk Q6: ``w.repeat_interleave(F)[e]`` == ``w[e // F]``."""
    w_rep = weights_row.repeat_interleave(num_frames)
    sel = w_rep[torch.tensor(active, device=weights_row.device)].float().contiguous()
    return ops.router_merge([to_channels_last_bf16(res_lists[e]) for e in active], sel)
