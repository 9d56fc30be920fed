"""Host-side building blocks of the H100 hot path.

Each class is an ``nn.Module`` used ONLY as a parameter container with the reference's / diffusers' parameter names
(so reference checkpoints load with ``load_state_dict``); ``forward`` never calls a PyTorch op on activations -- it
launches the sm_90a kernels of ``csrc/`` through ``ops``.  Activations are channels-last bf16.

Weights are repacked once (``pack()``, lazily on first use / after ``.to()``) into the kernel layouts:
conv weights ``[Cout, taps*Cin]`` (Cout and Cin zero padded to multiples of 8), fused QKV / KV projection matrices,
GEGLU rows interleaved per 256-wide N tile, head dims zero-padded to multiples of 64 (SD1.5 ControlNet heads are
40/80/160 wide), biases as fp32.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
from torch import nn

from . import ops
from .ops import ACT_GEGLU, ACT_NONE, ACT_SILU, BF16


def _pad64(d: int) -> int:
    return (d + 63) // 64 * 64


# ------------------------------------------------------------------------------------------------
# boundary helpers
# ------------------------------------------------------------------------------------------------
def to_channels_last_bf16(x: torch.Tensor, c_pad: Optional[int] = None) -> torch.Tensor:
    """logical NCHW (any memory format, bf16/fp32) -> physical [N, H, W, C] bf16 contiguous."""
    n, c, h, w = x.shape
    cp = c if c_pad is None else c_pad
    if x.dtype == BF16 and cp == c and x.permute(0, 2, 3, 1).is_contiguous():
        return x.permute(0, 2, 3, 1)
    if not x.is_contiguous():
        x = x.contiguous()
    if x.dtype not in (BF16, torch.float32):
        x = x.float()
    return ops.nchw_to_nhwc(x, cp)


def as_nchw(y: torch.Tensor) -> torch.Tensor:
    """physical NHWC -> logical NCHW view (channels_last memory format, no copy)."""
    return y.permute(0, 3, 1, 2)


def timestep_vector(timestep, n: int, device) -> torch.Tensor:
    """The forms accepted by adapter_spatial_temporal.py:190-198 -> fp32 device vector of length n.
    A device tensor is consumed without a host sync (the reference's torch.Tensor([t]) forces one, quirk Q17)."""
    if isinstance(timestep, (int, float)):
        return torch.full((n,), float(timestep), device=device, dtype=torch.float32)
    if not isinstance(timestep, torch.Tensor):
        raise TypeError(f"unsupported timestep type {type(timestep)}")
    t = timestep.to(device=device, dtype=torch.float32)
    if t.dim() == 0 or t.numel() == 1:
        return t.reshape(1).expand(n).contiguous()
    if t.dim() == 2:
        t = t.squeeze()
    return t.reshape(-1).contiguous()


def shared_timestep(timestep, device) -> torch.Tensor:
    """The step's ONE timestep as a [1] fp32 device tensor.  Every kernel path here shares a single timestep across the
    batch (the pipelines pass a 0-dim `t`); a tensor with several entries would be silently truncated, so it is refused
    instead (checking that the entries are equal would cost a host sync per call)."""
    if isinstance(timestep, torch.Tensor) and timestep.numel() > 1:
        raise NotImplementedError("per-sample timesteps: pass the step's single timestep (0-dim / 1-element / number)")
    return timestep_vector(timestep, 1, device)[:1].contiguous()


class _ConfigDict(dict):
    __getattr__ = dict.__getitem__


class Packable(nn.Module):
    """Mixin: caches kernel-format tensors; invalidated when parameters move / change dtype."""

    def __init__(self):
        super().__init__()
        self._pk = None
        self._pk_key = None

    def _key(self):
        p = next(self.parameters(), None)
        return None if p is None else (p.device, p.data_ptr(), p._version)

    def packed(self):
        k = self._key()
        if self._pk is None or self._pk_key != k:
            with torch.no_grad():
                self._pk = self.pack()
            self._pk_key = k
        return self._pk

    def pack(self):  # pragma: no cover - overridden
        raise NotImplementedError


def _f32(t: Optional[torch.Tensor]):
    return None if t is None else t.detach().to(BF16).float().contiguous()


def _bf(t: torch.Tensor):
    return t.detach().to(BF16).contiguous()


# ------------------------------------------------------------------------------------------------
class Linear(Packable):
    def __init__(self, i: int, o: int, bias: bool = True):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(o, i))
        self.bias = nn.Parameter(torch.empty(o)) if bias else None
        nn.init.normal_(self.weight, std=1.0 / math.sqrt(i))
        if bias:
            nn.init.zeros_(self.bias)

    def pack(self):
        return _bf(self.weight), _f32(self.bias)

    def forward(self, x2d, **kw):
        w, b = self.packed()
        return ops.linear(x2d, w, b, **kw)


class Conv2d(Packable):
    """3x3 / 1x1 convolution container (PyTorch weight layout [Cout, Cin, k, k]).  `pad` None: (k-1)/2 zeros on every
    side; (0, 1) with stride 2: one zero row / column after the bottom / right edge only (diffusers Downsample2D with
    padding=0, the VAE encoder's down-sampler)."""

    def __init__(self, i: int, o: int, k: int = 3, stride: int = 1, pad: Optional[tuple] = None):
        super().__init__()
        self.k, self.stride, self.cin, self.cout = k, stride, i, o
        self.pad = pad
        self.weight = nn.Parameter(torch.empty(o, i, k, k))
        self.bias = nn.Parameter(torch.zeros(o))
        nn.init.normal_(self.weight, std=1.0 / math.sqrt(i * k * k))

    def pack(self):
        """-> weight [ceil8(Cout), taps * Kp] bf16, bias [ceil8(Cout)] fp32.  Cin is zero padded to a multiple of 8
        (e.g. 4 latent / 3 image channels: the activations are zero padded to 8).  Cout is zero padded the same way (zero
        weight rows, zero bias) because the kernel stores 16-byte vectors: the output then has ceil8(Cout) channels, of
        which the first Cout are real and the rest are zeros (e.g. a UNet's 4-channel conv_out writes [N, H, W, 8])."""
        cin_eff = (self.cin + 7) // 8 * 8
        cout_eff = (self.cout + 7) // 8 * 8
        kpad = 64 if self.stride == 2 else 8
        w = self.weight.detach()
        b = _f32(self.bias)
        if cin_eff != self.cin:
            w = torch.nn.functional.pad(w, (0, 0, 0, 0, 0, cin_eff - self.cin))
        if cout_eff != self.cout:
            w = torch.nn.functional.pad(w, (0, 0, 0, 0, 0, 0, 0, cout_eff - self.cout))
            b = torch.nn.functional.pad(b, (0, cout_eff - self.cout))
        return ops.pack_conv_weight(w, kpad), b

    def forward(self, x, x2=None, **kw):
        w, b = self.packed()
        if self.pad is not None:
            kw["pad"] = self.pad
        return ops.conv2d(x, w, b, ksize=self.k, stride=self.stride, x2=x2, **kw)

    # ---- small-channel 3x3 convolutions: fold F adjacent pixels of a row into the channel axis ----------------------
    # The tensor-core kernel contracts 64 channels per tap; with C = 8 or 16 (ControlNet conditioning embedding at
    # 512 x 512) 7/8 or 3/4 of every MMA and of every staged tile is zero padding.  Viewing [N, H, W, C] as
    # [N, H, W/F, F*C] (the same memory) turns the layer into a 3x3 convolution with F*C = 64 input and F*Cout output
    # channels whose weight is block-banded:  W'[(jo, co), dy, dq, (ji, ci)] = W[co, ci, dy, dx]  with
    # dx = F*dq + ji - jo  in {-1, 0, 1}, zero otherwise.  Same arithmetic (zeros added), 4x fewer MMAs and staged bytes
    # per pixel, no kernel change; zero padding at the row ends is the folded image's own zero padding.
    def fold_factor(self, x) -> int:
        cs = x.shape[3]
        if self.k != 3 or self.stride != 1 or cs not in (8, 16, 32) or cs < self.cin:
            return 1
        f = 64 // cs
        return f if (x.shape[2] % f == 0 and (f * self.cout) % 8 == 0) else 1

    def packed_folded(self, f: int, cs: int):
        key = (self._key(), f, cs)
        cache = getattr(self, "_fold_cache", None)
        if cache is None or cache[0] != key:
            with torch.no_grad():
                w = self.weight.detach().float()                      # [Cout, Cin, 3, 3] (dy, dx)
                cout, cin = w.shape[:2]
                wf = torch.zeros(f, cout, f, cs, 3, 3, dtype=torch.float32, device=w.device)  # [jo, co, ji, ci, dy, dq]
                for jo in range(f):
                    for ji in range(f):
                        for dq in (-1, 0, 1):
                            dx = f * dq + ji - jo
                            if -1 <= dx <= 1:
                                wf[jo, :, ji, :cin, :, dq + 1] = w[:, :, :, dx + 1]
                wf = wf.reshape(f * cout, f * cs, 3, 3)
                bias = self.bias.detach().repeat(f)
                self._fold_cache = (key, ops.pack_conv_weight(wf, 8), _f32(bias))
        return self._fold_cache[1], self._fold_cache[2]

    def forward_folded(self, x, **kw):
        """x [N, H, W, Cs] -> [N, H, W, Cout]; falls back to forward() when the layer / shape does not qualify."""
        f = self.fold_factor(x)
        if f == 1:
            return self.forward(x, **kw)
        n, h, w_, cs = x.shape
        wp, bp = self.packed_folded(f, cs)
        y = ops.conv2d(x.reshape(n, h, w_ // f, f * cs), wp, bp, ksize=3, stride=1, **kw)
        return y.reshape(n, h, w_, self.cout)


class TemporalConv(Packable):
    """Conv3d (3,1,1) container (weight [Cout, Cin, 3, 1, 1])."""

    def __init__(self, i: int, o: int):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(o, i, 3, 1, 1))
        self.bias = nn.Parameter(torch.zeros(o))
        nn.init.normal_(self.weight, std=1.0 / math.sqrt(3 * i))

    def pack(self):
        return ops.pack_conv_weight(self.weight.detach()), _f32(self.bias)

    def forward(self, x, frames, **kw):
        w, b = self.packed()
        return ops.temporal_conv(x, w, b, frames, **kw)


class Norm(Packable):
    """GroupNorm / LayerNorm affine parameters."""

    def __init__(self, c: int, eps: float):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(c))
        self.bias = nn.Parameter(torch.zeros(c))

    def pack(self):
        return self.weight.detach().float().contiguous(), self.bias.detach().float().contiguous()

    def group_norm(self, x, **kw):
        g, b = self.packed()
        return ops.group_norm(x, g, b, self.eps, **kw)

    def layer_norm(self, x, **kw):
        g, b = self.packed()
        return ops.layer_norm(x, g, b, self.eps, **kw)


# ------------------------------------------------------------------------------------------------
class TimestepEmbedding(nn.Module):
    """linear_2(SiLU(linear_1(x))) -- diffusers TimestepEmbedding."""

    def __init__(self, i: int, d: int, out_dim: Optional[int] = None):
        super().__init__()
        self.linear_1 = Linear(i, d)
        self.linear_2 = Linear(d, out_dim or d)

    def forward(self, x2d):
        return self.linear_2(self.linear_1(x2d, act=ACT_SILU))


class Attention(Packable):
    """diffusers Attention (to_q / to_k / to_v bias-free, to_out.0 with bias); SDPA replaced by ca_attention."""

    def __init__(self, query_dim: int, cross_dim: Optional[int], heads: int, dim_head: int):
        super().__init__()
        self.heads, self.dim_head, self.query_dim = heads, dim_head, query_dim
        self.is_cross = cross_dim is not None
        inner = heads * dim_head
        cd = cross_dim if cross_dim is not None else query_dim
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(cd, inner, bias=False)
        self.to_v = nn.Linear(cd, inner, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim), nn.Dropout(0.0)])
        self._static_kv = None   # (ctx object, ctx._version, weight key, projected K/V) -- see cache_static_context()
        self._static_cv = None   # same for the single-token output vector

    def _static_hit(self, slot, ctx):
        return slot is not None and slot[0] is ctx and slot[1] == ctx._version and slot[2] == self._key()

    def _pad_rows(self, w):  # [heads*d, K] -> [heads*dp, K]
        d, dp = self.dim_head, _pad64(self.dim_head)
        if d == dp:
            return w
        w = w.reshape(self.heads, d, -1)
        return torch.nn.functional.pad(w, (0, 0, 0, dp - d)).reshape(self.heads * dp, -1)

    def pack(self):
        d, dp = self.dim_head, _pad64(self.dim_head)
        wq, wk, wv = (self._pad_rows(m.weight.detach()) for m in (self.to_q, self.to_k, self.to_v))
        wo = self.to_out[0].weight.detach()
        if d != dp:
            wo = torch.nn.functional.pad(wo.reshape(-1, self.heads, d), (0, dp - d)).reshape(-1, self.heads * dp)
        pk = {"wo": _bf(wo), "bo": _f32(self.to_out[0].bias)}
        if self.is_cross:
            pk["wq"] = _bf(wq)
            pk["wkv"] = _bf(torch.cat([wk, wv], 0))
            pk["wv"] = _bf(wv)
        else:
            pk["wqkv"] = _bf(torch.cat([wq, wk, wv], 0))
        return pk

    def forward(self, x, ctx=None, residual=None, kv=None, kv_batch_div: int = 1):
        """x [B, L, D] (normalised tokens); ctx [B, Lk, Dc]; returns to_out(attn) + residual, shape [B, L, D]."""
        pk = self.packed()
        b, l, dq = x.shape
        dp = _pad64(self.dim_head)
        inner = self.heads * dp
        if self.is_cross:
            q = ops.linear(x.reshape(b * l, dq), pk["wq"]).reshape(b, l, inner)
            if kv is None:
                # step-invariant context (the prompt embedding of a denoising loop): projected once, see
                # cache_static_context(); any other tensor object / in-place update / weight change misses
                kv = self._static_kv[3] if self._static_hit(self._static_kv, ctx) else self.project_kv(ctx)
            k, v = kv[:, :, :inner], kv[:, :, inner:]
        else:
            qkv = ops.linear(x.reshape(b * l, dq), pk["wqkv"]).reshape(b, l, 3 * inner)
            q, k, v = qkv[:, :, :inner], qkv[:, :, inner:2 * inner], qkv[:, :, 2 * inner:]
        o = ops.attention(q, k, v, self.heads, dp, self.dim_head ** -0.5, kv_batch_div=kv_batch_div if self.is_cross else 1)
        out = ops.linear(o.reshape(b * l, inner), pk["wo"], pk["bo"],
                         residual=None if residual is None else residual.reshape(b * l, dq))
        return out.reshape(b, l, dq)

    def single_token_output(self, ctx_vec, src=None):
        """Cross attention over ONE key/value token: softmax == 1, so every query receives to_out(to_v(ctx)).
        ctx_vec [1, Dc] -> [1, D] (exact, including the bf16 rounding points of the SDPA path).  `src` is the tensor
        object ctx_vec was sliced from: when it is the cached step-invariant context the stored vector is returned."""
        if src is not None and self._static_hit(self._static_cv, src) and self._static_cv[3].shape[0] == ctx_vec.shape[0]:
            return self._static_cv[3]
        pk = self.packed()
        return ops.linear(ops.linear(ctx_vec, pk["wv"]), pk["wo"], pk["bo"])

    def cache_static(self, ctx, ctx_vec=None):
        """Projects a step-invariant context once (K/V for the attention kernel, or the single-token output vector)."""
        if ctx_vec is not None:
            self._static_cv = None
            self._static_cv = (ctx, ctx._version, self._key(), self.single_token_output(ctx_vec))
        else:
            self._static_kv = (ctx, ctx._version, self._key(), self.project_kv(ctx))

    def project_kv(self, ctx):
        pk = self.packed()
        b, lk, dc = ctx.shape
        return ops.linear(ctx.reshape(b * lk, dc), pk["wkv"]).reshape(b, lk, -1)


def cache_static_context(root: nn.Module, ctx: torch.Tensor, single_token_rows: Optional[int] = None):
    """The cross-attention context of a denoising loop does not depend on the timestep or the latents, so its K/V
    projections are step-invariant (the reference recomputes them every step: e.g. attention_processor to_k / to_v
    under sdxl_controlnet_adapter_pipeline.py:1356).  This projects `ctx` once for every cross attention under `root`
    whose key width matches; forward() then uses the stored tensors whenever it is handed this very tensor object
    unmodified (identity + version check), and recomputes for anything else.  Exact: same kernels, same operands.
    `single_token_rows`: for single-token contexts, the number of leading rows the consumer slices ([:1] or [:B])."""
    if ctx.dtype != BF16 or not ctx.is_contiguous():
        raise ValueError("cache_static_context expects the bf16 contiguous tensor that will be passed to forward()")
    n = 0
    for m in root.modules():
        if isinstance(m, Attention) and m.is_cross and m.to_k.weight.shape[1] == ctx.shape[-1]:
            if single_token_rows is not None:
                m.cache_static(ctx, ctx.reshape(-1, ctx.shape[-1])[:single_token_rows].contiguous())
            else:
                m.cache_static(ctx)
            n += 1
    return n


class GEGLUProj(Packable):
    def __init__(self, i: int, inner: int):
        super().__init__()
        self.proj = nn.Linear(i, inner * 2)

    def pack(self):
        w, b = ops.pack_geglu_weight(self.proj.weight.detach(), self.proj.bias.detach(), 256)
        return _bf(w), _f32(b)


class FeedForward(nn.Module):
    """GEGLU feed-forward: net.0 = GEGLU proj, net.1 = dropout, net.2 = Linear."""

    def __init__(self, dim: int, dim_out: Optional[int] = None, mult: int = 4):
        super().__init__()
        inner = dim * mult
        self.net = nn.ModuleList([GEGLUProj(dim, inner), nn.Dropout(0.0), Linear(inner, dim_out or dim)])

    def forward(self, x2d, **kw):
        w, b = self.net[0].packed()
        h = ops.linear(x2d, w, b, act=ACT_GEGLU, bn=256)
        return self.net[2](h, **kw)


class BasicTransformerBlock(nn.Module):
    """norm1-attn1(self) / norm2-attn2(cross) / norm3-ff with residuals (diffusers BasicTransformerBlock)."""

    def __init__(self, dim: int, heads: int, head_dim: int, cross_dim: Optional[int]):
        super().__init__()
        self.norm1 = Norm(dim, 1e-5)
        self.attn1 = Attention(dim, None, heads, head_dim)
        self.norm2 = Norm(dim, 1e-5)
        self.attn2 = Attention(dim, cross_dim, heads, head_dim)
        self.norm3 = Norm(dim, 1e-5)
        self.ff = FeedForward(dim)

    def forward(self, h, ctx, ff_kw=None, kv_batch_div: int = 1):
        b, l, d = h.shape
        h = self.attn1(self.norm1.layer_norm(h), residual=h)
        h = self.attn2(self.norm2.layer_norm(h), ctx=ctx, residual=h, kv_batch_div=kv_batch_div)
        out = self.ff(self.norm3.layer_norm(h).reshape(b * l, d), residual=h.reshape(b * l, d), **(ff_kw or {}))
        return out.reshape(b, l, d)


class ResnetBlock2D(nn.Module):
    """GN-SiLU-[2x up]-conv3x3 (+temb) - GN-SiLU-conv3x3 (+1x1 shortcut) -- model/resnet_block_2d.py:164-221.
    Two-source input (x, x2) implements the UNet skip concat without materialising it."""

    def __init__(self, cin: int, cout: int, temb_channels: Optional[int], eps: float,
                 use_in_shortcut: Optional[bool] = None, up: bool = False):
        super().__init__()
        self.up = up
        self.norm1 = Norm(cin, eps)
        self.conv1 = Conv2d(cin, cout, 3)
        self.time_emb_proj = Linear(temb_channels, cout) if temb_channels is not None else None  # None: VAE resnets
        self.norm2 = Norm(cout, eps)
        self.conv2 = Conv2d(cout, cout, 3)
        shortcut = (cin != cout) if use_in_shortcut is None else use_in_shortcut
        self.conv_shortcut = Conv2d(cin, cout, 1) if shortcut else None

    def forward(self, x, temb_act, x2=None, temb_proj=None):
        """temb_act: SiLU(temb) [N, T] (shared by all resnets of a model) or a precomputed projection."""
        if temb_proj is None and self.time_emb_proj is not None:
            temb_proj = self.time_emb_proj(temb_act)
        h = self.norm1.group_norm(x, x2=x2, silu=True, up2x=self.up)
        h = self.conv1(h, rowvec=temb_proj)
        h = self.norm2.group_norm(h, silu=True)
        if self.conv_shortcut is not None:
            sc = self.conv_shortcut(x, x2=x2)  # 1x1 conv commutes exactly with nearest up-sampling
            if self.up:
                sc = ops.upsample2x(sc)
        else:
            assert x2 is None
            sc = ops.upsample2x(x) if self.up else x
        return self.conv2(h, residual=sc)


class Transformer2DModel(nn.Module):
    """GroupNorm(1e-6) - proj_in - N x BasicTransformerBlock - proj_out - +residual.  proj_in/out are 1x1 convs
    (SD1.5) or Linears (SDXL); on channels-last tokens both are the same GEMM."""

    def __init__(self, heads: int, head_dim: int, in_channels: int, num_layers: int, cross_dim: int, linear_proj: bool):
        super().__init__()
        inner = heads * head_dim
        self.linear_proj = linear_proj
        self.norm = Norm(in_channels, 1e-6)
        self.proj_in = Linear(in_channels, inner) if linear_proj else Conv2d(in_channels, inner, 1)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(inner, heads, head_dim, cross_dim)
                                                 for _ in range(num_layers)])
        self.proj_out = Linear(inner, in_channels) if linear_proj else Conv2d(inner, in_channels, 1)

    def _w(self, m):
        w, b = m.packed()
        return w, b

    def forward(self, x, ctx, kv_batch_div: int = 1):
        n, hh, ww, c = x.shape
        t = self.norm.group_norm(x, silu=False).reshape(n * hh * ww, c)
        w, b = self._w(self.proj_in)
        h = ops.linear(t, w, b).reshape(n, hh * ww, -1)
        for blk in self.transformer_blocks:
            h = blk(h, ctx, kv_batch_div=kv_batch_div)
        w, b = self._w(self.proj_out)
        out = ops.linear(h.reshape(n * hh * ww, -1), w, b, residual=x.reshape(n * hh * ww, c))
        return out.reshape(n, hh, ww, c)


# ------------------------------------------------------------------------------------------------
# diffusers' 2-D UNet block wiring, shared by the SDXL UNet, the SVD UNet and the ControlNet.  The blocks take their
# already-built resnets / attentions: ResnetBlock2D + Transformer2DModel, or SpatioTemporalResBlock +
# TransformerSpatioTemporalModel, whose forward()s take a trailing `frames` argument -- passed through as *frames.
# ------------------------------------------------------------------------------------------------
def _sampler(conv: Conv2d) -> nn.ModuleList:
    """Downsample2D / Upsample2D container (state-dict keys downsamplers.0.conv.* / upsamplers.0.conv.*)."""
    s = nn.Module()
    s.conv = conv
    return nn.ModuleList([s])


class DownBlock2D(nn.Module):
    """(CrossAttn)DownBlock2D: resnet [-> attention] per layer, then the optional stride-2 conv; every layer's output
    and the down-sampled one are skips."""

    def __init__(self, resnets, attentions=None, downsampler: Optional[Conv2d] = None):
        super().__init__()
        self.has_cross_attention = attentions is not None
        self.resnets = nn.ModuleList(resnets)
        if attentions is not None:
            self.attentions = nn.ModuleList(attentions)
        self.downsamplers = None if downsampler is None else _sampler(downsampler)

    def forward(self, x, temb_act, ctx, *frames):
        outs = []
        for i, r in enumerate(self.resnets):
            x = r(x, temb_act, *frames)
            if self.has_cross_attention:
                x = self.attentions[i](x, ctx, *frames)
            outs.append(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0].conv(x)
            outs.append(x)
        return x, outs


class MidBlock2D(nn.Module):
    """UNetMidBlock2DCrossAttn: resnet, then (attention, resnet) per attention."""

    def __init__(self, resnets, attentions):
        super().__init__()
        self.resnets = nn.ModuleList(resnets)
        self.attentions = nn.ModuleList(attentions)

    def forward(self, x, temb_act, ctx, *frames):
        x = self.resnets[0](x, temb_act, *frames)
        for attn, r in zip(self.attentions, self.resnets[1:]):
            x = r(attn(x, ctx, *frames), temb_act, *frames)
        return x


class UpBlock2D(nn.Module):
    """(CrossAttn)UpBlock2D: per layer, resnet on (x, the last skip) [-> attention]; then the optional 2x nearest
    up-sampling + conv.  The skip is the resnet's second input source, never concatenated in memory."""

    def __init__(self, resnets, attentions=None, upsampler: Optional[Conv2d] = None):
        super().__init__()
        self.has_cross_attention = attentions is not None
        self.resnets = nn.ModuleList(resnets)
        if attentions is not None:
            self.attentions = nn.ModuleList(attentions)
        self.upsamplers = None if upsampler is None else _sampler(upsampler)

    def forward(self, x, temb_act, ctx, *frames, skips):
        for i, r in enumerate(self.resnets):
            x = r(x, temb_act, *frames, x2=skips.pop())
            if self.has_cross_attention:
                x = self.attentions[i](x, ctx, *frames)
        if self.upsamplers is not None:
            x = self.upsamplers[0].conv(ops.upsample2x(x))
        return x


def add_residual(x, r: torch.Tensor):
    """x [B*F, H, W, C] + an adapter / ControlNet residual given as logical NCHW, 4-D "(b f) c h w" or 5-D "b c f h w"
    (any memory format)."""
    if r.dim() == 5:
        r = r.permute(0, 2, 1, 3, 4).flatten(0, 1)
    return ops.add(x, to_channels_last_bf16(r))


def add_skip_residuals(skips: list, residuals):
    """skips[i] = add_residual(skips[i], residuals[i]), truncated to the shorter list as the reference's zip() does."""
    for i, (s, r) in enumerate(zip(skips, residuals)):
        skips[i] = add_residual(s, r)
