"""H100 host mirror of diffusers' ``AutoencoderKL`` -- the VAE ``decode`` the reference pipelines call after the
denoising loop (/root/reference/sdxl/pipelines/sdxl_controlnet_adapter_pipeline.py:1414;
i2vgen_xl/pipelines/i2vgen_xl_controlnet_adapter_pipeline.py:398-418 ``decode_latents``; SURVEY.md section 8f row 1)
and the ``encode`` of the conditioning image before it (i2vgen pipeline :487-517, svd pipeline :214-235; section 8f
row 2).

Same constructor kwargs, ``encode()`` / ``decode()`` call forms and state-dict keys as the diffusers class
(``encoder.conv_in / down_blocks.N.{resnets,downsamplers} / mid_block / conv_norm_out / conv_out``, ``quant_conv.*``,
``post_quant_conv.*``, ``decoder.conv_in / mid_block.{resnets,attentions} / up_blocks.N.{resnets,upsamplers} /
conv_norm_out / conv_out``).  A checkpoint without a complete encoder half still loads its decoder (see ``_KLVae``).
Everything runs on the kernels of the denoising path: 3x3 / 1x1 convolutions on the implicit-GEMM kernel (the encoder's
down-samplers on its stride-2 parity view with bottom / right padding), GroupNorm(+SiLU) kernels, the 2x nearest
up-sampler; the mid block's single 512-wide attention head (outside ``attention_kernel``'s head dims, and run once per
generation) as QK^T GEMM (fp32) -> ``ca_softmax_rows`` -> PV GEMM, one image at a time; the posterior and the pipelines'
image-latent layouts in ``ca_vae_latents``.

``AutoencoderKLTemporalDecoder`` (decoder half) is the VAE of the SVD pipeline (svd/pipelines/
svd_controlnet_adapter_pipeline.py:265-292 ``decode_latents``): every decoder ResNet is a SpatioTemporalResBlock (spatial
ResnetBlock2D -> TemporalResnetBlock over the frames of the decode chunk, blended by a learned, switched alpha in the
GEMM epilogue), and a Conv3d (3,1,1) over the decoded RGB frames (``ca_frame_conv_small``) closes it.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import nn

from . import ops
from .adapter import AlphaBlender, TemporalResnetBlock
from .layers import BF16, Conv2d, Linear, Norm, Packable, ResnetBlock2D, _ConfigDict, to_channels_last_bf16
from .persistence import PretrainedMixin


class _VaeAttention(nn.Module):
    """diffusers ``Attention(heads=1, dim_head=C, norm_num_groups=32, residual_connection=True, bias=True)`` as built by
    UNetMidBlock2D for the VAE: GroupNorm -> q / k / v Linear (with bias) -> softmax(q k^T / sqrt(C)) v -> to_out + x."""

    def __init__(self, c: int, eps: float):
        super().__init__()
        self.group_norm = Norm(c, eps)
        self.to_q, self.to_k, self.to_v = Linear(c, c), Linear(c, c), Linear(c, c)
        self.to_out = nn.ModuleList([Linear(c, c), nn.Dropout(0.0)])
        self.scale = c ** -0.5

    def forward(self, x):
        n, h, w, c = x.shape
        hw = h * w
        t = self.group_norm.group_norm(x, silu=False).reshape(n * hw, c)
        q, k, v = self.to_q(t), self.to_k(t), self.to_v(t)
        o = torch.empty_like(q)
        for i in range(n):  # one image at a time: the [hw, hw] fp32 score matrix is 1 GB at 128 x 128 latents
            sl = slice(i * hw, (i + 1) * hw)
            s = ops.linear(q[sl], k[sl], None, out_fp32=True, out_scale=self.scale)          # [hw, hw] = q k^T * scale
            p = ops.softmax_rows(s)
            vt = ops.nhwc_to_nchw(v[sl].reshape(1, h, w, c)).reshape(c, hw)                   # v^T as the GEMM's B rows
            ops.linear(p, vt, None, out=o[sl])
        w_o, b_o = self.to_out[0].packed()
        return ops.linear(o, w_o, b_o, residual=x.reshape(n * hw, c)).reshape(n, h, w, c)


class _MidBlock(nn.Module):
    def __init__(self, c: int, eps: float):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, None, eps), ResnetBlock2D(c, c, None, eps)])
        self.attentions = nn.ModuleList([_VaeAttention(c, eps)])

    def forward(self, x):
        x = self.resnets[0](x, None)
        x = self.attentions[0](x)
        return self.resnets[1](x, None)


class _UpDecoderBlock(nn.Module):
    def __init__(self, cin: int, cout: int, layers: int, eps: float, add_upsample: bool):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, None, eps) for i in range(layers)])
        self.upsamplers = None
        if add_upsample:
            us = nn.Module()
            us.conv = Conv2d(cout, cout, 3)
            self.upsamplers = nn.ModuleList([us])

    def forward(self, x):
        for r in self.resnets:
            x = r(x, None)
        if self.upsamplers is not None:
            x = self.upsamplers[0].conv(ops.upsample2x(x))
        return x


class Decoder(nn.Module):
    def __init__(self, in_channels: int, out_channels: int, block_out_channels, layers_per_block: int, eps: float):
        super().__init__()
        rev = list(reversed(block_out_channels))
        self.conv_in = Conv2d(in_channels, rev[0], 3)
        self.mid_block = _MidBlock(rev[0], eps)
        blocks, prev = [], rev[0]
        for i, c in enumerate(rev):
            blocks.append(_UpDecoderBlock(prev, c, layers_per_block + 1, eps, i != len(rev) - 1))
            prev = c
        self.up_blocks = nn.ModuleList(blocks)
        self.conv_norm_out = Norm(rev[-1], eps)
        self.conv_out = Conv2d(rev[-1], out_channels, 3)
        self.out_channels = out_channels

    def forward(self, z_nhwc8):
        x = self.conv_in(z_nhwc8)
        x = self.mid_block(x)
        for blk in self.up_blocks:
            x = blk(x)
        return self.conv_out(self.conv_norm_out.group_norm(x, silu=True))  # [n, H, W, 8], the first out_channels are real


class DecoderOutput:
    def __init__(self, sample):
        self.sample = sample


# ---- encoder half (diffusers v0.27.2 models/autoencoders/vae.py Encoder with double_z=True) ---------------------------
class _DownEncoderBlock(nn.Module):
    """diffusers DownEncoderBlock2D: resnets (eps 1e-6, no time embedding), then Downsample2D(padding=0) -- a 3x3
    stride-2 convolution after one zero row / column at the bottom / right -- on every block but the last."""

    def __init__(self, cin: int, cout: int, layers: int, eps: float, add_downsample: bool):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, None, eps) for i in range(layers)])
        self.downsamplers = None
        if add_downsample:
            ds = nn.Module()
            ds.conv = Conv2d(cout, cout, 3, stride=2, pad=(0, 1))
            self.downsamplers = nn.ModuleList([ds])

    def forward(self, x):
        for r in self.resnets:
            x = r(x, None)
        if self.downsamplers is not None:
            x = self.downsamplers[0].conv(x)
        return x


class Encoder(nn.Module):
    """conv_in -> down blocks -> mid block (2 resnets + the single-head attention) -> GroupNorm + SiLU -> conv_out with
    2 * latent_channels outputs: the mean and log-variance of the diagonal Gaussian posterior."""

    def __init__(self, in_channels: int, latent_channels: int, block_out_channels, layers_per_block: int, eps: float):
        super().__init__()
        self.conv_in = Conv2d(in_channels, block_out_channels[0], 3)
        blocks, prev = [], block_out_channels[0]
        for i, c in enumerate(block_out_channels):
            blocks.append(_DownEncoderBlock(prev, c, layers_per_block, eps, i != len(block_out_channels) - 1))
            prev = c
        self.down_blocks = nn.ModuleList(blocks)
        self.mid_block = _MidBlock(block_out_channels[-1], eps)
        self.conv_norm_out = Norm(block_out_channels[-1], eps)
        self.conv_out = Conv2d(block_out_channels[-1], 2 * latent_channels, 3)

    def forward(self, x_nhwc8):
        x = self.conv_in(x_nhwc8)
        for blk in self.down_blocks:
            x = blk(x)
        x = self.mid_block(x)
        x = self.conv_norm_out.group_norm(x, silu=True)
        return self.conv_out(x)  # [n, h, w, 2 * latent_channels]


class DiagonalGaussianDistribution:
    """diffusers DiagonalGaussianDistribution over the quant_conv output: mean = channels 0-3, logvar = channels 4-7
    clamped to [-30, 20].  ``mode()`` / ``sample()`` run ``ca_vae_latents``; the result is bf16 [n, 4, h, w]."""

    def __init__(self, moments: torch.Tensor):
        self.moments = moments  # [n, h, w, 8] bf16, channels-last
        self.deterministic = False

    @property
    def mean(self):
        return self.mode()

    @property
    def logvar(self):
        return self.moments[..., 4:].permute(0, 3, 1, 2).float().clamp(-30.0, 20.0).to(self.moments.dtype)

    @property
    def std(self):
        return torch.exp(0.5 * self.logvar.float()).to(self.moments.dtype)

    @property
    def var(self):
        return torch.exp(self.logvar.float()).to(self.moments.dtype)

    def mode(self):
        return ops.vae_latents(self.moments, ops.VAE_POSTERIOR)

    def noise(self, generator=None):
        """The unit noise ``sample(generator)`` uses: drawn as diffusers' randn_tensor draws it (the posterior's shape and
        dtype, on the generator's device, the global RNG when generator is None), as fp32 on the moments' device."""
        n, h, w, _ = self.moments.shape
        if isinstance(generator, (list, tuple)):
            generator = generator[0]
        dev = generator.device if generator is not None else self.moments.device
        return torch.randn((n, 4, h, w), generator=generator, device=dev, dtype=self.moments.dtype).to(
            self.moments.device, torch.float32)

    def sample(self, generator=None, noise: Optional[torch.Tensor] = None):
        """mean + std * noise; `noise` (fp32 [n, 4, h, w]) replaces the draw."""
        return ops.vae_latents(self.moments, ops.VAE_POSTERIOR, noise=self.noise(generator) if noise is None else noise)


class AutoencoderKLOutput:
    def __init__(self, latent_dist):
        self.latent_dist = latent_dist


class _KLVae(PretrainedMixin, nn.Module):
    """What the two VAEs share: the encoder half, its loading rules and ``encode()``.

    A published checkpoint carries both halves.  The encoder half (``encoder.*``, ``quant_conv.*``) is loaded only when
    the state dict carries every one of its keys with the module's shapes; otherwise those keys are skipped, the decoder
    half loads as before, and ``encode()`` raises until a complete encoder is loaded.  A freshly constructed module can
    encode (with its random weights)."""

    encoder_prefixes = ("encoder.", "quant_conv.")

    def _init_encoder(self, in_channels, latent_channels, block_out_channels, layers_per_block):
        self.encoder = Encoder(in_channels, latent_channels, block_out_channels, layers_per_block, 1e-6)
        self.quant_conv = Conv2d(2 * latent_channels, 2 * latent_channels, 1)
        self.encoder_loaded = True

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        own = {k: tuple(v.shape) for k, v in self.state_dict().items() if k.startswith(self.encoder_prefixes)}
        complete = all(k in state_dict and tuple(state_dict[k].shape) == s for k, s in own.items())
        if complete:
            res = super().load_state_dict(state_dict, strict=strict, **kw)
            self.encoder_loaded = True
            return res
        sd = {k: v for k, v in state_dict.items() if not k.startswith(self.encoder_prefixes)}
        res = super().load_state_dict(sd, strict=False, **kw)
        missing = [k for k in res.missing_keys if not k.startswith(self.encoder_prefixes)]
        if strict and (missing or res.unexpected_keys):
            raise RuntimeError(f"Error(s) in loading state_dict for {type(self).__name__}: missing keys {missing}, "
                               f"unexpected keys {res.unexpected_keys}")
        self.encoder_loaded = False
        return type(res)(missing, res.unexpected_keys)

    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """x [N, 3, H, W] in [-1, 1] (fp32 or bf16, H and W multiples of 8) -> AutoencoderKLOutput(latent_dist=
        DiagonalGaussianDistribution) over [N, 4, H/8, W/8] latents."""
        if not self.encoder_loaded:
            raise ValueError(f"{type(self).__name__}.encode: the encoder weights were not loaded (the state dict did not "
                             f"carry a complete encoder.* / quant_conv.* set); load a full checkpoint to encode")
        f = 2 ** (len(self.config.block_out_channels) - 1)
        if x.dim() != 4 or x.shape[1] != self.config.in_channels:
            raise ValueError(f"encode expects [N, {self.config.in_channels}, H, W] images, got {tuple(x.shape)}")
        if x.shape[2] % f or x.shape[3] % f:
            raise ValueError(f"`height` and `width` have to be divisible by {f} but are {x.shape[2]} and {x.shape[3]}.")
        x = to_channels_last_bf16(x.to(self.device), 8)  # 3 -> 8 zero-padded channels
        moments = self.quant_conv(self.encoder(x))     # [N, h, w, 8] = (mean, logvar)
        post = DiagonalGaussianDistribution(moments)
        return AutoencoderKLOutput(post) if return_dict else (post,)


class AutoencoderKL(_KLVae):

    def __init__(self, in_channels: int = 3, out_channels: int = 3, down_block_types=("DownEncoderBlock2D",) * 4,
                 up_block_types=("UpDecoderBlock2D",) * 4, block_out_channels=(128, 256, 512, 512),
                 layers_per_block: int = 2, act_fn: str = "silu", latent_channels: int = 4, norm_num_groups: int = 32,
                 sample_size: int = 1024, scaling_factor: float = 0.13025, force_upcast: bool = True, **_ignored):
        super().__init__()
        if act_fn != "silu" or norm_num_groups != 32 or any(t != "UpDecoderBlock2D" for t in up_block_types) or \
                any(t != "DownEncoderBlock2D" for t in down_block_types):
            raise NotImplementedError("only the SD / SDXL AutoencoderKL topology is implemented")
        self.config = _ConfigDict(in_channels=in_channels, out_channels=out_channels,
                                  down_block_types=tuple(down_block_types), up_block_types=tuple(up_block_types),
                                  block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                                  act_fn=act_fn, latent_channels=latent_channels, norm_num_groups=norm_num_groups,
                                  sample_size=sample_size, scaling_factor=scaling_factor, force_upcast=force_upcast)
        self._init_encoder(in_channels, latent_channels, block_out_channels, layers_per_block)
        self.post_quant_conv = Conv2d(latent_channels, latent_channels, 1)
        self.decoder = Decoder(latent_channels, out_channels, block_out_channels, layers_per_block, 1e-6)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True, generator=None):
        """z [N, 4, h, w] (already divided by scaling_factor by the caller, as the pipelines do) -> images [N, 3, 8h, 8w]
        in [-1, 1] (logical NCHW, bf16)."""
        x = to_channels_last_bf16(z.to(BF16) if z.dtype not in (BF16, torch.float32) else z, 8)  # 4 -> 8 zero-padded channels
        y = self.decoder(self.post_quant_conv(x))  # 1x1 conv 4 -> 4 on the padded layout: [n, h, w, 8]
        img = ops.nhwc_to_nchw(y, self.config.out_channels)
        return DecoderOutput(img) if return_dict else (img,)


# ---- SVD: AutoencoderKLTemporalDecoder (diffusers models/autoencoders/autoencoder_kl_temporal_decoder.py) ---------------
class _SpatioTemporalResBlock(nn.Module):
    """diffusers SpatioTemporalResBlock as the temporal decoder builds it: temb_channels=None, eps=1e-6,
    temporal_eps=1e-5, merge_strategy="learned", merge_factor=0.0, switch_spatial_to_temporal_mix=True."""

    def __init__(self, cin: int, cout: int):
        super().__init__()
        self.spatial_res_block = ResnetBlock2D(cin, cout, None, 1e-6)
        self.temporal_res_block = TemporalResnetBlock(cout, None, 1e-5)
        self.time_mixer = AlphaBlender(0.0, switch_spatial_to_temporal_mix=True)

    def forward(self, x, frames: int):
        s = self.spatial_res_block(x, None)
        return self.temporal_res_block(s, frames, None, blend_src=s, blend_alpha=self.time_mixer.alpha())


class _MidBlockTemporalDecoder(nn.Module):
    def __init__(self, c: int, layers: int):
        super().__init__()
        self.resnets = nn.ModuleList([_SpatioTemporalResBlock(c, c) for _ in range(layers)])
        self.attentions = nn.ModuleList([_VaeAttention(c, 1e-6)])

    def forward(self, x, frames: int):
        x = self.resnets[0](x, frames)
        for resnet, attn in zip(self.resnets[1:], self.attentions):
            x = resnet(attn(x), frames)
        return x


class _UpBlockTemporalDecoder(nn.Module):
    def __init__(self, cin: int, cout: int, layers: int, add_upsample: bool):
        super().__init__()
        self.resnets = nn.ModuleList([_SpatioTemporalResBlock(cin if i == 0 else cout, cout) for i in range(layers)])
        self.upsamplers = None
        if add_upsample:
            us = nn.Module()
            us.conv = Conv2d(cout, cout, 3)
            self.upsamplers = nn.ModuleList([us])

    def forward(self, x, frames: int):
        for r in self.resnets:
            x = r(x, frames)
        if self.upsamplers is not None:
            x = self.upsamplers[0].conv(ops.upsample2x(x))
        return x


class _FrameConvSmall(Packable):
    """Conv3d(C, C, (3,1,1), padding (1,0,0)) on a handful of channels; its parameters travel to the kernel by value."""

    def __init__(self, c: int):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(c, c, 3, 1, 1))
        self.bias = nn.Parameter(torch.zeros(c))
        nn.init.normal_(self.weight, std=(3 * c) ** -0.5)

    def pack(self):
        co, ci = self.weight.shape[:2]
        return (self.weight.detach().to(BF16).float().reshape(co, ci, 3).cpu().contiguous(),
                self.bias.detach().to(BF16).float().cpu().contiguous())

    def forward(self, x_nhwc, frames: int):
        w, b = self.packed()
        return ops.frame_conv_small(x_nhwc, w, b, frames, w.shape[1])


class TemporalDecoder(nn.Module):
    def __init__(self, in_channels: int = 4, out_channels: int = 3, block_out_channels=(128, 256, 512, 512),
                 layers_per_block: int = 2):
        super().__init__()
        if out_channels > 4:
            raise NotImplementedError("time_conv_out is implemented for at most 4 image channels")
        rev = list(reversed(block_out_channels))
        self.conv_in = Conv2d(in_channels, rev[0], 3)
        self.mid_block = _MidBlockTemporalDecoder(rev[0], layers_per_block)
        blocks, prev = [], rev[0]
        for i, c in enumerate(rev):
            blocks.append(_UpBlockTemporalDecoder(prev, c, layers_per_block + 1, i != len(rev) - 1))
            prev = c
        self.up_blocks = nn.ModuleList(blocks)
        self.conv_norm_out = Norm(rev[-1], 1e-6)
        self.conv_out = Conv2d(rev[-1], out_channels, 3)
        self.time_conv_out = _FrameConvSmall(out_channels)

    def forward(self, z_nhwc8, frames: int):
        """z [B*F, h, w, 8] (frames of a clip contiguous) -> images [B*F, 3, 8h, 8w] bf16 (logical NCHW)."""
        x = self.conv_in(z_nhwc8)
        x = self.mid_block(x, frames)
        for blk in self.up_blocks:
            x = blk(x, frames)
        y = self.conv_out(self.conv_norm_out.group_norm(x, silu=True))  # [n, H, W, 8], the first out_channels are real
        return self.time_conv_out(y, frames)


class AutoencoderKLTemporalDecoder(_KLVae):
    """The SVD VAE (stabilityai/stable-video-diffusion-img2vid[-xt] ``vae``): same constructor kwargs,
    ``encode(x)`` / ``decode(z, num_frames)`` call forms and state-dict keys as the diffusers class.  Its encoder is the
    2-D ``Encoder`` of AutoencoderKL (with quant_conv); there is no post_quant_conv in this model."""

    def __init__(self, in_channels: int = 3, out_channels: int = 3, down_block_types=("DownEncoderBlock2D",) * 4,
                 block_out_channels=(128, 256, 512, 512), layers_per_block: int = 2, latent_channels: int = 4,
                 sample_size: int = 768, scaling_factor: float = 0.18215, force_upcast: bool = True, **_ignored):
        super().__init__()
        self.config = _ConfigDict(in_channels=in_channels, out_channels=out_channels,
                                  down_block_types=tuple(down_block_types), block_out_channels=tuple(block_out_channels),
                                  layers_per_block=layers_per_block, latent_channels=latent_channels,
                                  sample_size=sample_size, scaling_factor=scaling_factor, force_upcast=force_upcast)
        if any(t != "DownEncoderBlock2D" for t in down_block_types):
            raise NotImplementedError("only the SVD AutoencoderKLTemporalDecoder topology is implemented")
        self._init_encoder(in_channels, latent_channels, block_out_channels, layers_per_block)
        self.decoder = TemporalDecoder(latent_channels, out_channels, block_out_channels, layers_per_block)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, num_frames: int = 1, return_dict: bool = True):
        """z [B*F, 4, h, w] (already divided by scaling_factor, frames of a clip contiguous; B*F a multiple of
        num_frames) -> frames [B*F, 3, 8h, 8w] in [-1, 1] (logical NCHW, bf16)."""
        if z.shape[0] % num_frames:
            raise ValueError(f"batch {z.shape[0]} is not a multiple of num_frames={num_frames}")
        x = to_channels_last_bf16(z.to(BF16) if z.dtype not in (BF16, torch.float32) else z, 8)
        img = self.decoder(x, num_frames)
        return DecoderOutput(img) if return_dict else (img,)


def svd_decode_latents(vae: AutoencoderKLTemporalDecoder, latents: torch.Tensor, num_frames: int,
                       decode_chunk_size: int = 14):
    """svd pipeline :265-292: latents (B, F, 4, h, w) -> video (B, 3, F, H, W) fp32.  Frames are decoded
    ``decode_chunk_size`` at a time and, as in the reference, each chunk is ONE temporal unit for the decoder
    (``num_frames`` = the chunk's length), whatever clip its frames come from."""
    latents = latents.flatten(0, 1)
    latents = 1 / vae.config.scaling_factor * latents
    frames = []
    for i in range(0, latents.shape[0], decode_chunk_size):
        chunk = latents[i:i + decode_chunk_size].contiguous()
        frames.append(vae.decode(chunk, num_frames=chunk.shape[0]).sample)
    frames = torch.cat(frames, dim=0)
    frames = frames.reshape(-1, num_frames, *frames.shape[1:]).permute(0, 2, 1, 3, 4)
    return frames.float()


# ---- the pipelines' post-processing (diffusers VaeImageProcessor.postprocess / i2vgen tensor2vid) --------------------
def postprocess(image: torch.Tensor, output_type: str = "pil"):
    """[N, 3, H, W] in [-1, 1] -> "pt" tensor in [0, 1] / "np" NHWC float array / list of PIL images."""
    image = (image.float() / 2 + 0.5).clamp(0, 1)
    if output_type == "pt":
        return image
    arr = image.cpu().permute(0, 2, 3, 1).numpy()
    if output_type == "np":
        return arr
    if output_type == "pil":
        from PIL import Image
        return [Image.fromarray((a * 255).round().astype("uint8")) for a in arr]
    raise ValueError(f"{output_type} does not exist. Please choose one of ['np', 'pt', 'pil']")


def decode_latents(vae: AutoencoderKL, latents: torch.Tensor, decode_chunk_size: Optional[int] = None):
    """i2vgen pipeline :398-418: latents (B, 4, F, h, w) -> video (B, 3, F, H, W) fp32."""
    latents = 1 / vae.config.scaling_factor * latents
    b, c, f, h, w = latents.shape
    lat = latents.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)
    step = decode_chunk_size or lat.shape[0]
    frames = [vae.decode(lat[i:i + step].contiguous()).sample for i in range(0, lat.shape[0], step)]
    image = torch.cat(frames, dim=0)
    return image.reshape(b, f, -1, *image.shape[2:]).permute(0, 2, 1, 3, 4).float()


def tensor2vid(video: torch.Tensor, output_type: str = "np"):
    """i2vgen pipeline :81-99."""
    import numpy as np
    outs = [postprocess(video[i].permute(1, 0, 2, 3), output_type) for i in range(video.shape[0])]
    if output_type == "np":
        return np.stack(outs)
    if output_type == "pt":
        return torch.stack(outs)
    return outs
