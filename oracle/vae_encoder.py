"""ORACLE (test infrastructure): the encoder half of diffusers v0.27.2 ``AutoencoderKL`` /
``AutoencoderKLTemporalDecoder`` restated in plain PyTorch -- what ``self.vae.encode(image).latent_dist`` runs in
/root/reference/i2vgen_xl/pipelines/i2vgen_xl_controlnet_adapter_pipeline.py:496 and
svd/pipelines/svd_controlnet_adapter_pipeline.py:221.  Restated: models/autoencoders/vae.py ``Encoder`` (double_z=True)
and ``DiagonalGaussianDistribution``, models/unets/unet_2d_blocks.py ``DownEncoderBlock2D``, models/downsampling.py
``Downsample2D(padding=0)``, autoencoder_kl.py / autoencoder_kl_temporal_decoder.py ``encode``.  Parity unpinned like
oracle/vae.py; the structural pin is the published SD / SDXL VAE's total parameter count (83 653 863).

The classes here extend oracle/vae.py's decoders with ``encoder`` + ``quant_conv``, so the decoder-only classes (and the
key sets and seeded weights of the checks that use them) are unchanged.  Not imported by the product."""
from __future__ import annotations

import torch
from torch import nn

from .blocks import Downsample2D, ResnetBlock2D
from .vae import AutoencoderKL as _DecoderKL
from .vae import AutoencoderKLTemporalDecoder as _TemporalDecoderKL
from .vae import UNetMidBlock2D


class DownEncoderBlock2D(nn.Module):
    """DownEncoderBlock2D as the VAE Encoder builds it (temb_channels=None, resnet_eps=1e-6, downsample_padding=0):
    resnets, then Downsample2D(use_conv=True, padding=0, name="op") -- F.pad(x, (0, 1, 0, 1)) followed by a 3x3 stride-2
    convolution without padding."""

    def __init__(self, in_channels: int, out_channels: int, num_layers: int, eps: float, groups: int, add_downsample: bool):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(in_channels=in_channels if i == 0 else out_channels,
                                                    out_channels=out_channels, temb_channels=None, eps=eps, groups=groups)
                                      for i in range(num_layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(out_channels, use_conv=True, out_channels=out_channels, padding=0,
                                                        name="op")]) if add_downsample else None

    def forward(self, hidden_states):
        for resnet in self.resnets:
            hidden_states = resnet(hidden_states, temb=None)
        if self.downsamplers is not None:
            for ds in self.downsamplers:
                hidden_states = ds(hidden_states)
        return hidden_states


class Encoder(nn.Module):
    """vae.py Encoder: conv_in -> DownEncoderBlock2D x len(block_out_channels) -> UNetMidBlock2D (attention head dim =
    the last width) -> GroupNorm -> SiLU -> conv_out with 2 * out_channels (double_z)."""

    def __init__(self, in_channels=3, out_channels=4, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 norm_num_groups=32):
        super().__init__()
        self.conv_in = nn.Conv2d(in_channels, block_out_channels[0], kernel_size=3, stride=1, padding=1)
        self.down_blocks = nn.ModuleList([])
        out_c = block_out_channels[0]
        for i, c in enumerate(block_out_channels):
            prev, out_c = out_c, c
            self.down_blocks.append(DownEncoderBlock2D(prev, out_c, layers_per_block, 1e-6, norm_num_groups,
                                                       add_downsample=i != len(block_out_channels) - 1))
        self.mid_block = UNetMidBlock2D(block_out_channels[-1], 1e-6, norm_num_groups,
                                        attention_head_dim=block_out_channels[-1])
        self.conv_norm_out = nn.GroupNorm(num_channels=block_out_channels[-1], num_groups=norm_num_groups, eps=1e-6)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(block_out_channels[-1], 2 * out_channels, 3, padding=1)

    def forward(self, sample):
        sample = self.conv_in(sample)
        for down_block in self.down_blocks:
            sample = down_block(sample)
        sample = self.mid_block(sample)
        sample = self.conv_act(self.conv_norm_out(sample))
        return self.conv_out(sample)


class DiagonalGaussianDistribution:
    """vae.py DiagonalGaussianDistribution (deterministic=False).  ``sample(noise=...)`` takes the unit noise instead of
    drawing it with randn_tensor(mean.shape, generator, dtype=parameters.dtype)."""

    def __init__(self, parameters):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)

    def sample(self, generator=None, noise=None):
        if noise is None:
            noise = torch.randn(self.mean.shape, generator=generator, device=self.parameters.device,
                                dtype=self.parameters.dtype)
        return self.mean + self.std * noise.to(device=self.parameters.device, dtype=self.parameters.dtype)

    def mode(self):
        return self.mean


class _EncodeMixin:
    def _add_encoder(self, in_channels, latent_channels, block_out_channels, layers_per_block, norm_num_groups=32):
        self.encoder = Encoder(in_channels, latent_channels, block_out_channels, layers_per_block, norm_num_groups)
        self.quant_conv = nn.Conv2d(2 * latent_channels, 2 * latent_channels, 1)

    def encode(self, x, return_dict=False):
        """h = encoder(x); moments = quant_conv(h) -> (DiagonalGaussianDistribution(moments),)"""
        return (DiagonalGaussianDistribution(self.quant_conv(self.encoder(x))),)


class AutoencoderKL(_EncodeMixin, _DecoderKL):
    """Both halves of AutoencoderKL: oracle/vae.py's decode() plus encode()."""

    def __init__(self, in_channels=3, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 latent_channels=4, norm_num_groups=32, scaling_factor=0.13025, **_unused):
        super().__init__(in_channels=in_channels, out_channels=out_channels, block_out_channels=block_out_channels,
                         layers_per_block=layers_per_block, latent_channels=latent_channels,
                         norm_num_groups=norm_num_groups, scaling_factor=scaling_factor)
        self._add_encoder(in_channels, latent_channels, block_out_channels, layers_per_block, norm_num_groups)


class AutoencoderKLTemporalDecoder(_EncodeMixin, _TemporalDecoderKL):
    """Both halves of the SVD VAE: the 2-D Encoder + quant_conv (autoencoder_kl_temporal_decoder.py __init__ / encode)
    plus oracle/vae.py's temporal decode()."""

    def __init__(self, in_channels=3, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 latent_channels=4, scaling_factor=0.18215, **_unused):
        super().__init__(in_channels=in_channels, out_channels=out_channels, block_out_channels=block_out_channels,
                         layers_per_block=layers_per_block, latent_channels=latent_channels,
                         scaling_factor=scaling_factor)
        self._add_encoder(in_channels, latent_channels, block_out_channels, layers_per_block)

