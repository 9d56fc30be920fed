"""ORACLE (test infrastructure): the image-latent preparation of the two video pipelines restated on the oracle VAE
(oracle/vae_encoder.py), in the reference's own tensor-op order.  Not imported by the product.

* I2VGen-XL: /root/reference/i2vgen_xl/pipelines/i2vgen_xl_controlnet_adapter_pipeline.py:487-517
  ``prepare_image_latents`` (posterior sample * scaling_factor, position planes k / (F - 1) for frames 1..F-1,
  ``repeat(num_videos_per_prompt)``, ``cat([x] * 2)`` for classifier-free guidance), called at :805-812.
* SVD: svd/pipelines/svd_controlnet_adapter_pipeline.py:214-235 ``_encode_vae_image`` (posterior mode, ``cat([zeros, x])``
  then ``repeat(num_videos_per_prompt)``) and :580-583 (``unsqueeze(1).repeat(1, num_frames, 1, 1, 1)``); the image is
  noise-augmented first (:566-567): ``image + noise_aug_strength * randn_tensor(image.shape, generator)``.
"""
from __future__ import annotations

import torch


def i2vgen_prepare_image_latents(scaled_sample: torch.Tensor, num_frames: int, num_videos_per_prompt: int):
    """scaled_sample = vae.encode(image).latent_dist.sample() * scaling_factor, [n, 4, h, w] -> (2*n*nv, 4, F, h, w)"""
    image_latents = scaled_sample.unsqueeze(2)
    frame_position_mask = []
    for frame_idx in range(num_frames - 1):
        scale = (frame_idx + 1) / (num_frames - 1)
        frame_position_mask.append(torch.ones_like(image_latents[:, :, :1]) * scale)
    if frame_position_mask:
        image_latents = torch.cat([image_latents, torch.cat(frame_position_mask, dim=2)], dim=2)
    image_latents = image_latents.repeat(num_videos_per_prompt, 1, 1, 1, 1)
    return torch.cat([image_latents] * 2)


def svd_image_latents(mode: torch.Tensor, num_frames: int, num_videos_per_prompt: int):
    """mode = vae.encode(image).latent_dist.mode(), [n, 4, h, w] -> (2*n*nv, F, 4, h, w): zeros first, then the
    images, then repeat(nv) -- for nv > 1 that interleaves [0, L, 0, L] (SURVEY quirk table)."""
    image_latents = torch.cat([torch.zeros_like(mode), mode])
    image_latents = image_latents.repeat(num_videos_per_prompt, 1, 1, 1)
    return image_latents.unsqueeze(1).repeat(1, num_frames, 1, 1, 1)


def i2vgen_image_latents(vae, image: torch.Tensor, num_frames: int, num_videos_per_prompt: int, noise: torch.Tensor):
    """image: the VAE input [n, 3, H, W] in [-1, 1] (after _center_crop_wide + preprocess); noise: the posterior draw"""
    post = vae.encode(image)[0]
    return i2vgen_prepare_image_latents(post.sample(noise=noise) * vae.scaling_factor, num_frames, num_videos_per_prompt)


def svd_image_latents_from_image(vae, image: torch.Tensor, num_frames: int, num_videos_per_prompt: int,
                                 aug_noise: torch.Tensor, noise_aug_strength: float):
    """image: preprocess(image, height, width) in [-1, 1]; aug_noise: the pipeline generator's draw of image.shape"""
    image = image + noise_aug_strength * aug_noise
    return svd_image_latents(vae.encode(image)[0].mode(), num_frames, num_videos_per_prompt)
