"""The three pipeline classes ``inference.py`` imports (/root/reference/inference.py:351-367), under the reference's names
and with the reference's ``__init__`` / ``__call__`` signatures:

    sdxl.pipelines.sdxl_controlnet_adapter_pipeline.SDXLControlNetAdapterPipeline            (:235-275, :829-1434)
    i2vgen_xl.pipelines.i2vgen_xl_controlnet_adapter_pipeline.I2VGenXLControlNetAdapterPipeline   (:547-1143)
    svd.pipelines.svd_controlnet_adapter_pipeline.SVDControlNetAdapterPipeline                (:361-802)

What runs here is the denoising loop -- the hot path (SURVEY.md section 8): the loop classes of pipeline_sdxl /
pipeline_i2vgen / pipeline_svd on the H100 modules, CUDA-graph replayed.  Everything either side of the loop is a
different subsystem of the reference stack (CLIP text / vision encoders, the SD1.5 prompt helper, the VAE; SURVEY.md
section 8f) and is *duck-typed*: a pipeline uses whatever ``text_encoder`` / ``helper`` / ``image_encoder`` / ``vae``
objects it was constructed with (e.g. the diffusers / transformers ones where those libraries exist), and when one is
absent the caller passes that stage's OUTPUT instead -- ``prompt_embeds`` ... exactly as the reference signature already
allows, plus the keyword-only extensions listed in each ``__call__`` (``controlnet_prompt_embeds``, ``image_embeddings``,
``image_latents``, tensor ``control_images``).  ``output_type="latent"`` needs no VAE; with
``vae=ctrl_adapter_b200.vae.AutoencoderKL`` the SDXL and I2VGen-XL pipelines decode on the H100 kernels as well.
The two video pipelines also take the reference's ``image=`` (a PIL image, a list of them, or a [N, 3, H, W] tensor in
[0, 1]): the image latents are then built with ``self.vae.encode`` (our ``AutoencoderKL`` /
``AutoencoderKLTemporalDecoder`` on the H100 kernels, or any object with diffusers' ``encode()`` / ``config``) and the
image embeddings with the ``image_encoder`` + ``feature_extractor`` components, after the reference's own crop / resize
preprocessing (``encode_image`` of each pipeline).  Passed ``image_latents`` / ``image_embeddings`` keep priority.  Nothing
here falls back to a PyTorch implementation of the hot path.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import torch

from . import ops
from .controlnet import MultiControlNetModel
from .pipeline_i2vgen import I2VGenXLControlNetAdapterLoop
from .pipeline_sdxl import SDXLControlNetAdapterLoop
from .pipeline_svd import SVDControlNetAdapterLoop
from .vae import DiagonalGaussianDistribution, decode_latents, svd_decode_latents, tensor2vid
from .vae import postprocess as vae_postprocess

BF16 = torch.bfloat16


@dataclass
class StableDiffusionXLPipelineOutput:
    images: Any


@dataclass
class I2VGenXLPipelineOutput:
    frames: Any
    down_block_weights: Any = None
    mid_block_weights: Any = None


@dataclass
class StableVideoDiffusionPipelineOutput:
    frames: Any
    down_block_weights: Any = None
    mid_block_weights: Any = None


class DiffusionPipeline:
    """The slice of diffusers' DiffusionPipeline the three pipelines use (SURVEY.md section 8b row 1): module registry,
    ``to()``, ``_execution_device``, ``progress_bar``, ``from_pretrained`` with component overrides."""

    _unet_class = None      # set by the subclasses: the H100 UNet of the backbone
    _unet_subfolder = "unet"

    def __init__(self):
        self._modules_registry: Dict[str, Any] = {}
        self._progress_bar_config: Dict[str, Any] = {}
        self._interrupt = False

    def register_modules(self, **kwargs):
        for name, module in kwargs.items():
            self._modules_registry[name] = module
            setattr(self, name, module)

    @property
    def components(self) -> Dict[str, Any]:
        return dict(self._modules_registry)

    def to(self, *args, **kwargs):
        for name, m in self._modules_registry.items():
            if isinstance(m, torch.nn.Module):
                setattr(self, name, m.to(*args, **kwargs))
                self._modules_registry[name] = getattr(self, name)
        return self

    @property
    def device(self) -> torch.device:
        for m in self._modules_registry.values():
            if isinstance(m, torch.nn.Module):
                p = next(m.parameters(), None)
                if p is not None:
                    return p.device
        return torch.device("cpu")

    _execution_device = device

    def set_progress_bar_config(self, **kwargs):
        self._progress_bar_config = kwargs

    def progress_bar(self, iterable=None, total=None):
        from tqdm.auto import tqdm
        return tqdm(iterable, total=total, **self._progress_bar_config) if iterable is not None else \
            tqdm(total=total, **self._progress_bar_config)

    def maybe_free_model_hooks(self):
        pass

    def _controlnet_prompt_embeds(self, prompt, device, embeds, negative_embeds) -> torch.Tensor:
        """The SD1.5 ControlNet's prompt embeddings, negative half first: passed in, or from the helper's
        ``encode_controlnet_prompt``."""
        if embeds is None:
            helper = _need(self.helper, "controlnet_prompt_embeds", "SD1.5 prompt helper")
            embeds, negative_embeds, _, _ = helper.encode_controlnet_prompt(
                prompt, device, 1, True, negative_prompt=None, prompt_embeds=None, negative_prompt_embeds=None,
                lora_scale=None, clip_skip=None)
        _need(negative_embeds, "controlnet_negative_prompt_embeds", "SD1.5 prompt helper")
        return torch.cat([negative_embeds, embeds]).to(device)

    def _denoise(self, loop, num_inference_steps: int, use_cuda_graph: bool):
        with self.progress_bar(total=num_inference_steps) as bar:
            for i in range(num_inference_steps):
                (loop.step_graph if use_cuda_graph else loop.step)(i)
                bar.update()

    @property
    def interrupt(self):
        return self._interrupt

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, torch_dtype=None, **components):
        """``cls.from_pretrained(path, controlnet=..., adapter=..., helper=..., ...)`` as inference.py calls it.  The UNet
        is loaded from ``path/unet`` (config.json + safetensors, strict keys) unless passed; the encoder-stage components
        are whatever the caller passes (none are required for pre-encoded inputs)."""
        if "unet" not in components:
            folder = os.path.join(str(pretrained_model_name_or_path), cls._unet_subfolder)
            if not os.path.isdir(folder):
                raise FileNotFoundError(
                    f"{folder} not found: pass unet=... or a local snapshot folder (there is no hub access here)")
            components["unet"] = cls._unet_class.from_pretrained(folder, torch_dtype=torch_dtype)
        import inspect
        names = [p for p in inspect.signature(cls.__init__).parameters if p != "self"]
        kw = {n: components.pop(n, None) for n in names if n in components or
              inspect.signature(cls.__init__).parameters[n].default is inspect.Parameter.empty}
        if components:
            raise TypeError(f"unexpected components {sorted(components)}")
        return cls(**kw)


# ------------------------------------------------------------------------------------------------------------------
def _need(value, what: str, stage: str):
    if value is None:
        raise ValueError(f"{what} is required: this pipeline has no {stage} (the encoder stages are outside the H100 hot "
                         f"path) -- pass the pre-encoded tensor")
    return value


def _randn(shape, generator, device):
    if isinstance(generator, (list, tuple)):
        generator = generator[0]
    gdev = generator.device if generator is not None else torch.device("cpu")
    return torch.randn(shape, generator=generator, device=gdev, dtype=torch.float32).to(device)


def _first(v):
    """the reference's SDXL / SVD loops take one ControlNet: a list argument contributes its first entry"""
    return v[0] if isinstance(v, list) else v


def _per_frame(embeds: torch.Tensor, clips: int, frames: int) -> torch.Tensor:
    """ControlNet prompt embeddings with one row per clip -> one per frame-sample (i2vgen pipeline :871-874)."""
    return embeds.repeat_interleave(frames, dim=0) if embeds.shape[0] == clips else embeds


def _given_or_encoded(given, encoded):
    """(image_embeddings, image_latents): the passed tensors keep priority over the ones encode_image built"""
    return tuple(e if g is None else g for g, e in zip(given, encoded))


def _control_tensor(control_images, helper, n, width, height, device):
    """control images as the loops take them: [n, 3, H, W] in [0, 1], CFG-duplicated (negative half first)."""
    if torch.is_tensor(control_images):
        t = control_images.to(device)
        if t.dim() == 5:
            t = t.reshape(-1, *t.shape[2:])
        if t.shape[0] * 2 == n:
            t = torch.cat([t, t])
        if t.shape[0] != n:
            raise ValueError(f"control_images: expected {n // 2} or {n} images, got {t.shape[0]}")
        return t
    if helper is None:
        raise ValueError("control_images must be a tensor [N,3,H,W] in [0,1] when the pipeline has no helper "
                         "(ControlNetHelper.prepare_images does the PIL preprocessing in the reference)")
    imgs = helper.prepare_images(images=control_images, width=width, height=height, batch_size=1,
                                 num_images_per_prompt=1, device=device, dtype=BF16,
                                 do_classifier_free_guidance=True, guess_mode=False)
    return imgs.reshape(-1, *imgs.shape[-3:]) if imgs.dim() == 5 else imgs


def _vae(pipe):
    return _need(getattr(pipe, "vae", None), "a `vae` component (or output_type='latent')", "VAE")


# ---- conditioning-image preprocessing of the two video pipelines (restated from the reference and diffusers'
# VaeImageProcessor; i2vgen pipeline :1150-1203, svd pipeline :165-193, utils/utils_svd.py _resize_with_antialiasing) ----
def _image_list(image) -> list:
    """PIL image / list of them / [n, 3, H, W] (or [3, H, W]) tensor in [0, 1] -> list of PIL images"""
    from PIL import Image
    if isinstance(image, Image.Image):
        return [image]
    if torch.is_tensor(image):
        t = image.unsqueeze(0) if image.dim() == 3 else image
        arr = (t.detach().float().cpu().permute(0, 2, 3, 1).numpy() * 255).round().astype("uint8")
        return [Image.fromarray(a) for a in arr]
    if isinstance(image, (list, tuple)) and len(image) > 0:
        return [im for x in image for im in _image_list(x)]
    raise ValueError(f"`image` has to be a PIL image, a list of PIL images or a [N, 3, H, W] tensor, got {type(image)}")


def _center_crop_wide(image, resolution: Tuple[int, int]):
    """Resize (PIL BOX) so that the image covers `resolution` = (W, H) -- scale = min(w / W, h / H) of the first image,
    sizes round(w // scale) x round(h // scale) -- then crop the centred W x H box.  Tensors are converted to PIL first;
    a list comes back as a list."""
    from PIL import Image
    single = not isinstance(image, (list, tuple)) and not (torch.is_tensor(image) and image.dim() == 4)
    ims = _image_list(image)
    scale = min(ims[0].size[0] / resolution[0], ims[0].size[1] / resolution[1])
    ims = [u.resize((round(u.width // scale), round(u.height // scale)), resample=Image.BOX) for u in ims]
    x1, y1 = (ims[0].width - resolution[0]) // 2, (ims[0].height - resolution[1]) // 2
    ims = [u.crop((x1, y1, x1 + resolution[0], y1 + resolution[1])) for u in ims]
    return ims[0] if single else ims


def _resize_bilinear(image, resolution: Tuple[int, int]):
    from PIL import Image
    if isinstance(image, (list, tuple)):
        return [u.resize(resolution, Image.BILINEAR) for u in image]
    return image.resize(resolution, Image.BILINEAR)


def _pil_to_pt(images) -> torch.Tensor:
    """VaeImageProcessor.pil_to_numpy + numpy_to_pt: list of PIL -> [n, 3, H, W] fp32 in [0, 1]"""
    import numpy as np
    images = images if isinstance(images, (list, tuple)) else [images]
    arr = np.stack([np.array(im).astype(np.float32) / 255.0 for im in images])
    return torch.from_numpy(arr.transpose(0, 3, 1, 2))


def _vae_preprocess(image, height: Optional[int] = None, width: Optional[int] = None) -> torch.Tensor:
    """VaeImageProcessor.preprocess with do_normalize: PIL images are resized (Lanczos) to height x width when given,
    tensors in [0, 1] (nearest); then 2x - 1.  A tensor that already has negative values is taken as normalised."""
    from .helper import ControlNetHelper
    if torch.is_tensor(image):
        t = image.float().unsqueeze(0) if image.dim() == 3 else image.float()
        h, w = (height or t.shape[-2]), (width or t.shape[-1])
        t = ControlNetHelper._preprocess(t, h, w)
        return t if float(t.min()) < 0 else 2.0 * t - 1.0
    ims = _image_list(image)
    out = [ControlNetHelper._preprocess(im, height or im.height, width or im.width) for im in ims]
    return 2.0 * torch.cat(out) - 1.0


def _gaussian_window(size: int, sigma: float) -> torch.Tensor:
    x = torch.arange(size, dtype=torch.float32) - size // 2
    if size % 2 == 0:
        x = x + 0.5
    g = torch.exp(-x.pow(2.0) / (2 * sigma ** 2))
    return g / g.sum()


def _resize_with_antialiasing(x: torch.Tensor, size: Tuple[int, int]) -> torch.Tensor:
    """[n, C, H, W] fp32 -> [n, C, size]: separable Gaussian blur (sigma = max((factor - 1) / 2, 0.001) per axis, odd
    window of int(max(4 sigma, 3)) taps, reflect padding), then bicubic interpolation with align_corners=True -- the
    anti-aliased down-sizing the SVD pipeline applies before the CLIP image encoder."""
    import torch.nn.functional as F
    h, w = x.shape[-2:]
    sig = (max((h / size[0] - 1.0) / 2.0, 0.001), max((w / size[1] - 1.0) / 2.0, 0.001))
    ks = [int(max(2.0 * 2 * s, 3)) for s in sig]
    ks = [k + 1 if k % 2 == 0 else k for k in ks]
    n, c = x.shape[:2]
    for axis, (k, s) in ((1, (ks[1], sig[1])), (0, (ks[0], sig[0]))):   # x first, then y
        g = _gaussian_window(k, s).to(device=x.device, dtype=x.dtype)
        kern = g.view(1, 1, 1, k) if axis == 1 else g.view(1, 1, k, 1)
        lo = (k - 1) // 2
        pad = (lo, k - 1 - lo, 0, 0) if axis == 1 else (0, 0, lo, k - 1 - lo)
        xp = F.pad(x, pad, mode="reflect")
        x = F.conv2d(xp.reshape(n * c, 1, *xp.shape[-2:]), kern).reshape(n, c, h, w)
    return F.interpolate(x, size=size, mode="bicubic", align_corners=True)


def _clip_image_embeddings(image_encoder, feature_extractor, pixels: torch.Tensor, device, num_videos_per_prompt: int):
    """CLIP image embeddings as both pipelines' _encode_image builds them: pixels [n, 3, H, W] in [0, 1] -> normalised by
    the feature extractor -> image_encoder(...).image_embeds -> (2 * n * nv, 1, D), zeros for the unconditional half."""
    _need(image_encoder, "image_embeddings (or an `image_encoder` component)", "CLIP vision encoder")
    _need(feature_extractor, "image_embeddings (or a `feature_extractor` component)", "CLIP image processor")
    pv = feature_extractor(images=pixels, do_normalize=True, do_center_crop=False, do_resize=False, do_rescale=False,
                           return_tensors="pt").pixel_values
    dtype = next(image_encoder.parameters()).dtype
    emb = image_encoder(pv.to(device=device, dtype=dtype)).image_embeds.unsqueeze(1)
    bs, seq, _ = emb.shape
    emb = emb.repeat(1, num_videos_per_prompt, 1).view(bs * num_videos_per_prompt, seq, -1)
    return torch.cat([torch.zeros_like(emb), emb])


def _posterior(vae, image: torch.Tensor):
    return vae.encode(image).latent_dist


def i2vgen_image_latents(vae, image: torch.Tensor, num_frames: int, num_videos_per_prompt: int,
                         noise: Optional[torch.Tensor] = None) -> torch.Tensor:
    """i2vgen pipeline :487-517 prepare_image_latents: image [n, 3, H, W] in [-1, 1] -> (2*n*nv, 4, F, h, w) bf16:
    frame 0 = posterior sample * scaling_factor (noise from the global RNG unless given), frame k = k / (F - 1)."""
    post = _posterior(vae, image)
    if isinstance(post, DiagonalGaussianDistribution):
        return ops.vae_latents(post.moments, ops.VAE_I2VGEN, noise=post.noise() if noise is None else noise,
                               frames=num_frames, num_videos=num_videos_per_prompt, scale=vae.config.scaling_factor)
    # a diffusers-compatible VAE: the same assembly on its tensors
    x = (post.sample() * vae.config.scaling_factor).unsqueeze(2)
    pos = [torch.ones_like(x) * ((k + 1) / (num_frames - 1)) for k in range(num_frames - 1)]
    x = torch.cat([x] + pos, dim=2).repeat(num_videos_per_prompt, 1, 1, 1, 1)
    return torch.cat([x, x]).to(BF16)


def svd_image_latents(vae, image: torch.Tensor, num_frames: int, num_videos_per_prompt: int) -> torch.Tensor:
    """svd pipeline :214-235 _encode_vae_image + :580-583: image [n, 3, H, W] -> (2*n*nv, F, 4, h, w) bf16 = posterior
    mode (no scaling factor) after zeros, repeated nv times, then over the frames (for nv > 1 the batch order is
    [0, L, 0, L], the reference's)."""
    post = _posterior(vae, image)
    if isinstance(post, DiagonalGaussianDistribution):
        return ops.vae_latents(post.moments, ops.VAE_SVD, frames=num_frames, num_videos=num_videos_per_prompt)
    m = post.mode()
    x = torch.cat([torch.zeros_like(m), m]).repeat(num_videos_per_prompt, 1, 1, 1)
    return x.unsqueeze(1).repeat(1, num_frames, 1, 1, 1).to(BF16)


def sdxl_add_time_ids(batch, height, width, original_size=None, crops_coords_top_left=(0, 0), target_size=None,
                      negative_original_size=None, negative_crops_coords_top_left=(0, 0), negative_target_size=None):
    """SDXL micro-conditioning (sdxl pipeline :1185-1219): [2 * batch, 6] fp32 rows original_size +
    crops_coords_top_left + target_size, negative rows first.  Sizes are (height, width); both default to the
    generated image's."""
    original_size = original_size or (height, width)
    target_size = target_size or (height, width)
    ids = torch.tensor([list(original_size) + list(crops_coords_top_left) + list(target_size)], dtype=torch.float32)
    if negative_original_size is not None and negative_target_size is not None:
        nids = torch.tensor([list(negative_original_size) + list(negative_crops_coords_top_left) +
                             list(negative_target_size)], dtype=torch.float32)
    else:
        nids = ids
    return torch.cat([nids.repeat(batch, 1), ids.repeat(batch, 1)])


# ------------------------------------------------------------------------------------------------------------------
class SDXLControlNetAdapterPipeline(DiffusionPipeline):
    """sdxl/pipelines/sdxl_controlnet_adapter_pipeline.py:235-275 (constructor), :829-1434 (__call__)."""

    def __init__(self, vae, text_encoder, text_encoder_2, tokenizer, tokenizer_2, unet, scheduler, adapter, helper,
                 controlnet, image_encoder=None, feature_extractor=None, force_zeros_for_empty_prompt: bool = True,
                 add_watermarker: Optional[bool] = None):
        super().__init__()
        if isinstance(controlnet, (list, tuple)):
            controlnet = MultiControlNetModel(controlnet)
        self.register_modules(vae=vae, text_encoder=text_encoder, text_encoder_2=text_encoder_2, tokenizer=tokenizer,
                              tokenizer_2=tokenizer_2, unet=unet, scheduler=scheduler, image_encoder=image_encoder,
                              feature_extractor=feature_extractor, controlnet=controlnet, adapter=adapter, helper=helper)
        self.vae_scale_factor = 8
        self.default_sample_size = 128
        self.watermark = None

    @torch.no_grad()
    def __call__(self, prompt: Union[str, List[str]] = None, prompt_2=None, height: Optional[int] = None,
                 width: Optional[int] = None, num_inference_steps: int = 50, timesteps: List[int] = None,
                 denoising_end: Optional[float] = None, guidance_scale: float = 5.0, negative_prompt=None,
                 negative_prompt_2=None, num_images_per_prompt: Optional[int] = 1, eta: float = 0.0, generator=None,
                 latents: Optional[torch.Tensor] = None, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None,
                 pooled_prompt_embeds: Optional[torch.Tensor] = None,
                 negative_pooled_prompt_embeds: Optional[torch.Tensor] = None, ip_adapter_image=None,
                 ip_adapter_image_embeds=None, output_type: Optional[str] = "pil", return_dict: bool = True,
                 cross_attention_kwargs: Optional[Dict[str, Any]] = None, guidance_rescale: float = 0.0,
                 original_size: Optional[Tuple[int, int]] = None, crops_coords_top_left: Tuple[int, int] = (0, 0),
                 target_size: Optional[Tuple[int, int]] = None, negative_original_size=None,
                 negative_crops_coords_top_left: Tuple[int, int] = (0, 0), negative_target_size=None,
                 clip_skip: Optional[int] = None, callback_on_step_end: Optional[Callable] = None,
                 callback_on_step_end_tensor_inputs: List[str] = ["latents"],
                 # the reference's additions
                 skip_conv_in=False, skip_time_emb=False, control_images=None,
                 controlnet_conditioning_scale: Union[float, List[float]] = 1.0,
                 control_guidance_start: Union[float, List[float]] = 0.0,
                 control_guidance_end: Union[float, List[float]] = 1.0, guess_mode: bool = False, use_size_512=True,
                 inference_expert_masks=None,
                 # extensions: outputs of the encoder stages this package does not contain
                 controlnet_prompt_embeds: Optional[torch.Tensor] = None,
                 controlnet_negative_prompt_embeds: Optional[torch.Tensor] = None, use_cuda_graph: bool = True,
                 **kwargs):
        if isinstance(self.controlnet, MultiControlNetModel):
            raise Exception("not supported yet")  # the reference's own message (:1159)
        for name, v in dict(timesteps=timesteps, denoising_end=denoising_end, ip_adapter_image=ip_adapter_image,
                            ip_adapter_image_embeds=ip_adapter_image_embeds, cross_attention_kwargs=cross_attention_kwargs,
                            callback_on_step_end=callback_on_step_end).items():
            if v is not None:
                raise NotImplementedError(f"{name}: not on the Ctrl-Adapter inference path")
        if guidance_rescale or guess_mode or skip_conv_in or skip_time_emb:
            raise NotImplementedError("guidance_rescale / guess_mode / skip_* are unused by the SDXL scripts")
        height = height or self.default_sample_size * self.vae_scale_factor
        width = width or self.default_sample_size * self.vae_scale_factor
        device = self._execution_device
        # 3. prompt encodings (:1103-1143)
        if prompt_embeds is None:
            enc = _need(getattr(self, "encode_prompt", None), "prompt_embeds", "text encoder")
            prompt_embeds, negative_prompt_embeds, pooled_prompt_embeds, negative_pooled_prompt_embeds = enc(
                prompt=prompt, prompt_2=prompt_2, device=device, num_images_per_prompt=num_images_per_prompt,
                do_classifier_free_guidance=True, negative_prompt=negative_prompt, negative_prompt_2=negative_prompt_2)
        batch = prompt_embeds.shape[0]
        _need(negative_prompt_embeds, "negative_prompt_embeds", "text encoder")
        _need(pooled_prompt_embeds, "pooled_prompt_embeds", "text encoder")
        _need(negative_pooled_prompt_embeds, "negative_pooled_prompt_embeds", "text encoder")
        cpe = self._controlnet_prompt_embeds(prompt, device, controlnet_prompt_embeds,
                                             controlnet_negative_prompt_embeds)
        images = _control_tensor(_need(control_images, "control_images", "condition"), self.helper, 2 * batch, 512, 512,
                                 device)
        # 5. latents (:1170-1181): unit noise, scaled by init_noise_sigma inside the loop's prepare()
        shape = (batch * num_images_per_prompt, 4, height // self.vae_scale_factor, width // self.vae_scale_factor)
        # (user latents are scaled by init_noise_sigma as well, like the reference's prepare_latents)
        lat = latents.to(device).float() if latents is not None else _randn(shape, generator, device)
        add_time_ids = sdxl_add_time_ids(batch, height, width, original_size, crops_coords_top_left, target_size,
                                         negative_original_size, negative_crops_coords_top_left,
                                         negative_target_size).to(device)
        loop = SDXLControlNetAdapterLoop(
            self.controlnet, self.adapter, self.unet, num_inference_steps=num_inference_steps,
            guidance_scale=guidance_scale, controlnet_conditioning_scale=_first(controlnet_conditioning_scale),
            use_size_512=use_size_512, control_guidance_start=_first(control_guidance_start),
            control_guidance_end=_first(control_guidance_end))
        loop.prepare(latents=lat, prompt_embeds=torch.cat([negative_prompt_embeds, prompt_embeds]).to(device),
                     add_text_embeds=torch.cat([negative_pooled_prompt_embeds, pooled_prompt_embeds]).to(device),
                     add_time_ids=add_time_ids, controlnet_prompt_embeds=cpe, control_images=images)
        self._denoise(loop, num_inference_steps, use_cuda_graph)
        latents = loop.latents.to(prompt_embeds.dtype)
        if output_type == "latent":
            image = latents
        else:
            vae = _vae(self)  # ctrl_adapter_b200.vae.AutoencoderKL, or any object with diffusers' decode() / config
            image = vae.decode(latents / vae.config.scaling_factor, return_dict=False)[0]           # :1414
            proc = getattr(self, "image_processor", None)
            image = proc.postprocess(image, output_type=output_type) if proc is not None else \
                vae_postprocess(image, output_type)
        if not return_dict:
            return (image,)
        return StableDiffusionXLPipelineOutput(images=image), None, None  # (:1433) no router on the SDXL path


class I2VGenXLControlNetAdapterPipeline(DiffusionPipeline):
    """i2vgen_xl/pipelines/i2vgen_xl_controlnet_adapter_pipeline.py (__call__ :547-1143)."""

    def __init__(self, vae, text_encoder, tokenizer, image_encoder, feature_extractor, unet, scheduler, controlnet,
                 adapter, helper, router=None):
        super().__init__()
        if isinstance(controlnet, (list, tuple)):
            controlnet = MultiControlNetModel(controlnet)
        self.register_modules(vae=vae, text_encoder=text_encoder, tokenizer=tokenizer, image_encoder=image_encoder,
                              feature_extractor=feature_extractor, unet=unet, scheduler=scheduler, controlnet=controlnet,
                              adapter=adapter, helper=helper, router=router)
        self.vae_scale_factor = 8

    @torch.no_grad()
    def encode_image(self, image, height: int, width: int, num_frames: int, num_videos_per_prompt: int = 1,
                     device=None, embeddings: bool = True, latents: bool = True, noise: Optional[torch.Tensor] = None):
        """The conditioning image as the loop takes it (:795-812): (image_embeddings (2*n*nv, 1, D) or None,
        image_latents (2*n*nv, 4, F, h, w) bf16 or None) for n images.
        CLIP: _center_crop_wide to width x width, bilinear resize to the feature extractor's crop size, image_encoder.
        VAE: _center_crop_wide to width x height, 2x - 1, vae.encode, posterior sample (unit noise from the global RNG,
        as the reference draws it, unless `noise` [n, 4, h, w] fp32 is given) * scaling_factor, position planes."""
        device = device or self._execution_device
        emb = lat = None
        if embeddings:
            fe = _need(self.feature_extractor, "image_embeddings (or a `feature_extractor` component)",
                       "CLIP image processor")
            crop = fe.crop_size
            ims = _resize_bilinear(_center_crop_wide(_image_list(image), (width, width)), (crop["width"], crop["height"]))
            emb = _clip_image_embeddings(self.image_encoder, fe, _pil_to_pt(ims), device, num_videos_per_prompt)
        if latents:
            vae = _need(getattr(self, "vae", None), "image_latents (or a `vae` component)", "VAE")
            x = _vae_preprocess(_center_crop_wide(_image_list(image), (width, height))).to(device=device, dtype=BF16)
            lat = i2vgen_image_latents(vae, x, num_frames, num_videos_per_prompt, noise)
        return emb, lat

    @torch.no_grad()
    def __call__(self, prompt: Union[str, List[str]] = None, image=None, height: Optional[int] = 704,
                 width: Optional[int] = 1280, target_fps: Optional[int] = 16, num_frames: int = 16,
                 num_inference_steps: int = 50, guidance_scale: float = 9.0, negative_prompt=None, eta: float = 0.0,
                 num_videos_per_prompt: Optional[int] = 1, decode_chunk_size: Optional[int] = 1, generator=None,
                 latents: Optional[torch.Tensor] = None, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None, output_type: Optional[str] = "pil",
                 return_dict: bool = True, cross_attention_kwargs=None, clip_skip: Optional[int] = 1,
                 # the reference's additions
                 control_images=None, controlnet_conditioning_scale: Union[float, List[float]] = 1.0,
                 control_guidance_start: Union[float, List[float]] = 0.0,
                 control_guidance_end: Union[float, List[float]] = 1.0, num_images_per_prompt: Optional[int] = 1,
                 guess_mode: bool = False, crops_coords_top_left: Tuple[int, int] = (0, 0), negative_original_size=None,
                 negative_crops_coords_top_left: Tuple[int, int] = (0, 0), negative_target_size=None,
                 sparse_frames=None, skip_conv_in=False, skip_time_emb=False, fixed_controlnet_timestep=-1,
                 use_size_512=True, adapter_locations=None, inference_expert_masks=None, fixed_weights=None,
                 # extensions: outputs of the encoder stages this package does not contain
                 controlnet_prompt_embeds: Optional[torch.Tensor] = None,
                 controlnet_negative_prompt_embeds: Optional[torch.Tensor] = None,
                 image_embeddings: Optional[torch.Tensor] = None, image_latents: Optional[torch.Tensor] = None,
                 use_cuda_graph: bool = True):
        if cross_attention_kwargs is not None or guess_mode or fixed_weights is not None:
            raise NotImplementedError("cross_attention_kwargs / guess_mode / fixed_weights: not on the inference path")
        device = self._execution_device
        f = num_frames
        prompt_embeds = _need(prompt_embeds, "prompt_embeds", "text encoder")
        negative_prompt_embeds = _need(negative_prompt_embeds, "negative_prompt_embeds", "text encoder")
        b = prompt_embeds.shape[0]
        # image_embeddings (2B,1,1024) negative first (:808-815); image_latents (2B,4,F,h,w) (:818-833); built from
        # `image` when not passed
        if image is not None and (image_embeddings is None or image_latents is None):
            image_embeddings, image_latents = _given_or_encoded((image_embeddings, image_latents), self.encode_image(
                image, height, width, f, num_videos_per_prompt, device, embeddings=image_embeddings is None,
                latents=image_latents is None))
        image_embeddings = _need(image_embeddings, "image_embeddings (or `image`)", "CLIP vision encoder").to(device)
        image_latents = _need(image_latents, "image_latents (or `image`)", "VAE encoder").to(device)
        n = 2 * b * f
        cpe = _per_frame(self._controlnet_prompt_embeds(prompt, device, controlnet_prompt_embeds,
                                                        controlnet_negative_prompt_embeds), 2 * b, f)
        multi = isinstance(self.controlnet, MultiControlNetModel)
        _need(control_images, "control_images", "condition")
        if multi:
            images = [_control_tensor(ci, self.helper, n, 512, 512, device) for ci in control_images]
        else:
            images = _control_tensor(control_images, self.helper, n, 512, 512, device)
        shape = (b * num_videos_per_prompt, 4, f, height // self.vae_scale_factor, width // self.vae_scale_factor)
        lat = latents.to(device).float() if latents is not None else _randn(shape, generator, device)
        fps = torch.full((2 * b,), float(target_fps), device=device)
        loop = I2VGenXLControlNetAdapterLoop(
            self.controlnet, self.adapter, self.unet, self.router, num_inference_steps=num_inference_steps,
            guidance_scale=guidance_scale, controlnet_conditioning_scale=controlnet_conditioning_scale,
            inference_expert_masks=inference_expert_masks, skip_conv_in=skip_conv_in, skip_time_emb=skip_time_emb,
            sparse_frames=sparse_frames, use_size_512=use_size_512, control_guidance_start=control_guidance_start,
            control_guidance_end=control_guidance_end, fixed_controlnet_timestep=fixed_controlnet_timestep)
        loop.prepare(latents=lat, prompt_embeds=torch.cat([negative_prompt_embeds, prompt_embeds]).to(device),
                     image_latents=image_latents, image_embeddings=image_embeddings, fps=fps,
                     controlnet_prompt_embeds=cpe, control_images=images)
        self._denoise(loop, num_inference_steps, use_cuda_graph)
        latents = loop.latents_bcfhw().to(prompt_embeds.dtype)
        weights = (None, None)
        if self.router is not None and loop._router_w is not None:  # the reference logs them per step (:990-995)
            dw, mw = self.router(sparse_mask=inference_expert_masks)
            weights = ([dw.cpu().numpy().tolist()] * num_inference_steps,
                       [mw.cpu().numpy().tolist() if mw is not None else None] * num_inference_steps)
        if output_type == "latent":
            video = latents
        else:
            video = tensor2vid(decode_latents(_vae(self), latents, decode_chunk_size), output_type)  # :398-418, :1134-1135
        if not return_dict:
            return (video,)
        return I2VGenXLPipelineOutput(frames=video, down_block_weights=weights[0], mid_block_weights=weights[1])


class SVDControlNetAdapterPipeline(DiffusionPipeline):
    """svd/pipelines/svd_controlnet_adapter_pipeline.py (__call__ :361-802)."""

    def __init__(self, vae, image_encoder, unet, scheduler, feature_extractor, adapter, helper, controlnet):
        super().__init__()
        if isinstance(controlnet, (list, tuple)):
            controlnet = MultiControlNetModel(controlnet)
        self.register_modules(vae=vae, image_encoder=image_encoder, unet=unet, scheduler=scheduler,
                              feature_extractor=feature_extractor, controlnet=controlnet, adapter=adapter, helper=helper)
        self.vae_scale_factor = 8

    def decode_latents(self, latents: torch.Tensor, num_frames: int, decode_chunk_size: int = 14):
        """svd pipeline :265-292: (B, F, 4, h, w) latents -> (B, 3, F, H, W) fp32 frames in [-1, 1]."""
        return svd_decode_latents(_vae(self), latents, num_frames, decode_chunk_size)

    @torch.no_grad()
    def encode_image(self, image, height: int, width: int, num_frames: int, num_videos_per_prompt: int = 1,
                     noise_aug_strength: float = 0.02, generator=None, device=None, embeddings: bool = True,
                     latents: bool = True):
        """The conditioning image as the loop takes it (:553-583): (image_embeddings (2*n*nv, 1, D) or None,
        image_latents (2*n*nv, F, 4, h, w) bf16 or None) for n images.
        CLIP: 2x - 1, _resize_with_antialiasing to 224 x 224, (x + 1) / 2 (PIL input; a tensor goes to the feature
        extractor as it is, as in the reference), image_encoder.
        VAE: Lanczos resize to width x height, 2x - 1, + noise_aug_strength * randn(generator), vae.encode, posterior
        mode (no scaling factor), zeros for the unconditional half."""
        device = device or self._execution_device
        emb = lat = None
        if embeddings:
            if torch.is_tensor(image):
                pixels = image.float().unsqueeze(0) if image.dim() == 3 else image.float()
            else:
                pixels = (_resize_with_antialiasing(_pil_to_pt(_image_list(image)) * 2.0 - 1.0, (224, 224)) + 1.0) / 2.0
            emb = _clip_image_embeddings(self.image_encoder, _need(self.feature_extractor, "image_embeddings (or a "
                                         "`feature_extractor` component)", "CLIP image processor"), pixels, device,
                                         num_videos_per_prompt)
        if latents:
            vae = _need(getattr(self, "vae", None), "image_latents (or a `vae` component)", "VAE")
            x = _vae_preprocess(image, height, width).to(device)
            x = x + noise_aug_strength * _randn(tuple(x.shape), generator, device)
            lat = svd_image_latents(vae, x, num_frames, num_videos_per_prompt)
        return emb, lat

    @torch.no_grad()
    def __call__(self, image=None, prompt: str = "", height: int = 576, width: int = 1024,
                 num_frames: Optional[int] = None, num_inference_steps: int = 25, min_guidance_scale: float = 1.0,
                 max_guidance_scale: float = 3.0, fps: int = 7, motion_bucket_id: int = 127,
                 noise_aug_strength: float = 0.02, decode_chunk_size: Optional[int] = None,
                 num_videos_per_prompt: Optional[int] = 1, generator=None, latents: Optional[torch.Tensor] = None,
                 output_type: Optional[str] = "pil", callback_on_step_end: Optional[Callable] = None,
                 callback_on_step_end_tensor_inputs: List[str] = ["latents"], return_dict: bool = True,
                 # the reference's additions
                 sparse_frames=None, control_images=None, controlnet_conditioning_scale: Union[float, List[float]] = 1.0,
                 control_guidance_start: Union[float, List[float]] = 0.0,
                 control_guidance_end: Union[float, List[float]] = 1.0, guess_mode: bool = False,
                 crops_coords_top_left: Tuple[int, int] = (0, 0), negative_original_size=None,
                 negative_crops_coords_top_left: Tuple[int, int] = (0, 0), negative_target_size=None,
                 skip_conv_in=False, skip_time_emb=False, fixed_controlnet_timestep=-1, use_size_512=True,
                 adapter_locations=['A', 'B', 'C', 'D', 'M'], inference_expert_masks=None,
                 # extensions: outputs of the encoder stages this package does not contain
                 controlnet_prompt_embeds: Optional[torch.Tensor] = None,
                 controlnet_negative_prompt_embeds: Optional[torch.Tensor] = None,
                 image_embeddings: Optional[torch.Tensor] = None, image_latents: Optional[torch.Tensor] = None,
                 use_cuda_graph: bool = True):
        if isinstance(self.controlnet, MultiControlNetModel) or callback_on_step_end is not None or guess_mode:
            raise NotImplementedError("Multi-ControlNet / callbacks / guess_mode: not on the SVD inference path")
        device = self._execution_device
        f = num_frames if num_frames is not None else self.unet.config.num_frames
        # image_embeddings (2B,1,1024): zeros for the unconditional half (:497-503); image_latents (2B,F,4,h,w) (:566-583);
        # built from `image` when not passed.  The noise augmentation draws from `generator` before the latents do.
        if image is not None and (image_embeddings is None or image_latents is None):
            image_embeddings, image_latents = _given_or_encoded((image_embeddings, image_latents), self.encode_image(
                image, height, width, f, num_videos_per_prompt, noise_aug_strength, generator, device,
                embeddings=image_embeddings is None, latents=image_latents is None))
            # B below is image_embeddings.shape[0] // 2, which now counts every video of every image
            num_videos_per_prompt = 1
        image_embeddings = _need(image_embeddings, "image_embeddings (or `image`)", "CLIP vision encoder").to(device)
        image_latents = _need(image_latents, "image_latents (or `image`)", "VAE encoder").to(device)
        b = image_embeddings.shape[0] // 2
        n = 2 * b * f
        cpe = _per_frame(self._controlnet_prompt_embeds(prompt, device, controlnet_prompt_embeds,
                                                        controlnet_negative_prompt_embeds), 2 * b, f)
        images = _control_tensor(_need(control_images, "control_images", "condition"), self.helper, n,
                                 512 if use_size_512 else width, 512 if use_size_512 else height, device)
        # added time ids (:586-596): fps - 1 is what the model was conditioned on during training
        ids = torch.tensor([[float(fps - 1), float(motion_bucket_id), float(noise_aug_strength)]], device=device)
        added_time_ids = ids.repeat(2 * b * num_videos_per_prompt, 1)
        shape = (b * num_videos_per_prompt, f, 4, height // self.vae_scale_factor, width // self.vae_scale_factor)
        lat = latents.to(device).float() if latents is not None else _randn(shape, generator, device)
        loop = SVDControlNetAdapterLoop(
            self.controlnet, self.adapter, self.unet, num_inference_steps=num_inference_steps,
            min_guidance_scale=min_guidance_scale, max_guidance_scale=max_guidance_scale,
            controlnet_conditioning_scale=_first(controlnet_conditioning_scale), use_size_512=use_size_512,
            skip_conv_in=skip_conv_in, skip_time_emb=skip_time_emb, sparse_frames=sparse_frames,
            control_guidance_start=_first(control_guidance_start), control_guidance_end=_first(control_guidance_end))
        loop.prepare(latents=lat, image_latents=image_latents, image_embeddings=image_embeddings,
                     added_time_ids=added_time_ids, controlnet_prompt_embeds=cpe, control_images=images)
        self._denoise(loop, num_inference_steps, use_cuda_graph)
        latents = loop.latents.to(image_embeddings.dtype)
        if output_type == "latent":
            frames = latents
        else:
            # svd pipeline :495, :787-792: AutoencoderKLTemporalDecoder over chunks of decode_chunk_size frames
            chunk = decode_chunk_size if decode_chunk_size is not None else f
            frames = tensor2vid(self.decode_latents(latents, f, chunk), output_type)
        if not return_dict:
            return frames
        return StableVideoDiffusionPipelineOutput(frames=frames, down_block_weights=None, mid_block_weights=None)


def _bind_unets():
    from .unet_i2vgen import I2VGenXLUNet
    from .unet_sdxl import UNet2DConditionModel
    from .unet_svd import UNetSpatioTemporalConditionModel
    SDXLControlNetAdapterPipeline._unet_class = UNet2DConditionModel
    I2VGenXLControlNetAdapterPipeline._unet_class = I2VGenXLUNet
    SVDControlNetAdapterPipeline._unet_class = UNetSpatioTemporalConditionModel


_bind_unets()
