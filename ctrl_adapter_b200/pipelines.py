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
``vae=ctrl_adapter_b200.vae.AutoencoderKL`` the SDXL and I2VGen-XL pipelines decode on the H100 kernels as well.  Nothing
here falls back to a PyTorch implementation of the hot path.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import torch

from .controlnet import MultiControlNetModel
from .pipeline_i2vgen import I2VGenXLControlNetAdapterLoop
from .pipeline_sdxl import SDXLControlNetAdapterLoop
from .pipeline_svd import SVDControlNetAdapterLoop
from .vae import decode_latents, svd_decode_latents, tensor2vid
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
        original_size = original_size or (height, width)
        target_size = target_size or (height, width)
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
        if controlnet_prompt_embeds is None:
            helper = _need(self.helper, "controlnet_prompt_embeds", "SD1.5 prompt helper")
            controlnet_prompt_embeds, controlnet_negative_prompt_embeds, _, _ = helper.encode_controlnet_prompt(
                prompt, device, 1, True, negative_prompt=None, prompt_embeds=None, negative_prompt_embeds=None,
                lora_scale=None, clip_skip=None)
        _need(controlnet_negative_prompt_embeds, "controlnet_negative_prompt_embeds", "SD1.5 prompt helper")
        images = _control_tensor(_need(control_images, "control_images", "condition"), self.helper, 2 * batch, 512, 512,
                                 device)
        # 5. latents (:1170-1181): unit noise, scaled by init_noise_sigma inside the loop's prepare()
        shape = (batch * num_images_per_prompt, 4, height // self.vae_scale_factor, width // self.vae_scale_factor)
        # (user latents are scaled by init_noise_sigma as well, like the reference's prepare_latents)
        lat = latents.to(device).float() if latents is not None else _randn(shape, generator, device)
        # 7. micro-conditioning (:1185-1219)
        ids = torch.tensor([list(original_size) + list(crops_coords_top_left) + list(target_size)], dtype=torch.float32)
        if negative_original_size is not None and negative_target_size is not None:
            nids = torch.tensor([list(negative_original_size) + list(negative_crops_coords_top_left) +
                                 list(negative_target_size)], dtype=torch.float32)
        else:
            nids = ids
        add_time_ids = torch.cat([nids.repeat(batch, 1), ids.repeat(batch, 1)]).to(device)
        cscale = controlnet_conditioning_scale
        loop = SDXLControlNetAdapterLoop(
            self.controlnet, self.adapter, self.unet, num_inference_steps=num_inference_steps,
            guidance_scale=guidance_scale, controlnet_conditioning_scale=cscale[0] if isinstance(cscale, list) else cscale,
            use_size_512=use_size_512,
            control_guidance_start=control_guidance_start[0] if isinstance(control_guidance_start, list) else control_guidance_start,
            control_guidance_end=control_guidance_end[0] if isinstance(control_guidance_end, list) else control_guidance_end)
        loop.prepare(latents=lat, prompt_embeds=torch.cat([negative_prompt_embeds, prompt_embeds]).to(device),
                     add_text_embeds=torch.cat([negative_pooled_prompt_embeds, pooled_prompt_embeds]).to(device),
                     add_time_ids=add_time_ids,
                     controlnet_prompt_embeds=torch.cat([controlnet_negative_prompt_embeds,
                                                         controlnet_prompt_embeds]).to(device),
                     control_images=images)
        with self.progress_bar(total=num_inference_steps) as bar:
            for i in range(num_inference_steps):
                (loop.step_graph if use_cuda_graph else loop.step)(i)
                bar.update()
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
        # image_embeddings (2B,1,1024) negative first (:808-815); image_latents (2B,4,F,h,w) (:818-833)
        image_embeddings = _need(image_embeddings, "image_embeddings", "CLIP vision encoder").to(device)
        image_latents = _need(image_latents, "image_latents", "VAE encoder").to(device)
        if controlnet_prompt_embeds is None:
            helper = _need(self.helper, "controlnet_prompt_embeds", "SD1.5 prompt helper")
            controlnet_prompt_embeds, controlnet_negative_prompt_embeds, _, _ = helper.encode_controlnet_prompt(
                prompt, device, 1, True, negative_prompt=None, prompt_embeds=None, negative_prompt_embeds=None,
                lora_scale=None, clip_skip=None)
        _need(controlnet_negative_prompt_embeds, "controlnet_negative_prompt_embeds", "SD1.5 prompt helper")
        n = 2 * b * f
        cpe = torch.cat([controlnet_negative_prompt_embeds, controlnet_prompt_embeds]).to(device)
        if cpe.shape[0] == 2 * b:  # one row per clip -> one per frame-sample (:871-874)
            cpe = cpe.repeat_interleave(f, dim=0)
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
        with self.progress_bar(total=num_inference_steps) as bar:
            for i in range(num_inference_steps):
                (loop.step_graph if use_cuda_graph else loop.step)(i)
                bar.update()
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
        # image_embeddings (2B,1,1024): zeros for the unconditional half (:497-503); image_latents (2B,F,4,h,w) (:566-583)
        image_embeddings = _need(image_embeddings, "image_embeddings", "CLIP vision encoder").to(device)
        image_latents = _need(image_latents, "image_latents", "VAE encoder").to(device)
        b = image_embeddings.shape[0] // 2
        if controlnet_prompt_embeds is None:
            helper = _need(self.helper, "controlnet_prompt_embeds", "SD1.5 prompt helper")
            controlnet_prompt_embeds, controlnet_negative_prompt_embeds, _, _ = helper.encode_controlnet_prompt(
                prompt, device, 1, True, negative_prompt=None, prompt_embeds=None, negative_prompt_embeds=None,
                lora_scale=None, clip_skip=None)
        _need(controlnet_negative_prompt_embeds, "controlnet_negative_prompt_embeds", "SD1.5 prompt helper")
        n = 2 * b * f
        cpe = torch.cat([controlnet_negative_prompt_embeds, controlnet_prompt_embeds]).to(device)
        if cpe.shape[0] == 2 * b:
            cpe = cpe.repeat_interleave(f, dim=0)
        images = _control_tensor(_need(control_images, "control_images", "condition"), self.helper, n,
                                 512 if use_size_512 else width, 512 if use_size_512 else height, device)
        # added time ids (:586-596): fps - 1 is what the model was conditioned on during training
        ids = torch.tensor([[float(fps - 1), float(motion_bucket_id), float(noise_aug_strength)]], device=device)
        added_time_ids = ids.repeat(2 * b * num_videos_per_prompt, 1)
        shape = (b * num_videos_per_prompt, f, 4, height // self.vae_scale_factor, width // self.vae_scale_factor)
        lat = latents.to(device).float() if latents is not None else _randn(shape, generator, device)
        cs = controlnet_conditioning_scale
        loop = SVDControlNetAdapterLoop(
            self.controlnet, self.adapter, self.unet, num_inference_steps=num_inference_steps,
            min_guidance_scale=min_guidance_scale, max_guidance_scale=max_guidance_scale,
            controlnet_conditioning_scale=cs[0] if isinstance(cs, list) else cs, use_size_512=use_size_512,
            skip_conv_in=skip_conv_in, skip_time_emb=skip_time_emb, sparse_frames=sparse_frames,
            control_guidance_start=control_guidance_start[0] if isinstance(control_guidance_start, list) else control_guidance_start,
            control_guidance_end=control_guidance_end[0] if isinstance(control_guidance_end, list) else control_guidance_end)
        loop.prepare(latents=lat, image_latents=image_latents, image_embeddings=image_embeddings,
                     added_time_ids=added_time_ids, controlnet_prompt_embeds=cpe, control_images=images)
        with self.progress_bar(total=num_inference_steps) as bar:
            for i in range(num_inference_steps):
                (loop.step_graph if use_cuda_graph else loop.step)(i)
                bar.update()
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
