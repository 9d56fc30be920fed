"""What the three denoising loops share: the per-step control schedule (``controlnet_keep``), the pooling of the control
path to the ControlNet's 512x512 / 64x64 geometry, the video loops' key-frame adapter path, eager / CUDA-graph stepping.

Reference: the ``controlnet_keep`` list and ``cond_scale = controlnet_conditioning_scale * controlnet_keep[i]`` of
/root/reference/sdxl/pipelines/sdxl_controlnet_adapter_pipeline.py:1207-1211, :1296-1302 (identical code in
i2vgen_xl/...pipeline.py:844-850, :921-927 and svd/...pipeline.py:624-628, :652-658).  Every shipped inference script
passes ``--control_guidance_end`` < 1, so the steps past that fraction run with ``cond_scale == 0``: the reference then
drops the down-block residuals (:1346 ``if cond_scale == 0``).  A loop body is therefore parameterised by the step's
conditioning scale; one CUDA graph is captured per distinct scale value (normally two: the user's scale and 0) and the
per-step scalars (t, sigma, ...) live in device rows that a 16-byte copy refreshes before each replay.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Union

import torch

from . import ops
from .layers import BF16, as_nchw, to_channels_last_bf16

Scale = Union[float, tuple]


def controlnet_keep(num_steps: int, start: Sequence[float], end: Sequence[float]) -> List[List[float]]:
    """keeps[i][k] for ControlNet k at step i -- the reference's list comprehension, verbatim semantics."""
    return [[1.0 - float(i / num_steps < s or (i + 1) / num_steps > e) for s, e in zip(start, end)]
            for i in range(num_steps)]


def pool_control_images(images: torch.Tensor) -> torch.Tensor:
    """F.adaptive_avg_pool2d(images, (512, 512)) of the loop bodies (sdxl pipeline :1306-1312, svd :664-670).  It does
    not depend on the step, so the loops run it once in prepare().  images [N, 3, H, W] bf16, H and W multiples of
    512."""
    if tuple(images.shape[-2:]) == (512, 512):
        return images
    if images.shape[-2] % 512 or images.shape[-1] % 512:
        raise NotImplementedError("control images must be 512x512 or an integer multiple of it (adaptive pool windows)")
    return as_nchw(ops.avgpool(to_channels_last_bf16(images, 8), 512, 512))[:, :3].contiguous()


def pool_controlnet_input(latents: torch.Tensor) -> torch.Tensor:
    """F.adaptive_avg_pool2d(latents, (64, 64)): the ControlNet runs at 64x64 latents (512x512) whatever the backbone's
    resolution (same reference lines).  latents [N, 4, h, w] -> [N, 4, 64, 64], channels-last view."""
    return as_nchw(ops.avgpool(to_channels_last_bf16(latents, 8), 64, 64))[:, :4]


def check_geometry(loop: str, h: int, w: int, use_size_512: bool, control_images, *, multiple: int,
                   adapter_up: int) -> None:
    """Refuse, before any kernel runs, latents (h, w) or control images the loop body cannot carry through.

    The ControlNet runs at 64x64 latents when use_size_512 pools a latent size other than 64x64 (the reference's
    F.adaptive_avg_pool2d, here only at integer ratios), and at the latent size otherwise; its conditioning images are
    then 512x512 (pooled from integer multiples of 512) or 8 x the ControlNet's latent size.  The adapter returns its
    residuals at `adapter_up` x the ControlNet's size, and the UNet adds them to skips at the latent size, so the two
    must agree.  `multiple`: what the latent height and width must be multiples of (the UNet's down-samplers, the
    ControlNet's stride-2 convolutions when it runs at the latent size, I2VGen-XL's 32x32 image-latent pool).
    Domain of the three loops: SDXL (2x adapter) runs 128x128 latents with use_size_512; I2VGen-XL runs 64x64 with
    use_size_512, multiples of 32 without; SVD runs 64x64 with use_size_512, multiples of 8 without."""
    size = f"latents {h}x{w} (height {8 * h}, width {8 * w})"
    if h <= 0 or w <= 0 or h % multiple or w % multiple:
        raise ValueError(f"{loop}: height and width must be multiples of {8 * multiple} pixels (latent height and "
                         f"width multiples of {multiple}), got {size}")
    pool = use_size_512 and (h, w) != (64, 64)
    ch, cw = (64, 64) if pool else (h, w)
    if (ch * adapter_up, cw * adapter_up) != (h, w):
        why = "use_size_512 pools the ControlNet input to 64x64" if pool else "the ControlNet runs at the latent size"
        raise ValueError(f"{loop}: {size} with use_size_512={use_size_512} cannot be run: {why}, the adapter returns "
                         f"residuals at {ch * adapter_up}x{cw * adapter_up} and the UNet adds them at height x width "
                         f"{h}x{w}")
    for img in control_images if isinstance(control_images, (list, tuple)) else [control_images]:
        ih, iw = img.shape[-2:]
        if pool and (ih % 512 or iw % 512):
            raise ValueError(f"{loop}: control images of height {ih} and width {iw}: use_size_512 pools them to "
                             f"512x512, so height and width must be multiples of 512")
        if not pool and (ih, iw) != (8 * ch, 8 * cw):
            raise ValueError(f"{loop}: control images of height {ih} and width {iw}, expected height {8 * ch} and "
                             f"width {8 * cw} for {size}")


class DenoiseLoopBase:
    num_inference_steps: int

    def _init_control(self, conditioning_scale, control_guidance_start, control_guidance_end, num_nets: int):
        """Mirrors the reference's list alignment of start / end / scale (sdxl pipeline :1090-1105)."""
        s, e = control_guidance_start, control_guidance_end
        if not isinstance(s, (list, tuple)) and isinstance(e, (list, tuple)):
            s = len(e) * [s]
        elif not isinstance(e, (list, tuple)) and isinstance(s, (list, tuple)):
            e = len(s) * [e]
        elif not isinstance(s, (list, tuple)) and not isinstance(e, (list, tuple)):
            s, e = num_nets * [s], num_nets * [e]
        self._keep = controlnet_keep(self.num_inference_steps, list(s), list(e))
        self._multi = num_nets > 1
        if self._multi and not isinstance(conditioning_scale, (list, tuple)):
            conditioning_scale = [conditioning_scale] * num_nets
        self._scale = ([float(c) for c in conditioning_scale] if isinstance(conditioning_scale, (list, tuple))
                       else float(conditioning_scale))
        self._graphs: Dict[Scale, torch.cuda.CUDAGraph] = {}

    def _init_key_frames(self, clips: int, frames: int, device):
        """Rows of the `sparse_frames` key frames in the (clip, frame)-ordered batch of `clips` clips (None: all)."""
        self._sparse_rows = None
        if self.sparse_frames is not None:
            if not all(0 <= k < frames for k in self.sparse_frames):
                raise ValueError("sparse_frames must index frames of the clip")
            self._sparse_rows = torch.tensor([c * frames + k for c in range(clips) for k in self.sparse_frames],
                                             device=device)

    def _video_adapter(self, down, mid, t, n: int, mid_hw):
        """Ctrl-Adapter of the video loops (i2vgen pipeline :1024-1083, svd :700-750).  down / mid: the ControlNet's
        residuals for all n frame-samples, or down None when the step's conditioning scale is 0: every ControlNet output
        is then exactly zero and the down residuals are dropped, but the mid-block adapter's output (a function of t
        alone, on zeros of spatial size mid_hw) is still injected (quirk Q9).  With sparse_frames, only the key frames
        go through the adapter (host-side index gather over ControlNet-sized tensors) and are scattered into zero
        residuals; the reference's dense tensors are fp32 zeros, which only changes where the skip + residual sum is
        rounded (quirk Q21).  Returns (down residuals or None, mid residual or None)."""
        rows = self._sparse_rows
        nf = self.frames if rows is None else len(self.sparse_frames)
        if down is not None:
            if rows is not None:
                down = [d.index_select(0, rows) for d in down]
                mid = mid.index_select(0, rows) if mid is not None else None
            down, mid = self.adapter(down, mid_block_res_sample=mid, sparsity_masking=self.sparse_frames,
                                     num_frames=nf, timestep=t, encoder_hidden_states=self.adapter_ctx)
        else:
            mid0 = torch.zeros((n if rows is None else rows.numel(), *mid_hw, 1280), device=t.device,
                               dtype=BF16).permute(0, 3, 1, 2)
            mid = self.adapter.forward_mid(mid0, num_frames=nf, timestep=t, encoder_hidden_states=self.adapter_ctx)
        if rows is None:
            return down, mid

        def scatter(x):
            full = torch.zeros((n, *x.shape[1:]), device=x.device, dtype=x.dtype).contiguous(
                memory_format=torch.channels_last)
            full.index_copy_(0, rows, x)
            return full
        return ([scatter(d) for d in down] if down is not None else None), (scatter(mid) if mid is not None else None)

    def control_scale(self, i: int) -> Scale:
        """cond_scale of step i: a float for one ControlNet, a tuple for Multi-ControlNet (reference :1296-1302)."""
        keeps = self._keep[i]
        if self._multi:
            return tuple(c * k for c, k in zip(self._scale, keeps))
        c = self._scale[0] if isinstance(self._scale, list) else self._scale
        return c * keeps[0]

    # ---- subclass contract --------------------------------------------------------------------------------
    def _state(self) -> List[torch.Tensor]:  # tensors a body run mutates (restored after capture warm-ups)
        raise NotImplementedError

    def _load_step(self, i: int) -> None:    # refresh the device rows of step i
        raise NotImplementedError

    def _body(self, scale: Scale) -> None:   # one denoising iteration at conditioning scale `scale`
        raise NotImplementedError

    # ---- stepping -----------------------------------------------------------------------------------------
    @torch.no_grad()
    def step(self, i: Optional[int] = None):
        """One denoising iteration through the modules' public forward()s (eager launches)."""
        i = self.step_index if i is None else i
        self._load_step(i)
        self._body(self.control_scale(i))
        self.step_index = i + 1
        return self.latents

    @torch.no_grad()
    def capture(self, warmup: int = 2, scale: Optional[Scale] = None):
        """Record the step body at conditioning scale `scale` (default: step 0's) into a CUDA graph, after `warmup` eager
        runs that pack weights and set kernel attributes.  Loop state is restored afterwards."""
        scale = self.control_scale(0) if scale is None else scale
        saved = [t.clone() for t in self._state()]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                self._body(scale)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._body(scale)
        self._graphs[scale] = g
        for t, v in zip(self._state(), saved):
            t.copy_(v)
        return g

    @torch.no_grad()
    def step_graph(self, i: Optional[int] = None):
        i = self.step_index if i is None else i
        scale = self.control_scale(i)
        if scale not in self._graphs:
            self.capture(scale=scale)
        self._load_step(i)
        self._graphs[scale].replay()
        self.step_index = i + 1
        return self.latents

    @torch.no_grad()
    def run(self, use_graph: bool = True):
        for i in range(self.num_inference_steps):
            (self.step_graph if use_graph else self.step)(i)
        return self.latents
