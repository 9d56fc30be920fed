"""Host-side schedule tables for the fused CFG + scheduler kernels (tiny numpy math, done once per generation).

EulerDiscrete: the SDXL-base default scheduler used by the reference SDXL pipeline
(/root/reference/sdxl/pipelines/sdxl_controlnet_adapter_pipeline.py:1169,1285,1378; diffusers v0.27.2
EulerDiscreteScheduler with scaled_linear betas 0.00085..0.012, 1000 train steps, timestep_spacing="leading",
steps_offset=1, epsilon prediction, linear sigma interpolation).
DDIM: I2VGen-XL pipeline (/root/reference/i2vgen_xl/pipelines/i2vgen_xl_controlnet_adapter_pipeline.py:1112).
"""
from __future__ import annotations

import numpy as np


def _alphas_cumprod(beta_start=0.00085, beta_end=0.012, n=1000, schedule="scaled_linear"):
    if schedule == "scaled_linear":
        betas = np.linspace(beta_start ** 0.5, beta_end ** 0.5, n, dtype=np.float32) ** 2
    elif schedule == "linear":
        betas = np.linspace(beta_start, beta_end, n, dtype=np.float32)
    else:
        raise ValueError(schedule)
    return np.cumprod(1.0 - betas, axis=0)


def _check_steps(num_inference_steps: int, num_train_timesteps: int):
    """The "leading" spacing takes every (train // inference)-th training step: past num_train_timesteps the ratio is 0
    and every step would land on the same timestep."""
    if not 1 <= num_inference_steps <= num_train_timesteps:
        raise ValueError(f"num_inference_steps must be in 1..{num_train_timesteps} (num_train_timesteps), got "
                         f"{num_inference_steps}")


class EulerDiscreteSchedule:
    def __init__(self, num_inference_steps: int, num_train_timesteps: int = 1000, steps_offset: int = 1):
        _check_steps(num_inference_steps, num_train_timesteps)
        ac = _alphas_cumprod(n=num_train_timesteps)
        step_ratio = num_train_timesteps // num_inference_steps
        ts = (np.arange(0, num_inference_steps) * step_ratio).round()[::-1].copy().astype(np.float32) + steps_offset
        sig = ((1 - ac) / ac) ** 0.5
        sig = np.interp(ts, np.arange(0, len(sig)), sig).astype(np.float32)
        self.timesteps = ts                                   # fed to ControlNet / adapter / UNet
        self.sigmas = np.concatenate([sig, [0.0]]).astype(np.float32)
        self.init_noise_sigma = float((self.sigmas.max() ** 2 + 1) ** 0.5)  # "leading" spacing

    def input_scale(self, i: int) -> float:
        """scale_model_input: sample / sqrt(sigma_i^2 + 1)"""
        return float(1.0 / (self.sigmas[i] ** 2 + 1) ** 0.5)

    def table(self):
        """[steps, 4] fp32 rows (t, sigma, sigma_next, sqrt(sigma_next^2 + 1)) consumed by ca_cfg_euler; the last
        entry is the scale_model_input divisor of the NEXT step's model input (1 after the final step)."""
        n = len(self.timesteps)
        rows = np.zeros((n, 4), dtype=np.float32)
        for i in range(n):
            rows[i] = (self.timesteps[i], self.sigmas[i], self.sigmas[i + 1],
                       np.sqrt(np.float32(self.sigmas[i + 1]) ** 2 + np.float32(1.0)))
        return rows


def _betas_squaredcos_cap_v2(n: int, max_beta: float = 0.999):
    import math
    bar = lambda t: math.cos((t + 0.008) / 1.008 * math.pi / 2) ** 2  # noqa: E731
    return np.array([min(1 - bar((i + 1) / n) / bar(i / n), max_beta) for i in range(n)], dtype=np.float32)


def _rescale_zero_terminal_snr(betas: np.ndarray) -> np.ndarray:
    alphas = 1.0 - betas
    ac = np.cumprod(alphas, axis=0)
    s = np.sqrt(ac)
    s0, sT = s[0].copy(), s[-1].copy()
    s = (s - sT) * (s0 / (s0 - sT))
    ac = s ** 2
    alphas = np.concatenate([ac[0:1], ac[1:] / ac[:-1]])
    return (1.0 - alphas).astype(np.float32)


class DDIMSchedule:
    """DDIM, eta = 0, "leading" spacing, steps_offset 1, no sample clipping.  Defaults = the I2VGen-XL scheduler
    (ali-vilab/i2vgen-xl scheduler_config.json, restated from memory -- the file is not part of the reference repo):
    squaredcos_cap_v2 betas, rescale_betas_zero_snr, v_prediction, set_alpha_to_one."""

    def __init__(self, num_inference_steps: int, num_train_timesteps: int = 1000, steps_offset: int = 1,
                 beta_schedule: str = "squaredcos_cap_v2", rescale_betas_zero_snr: bool = True,
                 set_alpha_to_one: bool = True, prediction_type: str = "v_prediction"):
        if beta_schedule == "squaredcos_cap_v2":
            betas = _betas_squaredcos_cap_v2(num_train_timesteps)
        elif beta_schedule == "scaled_linear":
            betas = np.linspace(0.00085 ** 0.5, 0.012 ** 0.5, num_train_timesteps, dtype=np.float32) ** 2
        else:
            raise ValueError(beta_schedule)
        if rescale_betas_zero_snr:
            betas = _rescale_zero_terminal_snr(betas)
        self.ac = np.cumprod(1.0 - betas, axis=0).astype(np.float32)
        _check_steps(num_inference_steps, num_train_timesteps)
        step_ratio = num_train_timesteps // num_inference_steps
        self.timesteps = ((np.arange(0, num_inference_steps) * step_ratio).round()[::-1].copy().astype(np.int64)
                          + steps_offset)
        if self.timesteps[0] >= num_train_timesteps:
            # e.g. 1000 steps of 1000: the first timestep, 999 + steps_offset, has no alpha_prod_t
            raise ValueError(f"{num_inference_steps} DDIM steps with steps_offset {steps_offset} reach timestep "
                             f"{int(self.timesteps[0])}, past the last of {num_train_timesteps} training timesteps")
        self.step_ratio = step_ratio
        self.final_alpha = 1.0 if set_alpha_to_one else float(self.ac[0])
        self.init_noise_sigma = 1.0
        self.v_prediction = prediction_type == "v_prediction"

    def table(self):
        """[steps, 4] fp32 rows (t, alpha_prod_t, alpha_prod_prev, 0) consumed by ca_cfg_ddim."""
        rows = np.zeros((len(self.timesteps), 4), dtype=np.float32)
        for i, t in enumerate(self.timesteps):
            prev = t - self.step_ratio
            rows[i] = (t, self.ac[t], self.ac[prev] if prev >= 0 else self.final_alpha, 0.0)
        return rows


class EulerKarrasVSchedule:
    """EulerDiscreteScheduler as configured for Stable Video Diffusion (stabilityai/stable-video-diffusion-img2vid
    scheduler_config.json, restated from memory -- the file is not part of the reference repo): v_prediction,
    timestep_type "continuous" (t = 0.25 ln sigma), Karras sigmas (rho 7) between sigma_max 700 and sigma_min 0.002,
    "leading" spacing (init_noise_sigma = sqrt(sigma_max^2 + 1)).  Used by pipeline_svd (svd pipeline :600-602, :775)."""

    def __init__(self, num_inference_steps: int, sigma_min: float = 0.002, sigma_max: float = 700.0, rho: float = 7.0):
        _check_steps(num_inference_steps, 1000)  # the control timesteps step by 1000 // num_inference_steps
        ramp = np.linspace(0, 1, num_inference_steps)
        lo, hi = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
        sig = ((hi + ramp * (lo - hi)) ** rho).astype(np.float32)
        self.timesteps = (0.25 * np.log(sig)).astype(np.float32)       # fed to the UNet
        self.sigmas = np.concatenate([sig, [0.0]]).astype(np.float32)
        self.init_noise_sigma = float((self.sigmas.max() ** 2 + 1) ** 0.5)
        interval = 1000 // num_inference_steps
        # the ControlNet / adapter timestep is derived from the step index (svd pipeline :676-681)
        self.control_timesteps = np.array([1000 - (i + 1) * interval + 1 for i in range(num_inference_steps)],
                                          dtype=np.float32)

    def table(self):
        """[steps, 4] fp32 rows (t, sigma, sigma_next, sqrt(sigma_next^2 + 1)) consumed by ca_cfg_euler_v."""
        n = len(self.timesteps)
        rows = np.zeros((n, 4), dtype=np.float32)
        for i in range(n):
            rows[i] = (self.timesteps[i], self.sigmas[i], self.sigmas[i + 1],
                       np.sqrt(np.float32(self.sigmas[i + 1]) ** 2 + np.float32(1.0)))
        return rows
