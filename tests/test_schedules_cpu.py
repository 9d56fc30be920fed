"""CPU: the product's schedule tables (ctrl_adapter_b200/schedulers.py, what the fused CFG + scheduler kernels read) vs
the oracle's schedulers (oracle/pipeline_*.py, the diffusers v0.27.2 code the reference pipelines run, restated).  The
two are independent restatements of the same scheduler configurations, so they are compared directly for every step
count from 1 to 100 and for 250, 500 and 1000: timesteps, sigmas and init_noise_sigma (Euler, SVD's Karras Euler), the
rows (t, sigma, sigma_next, sqrt(sigma_next^2 + 1)) / (t, alpha_prod_t, alpha_prod_prev) the loops load, SVD's
ControlNet timesteps against the formula of oracle.pipeline_svd.svd_step, and DDIM's final_alpha where t - step_ratio
falls below 0.  A step count that makes a schedule degenerate is refused with ValueError by the loop's constructor.

Tolerances: timesteps are exact (Euler, DDIM: integers held in fp32 / int64); SVD's continuous timestep 0.25 ln(sigma)
is one fp32 log on each side, numpy's vs torch's, within 4 fp32 ulps.  The oracle builds its betas with torch.linspace
and its alphas_cumprod with torch.cumprod, whose CPU kernel accumulates fp32 in double; the product uses numpy, which
accumulates in fp32.  Sigmas and alphas_cumprod therefore differ by up to ~50 fp32 ulps (measured: 44 for Euler
sigmas, 29 for DDIM alphas), rtol 2^-16 here -- 500x below a bf16 ulp, which is the resolution the latents are kept at.
"""
import math

import numpy as np
import pytest
import torch

from ctrl_adapter_b200 import schedulers as S
from oracle.pipeline_i2vgen import DDIMScheduler
from oracle.pipeline_sdxl import EulerDiscreteScheduler
from oracle.pipeline_svd import EulerDiscreteSchedulerSVD

STEPS = list(range(1, 101)) + [250, 500, 1000]
RTOL = 2.0 ** -16


def _close(name, ours, ref, rtol=RTOL):
    ours, ref = np.asarray(ours, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert ours.shape == ref.shape, f"{name}: shape {ours.shape} vs {ref.shape}"
    err = np.abs(ours - ref)
    bad = err > rtol * np.abs(ref)
    assert not bad.any(), f"{name}: {int(bad.sum())} of {ours.size} off, worst at {int(err.argmax())}: " \
                          f"{ours.flat[err.argmax()]!r} vs {ref.flat[err.argmax()]!r}"


def _ulps(a, b):
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    return int(np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64)).max())


def oracle_rows(kind, n):
    """[n, 3 or 4] float64: the oracle scheduler's values for every step -- (t, sigma, sigma_next,
    sqrt(sigma_next^2 + 1)) for "euler" / "euler_v", (t, alpha_prod_t, alpha_prod_prev) for "ddim".  The last column of
    the Euler rows is the scale_model_input divisor as the oracle computes it, in fp32."""
    if kind == "ddim":
        o = DDIMScheduler()
        o.set_timesteps(n)
        ratio = o.num_train_timesteps // n
        rows = []
        for t in o.timesteps.tolist():
            prev = t - ratio
            rows.append((t, float(o.alphas_cumprod[t]),
                         float(o.alphas_cumprod[prev] if prev >= 0 else o.final_alpha_cumprod)))
        return np.array(rows, dtype=np.float64)
    o = EulerDiscreteScheduler() if kind == "euler" else EulerDiscreteSchedulerSVD()
    o.set_timesteps(n)
    s = o.sigmas
    div = (s[1:] ** 2 + 1) ** 0.5
    return np.stack([o.timesteps.double().numpy(), s[:-1].double().numpy(), s[1:].double().numpy(),
                     div.double().numpy()], axis=1)


def check_row(kind, n, i, row):
    """row: the 4 fp32 values a loop loaded for step i of an n-step schedule.  Raises AssertionError unless they are the
    oracle's (tolerances in the module docstring)."""
    ref = oracle_rows_cached(kind, n)[i]
    row = np.asarray(row, dtype=np.float64)
    what = f"{kind} {n} steps, row {i}: loaded {row.tolist()} vs oracle {ref.tolist()}"
    if kind == "euler_v":
        assert _ulps(row[0], ref[0]) <= 4, what
    else:
        assert row[0] == ref[0], what
    k = 3 if kind == "ddim" else 4
    _close(what, row[1:k], ref[1:k])


_CACHE = {}


def oracle_rows_cached(kind, n):
    if (kind, n) not in _CACHE:
        _CACHE[(kind, n)] = oracle_rows(kind, n)
    return _CACHE[(kind, n)]


@pytest.mark.parametrize("n", STEPS)
def test_euler_matches_oracle(n):
    ours = S.EulerDiscreteSchedule(n)
    o = EulerDiscreteScheduler()
    o.set_timesteps(n)
    assert np.array_equal(ours.timesteps, o.timesteps.numpy())
    assert ours.timesteps[-1] == 1 and len(ours.timesteps) == n
    _close("sigmas", ours.sigmas, o.sigmas.numpy())
    assert ours.sigmas[-1] == 0.0
    _close("init_noise_sigma", ours.init_noise_sigma, float(o.init_noise_sigma))
    tab = ours.table()
    assert tab.dtype == np.float32 and tab.shape == (n, 4)
    for i in range(n):
        check_row("euler", n, i, tab[i])
    assert tab[-1, 2] == 0.0 and tab[-1, 3] == 1.0  # the last step lands on sigma 0; the next "input" is unscaled


@pytest.mark.parametrize("n", STEPS)
def test_karras_v_matches_oracle(n):
    ours = S.EulerKarrasVSchedule(n)
    o = EulerDiscreteSchedulerSVD()
    o.set_timesteps(n)
    assert _ulps(ours.timesteps, o.timesteps.numpy()) <= 4
    assert np.array_equal(ours.sigmas, o.sigmas.numpy())  # the same float64 ramp rounded once to fp32 on both sides
    assert ours.sigmas[0] == np.float32(700.0) and ours.sigmas[-1] == 0.0
    if n > 1:
        assert ours.sigmas[-2] == np.float32(0.002)
    _close("init_noise_sigma", ours.init_noise_sigma, float(o.init_noise_sigma))
    tab = ours.table()
    for i in range(n):
        check_row("euler_v", n, i, tab[i])
    # the ControlNet / adapter timestep of step i, as oracle.pipeline_svd.svd_step computes it from the step index
    interval = 1000 // n
    want = [float(torch.Tensor([1000 - (i + 1) * interval + 1]).round()) for i in range(n)]
    assert ours.control_timesteps.tolist() == want
    assert ours.control_timesteps.dtype == np.float32 and min(want) >= 1


@pytest.mark.parametrize("n", [k for k in STEPS if k != 1000])
def test_ddim_matches_oracle(n):
    ours = S.DDIMSchedule(n)
    o = DDIMScheduler()
    o.set_timesteps(n)
    assert np.array_equal(ours.timesteps, o.timesteps.numpy())
    assert ours.step_ratio == 1000 // n and ours.final_alpha == float(o.final_alpha_cumprod) == 1.0
    assert ours.init_noise_sigma == o.init_noise_sigma == 1.0
    _close("alphas_cumprod", ours.ac, o.alphas_cumprod.numpy())
    tab = ours.table()
    for i in range(n):
        check_row("ddim", n, i, tab[i])
    # the last step's t - step_ratio is below 0 (t = 1): its alpha_prod_prev is final_alpha, exactly
    assert ours.timesteps[-1] - ours.step_ratio < 0 and tab[-1, 2] == 1.0
    # every earlier step reads alpha_prod at t - step_ratio
    prev = ours.timesteps[:-1] - ours.step_ratio
    assert (prev >= 0).all() and np.array_equal(tab[:-1, 2], ours.ac[prev])


def test_degenerate_step_counts_are_refused():
    """0 or more steps than training timesteps (step_ratio 0: every step on one timestep), and 1000 DDIM steps (the first
    timestep, 999 + steps_offset, is past the last alpha_prod_t: the oracle's own step() fails there with IndexError)"""
    o = DDIMScheduler()
    o.set_timesteps(1000)
    with pytest.raises(IndexError):
        o.step(torch.zeros(1), o.timesteps[0], torch.zeros(1))
    for make in (S.EulerDiscreteSchedule, S.EulerKarrasVSchedule, S.DDIMSchedule):
        for n in (0, -1, 1001, 5000):
            with pytest.raises(ValueError):
                make(n)
    with pytest.raises(ValueError, match="timestep 1000"):
        S.DDIMSchedule(1000)
    S.EulerDiscreteSchedule(1000)  # t = 1000 is in range for the sigma interpolation (clamped, as in the oracle)
    S.EulerKarrasVSchedule(1000)


@pytest.mark.parametrize("loop", ["sdxl", "i2vgen", "svd"])
def test_loops_refuse_degenerate_step_counts(loop):
    """the pipelines' loop classes build their schedule in the constructor: a degenerate step count fails there, before
    any module runs (the modules are not touched, so None stands in for them)"""
    from ctrl_adapter_b200.pipeline_i2vgen import I2VGenXLControlNetAdapterLoop
    from ctrl_adapter_b200.pipeline_sdxl import SDXLControlNetAdapterLoop
    from ctrl_adapter_b200.pipeline_svd import SVDControlNetAdapterLoop
    cls = {"sdxl": SDXLControlNetAdapterLoop, "i2vgen": I2VGenXLControlNetAdapterLoop,
           "svd": SVDControlNetAdapterLoop}[loop]
    for n in ([0, 1001] + ([1000] if loop == "i2vgen" else [])):
        with pytest.raises(ValueError):
            cls(None, None, None, num_inference_steps=n)


def test_row_check_flags_a_wrong_row():
    """check_row, which the schedule census runs on every row a loop loads, rejects a row one step off and a row whose
    sigma is off by 2^-14"""
    tab = S.EulerDiscreteSchedule(50).table()
    check_row("euler", 50, 7, tab[7])
    with pytest.raises(AssertionError):
        check_row("euler", 50, 7, tab[8])
    bad = tab[7].copy()
    bad[1] *= 1 + 2.0 ** -14
    with pytest.raises(AssertionError):
        check_row("euler", 50, 7, bad)
    dt = S.DDIMSchedule(50).table()
    check_row("ddim", 50, 49, dt[49])
    bad = dt[49].copy()
    bad[2] = bad[1]  # alpha_prev taken as alpha_t on the last step
    with pytest.raises(AssertionError):
        check_row("ddim", 50, 49, bad)
    assert math.isclose(oracle_rows("euler_v", 25)[0, 1], 700.0, rel_tol=1e-6)
