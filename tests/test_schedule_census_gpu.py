"""pytest -m gpu -s: the launch census (tests/launch_checks.py) over the runs the benchmark and the pipelines make, not only
one batch-1 step at conditioning scale 1 (tests/test_launch_census_gpu.py):

  * the benchmark batch sizes (SDXL 8, I2VGen-XL 4, SVD 2 at 72x128) on steps 0, 1, the middle one and the last, and
    every step of the three-ControlNet + router run;
  * whole schedules at batch 1 with control_guidance_end 0.5, so that the second half runs the scale-0 body (SDXL drops
    the down residuals, the video loops run only the mid-block adapter on zeros), and with sparse key frames on top
    (index_select, the adapter's temporal layers at 4 frames, the scatter).  Each body is a recorder context: a
    configuration both bodies launch is first-call checked on the data of each;
  * the CFG + scheduler updates get their verdict on every call (Recorder every_call), and the row the loop loaded for
    step i is compared with the oracle scheduler's values for step i (tests/test_schedules_cpu.check_row);
  * each case also counts the distinct configurations the step-0 / batch-1 census of the same workload never launches.

Then, outside any loop, every row of the real schedule tables (and of 1, 2, 7 and 30-step schedules) through the three
CFG + scheduler kernels at the benchmark's latent shapes and at the magnitudes each step sees, against the float64
chains of tests/kernel_checks.py; and four wrong variants of real ops that pass the step-0 / batch-1 census and fail
this one."""
import gc
import math
import time

import pytest
import torch

from tests import kernel_checks as kc
from tests import launch_checks as lc
from tests.test_launch_census_gpu import _step as _old_step
from tests.test_schedules_cpu import check_row

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
CFG_OPS = ("cfg_euler", "cfg_euler_v", "cfg_ddim")
KIND = {"sdxl": "euler", "svd": "euler_v", "i2vgen": "ddim", "multi": "ddim"}
I2VGEN_SPARSE, SVD_SPARSE = [0, 5, 10, 15], [0, 4, 8, 13]

# workload, batch, extra loop constructor arguments, steps (None: all of them; "ends": 0, 1, the middle one, the last)
CASES = {
    "sdxl_b8": ("sdxl", 8, {}, "ends"),
    "i2vgen_b4": ("i2vgen", 4, {}, "ends"),
    "svd_b2": ("svd", 2, {}, "ends"),
    "multi_b1": ("multi", 1, {}, None),
    "sdxl_end05": ("sdxl", 1, dict(control_guidance_end=0.5), None),
    "i2vgen_end05": ("i2vgen", 1, dict(control_guidance_end=0.5), None),
    "svd_end05": ("svd", 1, dict(control_guidance_end=0.5), None),
    "i2vgen_sparse": ("i2vgen", 1, dict(sparse_frames=I2VGEN_SPARSE, control_guidance_end=0.5), None),
    "svd_sparse": ("svd", 1, dict(sparse_frames=SVD_SPARSE, control_guidance_end=0.5), None),
}


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device is visible (there is no CPU fallback to test)")
    from ctrl_adapter_b200 import _lib
    _lib.check(_lib.load().ca_device_ok(), "ca_device_ok")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def build_loop(workload, batch, loop_kw):
    """bench.build_ours's loop; with loop_kw, a loop of the same class and settings around the same modules and
    inputs, with those constructor arguments added"""
    import bench
    loop, inp = bench.build_ours(workload, batch, 1024, "cuda", 0)
    if not loop_kw:
        return loop
    if workload == "sdxl":
        from ctrl_adapter_b200.pipeline_sdxl import SDXLControlNetAdapterLoop
        new = SDXLControlNetAdapterLoop(loop.controlnet, loop.adapter, loop.unet, num_inference_steps=50,
                                        guidance_scale=5.0, controlnet_conditioning_scale=1.0, **loop_kw)
    elif workload == "svd":
        from ctrl_adapter_b200.pipeline_svd import SVDControlNetAdapterLoop
        new = SVDControlNetAdapterLoop(loop.controlnet, loop.adapter, loop.unet, num_inference_steps=25,
                                       min_guidance_scale=1.0, max_guidance_scale=3.0, use_size_512=False,
                                       skip_conv_in=True, **loop_kw)
    else:
        from ctrl_adapter_b200.pipeline_i2vgen import I2VGenXLControlNetAdapterLoop
        new = I2VGenXLControlNetAdapterLoop(loop.controlnet, loop.adapter, loop.unet, loop.router,
                                            num_inference_steps=50, guidance_scale=9.0,
                                            inference_expert_masks=loop.masks, **loop_kw)
    new.prepare(**inp)
    return new


def _steps(loop, which):
    n = loop.num_inference_steps
    return list(range(n)) if which is None else sorted({0, 1, n // 2, n - 1})


_OLD_KEYS = {}


def old_keys(workload):
    """the configuration keys the step-0 / batch-1 census of `workload` launches (its body run under a second
    recorder)"""
    if workload not in _OLD_KEYS:
        with torch.no_grad(), lc.Recorder() as rec:
            _old_step(workload)
        torch.cuda.synchronize()
        _OLD_KEYS[workload] = {r.key for r in rec.rows.values()}
        del rec
        _free()
    return _OLD_KEYS[workload]


def run_case(workload, batch, loop_kw, which, steps=None):
    """the recorder over the loop's eager steps; returns (recorder, steps run, (step, row) pairs the CFG hook saw)"""
    seen, state = [], {}

    def on_call(name, a):
        i = state["i"]
        row = a["step_row"].cpu().tolist()
        check_row(KIND[workload], state["n"], i, row)
        seen.append((i, row))

    with torch.no_grad(), lc.Recorder(every_call=CFG_OPS, on_call=on_call) as rec:
        loop = build_loop(workload, batch, loop_kw)
        state["n"] = loop.num_inference_steps
        steps = _steps(loop, which) if steps is None else steps
        for i in steps:
            state["i"] = i
            if loop_kw:
                rec.context = f"scale {loop.control_scale(i)}"
            loop.step(i)
            if rec.failures():
                break
    torch.cuda.synchronize()
    del loop
    return rec, steps, seen


@pytest.mark.parametrize("case", list(CASES))
def test_schedule_census(case):
    workload, batch, loop_kw, which = CASES[case]
    torch.manual_seed(0)
    old = old_keys(workload)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    rec, steps, seen = run_case(workload, batch, loop_kw, which)
    wall = time.time() - t0
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    fam = rec.families()
    keys = {r.key for r in rec.rows.values()}
    new = keys - old
    cfg_verdicts = sum(r.verdicts for r in rec.rows.values() if r.op in CFG_OPS)
    contexts = sorted({r.context for r in rec.rows.values() if r.context is not None})
    print(f"\n== {case}: {len(steps)} steps ({steps[0]}..{steps[-1]}), {sum(v[0] for v in fam.values())} launches, "
          f"{len(rec.rows)} distinct configurations ({len(keys)} keys), {sum(v[2] for v in fam.values())} sampled, "
          f"{wall:.0f} s, peak device memory {peak:.1f} GiB")
    print(f"   configurations the step-0 / batch-1 `{workload}` census does not launch: {len(new)}; "
          f"CFG verdicts: {cfg_verdicts}; rows matched against the oracle scheduler: {len(seen)}"
          + (f"; contexts: {', '.join(contexts)}" if contexts else ""))
    for op, n in sorted(_count_ops(new).items()):
        print(f"   new {op}: {n}")
    print(rec.table())
    print("per op: " + "; ".join(f"{op} {n} launches / {d} configs / {s} sampled / worst err/tol {w:.3f}"
                                 for op, (n, d, s, w) in sorted(fam.items())))
    bad = rec.failures()
    assert not bad, "\n".join(f"{r.op} [{r.context}] {lc.key_summary(r.key)} [{r.where}]: {r.why}" for r in bad[:10])
    # one CFG + scheduler update per step, each with its verdict and its row checked
    assert cfg_verdicts == len(steps) == len(seen), (cfg_verdicts, len(steps), len(seen))
    assert [i for i, _ in seen] == steps
    del rec
    _free()


def _count_ops(keys):
    out = {}
    for k in keys:
        out[k[0]] = out.get(k[0], 0) + 1
    return out


# ----------------------------------------------------------------------------------------------------------------------
# every schedule row through the CFG + scheduler kernels, outside any loop
# ----------------------------------------------------------------------------------------------------------------------
SHAPES = {"euler": (8, 4, 128, 128), "euler_v": (2, 14, 4, 72, 128), "ddim": (4, 16, 4, 64, 64)}
GUIDANCE = {"euler": 5.0, "ddim": 9.0}


def _schedule(kind, n):
    from ctrl_adapter_b200 import schedulers as S
    return {"euler": S.EulerDiscreteSchedule, "euler_v": S.EulerKarrasVSchedule, "ddim": S.DDIMSchedule}[kind](n)


def _rand(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=g, device="cuda") * scale


@pytest.mark.parametrize("kind", ["euler", "euler_v", "ddim"])
def test_schedule_rows_through_the_kernels(kind):
    """every row of the 50 / 25 / 50-step tables the loops use and of 1, 2, 7 and 30-step tables; latents at the
    magnitude the step sees (noise at sigma_i: sqrt(sigma_i^2 + 1) for the Euler schedules -- init_noise_sigma at the
    first step, ~700 for SVD and ~13.2 for SDXL -- and O(1) for DDIM); bf16-valued and fp32 latents, with and without
    the next model input, written in place and into a separate buffer; each against the float64 chain of
    kernel_checks.cfg_euler_verdict / cfg_ddim_verdict"""
    from ctrl_adapter_b200 import ops
    shape = SHAPES[kind]
    main = {"euler": 50, "euler_v": 25, "ddim": 50}[kind]
    eu, et = _rand(shape, 1).to(BF16), _rand(shape, 2).to(BF16)
    noise = _rand(shape, 3)
    f = shape[1]
    g_frames = torch.linspace(1.0, 3.0, f, device="cuda").to(BF16).float().contiguous()
    worst, calls, bad = 0.0, 0, []
    for n in (main, 1, 2, 7, 30):
        sch = _schedule(kind, n)
        table = torch.from_numpy(sch.table()).cuda()
        row = table[0].clone()
        for i in range(n):
            row.copy_(table[i])
            mag = 1.0 if kind == "ddim" else math.sqrt(float(sch.sigmas[i]) ** 2 + 1.0)
            for combo in range(8):
                round_bf16, with_next, in_place = bool(combo & 1), bool(combo & 2), bool(combo & 4)
                lat = noise * mag
                if round_bf16:
                    lat = lat.to(BF16).float()
                pre = lat.clone()
                nxt = torch.full(shape, math.nan, device="cuda", dtype=BF16) if with_next else None
                call = dict(eps_uncond=eu, eps_text=et, latents=lat, step_row=row,
                            latents_out=lat if in_place else None, model_in_next=nxt, round_latents_bf16=round_bf16)
                if kind == "euler":
                    out = ops.cfg_euler(guidance=GUIDANCE[kind], **call)
                elif kind == "euler_v":
                    out = ops.cfg_euler_v(guidance_per_frame=g_frames, frames=f, **call)
                else:
                    out = ops.cfg_ddim(guidance=GUIDANCE[kind], v_prediction=sch.v_prediction, **call)
                torch.cuda.synchronize()
                a = dict(call, latents=pre, guidance=GUIDANCE.get(kind), frames=f, guidance_per_frame=g_frames,
                         v_prediction=True)
                if kind == "ddim":
                    r = kc.cfg_ddim_verdict(kind, a, out, nxt)
                else:
                    r = kc.cfg_euler_verdict(kind, a, out, nxt, v_prediction=kind == "euler_v")
                calls += 1
                worst = max(worst, r["max_err_over_tol"])
                if not r["ok"] or (in_place and out.data_ptr() != lat.data_ptr()):
                    bad.append(f"{n} steps, row {i} {table[i].tolist()}, round {round_bf16}, next {with_next}, "
                               f"in place {in_place}: err/tol {r['max_err_over_tol']:.3g}")
    print(f"\n{kind} {list(shape)}: {calls} calls, worst err/tol {worst:.3f}")
    assert not bad, "\n".join(bad[:10])


# ----------------------------------------------------------------------------------------------------------------------
# wrong variants of real ops: each passes the step-0 / batch-1 census and fails this one
# ----------------------------------------------------------------------------------------------------------------------
def _real(name):
    from ctrl_adapter_b200 import ops
    return getattr(ops, name)


def _conv_rowvec_mod2(real):
    def conv2d(x, w_packed, bias, *, rowvec=None, **kw):
        """the time-embedding row vector of image i taken from image i % 2 (the same at batch 1 with CFG)"""
        if rowvec is not None and rowvec.shape[0] > 2:
            rowvec = rowvec[torch.arange(rowvec.shape[0], device=rowvec.device) % 2].contiguous()
        return real(x, w_packed, bias, rowvec=rowvec, **kw)
    return conv2d


def _ta_short_last_frame(real):
    def temporal_attention(q, k, v, clips, frames, hw, heads, scale, out=None, row_stride=None):
        """with fewer than 8 frames, the last frame's output left at zero"""
        o = real(q, k, v, clips, frames, hw, heads, scale, out=out, row_stride=row_stride)
        if frames < 8:
            o.unflatten(0, (clips, frames, hw))[:, frames - 1].zero_()
        return o
    return temporal_attention


def _gn_zero_input(real):
    def group_norm(x, gamma, beta, eps, **kw):
        """an all-zero input (the mid-block adapter of the scale-0 body) normalised to beta + 1 instead of beta"""
        o = real(x, gamma, beta, eps, **kw)
        o.add_((x == 0).all().to(o.dtype))  # on the device: no host branch, no extra launch of the kernel
        return o
    return group_norm


# variant -> (op, wrapper, step-0 / batch-1 workload, new case, steps of the new case it needs)
VARIANTS = {
    "conv2d: time-embedding row vector of image i from image i % 2": ("conv2d", _conv_rowvec_mod2, "sdxl",
                                                                      "sdxl_b8", [0]),
    "temporal_attention: last frame dropped below 8 frames": ("temporal_attention", _ta_short_last_frame, "i2vgen",
                                                              "i2vgen_sparse", [0]),
    "group_norm: all-zero input off by one (scale-0 body)": ("group_norm", _gn_zero_input, "i2vgen", "i2vgen_end05",
                                                             [0, 25]),
}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_schedule_census_catches_wrong_variant(variant, monkeypatch):
    from ctrl_adapter_b200 import ops
    name, wrap, old_workload, case, steps = VARIANTS[variant]
    monkeypatch.setattr(ops, name, wrap(_real(name)))
    with torch.no_grad(), lc.Recorder() as old:
        _old_step(old_workload)
    torch.cuda.synchronize()
    old_bad = old.failures()
    del old
    _free()
    workload, batch, loop_kw, _ = CASES[case]
    rec, _, _ = run_case(workload, batch, loop_kw, None, steps=steps)
    bad = rec.failures()
    print(f"\n{variant}: step-0 / batch-1 `{old_workload}` census: {'FAILS' if old_bad else 'passes'}; {case}: caught by "
          + ("; ".join(f"{r.op} [{r.context}] {lc.key_summary(r.key)} [{r.where}]" for r in bad[:3]) or "NOTHING"))
    del rec
    _free()
    assert not old_bad, [f"{r.op} {lc.key_summary(r.key)}: {r.why}" for r in old_bad[:3]]
    assert bad, f"the schedule census does not notice: {variant}"
