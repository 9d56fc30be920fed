"""CPU: the launch census (tests/launch_checks.py) can pass and can fail.  With the emulated op layer
(tests/ops_emulator.py) standing in for the kernels, the recorder runs over the ControlNet, the video adapter, the VAE
decoder and encoder at reduced size and over direct calls of the remaining entry points: every launch passes, every
`ops` function that launches a kernel has a verifier that ran, and each deliberately wrong variant of an emulated op
below fails at least one launch, printed with -s."""
import ast
import functools
import inspect

import pytest
import torch
import torch.nn.functional as F

from oracle import cases
from oracle.weights import seeded_init_, seeded_tensor
from tests import kernel_checks as kc
from tests import launch_checks as lc
from tests import ops_emulator as emu

BF16 = torch.bfloat16
VAE_KW = dict(block_out_channels=(32, 64, 64, 64), layers_per_block=1)


@pytest.fixture(scope="module", autouse=True)
def _cpu_device():
    saved = kc.DEVICE
    kc.DEVICE = "cpu"
    torch.set_grad_enabled(False)
    yield
    kc.DEVICE = saved
    torch.set_grad_enabled(True)


def _ours(make_oracle, make_ours, seed):
    sd = seeded_init_(make_oracle(), seed).state_dict()
    m = make_ours()
    m.load_state_dict(sd)
    return m.to(BF16).eval()


@functools.lru_cache(maxsize=None)
def _modules():
    from ctrl_adapter_b200 import vae
    from ctrl_adapter_b200.adapter import ControlNetAdapter
    from ctrl_adapter_b200.controlnet import ControlNetModel
    from oracle import vae_encoder as ov
    from oracle.adapter import ControlNetAdapter as OA
    from oracle.controlnet import ControlNetModel as OC
    return dict(
        controlnet=_ours(lambda: OC(**cases.CONTROLNET_KW), lambda: ControlNetModel(**cases.CONTROLNET_KW), 4),
        adapter=_ours(lambda: OA(**cases.ADAPTER_VIDEO_KW), lambda: ControlNetAdapter(**cases.ADAPTER_VIDEO_KW), 2),
        vae=_ours(lambda: ov.AutoencoderKL(**VAE_KW), lambda: vae.AutoencoderKL(**VAE_KW), 20))


def _r(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(BF16)


def _direct_calls(ops):
    """the entry points and variants the modules above do not reach at this size: the UNet up-blocks' concatenated
    sources, a row vector every 48 rows, the schedulers, the router, the VAE latent layouts and the small kernels"""
    x, x2 = _r(2, 9, 16, 64, seed=1), _r(2, 9, 16, 64, seed=2)
    w = ops.pack_conv_weight(_r(64, 128, 3, 3, seed=3, scale=128 ** -0.5 / 3))
    ops.conv2d(x, w, ops.bias_f32(_r(64, seed=4)), x2=x2, residual=_r(2, 9, 16, 64, seed=5))
    ops.group_norm(x, torch.ones(128) * 1.1, torch.zeros(128) + 0.1, 1e-5, x2=x2 - 2.0, silu=True, up2x=True)
    ops.linear(_r(192, 64, seed=6), _r(128, 64, seed=7, scale=0.125), None, rowvec=_r(4, 128, seed=8), rows_per_vec=48)
    eu, et = _r(2, 3, 4, 6, 8, seed=9), _r(2, 3, 4, 6, 8, seed=10)
    lat = _r(2, 3, 4, 6, 8, seed=11, scale=8.0).float()
    row = torch.tensor([900.0, 11.3, 9.7, (9.7 ** 2 + 1) ** 0.5])
    nxt = torch.empty(2, 3, 4, 6, 8, dtype=BF16)
    ops.cfg_euler_v(eu, et, lat, torch.tensor([1.0, 2.0, 3.0]), 3, row, latents_out=lat, model_in_next=nxt)
    ops.cfg_euler(eu, et, lat.clone(), 5.0, row, model_in_next=nxt)
    ops.cfg_ddim(eu, et, lat.clone(), 9.0, torch.tensor([500.0, 0.3, 0.45, 0.0]), model_in_next=nxt,
                 round_latents_bf16=False, v_prediction=True)
    ops.router_merge([_r(2, 4, 4, 64, seed=20 + i) for i in range(3)],
                     ops.router_weights(_r(1, 7, seed=12).float(), torch.tensor([1, 1, 0, 1, 0, 0, 0], dtype=torch.uint8))[0, [0, 1, 3]].contiguous())
    mom, noise = _r(2, 6, 10, 8, seed=13), torch.randn(2, 4, 6, 10, generator=torch.Generator().manual_seed(14))
    ops.vae_latents(mom, ops.VAE_I2VGEN, noise, 4, 2, 0.18215)
    ops.vae_latents(mom, ops.VAE_SVD, None, 3, 1)
    ops.vae_latents(mom, ops.VAE_POSTERIOR, noise)
    xs = _r(6, 5, 7, 8, seed=15)
    ops.frame_conv_small(xs, torch.randn(3, 3, 3, generator=torch.Generator().manual_seed(16)) * 0.5,
                         torch.tensor([0.1, -0.2, 0.3]), 3, 3)
    params = torch.randn(288, generator=torch.Generator().manual_seed(17)).to(BF16).float() * 0.5
    params[:4] += 1.0
    ops.i2vgen_latent_encoder(xs, 2, 3, params)
    ops.softmax_rows(torch.randn(5, 300, generator=torch.Generator().manual_seed(18)) * 4.0)
    y = ops.avgpool(_r(2, 16, 16, 8, seed=19), 8, 8)
    ops.nhwc_to_nchw(ops.upsample2x(ops.add(ops.silu(y), y)), 6)
    ops.nchw_to_nhwc(_r(2, 3, 5, 7, seed=21), 8)


def _run(wrong=None):
    """the emulated workload under the recorder, `wrong` ({op: function}) patched over the emulation"""
    from ctrl_adapter_b200.vae import AutoencoderKL  # noqa: F401  (imports the module before ops is patched)
    m = _modules()
    with emu.patched_ops() as ops:
        for name, fn in (wrong or {}).items():
            setattr(ops, name, fn)
        with lc.Recorder() as rec:
            m["controlnet"](**{k: (v.to(BF16) if torch.is_tensor(v) and v.is_floating_point() else v)
                               for k, v in dict(cases.controlnet_inputs(2, 8), conditioning_scale=0.75).items()})
            inp = cases.adapter_video_inputs(1, 4, 8)
            inp["down_block_res_samples"] = [t.to(BF16) for t in inp["down_block_res_samples"]]
            inp["mid_block_res_sample"] = inp["mid_block_res_sample"].to(BF16)
            inp["encoder_hidden_states"] = inp["encoder_hidden_states"].to(BF16)
            m["adapter"](**inp)
            m["vae"].decode(seeded_tensor("vae_z", (1, 4, 9, 16)).to(BF16))
            m["vae"].encode(torch.tanh(seeded_tensor("enc_x", (1, 3, 48, 80))).to(BF16)).latent_dist.mode()
            _direct_calls(ops)
    return rec


def test_census_passes_on_emulator():
    rec = _run()
    print("\n" + rec.table())
    bad = rec.failures()
    assert not bad, "\n".join(f"{r.op} {lc.key_summary(r.key)}: {r.why}" for r in bad[:5])
    assert {r.op for r in rec.rows.values()} == set(lc.OPS), set(lc.OPS) - {r.op for r in rec.rows.values()}


def test_every_launching_entry_point_has_a_verifier():
    from ctrl_adapter_b200 import ops
    tree = ast.parse(inspect.getsource(ops))
    launching = {f.name for f in tree.body if isinstance(f, ast.FunctionDef) and f.name != "_launch" and any(
        isinstance(n, ast.Call) and getattr(n.func, "id", None) == "_launch" for n in ast.walk(f))}
    assert launching == set(lc.OPS) == set(lc.VERIFIERS), launching ^ set(lc.OPS)


# ---- wrong variants of the emulated ops (each a small wrapper around the correct emulation) ----
def _into(y, out):
    if out is None:
        return y
    out.copy_(y)
    return out


def _conv_symmetric_pad(x, w_packed, bias, *, pad=None, **kw):
    """pad (0, 1) done as symmetric padding"""
    return emu.conv2d(x, w_packed, bias, **kw)


def _conv_last_box_rows_zero(x, w_packed, bias, *, out=None, **kw):
    """rows past the last full box row (ho % bh of ops.choose_box) left at zero"""
    from ctrl_adapter_b200 import ops
    y = emu.conv2d(x, w_packed, bias, **kw)
    bh = ops.choose_box(y.shape[2], y.shape[1], y.shape[0])[1]
    y[:, y.shape[1] // bh * bh:] = 0
    return _into(y, out)


def _conv_x2_late(x, w_packed, bias, *, x2=None, **kw):
    """the second source read 8 channels late"""
    if x2 is not None:
        x2 = F.pad(x2[..., 8:], (0, 8))
    return emu.conv2d(x, w_packed, bias, x2=x2, **kw)


def _temporal_taps_reversed(x, w_packed, bias, frames, **kw):
    """frame taps t-1 and t+1 exchanged"""
    w = w_packed
    return emu.temporal_conv(x, w.reshape(w.shape[0], 3, -1).flip(1).reshape(w.shape), bias, frames, **kw)


def _gn_first_source_stats(x, gamma, beta, eps, *, x2=None, groups=32, silu=False, up2x=False, imgs_per_sample=1,
                           out=None):
    """with x2: the statistics summed over the first source only (x2 read as zeros), then applied to both"""
    y = emu.group_norm(x, gamma, beta, eps, groups=groups, silu=silu, up2x=up2x, x2=x2, imgs_per_sample=imgs_per_sample)
    if x2 is not None:
        xin = torch.cat([x, x2], dim=3).float()
        n, h, w, c = xin.shape
        t = torch.cat([x, torch.zeros_like(x2)], dim=3).float().reshape(n // imgs_per_sample, -1, groups, c // groups)
        mean, var = t.mean(dim=(1, 3), keepdim=True), t.var(dim=(1, 3), unbiased=False, keepdim=True)
        v = ((xin.reshape(t.shape) - mean) * torch.rsqrt(var + eps)).reshape(n, h, w, c) * gamma.float() + beta.float()
        v = F.silu(v) if silu else v
        y = (v.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2) if up2x else v).to(BF16)
    return _into(y, out)


def _gn_no_ips(*args, imgs_per_sample=1, **kw):
    """imgs_per_sample ignored: per-image statistics"""
    return emu.group_norm(*args, **kw)


def _ln_rowvec_modulo(x, gamma, beta, eps=1e-5, *, add_rowvec=None, rows_per_vec=0, return_sum=False):
    """row vector indexed by row % (number of vectors) instead of row // rows_per_vec"""
    if add_rowvec is not None:
        rows = x.numel() // x.shape[-1]
        add_rowvec = add_rowvec[torch.arange(rows) % add_rowvec.shape[0]]
        rows_per_vec = 1
    return emu.layer_norm(x, gamma, beta, eps, add_rowvec=add_rowvec, rows_per_vec=rows_per_vec, return_sum=return_sum)


def _linear_rowvec_tile_origin(x, w, bias=None, *, rowvec=None, rows_per_vec=0, **kw):
    """row vector of row r taken at the origin of r's 128-row tile"""
    if rowvec is not None:
        rowvec = rowvec[(torch.arange(x.shape[0]) // 128 * 128) // rows_per_vec]
        rows_per_vec = 1
    return emu.linear(x, w, bias, rowvec=rowvec, rows_per_vec=rows_per_vec, **kw)


def _attention_last_tile_zero(q, k, v, heads, head_dim_pad, scale, out=None, kv_batch_div=1):
    """the last partial 128-row query tile left at zero"""
    y = emu.attention(q, k, v, heads, head_dim_pad, scale, kv_batch_div=kv_batch_div)
    lq = q.shape[1]
    if lq % 128:
        y[:, lq // 128 * 128:] = 0
    return _into(y, out)


def _euler_v_guidance_per_clip(eps_uncond, eps_text, latents, guidance_per_frame, frames, step_row, latents_out=None,
                               model_in_next=None, round_latents_bf16=True):
    """guidance indexed by clip instead of frame: every frame of clip c uses guidance[c]"""
    eu, et, lat, g = eps_uncond, eps_text, latents, guidance_per_frame
    ys = [emu.cfg_euler_v(eu[c:c + 1], et[c:c + 1], lat[c:c + 1], g[min(c, frames - 1)].expand(frames), frames,
                          step_row, round_latents_bf16=round_latents_bf16) for c in range(lat.shape[0])]
    y = torch.cat(ys)
    if model_in_next is not None:
        model_in_next.copy_((y / float(step_row[3].to(BF16))).to(BF16))
    if latents_out is None:
        return y
    latents_out.copy_(y)
    return latents_out


def _vae_latents_halves_swapped(moments, layout=0, noise=None, frames=1, num_videos=1, scale=1.0):
    """SVD layout with the halves in the order [latent, 0]"""
    y = emu.vae_latents(moments, layout, noise, frames, num_videos, scale)
    if layout == 2:
        n = moments.shape[0]
        y = y.reshape(num_videos, 2, n, *y.shape[1:]).flip(1).reshape(y.shape)
    return y


VARIANTS = {
    "conv2d: pad (0, 1) as symmetric padding": {"conv2d": _conv_symmetric_pad},
    "conv2d: rows past the last full box row left at zero": {"conv2d": _conv_last_box_rows_zero},
    "conv2d: second source read 8 channels late": {"conv2d": _conv_x2_late},
    "temporal_conv: frame taps reversed": {"temporal_conv": _temporal_taps_reversed},
    "group_norm: statistics of the first source only with x2": {"group_norm": _gn_first_source_stats},
    "group_norm: imgs_per_sample ignored": {"group_norm": _gn_no_ips},
    "layer_norm: row vector at row % vectors": {"layer_norm": _ln_rowvec_modulo},
    "linear: row vector at the 128-row tile origin": {"linear": _linear_rowvec_tile_origin},
    "attention: last partial query tile zeroed": {"attention": _attention_last_tile_zero},
    "cfg_euler_v: guidance by clip instead of frame": {"cfg_euler_v": _euler_v_guidance_per_clip},
    "vae_latents: SVD halves in the order [L, 0]": {"vae_latents": _vae_latents_halves_swapped},
}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_census_catches_wrong_variant(variant):
    rec = _run(VARIANTS[variant])
    bad = rec.failures()
    print(f"\n{variant}: caught by " + ("; ".join(f"{r.op} {lc.key_summary(r.key)} [{r.where}]" for r in bad[:3])
                                       or "NOTHING"))
    assert bad, f"no launch notices: {variant}"


# ---- the CFG + scheduler updates over whole schedules: a verdict on every call (Recorder every_call) ----
CFG_OPS = ("cfg_euler", "cfg_euler_v", "cfg_ddim")


def _schedule_updates(kind, steps, wrong=None, every_call=()):
    """the last launch of a loop's step over the steps `steps` of its schedule, made as the loop makes it: one step row
    refreshed from the table before each call, the latents updated in place, the next model input written"""
    from ctrl_adapter_b200 import schedulers as S
    sch = {"euler": lambda: S.EulerDiscreteSchedule(50), "euler_v": lambda: S.EulerKarrasVSchedule(25),
           "ddim": lambda: S.DDIMSchedule(50)}[kind]()
    shape = (2, 3, 4, 6, 8)
    eu, et = _r(*shape, seed=30), _r(*shape, seed=31)
    table = torch.from_numpy(sch.table())
    row = table[0].clone()
    lat = (torch.randn(*shape, generator=torch.Generator().manual_seed(32)) * sch.init_noise_sigma).to(BF16).float()
    nxt = torch.empty(shape, dtype=BF16)
    with emu.patched_ops() as ops:
        for name, fn in (wrong or {}).items():
            setattr(ops, name, fn)
        with lc.Recorder(every_call=every_call) as rec:
            for i in steps:
                row.copy_(table[i])
                if kind == "euler":
                    ops.cfg_euler(eu, et, lat, 5.0, row, latents_out=lat, model_in_next=nxt)
                elif kind == "euler_v":
                    ops.cfg_euler_v(eu, et, lat, torch.linspace(1.0, 3.0, 3).to(BF16).float(), 3, row, latents_out=lat,
                                    model_in_next=nxt)
                else:
                    ops.cfg_ddim(eu, et, lat, 9.0, row, latents_out=lat, model_in_next=nxt, v_prediction=True)
    return rec, len(table)


@pytest.mark.parametrize("kind", ["euler", "euler_v", "ddim"])
def test_every_call_verdict_covers_every_row(kind):
    """with every_call, each call of a whole schedule gets its verdict (one key, as many verdicts as steps); without it
    only the first does, as before"""
    rec, n = _schedule_updates(kind, range({"euler_v": 25}.get(kind, 50)), every_call=CFG_OPS)
    assert not rec.failures(), rec.table()
    assert len(rec.rows) == 1 and [r.verdicts for r in rec.rows.values()] == [n]
    rec, n = _schedule_updates(kind, range(n))
    assert not rec.failures() and [(r.launches, r.verdicts) for r in rec.rows.values()] == [(n, 1)]


def _euler_sigma_next_zero_no_step(eps_uncond, eps_text, latents, guidance, step_row, latents_out=None,
                                   model_in_next=None, round_latents_bf16=True):
    """sigma_next == 0 (the last step) treated as "no step": the latents are left as they are"""
    if float(step_row[2]) != 0.0:
        return emu.cfg_euler(eps_uncond, eps_text, latents, guidance, step_row, latents_out, model_in_next,
                             round_latents_bf16)
    y = latents.clone()
    if model_in_next is not None:
        model_in_next.copy_((y / float(step_row[3].to(BF16))).to(BF16))
    return _into(y, latents_out)


def _ddim_final_alpha_as_alpha_t(eps_uncond, eps_text, latents, guidance, step_row, latents_out=None,
                                 model_in_next=None, round_latents_bf16=True, v_prediction=False):
    """alpha_prod_prev == 1 (set_alpha_to_one on the last step) replaced by alpha_prod_t"""
    if float(step_row[2]) == 1.0:
        step_row = step_row.clone()
        step_row[2] = step_row[1]
    return emu.cfg_ddim(eps_uncond, eps_text, latents, guidance, step_row, latents_out, model_in_next,
                        round_latents_bf16, v_prediction)


SCHEDULE_VARIANTS = {
    "cfg_euler: sigma_next == 0 taken as no step": ("euler", {"cfg_euler": _euler_sigma_next_zero_no_step}),
    "cfg_ddim: alpha_prev == 1 replaced by alpha_t": ("ddim", {"cfg_ddim": _ddim_final_alpha_as_alpha_t}),
}


@pytest.mark.parametrize("variant", list(SCHEDULE_VARIANTS))
def test_every_call_verdict_catches_end_of_schedule_variant(variant):
    """special-cased end-of-schedule arithmetic: invisible to the step-0 census (first call of the key only), caught
    when every step's update gets its verdict"""
    kind, wrong = SCHEDULE_VARIANTS[variant]
    old, n = _schedule_updates(kind, [0], wrong)
    assert not old.failures(), f"the step-0 census should not see it: {variant}"
    rec, _ = _schedule_updates(kind, range(n), wrong, every_call=CFG_OPS)
    bad = rec.failures()
    print(f"\n{variant}: step-0 census passes; every-call census caught by "
          + ("; ".join(f"{r.op} {lc.key_summary(r.key)} [{r.where}] after {r.verdicts} verdicts" for r in bad[:3])
             or "NOTHING"))
    assert bad, f"no verdict notices: {variant}"


@pytest.mark.parametrize("wrong", [None, "linear: row vector at the 128-row tile origin"])
def test_linear_rows_sampled(wrong, monkeypatch):
    """linear launches too large for a whole float64 reference (the video UNets at benchmark batch) are verified on the
    rows of their first, middle and last image: the emulated census passes that way, and a wrong row vector is still
    caught"""
    monkeypatch.setattr(lc, "LINEAR_SAMPLE_BYTES", 0)
    rec = _run(VARIANTS[wrong] if wrong else None)
    linear = [r for r in rec.rows.values() if r.op == "linear"]
    assert linear and all(r.sampled for r in linear)
    bad = rec.failures()
    print(f"\nlinear rows sampled, {wrong or 'correct emulation'}: "
          + ("; ".join(f"{r.op} {lc.key_summary(r.key)}: {r.why}" for r in bad[:2]) or "passes"))
    assert bool(bad) == bool(wrong)
