"""Launch census: every distinct kernel launch a real run makes, each checked against a float64 reference of its op.

`Recorder` is a context manager that wraps the entry points of `ctrl_adapter_b200.ops` that launch kernels (the host
modules call `ops.X` through the module, so replacing the attribute is enough, as ops_emulator.patched_ops does).  Each
call is keyed by its configuration: the op; shape, strides, dtype, 16-byte alignment and aliasing of every tensor
argument; every scalar argument.  The first call with a key:
  1. clones its inputs, keeping strides, alignment and aliasing (views of a wider buffer stay views of a buffer of the
     same width);
  2. runs the real kernel and synchronises;
  3. checks what it wrote against the op's reference (VERIFIERS: the per-launch verdicts of tests/kernel_checks.py, so
     the layout checks and the census share one reference per op) and, for an `out=` view, that the bytes around it in
     its buffer are unchanged;
  4. replays the call on the clones -- into NaN-filled outputs where the op takes them -- and requires the replay to be
     bit-identical to the in-step output; group_norm, whose statistics are summed with float atomics, must pass its
     reference again instead.
Later calls with the same key are only counted.  A call without a verifier, or one its verifier cannot handle, fails.
Where the float64 reference of a whole launch would be too large, it is evaluated on the first, middle and last image /
batch entry / sample (never on part of an image) and the row says so.

tests/test_launch_census_gpu.py runs one step of each benchmark workload and the VAE at the pipelines' geometry under
it; tests/test_launch_checks_cpu.py runs it over the emulated op layer and shows that it flags wrong variants.
"""
from __future__ import annotations

import inspect
import math

import torch
import torch.nn.functional as F

from tests import kernel_checks as kc

F64 = torch.float64
BF16 = torch.bfloat16
OPS = ("linear", "conv2d", "temporal_conv", "attention", "temporal_attention", "group_norm", "layer_norm",
       "timestep_embedding", "silu", "add", "nchw_to_nhwc", "nhwc_to_nchw", "avgpool", "upsample2x", "softmax_rows",
       "frame_conv_small", "router_weights", "router_merge", "cfg_euler", "cfg_euler_v", "cfg_ddim",
       "i2vgen_latent_encoder", "vae_latents")
OUT_ARGS = ("out", "latents_out", "model_in_next")
SAMPLE_BYTES = 3 << 29  # float64 reference of a launch above this: evaluated on the first, middle and last entry


def _ops():
    from ctrl_adapter_b200 import ops
    return ops


def _signatures():
    """the parameter lists of the real entry points (the recorder may wrap an emulation with fewer parameters)"""
    ops = _ops()
    return {name: inspect.signature(getattr(ops, name)) for name in OPS}


_SIGS = _signatures()


def _sample(n, bytes_per_item):
    """indices of the entries the float64 reference is evaluated on: None (all), or the first, middle and last"""
    return None if n <= 3 or n * bytes_per_item <= SAMPLE_BYTES else [0, n // 2, n - 1]


# ----------------------------------------------------------------------------------------------------------------------
# verifiers: (a = the call's arguments on the pre-call clones, out = what the launch returned, rerun = the same call
# with some arguments changed) -> (records, sampled)
# ----------------------------------------------------------------------------------------------------------------------
def _v_linear(a, out, rerun):
    return kc.linear_verdict("linear", a, out, rerun), False


def _v_conv2d(a, out, rerun):
    n, ho, wo, cout = out.shape
    ct = a["x"].shape[3] + (0 if a["x2"] is None else a["x2"].shape[3])
    rows = _sample(n, 8 * max(ho * wo * cout, a["x"].shape[1] * a["x"].shape[2] * ct) * 3)
    return kc.conv2d_verdict("conv2d", a, out, rerun, rows=rows), rows is not None


def _v_temporal_conv(a, out, rerun):
    bf, h, w, c = a["x"].shape
    f = a["frames"]
    frames = _sample(f, 8 * (bf // f) * h * w * max(c, out.shape[3]) * 6)  # whole frames: first, middle, last
    return [kc.temporal_conv_verdict("temporal_conv", a, out, frames=frames)], frames is not None


def _v_attention(a, out, rerun):
    q, k, v, heads, dp = a["q"], a["k"], a["v"], a["heads"], a["head_dim_pad"]
    b, lq = q.shape[:2]
    lk = k.shape[1]
    rows = _sample(b, 8 * heads * lq * lk)
    ii = torch.arange(b, device=q.device) if rows is None else torch.tensor(rows, device=q.device)
    nb = ii.numel()
    q4 = q[ii].reshape(nb, lq, heads, dp)
    k4, v4 = (t.reshape(t.shape[0], lk, heads, dp) for t in (k, v))
    o4 = out[ii].reshape(nb, lq, heads, dp)
    rec = kc._attn_verdict("attention", q4, k4, v4, ii // a["kv_batch_div"], a["scale"], o4, rows=rows)
    return [rec], rows is not None


def _v_temporal_attention(a, out, rerun):
    return [kc.temporal_attention_verdict("temporal_attention", a["q"], a["k"], a["v"], a["clips"], a["frames"], a["hw"],
                                          a["heads"], a["scale"], out)], False


def _v_group_norm(a, out, rerun):
    n, h, w, c = a["x"].shape
    ct = c + (0 if a["x2"] is None else a["x2"].shape[3])
    ips = a["imgs_per_sample"]
    samples = _sample(n // ips, 8 * ips * h * w * ct * (4 if a["up2x"] else 1) * 4)
    return [kc.groupnorm_verdict("group_norm", a, out, samples=samples)], samples is not None


def _v_layer_norm(a, out, rerun):
    return kc.layernorm_verdict("layer_norm", a, out), False


def _v_timestep_embedding(a, out, rerun):
    t = a["t"].to(F64)
    if a["round_t_bf16"]:
        t = kc._r64(t)
    dim = a["dim"]
    half = dim // 2
    freq = torch.exp(-math.log(10000.0) * torch.arange(half, device=t.device, dtype=F64) / (half - a["freq_shift"]))
    arg = t[:, None] * freq[None, :]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)] if a["flip_sin_to_cos"] else [torch.sin(arg), torch.cos(arg)], -1)
    return [kc._report("timestep_embedding", out, kc._r64(ref), 2 ** -7, 4e-3, dims=("t", "ch"))], False


def _v_silu(a, out, rerun):
    return [kc._report("silu", out, kc._r64(F.silu(a["x"].to(F64))), 2 ** -7, 1e-3)], False


def _v_add(a, out, rerun):
    return [kc._report("add", out, kc._r64(a["a"].to(F64) + a["b"].to(F64)), 0.0, 0.0)], False


def _v_nchw_to_nhwc(a, out, rerun):
    x = a["x"]
    ref = F.pad(x.to(BF16).permute(0, 2, 3, 1), (0, out.shape[3] - x.shape[1]))
    return [kc._report("nchw_to_nhwc", out, ref, 0.0, 0.0, dims=("img", "y", "x", "ch"))], False


def _v_nhwc_to_nchw(a, out, rerun):
    x = a["x"]
    c = x.shape[3] if a["c"] is None else a["c"]
    ref = x[..., :c].permute(0, 3, 1, 2)
    return [kc._report("nhwc_to_nchw", out, ref, 0.0, 0.0, dims=("img", "ch", "y", "x"))], False


def _v_avgpool(a, out, rerun):
    ref = F.adaptive_avg_pool2d(a["x"].to(F64).permute(0, 3, 1, 2), (a["oh"], a["ow"])).permute(0, 2, 3, 1)
    return [kc._report("avgpool", out, kc._r64(ref), 2 ** -7, 1e-3, dims=("img", "y", "x", "ch"))], False


def _v_upsample2x(a, out, rerun):
    ref = a["x"].repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    return [kc._report("upsample2x", out, ref, 0.0, 0.0, dims=("img", "y", "x", "ch"))], False


def _v_softmax_rows(a, out, rerun):
    return [kc._report("softmax_rows", out, torch.softmax(a["x"].to(F64), dim=-1), 2 ** -8, 1e-6,
                       dims=("row", "col"))], False


def _v_frame_conv_small(a, out, rerun):
    x, f, cin = a["x"], a["frames"], a["cin"]
    bf, h, w, _ = x.shape
    xs = x[..., :cin].to(F64).reshape(bf // f, f, h, w, cin).permute(0, 4, 1, 2, 3)
    b = a["bias_host"]
    ref = F.conv3d(xs, a["w_host"].to(x.device, F64)[:, :, :, None, None],
                   None if b is None else b.to(x.device, F64), padding=(1, 0, 0))
    ref = ref.permute(0, 2, 1, 3, 4).reshape(bf, -1, h, w)
    return [kc._report("frame_conv_small", out, kc._r64(ref), 2 ** -7, 2e-3, dims=("img", "ch", "y", "x"))], False


def _v_router_weights(a, out, rerun):
    lg = a["logits"].to(F64)
    if a["mask"] is not None:
        lg = torch.where(a["mask"].bool()[None, :], lg, lg - 1e6)
    return [kc._report("router_weights", out, torch.softmax(lg, dim=-1), 1e-5, 1e-7, dims=("row", "expert"))], False


def _v_router_merge(a, out, rerun):
    acc = None
    for x, wk in zip(a["xs"], a["w"].to(F64)):
        term = kc._r64(x.to(F64) * kc._r64(wk))
        acc = term if acc is None else kc._r64(acc + term)
    return [kc._report("router_merge", out, acc, 0.0, 0.0)], False


def _v_cfg_euler(a, out, rerun):
    return [kc.cfg_euler_verdict("cfg_euler", a, out, a["model_in_next"])], False


def _v_cfg_euler_v(a, out, rerun):
    return [kc.cfg_euler_verdict("cfg_euler_v", a, out, a["model_in_next"], v_prediction=True)], False


def _v_cfg_ddim(a, out, rerun):
    return [kc.cfg_ddim_verdict("cfg_ddim", a, out, a["model_in_next"])], False


def _v_latent_encoder(a, out, rerun):
    return kc.latent_encoder_verdict("i2vgen_latent_encoder", a["x"], a["clips"], a["frames"], a["params"], out), False


def _v_vae_latents(a, out, rerun):
    return [kc.vae_latents_verdict("vae_latents", a, out)], False


VERIFIERS = {"linear": _v_linear, "conv2d": _v_conv2d, "temporal_conv": _v_temporal_conv, "attention": _v_attention,
             "temporal_attention": _v_temporal_attention, "group_norm": _v_group_norm, "layer_norm": _v_layer_norm,
             "timestep_embedding": _v_timestep_embedding, "silu": _v_silu, "add": _v_add,
             "nchw_to_nhwc": _v_nchw_to_nhwc, "nhwc_to_nchw": _v_nhwc_to_nchw, "avgpool": _v_avgpool,
             "upsample2x": _v_upsample2x, "softmax_rows": _v_softmax_rows, "frame_conv_small": _v_frame_conv_small,
             "router_weights": _v_router_weights, "router_merge": _v_router_merge, "cfg_euler": _v_cfg_euler,
             "cfg_euler_v": _v_cfg_euler_v, "cfg_ddim": _v_cfg_ddim, "i2vgen_latent_encoder": _v_latent_encoder,
             "vae_latents": _v_vae_latents}


# ----------------------------------------------------------------------------------------------------------------------
# cloning with strides, alignment and aliasing kept
# ----------------------------------------------------------------------------------------------------------------------
def _flat_tensors(args):
    """[(label, tensor)] of the tensor arguments, list arguments (router_merge's xs) element by element"""
    out = []
    for k, v in args.items():
        if torch.is_tensor(v):
            out.append((k, v))
        elif isinstance(v, (list, tuple)):
            out += [(f"{k}[{i}]", t) for i, t in enumerate(v) if torch.is_tensor(t)]
    return out


def _byte_range(t):
    es = t.element_size()
    lo = t.storage_offset() * es
    span = 1 + sum((s - 1) * st for s, st in zip(t.shape, t.stride())) if t.numel() else 0
    return lo, lo + span * es


def _storage_key(t):
    return (t.device, t.untyped_storage().data_ptr())


def _bytes(storage, device, lo, hi):
    return torch.empty(0, dtype=torch.uint8, device=device).set_(storage, lo, (hi - lo,))


class _Clone:
    """copies of the argument tensors: per storage, one buffer holding the byte range the call's views of it cover, at
    the same address modulo 16; every view re-created on it with its own shape and strides"""

    def __init__(self, args):
        self.groups = {}
        for _, t in _flat_tensors(args):
            lo, hi = _byte_range(t)
            g = self.groups.setdefault(_storage_key(t), [t.untyped_storage(), lo, hi])
            g[1], g[2] = min(g[1], lo), max(g[2], hi)
        self.bufs = {}
        for key, (st, lo, hi) in self.groups.items():
            buf = torch.empty(hi - lo + 16, dtype=torch.uint8, device=key[0])
            shift = (st.data_ptr() + lo - buf.data_ptr()) % 16
            buf[shift:shift + hi - lo].copy_(_bytes(st, key[0], lo, hi))
            self.bufs[key] = (buf, shift)

    def view(self, t):
        buf, shift = self.bufs[_storage_key(t)]
        lo = self.groups[_storage_key(t)][1]
        off = shift + t.storage_offset() * t.element_size() - lo
        assert off % t.element_size() == 0
        return torch.empty(0, dtype=t.dtype, device=t.device).set_(
            buf.untyped_storage(), off // t.element_size(), t.shape, t.stride())

    def args(self, args):
        out = {}
        for k, v in args.items():
            if torch.is_tensor(v):
                out[k] = self.view(v)
            elif isinstance(v, (list, tuple)) and any(torch.is_tensor(t) for t in v):
                out[k] = type(v)(self.view(t) if torch.is_tensor(t) else t for t in v)
            else:
                out[k] = v
        return out

    def untouched_around(self, t, written):
        """the bytes of t's buffer range outside the views in `written` are what they were before the call"""
        key = _storage_key(t)
        st, lo, hi = self.groups[key]
        buf, shift = self.bufs[key]
        now = _bytes(st, key[0], lo, hi).clone()
        for w in written:  # put the pre-call values back where the call was allowed to write
            if _storage_key(w) == key:
                es = w.element_size()
                dst = torch.empty(0, dtype=w.dtype, device=w.device).set_(
                    now.untyped_storage(), (w.storage_offset() * es - lo) // es, w.shape, w.stride())
                dst.copy_(self.view(w))
        return torch.equal(now, buf[shift:shift + hi - lo])


# ----------------------------------------------------------------------------------------------------------------------
def config_key(name, args):
    """(op, per tensor argument: shape, strides, dtype, data_ptr % 16, the argument it aliases; every scalar argument)"""
    parts, first = [name], {}
    for label, v in list(args.items()):
        tensors = _flat_tensors({label: v})
        if tensors:
            for lb, t in tensors:
                alias = first.setdefault(_storage_key(t), lb)
                parts.append((lb, tuple(t.shape), tuple(t.stride()), str(t.dtype).replace("torch.", ""),
                              t.data_ptr() % 16, None if alias == lb else alias))
        elif label == "out_scale":
            parts.append((label, float(v) != 1.0))
        else:
            parts.append((label, tuple(v) if isinstance(v, list) else v))
    return tuple(parts)


def key_summary(key):
    """short text of a key: tensor shapes (strides when not contiguous, alignment when not 16, aliases), scalars"""
    out = []
    for p in key[1:]:
        if len(p) == 6:
            lb, shape, stride, dtype, al, alias = p
            contig = list(stride) == [math.prod(shape[i + 1:]) for i in range(len(shape))]
            s = f"{lb}{list(shape)}{'' if dtype == 'bfloat16' else dtype}"
            s += "" if contig else f"s{list(stride)}"
            s += "" if al == 0 else f"@{al}"
            s += "" if alias is None else f"={alias}"
            out.append(s)
        elif p[1] is not None and p[1] is not False and not (p[0] in ("bn", "rows_per_vec", "act") and p[1] == 0):
            out.append(f"{p[0]}={p[1]:.4g}" if isinstance(p[1], float) else f"{p[0]}={p[1]}")
    return " ".join(out)


def _tensor_outputs(ret, args):
    """the tensors a call wrote: its return value(s) and its out-style arguments"""
    outs = [t for t in (ret if isinstance(ret, tuple) else (ret,)) if torch.is_tensor(t)]
    for k in OUT_ARGS:
        t = args.get(k)
        if torch.is_tensor(t) and not any(t is o for o in outs):
            outs.append(t)
    return outs


def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))


class Row:
    def __init__(self, op, key):
        self.op, self.key, self.launches = op, key, 0
        self.worst, self.where, self.sampled, self.ok, self.why = 0.0, "", False, True, []
        self.notes = {}

    def fail(self, why):
        self.ok = False
        self.why.append(why)

    def add(self, recs):
        for r in recs:
            for k in ("torch_fp32_max_err", "sdpa_bf16_max_err"):  # the error of torch's own kernel, for scale
                if k in r:
                    self.notes[k] = max(self.notes.get(k, 0.0), r[k])
            ratio = max(r.get("max_err_over_tol", 0.0), r.get("max_bh_err_over_2x_sdpa", 0.0))
            if not r["ok"]:
                self.fail(f"{r['check']}: {r.get('why') or 'out of tolerance'}")
                ratio = max(ratio, 1.0 + 1e-9) if ratio <= 1.0 else ratio
            if ratio >= self.worst:
                self.worst, self.where = ratio, r.get("where") or r.get("worst_bh") or ""


class Recorder:
    """with Recorder() as rec: ... -- every launch through ctrl_adapter_b200.ops is keyed, the first of each key checked"""

    def __init__(self, sync=None):
        self.rows = {}
        self._busy = False
        self._saved = {}
        self._sync = sync or kc._sync

    def __enter__(self):
        ops = _ops()
        for name in OPS:
            fn = getattr(ops, name)
            self._saved[name] = fn
            setattr(ops, name, self._wrap(name, fn))
        return self

    def __exit__(self, *exc):
        ops = _ops()
        for name, fn in self._saved.items():
            setattr(ops, name, fn)
        self._saved = {}
        return False

    def _wrap(self, name, fn):
        sig = _SIGS[name]

        def wrapped(*args, **kw):
            if self._busy:
                return fn(*args, **kw)
            bound = sig.bind(*args, **kw)
            bound.apply_defaults()
            a = dict(bound.arguments)
            key = config_key(name, a)
            row = self.rows.get(key)
            if row is not None:
                row.launches += 1
                return fn(*args, **kw)
            row = self.rows[key] = Row(name, key)
            row.launches = 1
            self._busy = True
            try:
                return self._first(name, fn, a, row)
            finally:
                self._busy = False
        return wrapped

    def _first(self, name, fn, a, row):
        clone = _Clone(a)
        # the verifiers read the inputs as they were before the call and the out-style arguments as it left them
        pre = {**clone.args(a), **{k: a[k] for k in OUT_ARGS if k in a}}
        ret = fn(**a)
        self._sync()
        outs = _tensor_outputs(ret, a)
        verify = VERIFIERS.get(name)
        try:
            if verify is None:
                raise NotImplementedError(f"no verifier for ops.{name}")
            recs, row.sampled = verify(pre, ret, lambda **changes: fn(**{**clone.args(a), **changes}))
            row.add(recs)
            for k in OUT_ARGS:
                t = a.get(k)
                if torch.is_tensor(t) and not clone.untouched_around(t, outs):
                    row.fail(f"{k}: bytes around the output view changed")
            # replay on the clones: out-style arguments that alias no input start as NaN
            rp = clone.args(a)
            in_keys = {_storage_key(t) for lb, t in _flat_tensors({k: v for k, v in a.items() if k not in OUT_ARGS})}
            for k in OUT_ARGS:
                t = rp.get(k)
                if torch.is_tensor(t) and t.is_floating_point() and _storage_key(a[k]) not in in_keys:
                    t.fill_(math.nan)
            ret2 = fn(**rp)
            self._sync()
            if name == "group_norm":  # float atomics in the statistics: the replay must pass the reference again
                recs2, _ = verify({**pre, "out": rp["out"]}, ret2, None)
                row.add(recs2)
            else:
                outs2 = _tensor_outputs(ret2, rp)
                if len(outs2) != len(outs) or not all(_same_bits(x, y) for x, y in zip(outs, outs2)):
                    row.fail("replay not bit-identical to the in-step launch")
        except Exception as e:  # a launch its verifier cannot handle fails its row
            row.fail(f"{type(e).__name__}: {e}"[:300])
        return ret

    # ---- report ------------------------------------------------------------------------------------------------------
    def table(self):
        lines = [f"{'op':<22} {'launches':>8} {'err/tol':>8}  {'sampled':<7} {'where':<28} configuration"]
        for row in sorted(self.rows.values(), key=lambda r: (r.op, -r.worst)):
            lines.append(f"{row.op:<22} {row.launches:>8} {row.worst:>8.3f}  {'yes' if row.sampled else '':<7} "
                         f"{row.where[:28]:<28} {key_summary(row.key)}" +
                         "".join(f" {k}={v:.3g}" for k, v in row.notes.items()) + ("" if row.ok else f"  FAIL {row.why}"))
        return "\n".join(lines)

    def failures(self):
        return [r for r in self.rows.values() if not r.ok]

    def families(self):
        """{op: (launches, distinct configurations, sampled configurations, worst err/tol)}"""
        fam = {}
        for r in self.rows.values():
            n, d, s, w = fam.get(r.op, (0, 0, 0, 0.0))
            fam[r.op] = (n + r.launches, d + 1, s + int(r.sampled), max(w, r.worst))
        return fam
