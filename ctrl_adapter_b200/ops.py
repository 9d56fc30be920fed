"""Torch-tensor front end of the C ABI: builds the descriptors (boxes, taps, strides) and launches on the
current CUDA stream.  PyTorch is used only for device memory and streams; every computation below runs in
the hand-written sm_90a kernels of ``csrc/`` (no fallback path).

Layouts: activations are channels-last, ``[N, H, W, C]`` / ``[tokens, C]`` bf16 contiguous.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import ACT_GEGLU, ACT_NONE, ACT_SILU, AttentionDesc, GemmDesc, check

BF16 = torch.bfloat16


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _req(t: torch.Tensor, dtype=BF16):
    if not t.is_cuda:
        raise ValueError("ctrl_adapter_b200 ops need CUDA tensors (there is no CPU path)")
    if t.dtype != dtype:
        raise ValueError(f"expected {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError("expected a contiguous tensor")


# ----------------------------------------------------------------------------------------------
# launch accounting: every kernel launch goes through _launch(); PROFILER (off by default) brackets each launch
# with CUDA events on the launching stream and records algorithmic FLOPs / bytes per kernel family, which is what
# bench.py's roofline block is computed from.
# ----------------------------------------------------------------------------------------------
class _Profiler:
    def __init__(self):
        self.active = False
        self.launches = 0
        self.records = []

    def start(self):
        self.records = []
        self.active = True

    def stop(self):
        self.active = False

    def summary(self):
        """-> {family: {"launches", "ms", "flops", "bytes"}} (synchronises)."""
        torch.cuda.synchronize()
        out = {}
        for fam, flops, nbytes, e0, e1, _note in self.records:
            d = out.setdefault(fam, {"launches": 0, "ms": 0.0, "flops": 0.0, "bytes": 0.0})
            d["launches"] += 1
            d["ms"] += e0.elapsed_time(e1)
            d["flops"] += flops
            d["bytes"] += nbytes
        return out


    def launches_table(self, top: int = 60):
        """Per-(family, shape note) aggregation sorted by time: [{"fam","note","n","ms","tflops"}]."""
        torch.cuda.synchronize()
        agg = {}
        for fam, flops, nbytes, e0, e1, note in self.records:
            d = agg.setdefault((fam, note), {"fam": fam, "note": note, "n": 0, "ms": 0.0, "flops": 0.0, "bytes": 0.0})
            d["n"] += 1
            d["ms"] += e0.elapsed_time(e1)
            d["flops"] += flops
            d["bytes"] += nbytes
        rows = sorted(agg.values(), key=lambda r: -r["ms"])[:top]
        for r in rows:
            r["tflops"] = round(r["flops"] / (r["ms"] * 1e9), 1) if r["ms"] > 0 and r["flops"] else None
            r["gbs"] = round(r["bytes"] / (r["ms"] * 1e6), 1) if r["ms"] > 0 and r["bytes"] else None
            r["ms"] = round(r["ms"], 3)
            del r["flops"], r["bytes"]
        return rows


PROFILER = _Profiler()
NOTE = [""]  # shape note of the launch being issued (set by the GEMM / attention wrappers when profiling)


def _launch(fam: str, flops: float, nbytes: float, name: str, *args):
    lib = _lib.load()
    PROFILER.launches += 1
    if PROFILER.active:
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        st = getattr(lib, name)(*args)
        e1.record()
        PROFILER.records.append((fam, flops, nbytes, e0, e1, NOTE[0]))
        NOTE[0] = ""
    else:
        st = getattr(lib, name)(*args)
    check(st, name)


# ----------------------------------------------------------------------------------------------
# weight packing (host side, once at load time)
# ----------------------------------------------------------------------------------------------
def pack_conv_weight(w: torch.Tensor, k_pad_to: int = 8) -> torch.Tensor:
    """[Cout, Cin, kh, kw] (or [Cout, Cin, kt, 1, 1]) -> [Cout, taps * Kp] with K = Cin zero padded to `k_pad_to`."""
    cout, cin = w.shape[0], w.shape[1]
    taps = w[0, 0].numel()
    wp = w.reshape(cout, cin, taps).permute(0, 2, 1)  # [Cout, taps, Cin]
    kp = (cin + k_pad_to - 1) // k_pad_to * k_pad_to
    if kp != cin:
        wp = torch.nn.functional.pad(wp, (0, kp - cin))
    return wp.reshape(cout, taps * kp).contiguous().to(BF16)


def pack_geglu_weight(w: torch.Tensor, b: Optional[torch.Tensor], bn: int = 256):
    """GEGLU proj [2*D, K] (value rows then gate rows) -> rows interleaved per n-tile of `bn`."""
    d = w.shape[0] // 2
    half = bn // 2
    assert d % half == 0
    wv, wg = w[:d].reshape(d // half, half, -1), w[d:].reshape(d // half, half, -1)
    wi = torch.cat([wv, wg], dim=1).reshape(2 * d, -1).contiguous()
    bi = None
    if b is not None:
        bv, bg = b[:d].reshape(d // half, half), b[d:].reshape(d // half, half)
        bi = torch.cat([bv, bg], dim=1).reshape(2 * d).contiguous()
    return wi, bi


def bias_f32(b: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """Biases are consumed as fp32 holding the bf16-rounded value (autocast casts them to bf16)."""
    return None if b is None else b.to(BF16).float().contiguous()


# ----------------------------------------------------------------------------------------------
# box heuristics: split the 128-row tile over (x, y, n) minimising padded work
# ----------------------------------------------------------------------------------------------
def choose_box(w: int, h: int, n: int):
    best = None
    for lw in range(8):
        bw = 1 << lw
        for lh in range(8 - lw):
            bh = 1 << lh
            bn_ = 128 // (bw * bh)
            tiles = math.ceil(w / bw) * math.ceil(h / bh) * math.ceil(n / bn_)
            key = (tiles, -bw, -bh)
            if best is None or key < best[0]:
                best = (key, (bw, bh, bn_))
    return best[1]


# ----------------------------------------------------------------------------------------------
# GEMM family
# ----------------------------------------------------------------------------------------------
def _fill_epilogue(d: GemmDesc, *, bias, act, out_scale, rowvec, rowvec_strides, residual, blend_src, res_strides,
                   blend_alpha):
    d.bias = _ptr(bias)
    d.act = act
    d.out_scale = float(out_scale)
    d.rowvec = _ptr(rowvec)
    d.residual = _ptr(residual)
    d.blend_src = _ptr(blend_src)
    d.blend_alpha = _ptr(blend_alpha)
    for i in range(4):
        d.rowvec_strides[i] = rowvec_strides[i] if rowvec_strides else 0
        d.res_strides[i] = res_strides[i] if res_strides else 0


def _epilogue_note(w_rows, act, bn, residual, rowvec, blend_src):
    """Profiler shape note of a GEMM's N tile and epilogue operands.  bn 0 is resolved by ca_gemm's rule."""
    if bn == 0:
        bn = next((b for b in (256, 160, 128) if w_rows % b == 0), 64 if w_rows <= 64 else 128 if w_rows <= 128 else 256)
        bn = 256 if act == ACT_GEGLU else bn
    return (f"bn{bn} res{int(residual is not None)} rv{int(rowvec is not None)} "
            f"blend{int(blend_src is not None)}")


def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, act: int = ACT_NONE,
           residual: Optional[torch.Tensor] = None, rowvec: Optional[torch.Tensor] = None, rows_per_vec: int = 0,
           blend_src: Optional[torch.Tensor] = None, blend_alpha: Optional[torch.Tensor] = None,
           out_scale: float = 1.0, out: Optional[torch.Tensor] = None, out_fp32: bool = False, bn: int = 0):
    """y[M, N] = epilogue(x[M, K] @ w[N, K]^T).  `rowvec` [M / rows_per_vec, N] is broadcast over consecutive rows."""
    _req(x); _req(w)
    m, k = x.shape
    wr = w.shape[0]
    n_out = wr // 2 if act == ACT_GEGLU else wr
    if out is None:
        out = torch.empty((m, n_out), device=x.device, dtype=torch.float32 if out_fp32 else BF16)
    d = GemmDesc()
    d.nsrc = 1
    d.a[0] = x.data_ptr()
    d.a_channels[0] = k; d.a_c_off[0] = 0; d.a_c_len[0] = k
    d.a_dims[0], d.a_dims[1], d.a_dims[2], d.a_dims[3] = m, 1, 1, 1
    st = (k, m * k, m * k, m * k)
    for i in range(4):
        d.a_strides[0][i] = st[i]
    d.box[0], d.box[1], d.box[2], d.box[3] = 128, 1, 1, 1
    d.ntaps = 1
    d.w = w.data_ptr(); d.w_rows = wr; d.w_k_per_tap = w.shape[1]
    d.out = out.data_ptr(); d.out_fp32 = int(out_fp32); d.n_out = n_out
    d.out_dims[0], d.out_dims[1], d.out_dims[2], d.out_dims[3] = m, 1, 1, 1
    d.out_strides[0] = out.stride(0)
    d.bn = bn
    if rowvec is not None:
        # rowvec index = row // rows_per_vec: expressed by splitting the row space as (rows_per_vec, M/rows_per_vec)
        if rows_per_vec <= 0 or m % rows_per_vec != 0:
            raise ValueError("rows_per_vec must divide M")
    rs = (residual.stride(0), 0, 0, 0) if residual is not None else (blend_src.stride(0), 0, 0, 0) if blend_src is not None else None
    if rowvec is not None:
        # re-express rows as (r % rpv, r // rpv): tile box stays 128 x 1 when rpv is a multiple of 128, otherwise
        # use a 2-D box so that tiles do not straddle rowvec boundaries
        rpv = rows_per_vec
        nv = m // rpv
        if rpv >= 128:
            b0 = 128
            b1 = 1
        else:
            b0 = 1 << (rpv.bit_length() - 1)  # largest power of two <= rpv
            b1 = 128 // b0
        d.a_dims[0], d.a_dims[1] = rpv, nv
        d.a_strides[0][0], d.a_strides[0][1] = k, rpv * k
        d.box[0], d.box[1] = b0, b1
        d.out_dims[0], d.out_dims[1] = rpv, nv
        d.out_strides[0], d.out_strides[1] = out.stride(0), rpv * out.stride(0)
        rvs = (0, rowvec.stride(0), 0, 0)
        if rs is not None:
            rs = (rs[0], rpv * rs[0], 0, 0)
    else:
        rvs = None
    _fill_epilogue(d, bias=bias, act=act, out_scale=out_scale, rowvec=rowvec, rowvec_strides=rvs, residual=residual,
                   blend_src=blend_src, res_strides=rs, blend_alpha=blend_alpha)
    if PROFILER.active:
        NOTE[0] = f"linear m{m} k{k} n{wr} act{act} {_epilogue_note(wr, act, bn, residual, rowvec, blend_src)}"
    _launch("gemm", 2.0 * m * k * wr, 2.0 * (m * k + wr * k + m * n_out), "ca_gemm", C.byref(d), _stream())
    return out


_TAPS_3X3 = [(dy, dx) for dy in range(3) for dx in range(3)]


def conv2d(x: torch.Tensor, w_packed: torch.Tensor, bias: Optional[torch.Tensor], *, ksize: int = 3, stride: int = 1,
           x2: Optional[torch.Tensor] = None, act: int = ACT_NONE, out_scale: float = 1.0,
           rowvec: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
           blend_src: Optional[torch.Tensor] = None, blend_alpha: Optional[torch.Tensor] = None,
           out: Optional[torch.Tensor] = None, out_fp32: bool = False, bn: int = 0, k_per_tap: Optional[int] = None,
           pad: Optional[Tuple[int, int]] = None):
    """Channels-last conv: x [N,H,W,C] (+ optional x2 [N,H,W,C2] concatenated on C), w_packed [Cout, taps*Kp].
    ksize 1 or 3 (padding (ksize-1)/2), stride 1 or 2 (3x3 only).  rowvec [N, Cout] is broadcast per sample
    (time-embedding add); residual / blend_src are [N, Ho, Wo, Cout].
    pad: zero padding (before, after) of both spatial axes; None is (ksize-1)/2 on every side.  Stride 2 also takes
    (0, 1): one zero row / column at the bottom / right only (diffusers Downsample2D(padding=0) of the VAE encoder)."""
    _req(x); _req(w_packed)
    if pad is not None and tuple(pad) != (ksize // 2, ksize // 2) and not (stride == 2 and tuple(pad) == (0, 1)):
        raise ValueError(f"conv2d: pad {tuple(pad)} is not supported at ksize {ksize}, stride {stride}")
    pad_after_only = pad is not None and tuple(pad) == (0, 1)
    n, h, w_, c = x.shape
    c2 = 0
    if x2 is not None:
        _req(x2)
        c2 = x2.shape[3]
        assert x2.shape[:3] == x.shape[:3]
    cout = w_packed.shape[0]
    ntaps = ksize * ksize
    kpt = k_per_tap if k_per_tap is not None else w_packed.shape[1] // ntaps
    ho, wo = (h, w_) if stride == 1 else (h // 2, w_ // 2)
    if out is None:
        out = torch.empty((n, ho, wo, cout), device=x.device, dtype=torch.float32 if out_fp32 else BF16)
    d = GemmDesc()
    d.nsrc = 2 if x2 is not None else 1
    d.a[0] = x.data_ptr()
    d.a_c_off[0] = 0; d.a_c_len[0] = c
    if x2 is not None:
        d.a[1] = x2.data_ptr(); d.a_c_off[1] = 0; d.a_c_len[1] = c2
    bw, bh, bnn = choose_box(wo, ho, n)
    if stride == 1:
        d.a_channels[0] = c; d.a_channels[1] = c2
        d.a_dims[0], d.a_dims[1], d.a_dims[2], d.a_dims[3] = w_, h, n, 1
        for s_, cc in ((0, c), (1, c2)):
            if s_ == 1 and x2 is None:
                break
            d.a_strides[s_][0], d.a_strides[s_][1], d.a_strides[s_][2], d.a_strides[s_][3] = cc, w_ * cc, h * w_ * cc, n * h * w_ * cc
        d.box[0], d.box[1], d.box[2], d.box[3] = bw, bh, bnn, 1
        d.ntaps = ntaps
        if ksize == 3:
            for t, (dy, dx) in enumerate(_TAPS_3X3):
                d.tap_off[t][0], d.tap_off[t][1] = dx - 1, dy - 1
        d.out_dims[0], d.out_dims[1], d.out_dims[2], d.out_dims[3] = wo, ho, n, 1
        os_ = (cout, wo * cout, ho * wo * cout, 0)
        rvs = (0, 0, rowvec.stride(0) if (rowvec is not None and rowvec.shape[0] > 1) else 0, 0)
    else:
        if ksize != 3 or x2 is not None or h % 2 or w_ % 2:
            raise ValueError(f"conv2d: stride 2 takes one source, a 3x3 kernel and an even height and width, got "
                             f"ksize {ksize}, {2 if x2 is not None else 1} sources, height {h}, width {w_}")
        # parity view: channel axis [x parity][C], row dims (x/2, y parity, y/2, n)
        d.a_channels[0] = 2 * c
        d.a_dims[0], d.a_dims[1], d.a_dims[2], d.a_dims[3] = w_ // 2, 2, h // 2, n
        d.a_strides[0][0], d.a_strides[0][1], d.a_strides[0][2], d.a_strides[0][3] = 2 * c, w_ * c, 2 * w_ * c, h * w_ * c
        d.box[0], d.box[1], d.box[2], d.box[3] = bw, 1, bh, bnn
        d.ntaps = 9
        # input row 2*oy + dy - 1: dy=0 -> (parity 1, oy-1); dy=1 -> (0, oy); dy=2 -> (1, oy).
        # pad (0, 1): input row 2*oy + dy: dy=0 -> (0, oy); dy=1 -> (1, oy); dy=2 -> (0, oy+1), zero filled at oy+1 = H/2
        taps = ((0, 0), (1, 0), (0, 1)) if pad_after_only else ((1, -1), (0, 0), (1, 0))
        for t, (dy, dx) in enumerate(_TAPS_3X3):
            py, oyo = taps[dy]
            px, oxo = taps[dx]
            d.tap_off[t][0], d.tap_off[t][1], d.tap_off[t][2], d.tap_off[t][3] = oxo, py, oyo, 0
            d.tap_c_off[t] = px * c
        d.out_dims[0], d.out_dims[1], d.out_dims[2], d.out_dims[3] = wo, 1, ho, n
        os_ = (cout, 0, wo * cout, ho * wo * cout)
        rvs = (0, 0, 0, rowvec.stride(0) if (rowvec is not None and rowvec.shape[0] > 1) else 0)
    for i in range(4):
        d.out_strides[i] = os_[i]
    d.w = w_packed.data_ptr(); d.w_rows = cout; d.w_k_per_tap = kpt
    d.out = out.data_ptr(); d.out_fp32 = int(out_fp32); d.n_out = cout
    d.bn = bn
    _fill_epilogue(d, bias=bias, act=act, out_scale=out_scale, rowvec=rowvec, rowvec_strides=rvs if rowvec is not None else None,
                   residual=residual, blend_src=blend_src,
                   res_strides=os_ if (residual is not None or blend_src is not None) else None, blend_alpha=blend_alpha)
    if PROFILER.active:
        NOTE[0] = (f"conv{ksize} s{stride} n{n} {h}x{w_} c{c}+{c2}->{cout} box{bw}x{bh}x{bnn} "
                   f"{_epilogue_note(cout, act, bn, residual, rowvec, blend_src)}")
    _launch("gemm", 2.0 * n * ho * wo * ntaps * (c + c2) * cout,
            2.0 * (n * h * w_ * (c + c2) + w_packed.numel() + n * ho * wo * cout), "ca_gemm", C.byref(d), _stream())
    return out


def temporal_conv(x: torch.Tensor, w_packed: torch.Tensor, bias: Optional[torch.Tensor], frames: int, *,
                  rowvec: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
                  blend_src: Optional[torch.Tensor] = None, blend_alpha: Optional[torch.Tensor] = None,
                  out: Optional[torch.Tensor] = None):
    """Conv3d kernel (3,1,1), padding (1,0,0) over the frame axis of x [B*F, H, W, C] (frames contiguous per clip).
    rowvec [B*F, Cout] is broadcast per frame."""
    _req(x); _req(w_packed)
    bf, h, w_, c = x.shape
    b = bf // frames
    hw = h * w_
    cout = w_packed.shape[0]
    if out is None:
        out = torch.empty((bf, h, w_, cout), device=x.device, dtype=BF16)
    d = GemmDesc()
    d.nsrc = 1
    d.a[0] = x.data_ptr(); d.a_channels[0] = c; d.a_c_off[0] = 0; d.a_c_len[0] = c
    d.a_dims[0], d.a_dims[1], d.a_dims[2], d.a_dims[3] = hw, frames, b, 1
    d.a_strides[0][0], d.a_strides[0][1], d.a_strides[0][2], d.a_strides[0][3] = c, hw * c, frames * hw * c, bf * hw * c
    bp = min(128, 1 << (hw.bit_length() - 1)) if hw < 128 else 128
    bfm = 128 // bp
    d.box[0], d.box[1], d.box[2], d.box[3] = bp, bfm, 1, 1
    d.ntaps = 3
    for t in range(3):
        d.tap_off[t][1] = t - 1
    d.out_dims[0], d.out_dims[1], d.out_dims[2], d.out_dims[3] = hw, frames, b, 1
    os_ = (cout, hw * cout, frames * hw * cout, 0)
    for i in range(4):
        d.out_strides[i] = os_[i]
    d.w = w_packed.data_ptr(); d.w_rows = cout; d.w_k_per_tap = w_packed.shape[1] // 3
    d.out = out.data_ptr(); d.n_out = cout
    _fill_epilogue(d, bias=bias, act=ACT_NONE, out_scale=1.0, rowvec=rowvec,
                   rowvec_strides=((0, rowvec.stride(0), frames * rowvec.stride(0), 0) if rowvec.shape[0] > 1 else (0, 0, 0, 0)) if rowvec is not None else None,
                   residual=residual,
                   blend_src=blend_src, res_strides=os_ if (residual is not None or blend_src is not None) else None,
                   blend_alpha=blend_alpha)
    _launch("gemm", 2.0 * bf * hw * 3 * c * cout, 2.0 * (bf * hw * (c + cout) + w_packed.numel()), "ca_gemm", C.byref(d), _stream())
    return out


# ----------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------
def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, head_dim_pad: int, scale: float,
              out: Optional[torch.Tensor] = None, kv_batch_div: int = 1):
    """q [B, Lq, heads*Dp], k/v [B / kv_batch_div, Lk, heads*Dp] (last dim contiguous, row/batch strided views
    allowed).  kv_batch_div > 1: consecutive query batches (the frames of a clip) share one K/V context."""
    b, lq, ctot = q.shape
    lk = k.shape[1]
    assert ctot == heads * head_dim_pad and q.stride(2) == 1 and k.stride(2) == 1 and v.stride(2) == 1
    if out is None:
        out = torch.empty((b, lq, ctot), device=q.device, dtype=BF16)
    d = AttentionDesc()
    d.q, d.k, d.v, d.out = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr()
    d.batch, d.heads, d.lq, d.lk = b, heads, lq, lk
    d.head_dim_pad = head_dim_pad
    d.scale = float(scale)
    d.q_row_stride, d.q_batch_stride = q.stride(1), q.stride(0)
    d.k_row_stride, d.k_batch_stride = k.stride(1), k.stride(0)
    d.v_row_stride, d.v_batch_stride = v.stride(1), v.stride(0)
    d.out_row_stride, d.out_batch_stride = out.stride(1), out.stride(0)
    d.kv_batch_div = kv_batch_div
    if PROFILER.active:
        NOTE[0] = f"attn b{b} h{heads} lq{lq} lk{lk} dp{head_dim_pad}"
    _launch("attention", 4.0 * b * heads * lq * lk * head_dim_pad, 2.0 * b * (2 * lq + 2 * lk) * ctot, "ca_attention", C.byref(d), _stream())
    return out


def temporal_attention(q, k, v, clips: int, frames: int, hw: int, heads: int, scale: float, out=None,
                       row_stride: Optional[int] = None):
    """q/k/v: [clips*frames*hw, heads*64] rows (row stride `row_stride` elements, e.g. views of a fused QKV buffer)."""
    c = heads * 64
    rs = c if row_stride is None else row_stride
    if out is None:
        out = torch.empty((clips * frames * hw, c), device=q.device, dtype=BF16)
    _launch("temporal_attention", 4.0 * clips * hw * heads * frames * frames * 64, 2.0 * 4 * clips * frames * hw * c, "ca_temporal_attention", q.data_ptr(), k.data_ptr(), v.data_ptr(), clips, frames, hw, heads,
                                            float(scale), rs, out.data_ptr(), _stream())
    return out


# ----------------------------------------------------------------------------------------------
# norms
# ----------------------------------------------------------------------------------------------
_gn_scratch = {}


def _gn_sums(device, n: int, groups: int) -> torch.Tensor:
    key = (device.index, torch.cuda.current_stream().cuda_stream)
    need = n * groups * 2
    buf = _gn_scratch.get(key)
    if buf is None or buf.numel() < need:
        buf = torch.empty(max(need, 8192), device=device, dtype=torch.float64)
        _gn_scratch[key] = buf
    return buf


def group_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, *, groups: int = 32,
               silu: bool = False, up2x: bool = False, x2: Optional[torch.Tensor] = None, imgs_per_sample: int = 1,
               out: Optional[torch.Tensor] = None):
    """x [N, H, W, C] (+x2 concatenated on C).  imgs_per_sample > 1: statistics span that many consecutive images
    (the 5-D GroupNorm of the temporal ResNet)."""
    _req(x)
    n, h, w_, c = x.shape
    c2 = x2.shape[3] if x2 is not None else 0
    ct = c + c2
    nsamp = n // imgs_per_sample
    sums = torch.empty(nsamp * groups * 2, device=x.device, dtype=torch.float64)
    if PROFILER.active:
        NOTE[0] = f"gn_stats n{n} {h}x{w_} c{c}+{c2}"
    _launch("groupnorm", 0.0, 2.0 * n * h * w_ * ct, "ca_groupnorm_stats", x.data_ptr(), c, _ptr(x2), c2, nsamp,
            imgs_per_sample * h * w_, groups, sums.data_ptr(), _stream())
    if out is None:
        out = torch.empty((n, h * 2, w_ * 2, ct) if up2x else (n, h, w_, ct), device=x.device, dtype=BF16)
    if PROFILER.active:
        NOTE[0] = f"gn_apply n{n} {h}x{w_} c{c}+{c2} silu{int(silu)} up{int(up2x)}"
    _launch("groupnorm", 0.0, 2.0 * n * h * w_ * ct * (5 if up2x else 2), "ca_groupnorm_apply", x.data_ptr(), c,
            _ptr(x2), c2, n, h, w_, imgs_per_sample, groups, float(eps), sums.data_ptr(), gamma.data_ptr(),
            beta.data_ptr(), int(silu), int(up2x), out.data_ptr(), _stream())
    return out


def layer_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5, *,
               add_rowvec: Optional[torch.Tensor] = None, rows_per_vec: int = 0, return_sum: bool = False):
    _req(x)
    c = x.shape[-1]
    rows = x.numel() // c
    y = torch.empty_like(x)
    ysum = torch.empty_like(x) if (add_rowvec is not None and return_sum) else None
    if PROFILER.active:
        NOTE[0] = f"layernorm rows{rows} c{c} rv{int(add_rowvec is not None)}"
    _launch("layernorm", 0.0, 2.0 * 2 * x.numel(), "ca_layernorm", x.data_ptr(), rows, c, float(eps), gamma.data_ptr(), beta.data_ptr(),
                                   _ptr(add_rowvec), rows_per_vec, _ptr(ysum), y.data_ptr(), _stream())
    return (y, ysum) if return_sum else y


# ----------------------------------------------------------------------------------------------
# small kernels
# ----------------------------------------------------------------------------------------------
def timestep_embedding(t: torch.Tensor, dim: int, *, flip_sin_to_cos: bool = True, freq_shift: float = 0.0,
                       round_t_bf16: bool = False):
    _req(t, torch.float32)
    n = t.numel()
    out = torch.empty((n, dim), device=t.device, dtype=BF16)
    _launch("timestep_embedding", 0.0, 0.0, "ca_timestep_embedding", t.data_ptr(), n, dim, int(flip_sin_to_cos), float(freq_shift),
                                            int(round_t_bf16), out.data_ptr(), _stream())
    return out


def silu(x: torch.Tensor):
    _req(x)
    y = torch.empty_like(x)
    _launch("silu", 0.0, 2.0 * 2 * x.numel(), "ca_silu", x.data_ptr(), x.numel(), y.data_ptr(), _stream())
    return y


def add(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None):
    _req(a); _req(b)
    y = torch.empty_like(a) if out is None else out
    _launch("add", 0.0, 2.0 * 3 * a.numel(), "ca_add", a.data_ptr(), b.data_ptr(), a.numel(), y.data_ptr(), _stream())
    return y


def nchw_to_nhwc(x: torch.Tensor, c_pad: Optional[int] = None):
    """[N, C, H, W] bf16/fp32 contiguous -> [N, H, W, c_pad] bf16 (extra channels zero)."""
    if not x.is_contiguous():
        raise ValueError("expected contiguous NCHW")
    n, c, h, w_ = x.shape
    cp = c if c_pad is None else c_pad
    y = torch.empty((n, h, w_, cp), device=x.device, dtype=BF16)
    if x.dtype not in (BF16, torch.float32):
        raise ValueError("nchw_to_nhwc: bf16 or fp32 input")
    _launch("nchw_to_nhwc", 0.0, 2.0 * 2 * x.numel(), "ca_nchw_to_nhwc", x.data_ptr(), int(x.dtype == torch.float32), n, c, h * w_, cp, y.data_ptr(),
                                      _stream())
    return y


def nhwc_to_nchw(x: torch.Tensor, c: Optional[int] = None, fp32: bool = False):
    _req(x)
    n, h, w_, cs = x.shape
    cc = cs if c is None else c
    y = torch.empty((n, cc, h, w_), device=x.device, dtype=torch.float32 if fp32 else BF16)
    _launch("nhwc_to_nchw", 0.0, 2.0 * 2 * x.numel(), "ca_nhwc_to_nchw", x.data_ptr(), n, cc, cs, h * w_, y.data_ptr(), int(fp32), _stream())
    return y


def avgpool(x: torch.Tensor, oh: int, ow: int):
    _req(x)
    n, h, w_, c = x.shape
    y = torch.empty((n, oh, ow, c), device=x.device, dtype=BF16)
    _launch("avgpool", 0.0, 2.0 * x.numel(), "ca_avgpool", x.data_ptr(), n, h, w_, c, oh, ow, y.data_ptr(), _stream())
    return y


def upsample2x(x: torch.Tensor):
    _req(x)
    n, h, w_, c = x.shape
    y = torch.empty((n, 2 * h, 2 * w_, c), device=x.device, dtype=BF16)
    _launch("upsample2x", 0.0, 2.0 * 5 * x.numel(), "ca_upsample2x", x.data_ptr(), n, h, w_, c, y.data_ptr(), _stream())
    return y


def softmax_rows(x: torch.Tensor):
    """fp32 [rows, cols] -> bf16 softmax over the last axis (fp32 math, one rounding)."""
    _req(x, torch.float32)
    rows, cols = x.shape
    y = torch.empty((rows, cols), device=x.device, dtype=BF16)
    _launch("softmax_rows", 0.0, 6.0 * x.numel(), "ca_softmax_rows", x.data_ptr(), rows, cols, y.data_ptr(), _stream())
    return y


def frame_conv_small(x: torch.Tensor, w_host: torch.Tensor, bias_host: Optional[torch.Tensor], frames: int, cin: int):
    """Conv3d (3,1,1), padding (1,0,0) over the frame axis for <= 4 channels (the temporal VAE decoder's time_conv_out).
    x [B*F, H, W, Cs] channels-last bf16 (the first `cin` channels are read); w_host [Cout, Cin, 3] / bias_host [Cout]:
    fp32 HOST tensors (passed to the kernel by value).  Returns [B*F, Cout, H, W] bf16 (logical NCHW, contiguous)."""
    _req(x)
    if w_host.device.type != "cpu" or w_host.dtype != torch.float32 or not w_host.is_contiguous():
        raise ValueError("frame_conv_small: weights must be a contiguous fp32 host tensor")
    bf, h, w_, cs = x.shape
    cout = w_host.shape[0]
    if tuple(w_host.shape) != (cout, cin, 3) or bf % frames:
        raise ValueError("frame_conv_small: weight shape / frame count mismatch")
    y = torch.empty((bf, cout, h, w_), device=x.device, dtype=BF16)
    bptr = None
    if bias_host is not None:
        if bias_host.device.type != "cpu" or bias_host.dtype != torch.float32 or bias_host.numel() != cout:
            raise ValueError("frame_conv_small: bias must be an fp32 host tensor of Cout elements")
        bptr = bias_host.data_ptr()
    _launch("frame_conv_small", 0.0, 2.0 * (x.numel() + y.numel()), "ca_frame_conv_small", x.data_ptr(), bf // frames, frames,
            h * w_, cs, cin, cout, w_host.data_ptr(), bptr, y.data_ptr(), _stream())
    return y


def router_weights(logits: torch.Tensor, mask: Optional[torch.Tensor]):
    """logits [R, E] fp32, mask [E] uint8 (0 = masked) -> softmax weights [R, E] fp32."""
    _req(logits, torch.float32)
    r, e = logits.shape
    out = torch.empty_like(logits)
    _launch("router_weights", 0.0, 0.0, "ca_router_weights", logits.data_ptr(), _ptr(mask), r, e, out.data_ptr(), _stream())
    return out


def router_merge(xs: Sequence[torch.Tensor], w: torch.Tensor):
    """y = sum_k w[k] * xs[k] (bf16 rounding after every multiply / add as in the reference loop)."""
    for x in xs:
        _req(x)
    _req(w, torch.float32)
    if not 1 <= len(xs) <= 8:
        raise ValueError("router_merge takes 1..8 expert tensors")
    ptrs = (C.c_void_p * len(xs))(*[x.data_ptr() for x in xs])  # host array: pointers are passed to the kernel by value
    y = torch.empty_like(xs[0])
    _launch("router_merge", 0.0, 2.0 * (len(xs) + 1) * xs[0].numel(), "ca_router_merge", ptrs, w.data_ptr(), len(xs),
            xs[0].numel(), y.data_ptr(), _stream())
    return y


def cfg_euler(eps_uncond, eps_text, latents, guidance, step_row, latents_out=None, model_in_next=None,
              round_latents_bf16: bool = True):
    """step_row: device fp32 [4] = (t, sigma, sigma_next, sqrt(sigma_next^2+1))."""
    _req(eps_uncond); _req(eps_text); _req(latents, torch.float32); _req(step_row, torch.float32)
    if latents_out is None:
        latents_out = torch.empty_like(latents)
    _launch("cfg_euler", 0.0, 0.0, "ca_cfg_euler", eps_uncond.data_ptr(), eps_text.data_ptr(), latents.data_ptr(), latents.numel(),
                                   float(guidance), step_row.data_ptr(), int(round_latents_bf16),
                                   latents_out.data_ptr(), _ptr(model_in_next), _stream())
    return latents_out


def cfg_euler_v(eps_uncond, eps_text, latents, guidance_per_frame, frames: int, step_row, latents_out=None,
                model_in_next=None, round_latents_bf16: bool = True):
    """SVD loop update: latents fp32 [clips, frames, C, H, W]; guidance_per_frame device fp32 [frames];
    step_row: device fp32 [4] = (t, sigma, sigma_next, sqrt(sigma_next^2+1))."""
    _req(eps_uncond); _req(eps_text); _req(latents, torch.float32); _req(step_row, torch.float32)
    _req(guidance_per_frame, torch.float32)
    if latents_out is None:
        latents_out = torch.empty_like(latents)
    frame_elems = latents.numel() // (latents.shape[0] * frames)
    _launch("cfg_euler", 0.0, 0.0, "ca_cfg_euler_v", eps_uncond.data_ptr(), eps_text.data_ptr(), latents.data_ptr(),
            latents.numel(), guidance_per_frame.data_ptr(), int(frames), int(frame_elems), step_row.data_ptr(),
            int(round_latents_bf16), latents_out.data_ptr(), _ptr(model_in_next), _stream())
    return latents_out


def cfg_ddim(eps_uncond, eps_text, latents, guidance, step_row, latents_out=None, model_in_next=None,
             round_latents_bf16: bool = True, v_prediction: bool = False):
    """step_row: device fp32 [4] = (t, alpha_prod_t, alpha_prod_prev, -)."""
    _req(eps_uncond); _req(eps_text); _req(latents, torch.float32); _req(step_row, torch.float32)
    if latents_out is None:
        latents_out = torch.empty_like(latents)
    _launch("cfg_ddim", 0.0, 0.0, "ca_cfg_ddim", eps_uncond.data_ptr(), eps_text.data_ptr(), latents.data_ptr(), latents.numel(),
                                  float(guidance), step_row.data_ptr(), int(round_latents_bf16), int(v_prediction),
                                  latents_out.data_ptr(), _ptr(model_in_next), _stream())
    return latents_out


def i2vgen_latent_encoder(x: torch.Tensor, clips: int, frames: int, params: torch.Tensor):
    """x [clips*frames, H, W, Cs] bf16 (first 4 channels used); params fp32 [288] (layout: include/ctrl_adapter_b200.h)."""
    _req(x); _req(params, torch.float32)
    bf, h, w_, cs = x.shape
    y = torch.zeros_like(x)
    _launch("i2vgen_latent_encoder", 0.0, 4.0 * x.numel(), "ca_i2vgen_latent_encoder", x.data_ptr(), clips, frames,
            h * w_, cs, params.data_ptr(), y.data_ptr(), _stream())
    return y


VAE_POSTERIOR, VAE_I2VGEN, VAE_SVD = 0, 1, 2


def vae_latents(moments: torch.Tensor, layout: int = VAE_POSTERIOR, noise: Optional[torch.Tensor] = None,
                frames: int = 1, num_videos: int = 1, scale: float = 1.0):
    """VAE posterior -> latents (layouts: include/ctrl_adapter_b200.h ``ca_vae_latents``).  moments [n, h, w, 8] bf16
    (mean, logvar); noise fp32 [n, 4, h, w] or None (the posterior's mode).  Returns bf16
    VAE_POSTERIOR [n, 4, h, w] / VAE_I2VGEN [2*n*nv, 4, F, h, w] / VAE_SVD [2*n*nv, F, 4, h, w]."""
    _req(moments)
    n, h, w_, cm = moments.shape
    if cm != 8:
        raise ValueError(f"vae_latents: moments carry {cm} channels, expected 8 (mean and logvar of 4 latent channels)")
    if noise is not None:
        _req(noise, torch.float32)
        if tuple(noise.shape) != (n, 4, h, w_):
            raise ValueError(f"vae_latents: noise shape {tuple(noise.shape)}, expected {(n, 4, h, w_)}")
    rows = n if layout == VAE_POSTERIOR else 2 * n * num_videos
    shape = {VAE_POSTERIOR: (n, 4, h, w_), VAE_I2VGEN: (rows, 4, frames, h, w_),
             VAE_SVD: (rows, frames, 4, h, w_)}.get(layout)
    if shape is None or min(shape) < 1:
        raise ValueError(f"vae_latents: layout {layout}, frames {frames}, num_videos {num_videos}")
    out = torch.empty(shape, device=moments.device, dtype=BF16)
    _launch("vae_latents", 0.0, 2.0 * (moments.numel() + out.numel()), "ca_vae_latents", moments.data_ptr(),
            _ptr(noise), n, h * w_, 4, layout, frames, num_videos, float(scale), out.data_ptr(), _stream())
    return out
