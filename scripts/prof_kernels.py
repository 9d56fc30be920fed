"""Launches single hot kernels at the BASELINE config-2 shapes (for ncu captures and quick CUDA-event timings).
usage: python scripts/prof_kernels.py attn|attn1k|attn77|geglu|lin_small|lin_res|conv [--time] [--no-res]
--no-res drops the residual of lin_small / lin_res: the same GEMM with a plain epilogue."""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ctrl_adapter_b200 import ops  # noqa: E402

BF16 = torch.bfloat16
which = sys.argv[1]
do_time = "--time" in sys.argv
no_res = "--no-res" in sys.argv
torch.manual_seed(0)
dev = "cuda"


def rnd(*s, scale=1.0):
    return (torch.randn(*s, device=dev) * scale).to(BF16)


if which.startswith("attn"):
    b, h, l, lk = {"attn": (16, 5, 16384, 16384), "attn4k": (16, 10, 4096, 4096), "attn1k": (16, 20, 1024, 1024),
                   "attn77": (16, 20, 1024, 77)}[which]
    qkv = rnd(b, l, 3 * h * 64)
    kv = rnd(b, lk, 2 * h * 64)
    q = qkv[:, :, : h * 64]
    k, v = (qkv[:, :, h * 64: 2 * h * 64], qkv[:, :, 2 * h * 64:]) if lk == l else (kv[:, :, : h * 64], kv[:, :, h * 64:])
    fn = lambda: ops.attention(q, k, v, h, 64, 0.125)  # noqa: E731
    flops = 4.0 * b * h * l * lk * 64
elif which == "geglu":
    x, w, bias = rnd(16384, 1280), rnd(10240, 1280, scale=1 / math.sqrt(1280)), torch.zeros(10240, device=dev)
    fn = lambda: ops.linear(x, w, bias, act=ops.ACT_GEGLU, bn=256)  # noqa: E731
    flops = 2.0 * 16384 * 1280 * 10240
elif which == "lin_small":
    x, w, bias = rnd(65536, 640), rnd(640, 640, scale=1 / math.sqrt(640)), torch.zeros(640, device=dev)
    res = None if no_res else rnd(65536, 640)
    fn = lambda: ops.linear(x, w, bias, residual=res)  # noqa: E731
    flops = 2.0 * 65536 * 640 * 640
elif which == "lin_res":
    x, w, bias = rnd(16384, 1280), rnd(1280, 1280, scale=1 / math.sqrt(1280)), torch.zeros(1280, device=dev)
    res = None if no_res else rnd(16384, 1280)
    fn = lambda: ops.linear(x, w, bias, residual=res)  # noqa: E731
    flops = 2.0 * 16384 * 1280 * 1280
elif which.startswith("conv"):  # conv or conv:<bn>
    bn = int(which.split(":")[1]) if ":" in which else 0
    x = rnd(16, 128, 128, 320)
    w = ops.pack_conv_weight(rnd(320, 320, 3, 3, scale=1 / math.sqrt(2880)))
    bias = torch.zeros(320, device=dev)
    fn = lambda: ops.conv2d(x, w, bias, bn=bn)  # noqa: E731
    flops = 2.0 * 16 * 128 * 128 * 2880 * 320
elif which.startswith("tattn"):  # temporal attention at config 3's adapter-A shape (8 clips x 16 frames x 64^2 pixels, 5 heads)
    clips, frames, hw, heads = {"tattn": (8, 16, 4096, 5), "tattn14": (4, 14, 9216, 5), "tattn20": (8, 16, 256, 20)}[which]
    inner = heads * 64
    qkv = rnd(clips * frames * hw, 3 * inner)
    fn = lambda: ops.temporal_attention(qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:], clips, frames, hw,  # noqa: E731
                                        heads, 0.125, row_stride=3 * inner)
    flops = 4.0 * clips * hw * heads * frames * frames * 64
    nbytes = 4.0 * clips * frames * hw * inner * 2
elif which in ("ln", "ln640", "ln320"):
    rows, c = {"ln": (16384, 1280), "ln640": (65536, 640), "ln320": (131072, 320)}[which]
    xs = [rnd(rows, c) for _ in range(8)]   # 8 x 42 MB rotate through the 50 MB L2: every launch reads from HBM
    g, b = torch.ones(c, device=dev), torch.zeros(c, device=dev)
    _i = [0]

    def fn():
        _i[0] += 1
        return ops.layer_norm(xs[_i[0] % 8], g, b)
    flops = 0.0
    nbytes = 2.0 * rows * c * 2
elif which == "gn":
    x = rnd(16, 128, 128, 320)
    g, b = torch.ones(320, device=dev), torch.zeros(320, device=dev)
    fn = lambda: ops.group_norm(x, g, b, 1e-5, silu=True)  # noqa: E731
    flops = 0.0
else:
    raise SystemExit(which)

for _ in range(5):
    fn()
torch.cuda.synchronize()
if do_time:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 10
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    extra = f"  {nbytes / ms / 1e6:.0f} GB/s" if which.startswith(("tattn", "ln")) else ""
    print(f"{which}: {ms:.3f} ms  {flops / ms / 1e9:.1f} TFLOP/s{extra}")
