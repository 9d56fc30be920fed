"""Bytes of the GEMM's bf16 epilogues on seeded inputs, for checking that two builds of the library compute the same
bits.
usage: python scripts/gemm_epilogue_ab.py save DIR [--lib PATH]   (PATH: a libctrl_adapter_b200.so, default in-tree)
       python scripts/gemm_epilogue_ab.py compare DIR_A DIR_B
Cases: prof_kernels.py's lin_res, lin_small (each with and without residual), conv and geglu; a scale-0.5 conv with and
without residual; a conv with a row vector, with and without residual; a SiLU linear with and without scale; an
AlphaBlender linear; a linear without bias at each BN."""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def cases(ops, torch):
    dev = "cuda"
    bf16 = torch.bfloat16
    g = torch.Generator(device=dev)

    def rnd(*s, scale=1.0, seed):
        g.manual_seed(seed)
        return (torch.randn(*s, generator=g, device=dev) * scale).to(bf16)

    def bias(n, seed):  # fp32 biases that are not bf16-valued
        g.manual_seed(seed)
        return torch.randn(n, generator=g, device=dev)

    x1, w1, b1, r1 = rnd(16384, 1280, seed=1), rnd(1280, 1280, scale=1 / math.sqrt(1280), seed=2), bias(1280, 3), \
        rnd(16384, 1280, seed=4)
    x2, w2, b2, r2 = rnd(65536, 640, seed=5), rnd(640, 640, scale=1 / math.sqrt(640), seed=6), bias(640, 7), \
        rnd(65536, 640, seed=8)
    wg, bg = rnd(10240, 1280, scale=1 / math.sqrt(1280), seed=9), bias(10240, 10)
    xc, bc, rc = rnd(16, 128, 128, 320, seed=11), bias(320, 13), rnd(16, 128, 128, 320, seed=14)
    wc = ops.pack_conv_weight(rnd(320, 320, 3, 3, scale=1 / math.sqrt(2880), seed=12))
    alpha = torch.sigmoid(torch.tensor([0.3], device=dev)).to(bf16).float()
    yield "lin_res", lambda: ops.linear(x1, w1, b1, residual=r1)
    yield "lin_res_nores", lambda: ops.linear(x1, w1, b1)
    yield "lin_small", lambda: ops.linear(x2, w2, b2, residual=r2)
    yield "lin_small_nores", lambda: ops.linear(x2, w2, b2)
    yield "conv", lambda: ops.conv2d(xc, wc, bc)
    yield "geglu", lambda: ops.linear(x1, wg, bg, act=ops.ACT_GEGLU, bn=256)
    yield "conv_scale05_res", lambda: ops.conv2d(xc, wc, bc, residual=rc, out_scale=0.5)
    yield "conv_scale05", lambda: ops.conv2d(xc, wc, None, out_scale=0.5)
    yield "lin_silu", lambda: ops.linear(x2, w2, b2, act=ops.ACT_SILU)
    yield "lin_silu_scale05", lambda: ops.linear(x2, w2, b2, act=ops.ACT_SILU, out_scale=0.5)
    rv = rnd(16, 320, seed=15)
    yield "conv_rowvec", lambda: ops.conv2d(xc, wc, bc, rowvec=rv)
    yield "conv_rowvec_res", lambda: ops.conv2d(xc, wc, bc, rowvec=rv, residual=rc)
    yield "lin_blend", lambda: ops.linear(x2, w2, b2, residual=r2, blend_src=x2, blend_alpha=alpha)
    for bn in (64, 128, 160, 256):
        yield f"lin_nobias_bn{bn}", lambda bn=bn: ops.linear(x2[:50001], w2[:600], None, bn=bn)


def main():
    if sys.argv[1] == "compare":
        a, b = sys.argv[2], sys.argv[3]
        names = sorted(f for f in os.listdir(a) if f.endswith(".npy"))
        bad = [f for f in names if not np.array_equal(np.load(os.path.join(a, f)), np.load(os.path.join(b, f)))]
        for f in names:
            print(f"{f[:-4]}: {'DIFFERENT' if f in bad else 'identical'}")
        sys.exit(1 if bad or not names else 0)
    out_dir = sys.argv[2]
    if "--lib" in sys.argv:
        from ctrl_adapter_b200 import _lib
        _lib.LIB_PATH = os.path.abspath(sys.argv[sys.argv.index("--lib") + 1])
    import torch
    from ctrl_adapter_b200 import ops
    if not torch.cuda.is_available():
        raise SystemExit("gemm_epilogue_ab.py save needs a CUDA device")
    os.makedirs(out_dir, exist_ok=True)
    for name, fn in cases(ops, torch):
        y = fn()
        torch.cuda.synchronize()
        np.save(os.path.join(out_dir, name + ".npy"), y.view(torch.int16).cpu().numpy())


if __name__ == "__main__":
    main()
