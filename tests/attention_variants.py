"""Wrong attention variants for the direction tests (tests/test_error_bias_cpu.py, tests/test_error_bias_gpu.py):
flash-style attention whose unnormalised probabilities come from a replaceable function, with the probabilities
truncated to bf16 or exp2 from a short polynomial.  Test infrastructure, never imported by the product."""
import math

import numpy as np
import torch

BF16 = torch.bfloat16


def trunc_bf16(t):
    """fp32 -> bf16 rounded toward zero (the low 16 bits dropped)"""
    return (t.float().contiguous().view(torch.int32) & -65536).view(torch.float32).to(BF16)


def flash(p_of, q, k, v, heads, head_dim_pad, scale, out=None, kv_batch_div=1):
    """ops.attention's arguments; the probabilities p = p_of(score - row max) (unnormalised), normalised by their fp32
    sum"""
    b, lq, _ = q.shape
    qh = q.float().reshape(b, lq, heads, head_dim_pad).permute(0, 2, 1, 3)
    kb = torch.arange(b, device=q.device) // kv_batch_div
    kh = k.float().reshape(k.shape[0], -1, heads, head_dim_pad).permute(0, 2, 1, 3)[kb]
    vh = v.float().reshape(v.shape[0], -1, heads, head_dim_pad).permute(0, 2, 1, 3)[kb]
    s = qh @ kh.transpose(-1, -2) * scale
    p, l = p_of(s - s.amax(dim=-1, keepdim=True))
    y = ((p @ vh) / l).permute(0, 2, 1, 3).reshape(b, lq, heads * head_dim_pad).to(BF16)
    if out is None:
        return y
    out.copy_(y)
    return out


def p_trunc(z):
    """P truncated to bf16 before P.V, the sum taken of the unrounded P"""
    p = torch.exp(z)
    return trunc_bf16(p).float(), p.sum(dim=-1, keepdim=True)


def poly2_exp2():
    """exp via 2^f on [0, 1) by the least-squares quadratic: relative error up to ~2e-3, a function of the fraction"""
    f = np.linspace(0.0, 1.0, 4097)
    c = np.polyfit(f, np.exp2(f), 2)

    def p_of(z):
        t = z * math.log2(math.e)
        i = torch.floor(t)
        fr = t - i
        p = torch.ldexp(c[0] * fr * fr + c[1] * fr + c[2], i.to(torch.int32))
        return p, p.sum(dim=-1, keepdim=True)
    return p_of
