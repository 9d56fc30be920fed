"""Wall time and peak memory of ``vae.encode`` (the conditioning image of the two video pipelines, run once per call) on
our kernels vs the restated diffusers encoder run eagerly in bf16 autocast, in the same process.

    python scripts/encode_timing.py [--iters 10] [--json out.json]

Cases: one 704x1280 image through AutoencoderKL (I2VGen-XL's default size) and one 576x1024 image through
AutoencoderKLTemporalDecoder (SVD's).  Both encoders get the same name-seeded weights.  Times are CUDA events around
``iters`` calls after two warm-up calls; peak memory is torch.cuda.max_memory_allocated over one call minus what was
allocated before it.  The card's name, power limit and max SM clock are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BF16 = torch.bfloat16


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        q = f"unknown ({e})"
    return q


def _time(fn, iters):
    fn(); fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from ctrl_adapter_b200 import vae
    from oracle import vae_encoder as ov
    from oracle.weights import seeded_init_, seeded_tensor
    torch.backends.cuda.matmul.allow_tf32 = False
    rows = []
    for name, ours_cls, ref_cls, h, w in (("AutoencoderKL 1x704x1280", vae.AutoencoderKL, ov.AutoencoderKL, 704, 1280),
                                          ("AutoencoderKLTemporalDecoder 1x576x1024", vae.AutoencoderKLTemporalDecoder,
                                           ov.AutoencoderKLTemporalDecoder, 576, 1024)):
        with torch.device("cuda"):
            ref = ref_cls()
        ref = seeded_init_(ref.cuda(), 16).to(BF16).eval()
        with torch.device("cuda"):
            ours = ours_cls()
        ours.load_state_dict(ref.state_dict())
        ours = ours.to(BF16).eval()
        x = torch.tanh(seeded_tensor("timing_x", (1, 3, h, w))).to(BF16).cuda()

        def run_ours():
            return ours.encode(x).latent_dist.mode()

        def run_ref():
            with torch.no_grad(), torch.autocast("cuda", dtype=BF16):
                return ref.encode(x)[0].mode()
        a, b = run_ours().float(), run_ref().float()
        rel = float((a - b).norm() / b.norm())
        row = {"case": name, "ours_ms": round(_time(run_ours, args.iters), 2),
               "eager_bf16_ms": round(_time(run_ref, args.iters), 2),
               "ours_peak_mib": round(_peak(run_ours), 1), "eager_bf16_peak_mib": round(_peak(run_ref), 1),
               "rel_fro_ours_vs_eager": round(rel, 5)}
        print(json.dumps(row))
        rows.append(row)
        del ref, ours
        torch.cuda.empty_cache()
    res = {"card": _card(), "iters": args.iters, "rows": rows}
    print(json.dumps(res))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
