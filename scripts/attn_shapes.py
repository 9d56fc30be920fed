"""Per-shape time of the attention family in one eager step of bench.py's flagship workload (SDXL 1024^2, batch 8).
usage: python scripts/attn_shapes.py [--top N] [--json PATH]
Prints one row per distinct launch shape (the note says batch, heads, lq, lk and the padded head dim): launches,
CUDA-event ms, TFLOP/s and share of the step's event time."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import WORKLOADS, build_ours  # noqa: E402
from ctrl_adapter_b200 import ops  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--top", type=int, default=25)
    ap.add_argument("--json", default=None, help="also write every attention row here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_shapes.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.manual_seed(1234)
    loop, _ = build_ours("sdxl", WORKLOADS["sdxl"]["batch"], 1024, dev, 1234)
    loop.step(0)  # packs weights, sets kernel attributes
    loop.step(1)
    torch.cuda.synchronize()
    ops.PROFILER.start()
    loop.step(0)
    ops.PROFILER.stop()
    rows = ops.PROFILER.launches_table(top=10 ** 6)
    step_ms = sum(r["ms"] for r in rows)
    attn = [r for r in rows if r["fam"] == "attention"]
    attn_ms = sum(r["ms"] for r in attn)
    print(f"step (sum of launch events) {step_ms:.1f} ms; attention {attn_ms:.1f} ms in {sum(r['n'] for r in attn)} "
          f"launches ({100 * attn_ms / step_ms:.1f}%), {len(attn)} shapes")
    print(f"{'launches':>8} {'ms':>8} {'TFLOP/s':>8} {'share':>6}  shape")
    for r in attn[:a.top]:
        print(f"{r['n']:>8} {r['ms']:>8.3f} {r['tflops'] or 0:>8.1f} {100 * r['ms'] / step_ms:>5.1f}%  {r['note']}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"step_ms": step_ms, "attn_ms": attn_ms, "rows": attn}, f, indent=1)


if __name__ == "__main__":
    main()
