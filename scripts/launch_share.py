"""Aggregates an ncu launch list (`--metrics gpu__time_duration.sum[,dram__bytes_read.sum,dram__bytes_write.sum] --csv`)
per kernel: launches, total time, share and (when captured) average DRAM bytes per launch.
usage: python scripts/launch_share.py launches.csv [skip_launches] [traffic.json] > launch_shares.md
The optional third argument writes {kernel base name: {"launches", "dram_bytes_per_launch"}}.

The per-launch times of such a pass are cold-cache and serialised, so only the SHARE of each kernel is meaningful; the
absolute step time comes from bench.py's CUDA events."""
import csv
import re
import sys
from collections import defaultdict


def short(name):
    name = re.sub(r"^void ", "", name)
    name = re.sub(r"\(.*$", "", name)
    return name if len(name) < 110 else name[:107] + "..."


def main():
    import json
    path = sys.argv[1]
    skip = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    with open(path, newline="") as f:
        lines = [ln for ln in f if ln.startswith('"')]
    rd = csv.reader(lines)
    hdr = next(rd)
    i_name, i_metric, i_val, i_id, i_unit = (hdr.index(k) for k in ("Kernel Name", "Metric Name", "Metric Value", "ID",
                                                                     "Metric Unit"))
    scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1.0, "us": 1e3, "ms": 1e6, "nsecond": 1.0,
             "usecond": 1e3, "msecond": 1e6, "second": 1e9}
    agg = defaultdict(lambda: [0, 0.0, 0.0])  # launches, ns, dram bytes
    n_rows = 0
    for r in rd:
        if int(r[i_id]) < skip:
            continue
        name = short(r[i_name])
        val = float(r[i_val].replace(",", "")) * scale.get(r[i_unit], 1.0)
        if r[i_metric] == "gpu__time_duration.sum":
            agg[name][0] += 1
            agg[name][1] += val
            n_rows += 1
        elif r[i_metric] in ("dram__bytes_read.sum", "dram__bytes_write.sum"):
            agg[name][2] += val
    total = sum(v[1] for v in agg.values())
    print(f"source: `{path}` -- {n_rows} launches, {total / 1e6:.2f} ms summed (serialised, cold cache)\n")
    print("| kernel | launches | total ms | share | avg DRAM MB / launch |")
    print("|---|---:|---:|---:|---:|")
    for n, (c, ns, by) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"| `{n}` | {c} | {ns / 1e6:.3f} | {100 * ns / total:.1f}% | {by / c / 1e6:.2f} |")
    if len(sys.argv) > 3:
        out = {}
        for n, (c, ns, by) in agg.items():
            base = re.sub(r"<.*$", "", n).split("::")[-1]
            o = out.setdefault(base, {"launches": 0, "dram_bytes": 0.0, "ns": 0.0})
            o["launches"] += c
            o["dram_bytes"] += by
            o["ns"] += ns
        for o in out.values():
            o["dram_bytes_per_launch"] = o["dram_bytes"] / o["launches"]
        json.dump(out, open(sys.argv[3], "w"), indent=1)


if __name__ == "__main__":
    main()
