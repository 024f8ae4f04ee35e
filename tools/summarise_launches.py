"""Per-kernel totals of an `ncu --metrics gpu__time_duration.sum --csv` launch list.

usage: python tools/summarise_launches.py final_launches.csv [last_n_launches | step:K] > summary.csv
With last_n_launches the summary covers only the tail of the list; with `step:K` (e.g. step:-3) it
covers exactly one train step: the launches between the K-th and (K+1)-th optimizer kernel
(`k_sgd_momentum`) of the run — bench.py's tail is the roofline replay, not a step.
"""
import csv
import sys
from collections import defaultdict


def main():
    path = sys.argv[1]
    arg = sys.argv[2] if len(sys.argv) > 2 else "0"
    step = int(arg.split(":")[1]) if arg.startswith("step:") else None
    last = 0 if step is not None else int(arg)
    rows = []
    with open(path, newline="") as f:
        lines = [l for l in f if l.startswith('"')]
    for r in csv.DictReader(lines):
        if r.get("Metric Name") == "gpu__time_duration.sum":
            rows.append((r["Kernel Name"], float(r["Metric Value"].replace(",", "")) / 1e3))
    if step is not None:
        marks = [i for i, (k, _) in enumerate(rows) if "k_sgd_momentum" in k]
        rows = rows[marks[step] + 1:marks[step + 1] + 1]
    if last:
        rows = rows[-last:]
    tot = defaultdict(float)
    cnt = defaultdict(int)
    for k, us in rows:
        k = k[:110]
        tot[k] += us
        cnt[k] += 1
    total = sum(tot.values())
    edb = sum(v for k, v in tot.items() if "edb::" in k)
    print(f"# {path}: {len(rows)} launches, {total / 1e3:.2f} ms of kernel time (cold-cache, serialised under ncu); "
          f"edb:: kernels {edb / total:.3f} of it")
    print("kernel,launches,total_us,avg_us,share")
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1]):
        print(f'"{k}",{cnt[k]},{v:.1f},{v / cnt[k]:.2f},{v / total:.4f}')


if __name__ == "__main__":
    main()
