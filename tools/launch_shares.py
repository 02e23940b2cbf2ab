"""Per-kernel shares of one mastering step from an ncu launch list (CSV of gpu__time_duration.sum) next
to the bench line's CUDA-event figures.  usage: python tools/launch_shares.py launches.csv bench.json [steps]"""
import csv
import json
import sys
from collections import defaultdict

PIPELINE = ("analyze_kernel", "spectrum_mean_kernel", "smooth_operator_kernel", "design_kernel", "convolve",
            "loud_sumsq_kernel", "correction_final_kernel", "limiter_kernel")

steps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
rows = [r for r in csv.reader(l for l in open(sys.argv[1]) if l.startswith('"'))]
hdr = rows[0]
name_i, val_i = hdr.index("Kernel Name"), hdr.index("Metric Value")
tot = defaultdict(float)
cnt = defaultdict(int)
for r in rows[1:]:
    short = next((k for k in PIPELINE if k in r[name_i]), None)
    if short is None:
        continue
    key = "convolve_kernel" if short == "convolve" else short
    tot[key] += float(r[val_i]) / 1e3
    cnt[key] += 1
# plan building launches design kernels too: keep the last `steps` steps' worth by count ratio
bench = json.loads(open(sys.argv[2]).read().strip().splitlines()[-1])
kern = bench["kernels"]
ncu_step = {k: tot[k] / cnt[k] * kern[k]["launches_per_step"] for k in kern if cnt.get(k)}
ncu_sum = sum(ncu_step.values())
ev_sum = sum(v["ms_per_step"] for v in kern.values()) * 1e3
print(f"{'kernel':26s} {'launches':>8s} {'events us':>10s} {'share':>7s} {'ncu us':>8s} {'share':>7s}")
for k, v in sorted(kern.items(), key=lambda kv: -kv[1]["ms_per_step"]):
    ev = v["ms_per_step"] * 1e3
    print(f"{k:26s} {v['launches_per_step']:8.0f} {ev:10.1f} {100 * ev / ev_sum:6.1f}% {ncu_step.get(k, 0):8.1f} "
          f"{100 * ncu_step.get(k, 0) / ncu_sum:6.1f}%")
print(f"{'sum':26s} {'':8s} {ev_sum:10.1f} {'':7s} {ncu_sum:8.1f}")
