"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list: the LAST learner step in the file
(from the last k_tree_sample launch to the launch before the next one / end), kernels grouped by name.
    python tools/summarize_launches.py launches.csv [title] > launches_step.txt"""
import csv
import re
import sys

rows = []
with open(sys.argv[1], newline="") as f:
    lines = [ln for ln in f if ln.startswith('"')]
for r in csv.DictReader(lines):
    if r.get("Metric Name") != "gpu__time_duration.sum":
        continue
    v = float(r["Metric Value"].replace(",", ""))
    unit = r["Metric Unit"]
    us = v / 1e3 if unit in ("nsecond", "ns") else v if unit in ("usecond", "us") else v * 1e3
    rows.append((r["Kernel Name"], us))
starts = [i for i, (k, _) in enumerate(rows) if "k_tree_sample" in k]
if len(starts) >= 2:
    step = rows[starts[-2]:starts[-1]]
elif starts:
    step = rows[starts[-1]:]
else:
    step = rows


def short(name):
    name = re.sub(r"^void ", "", name)
    name = re.sub(r"\(.*$", "", name)
    name = name.replace("b2rl::", "")
    return name[:100]


agg = {}
for k, us in step:
    a = agg.setdefault(short(k), [0.0, 0])
    a[0] += us; a[1] += 1
tot = sum(a[0] for a in agg.values())
mine = sum(a[0] for k, a in agg.items() if not (k.startswith("at::") or "cutlass" in k or "cudnn" in k or "Nhwc" in k
                                                 or "nhwc" in k or "convertTensor" in k or k.startswith("Memset")))
print(f"# {sys.argv[2] if len(sys.argv) > 2 else ''}")
print(f"# kernels in step: {len(step)}   sum of durations: {tot:.1f} us   libb2rl share: {100 * mine / tot:.1f} %")
print("# (per-launch times under ncu are cold-cache and serialised: compare SHARES; in the graph the forward passes overlap)\n")
print("time_us  share%  launches  kernel")
for k, (us, n) in sorted(agg.items(), key=lambda kv: -kv[1][0]):
    print(f"{us:8.1f} {100 * us / tot:6.1f} {n:9d}  {k}")
