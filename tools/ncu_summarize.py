"""Aggregate an `ncu --metrics gpu__time_duration.sum --csv` launch list by kernel name -> share of the profiled window."""
import csv
import re
import sys
from collections import defaultdict

path = sys.argv[1]
rows = []
with open(path, newline="") as f:
    lines = [l for l in f if not l.startswith("==")]
rd = csv.DictReader(lines)
tot = defaultdict(float)
cnt = defaultdict(int)
for r in rd:
    if r.get("Metric Name") != "gpu__time_duration.sum":
        continue
    name = r["Kernel Name"]
    name = re.sub(r"\(.*$", "", name)
    name = re.sub(r"<.*$", "", name) if not name.startswith("dvla::gemm") and "gemm_wgmma" not in name else name
    v = float(r["Metric Value"].replace(",", ""))
    unit = r.get("Metric Unit", "ns")
    if unit in ("us", "usecond"):
        v *= 1e3
    elif unit in ("ms", "msecond"):
        v *= 1e6
    tot[name] += v
    cnt[name] += 1
total = sum(tot.values())
print(f"total {total/1e6:.3f} ms over {sum(cnt.values())} launches")
for name, t in sorted(tot.items(), key=lambda kv: -kv[1])[:40]:
    print(f"{t/1e6:9.3f} ms {100*t/total:5.1f}% n={cnt[name]:5d} avg={t/cnt[name]/1e3:8.1f} us  {name[:110]}")
