"""Summarise an ncu launch list (--metrics gpu__time_duration.sum --csv): per-kernel totals and shares.
    python tools/launch_summary.py out/r01_launches.csv [--top 25] [--by-grid]
"""
import argparse
import csv
import io
import re
from collections import defaultdict


def load(path):
    txt = open(path, errors="replace").read()
    start = txt.find('"ID"')
    if start < 0:
        raise SystemExit("no CSV header found in " + path)
    rows = list(csv.DictReader(io.StringIO(txt[start:])))
    out = []
    for r in rows:
        if r.get("Metric Name") != "gpu__time_duration.sum":
            continue
        val = float(r["Metric Value"].replace(",", ""))
        unit = r.get("Metric Unit", "ns")
        ns = val * {"ns": 1, "us": 1e3, "ms": 1e6, "s": 1e9, "nsecond": 1, "usecond": 1e3, "msecond": 1e6}.get(unit, 1)
        name = r["Kernel Name"]
        name = re.sub(r"^void ", "", name)
        name = re.sub(r"\(.*$", "", name)
        name = name.replace("mgb::", "")
        out.append((name, r.get("Grid Size", ""), r.get("Block Size", ""), ns))
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("--top", type=int, default=30)
    ap.add_argument("--by-grid", action="store_true")
    ap.add_argument("--last-step", action="store_true", help="only the launches from the last select_step_kernel on")
    a = ap.parse_args()
    rows = load(a.csv)
    if a.last_step:
        idx = [i for i, r in enumerate(rows) if r[0].startswith("select_step_kernel")]
        if idx:
            rows = rows[idx[-1]:]
    tot = sum(r[3] for r in rows)
    agg = defaultdict(lambda: [0, 0.0])
    for name, grid, block, ns in rows:
        key = (name, grid) if a.by_grid else (name,)
        agg[key][0] += 1
        agg[key][1] += ns
    print(f"{len(rows)} launches, {tot / 1e6:.3f} ms total device time (serialised, cold-cache)")
    for key, (n, ns) in sorted(agg.items(), key=lambda kv: -kv[1][1])[: a.top]:
        print(f"{ns / 1e3:10.1f} us  {100 * ns / tot:5.1f}%  n={n:4d}  avg={ns / n / 1e3:8.1f} us  {' '.join(key)}")
