"""Aggregate an `ncu --csv` launch list of one benchmark step into per-kernel-family time, share, DRAM bytes and the
TIME-WEIGHTED tensor-pipe activity of the whole step (VERDICT r1 item 4: the north_star's ">= 40 % tensor pipe" answered
directly instead of through a FLOP fraction).

    ncu --metrics gpu__time_duration.sum,sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed,dram__bytes_read.sum,dram__bytes_write.sum \
        --clock-control none --csv --log-file step_metrics.csv \
        python bench.py --steps 1 --warmup 1 --no-e2e --no-cpu-baseline --no-gpu-baseline
    python tools/step_profile.py step_metrics.csv [--md step_profile.md]

The LAST step is the run of launches between the last two `adamw_multi_kernel` launches.  ncu serialises the launches
and runs each cold at the unthrottled clock: compare shares, not absolutes, with bench.py's live numbers."""
import argparse
import csv
import io
import json
import re
import sys
from collections import OrderedDict, defaultdict


def read_launches(path):
    text = open(path, errors="replace").read()
    start = text.find('"ID"')
    rows = csv.DictReader(io.StringIO(text[start:]))
    launches = OrderedDict()
    for r in rows:
        try:
            lid = int(r["ID"])
        except (KeyError, ValueError, TypeError):
            continue
        ent = launches.setdefault(lid, {"name": r["Kernel Name"], "m": {}})
        try:
            v = float(r["Metric Value"].replace(",", ""))
        except ValueError:
            continue
        unit = r.get("Metric Unit", "")
        name = r["Metric Name"]
        if name == "gpu__time_duration.sum":
            v *= {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3, "nsecond": 1e-6, "usecond": 1e-3, "msecond": 1.0,
                  "second": 1e3}.get(unit, 1e-6)
        if name.startswith("dram__bytes"):
            v *= {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "B": 1.0, "KB": 1e3, "MB": 1e6, "GB": 1e9}.get(unit, 1.0)
        ent["m"][name] = v
    return list(launches.values())


def family(name):
    name = re.sub(r"^void ", "", name)
    name = re.sub(r"\(.*$", "", name)
    name = re.sub(r"egovlp::\(anonymous namespace\)::|egovlp::<unnamed>::|egovlp::", "", name)
    return name[:90]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("--md", default="")
    ap.add_argument("--json", default="")
    ap.add_argument("--marker", default="adamw_multi_kernel")
    a = ap.parse_args()
    L = read_launches(a.csv)
    marks = [i for i, l in enumerate(L) if a.marker in l["name"]]
    step = L[marks[-2] + 1: marks[-1] + 1] if len(marks) >= 2 else L
    fam = defaultdict(lambda: {"n": 0, "ms": 0.0, "tensor_ms": 0.0, "dram": 0.0})
    T = "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed"
    for l in step:
        m = l["m"]
        ms = m.get("gpu__time_duration.sum", 0.0)
        f = fam[family(l["name"])]
        f["n"] += 1
        f["ms"] += ms
        f["tensor_ms"] += ms * m.get(T, 0.0) / 100.0
        f["dram"] += m.get("dram__bytes_read.sum", 0.0) + m.get("dram__bytes_write.sum", 0.0)
    total = sum(f["ms"] for f in fam.values())
    tens = sum(f["tensor_ms"] for f in fam.values())
    out = {"launches": len(step), "kernel_ms": total, "tensor_pipe_active_pct_time_weighted": 100.0 * tens / total if total else None,
           "dram_gb": sum(f["dram"] for f in fam.values()) / 1e9,
           "families": [{"kernel": k, "launches": f["n"], "ms": f["ms"], "share": f["ms"] / total,
                         "tensor_pipe_pct": 100.0 * f["tensor_ms"] / f["ms"] if f["ms"] else 0.0,
                         "dram_gb": f["dram"] / 1e9, "dram_gbs": f["dram"] / f["ms"] / 1e6 if f["ms"] else 0.0}
                        for k, f in sorted(fam.items(), key=lambda kv: -kv[1]["ms"])]}
    lines = [f"launches {out['launches']}, kernel time {total:.2f} ms, time-weighted tensor-pipe activity "
             f"{out['tensor_pipe_active_pct_time_weighted']:.1f} %, DRAM traffic {out['dram_gb']:.1f} GB", "",
             "| kernel | launches | ms | share | tensor pipe % | DRAM GB | DRAM GB/s |", "|---|---:|---:|---:|---:|---:|---:|"]
    for f in out["families"]:
        if f["ms"] / total < 0.001:
            continue
        lines.append(f"| `{f['kernel']}` | {f['launches']} | {f['ms']:.2f} | {100 * f['share']:.1f}% | {f['tensor_pipe_pct']:.1f} | "
                     f"{f['dram_gb']:.2f} | {f['dram_gbs']:.0f} |")
    print("\n".join(lines))
    if a.md:
        open(a.md, "w").write("\n".join(lines) + "\n")
    if a.json:
        json.dump(out, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    sys.exit(main())
