"""Cost and reproducibility of the deterministic mode (torch.use_deterministic_algorithms(True)) on bench.py's workloads.

    python tools/bench_deterministic.py [--pairs 2] [--cfg2-pairs 1] [--steps 8] [--warmup 3] [--parent DIR]
                                        [--out DIR]
    python tools/bench_deterministic.py --profile     (where the flag's time goes: torch.profiler, kernel time)

Runs bench.py's own main (runpy, --no-cpu-baseline --no-gpu-baseline --no-e2e --dump-outputs) in a fresh process per
run, alternating flag-off and flag-on runs (CUBLAS_WORKSPACE_CONFIG=:4096:8 for the flagged ones), cfg3 `--pairs`
times and cfg2 `--cfg2-pairs` times.  --parent DIR: a built checkout of another revision; its flag-off run joins each
cfg3 pair, so the default path's rate is compared with that build's in the same alternation.  Reports clips/s, peak
allocated memory, the card, its power limit and the median SM clock, and checks:
  * the output dumps of the flagged runs are byte-identical;
  * flag-off runs differ from the flagged ones by no more than they differ from each other;
  * the flag-off rate matches the parent build's within the spread of the alternated runs (with --parent).
Prints one JSON line; exits non-zero if a check fails."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

RUNNER = r"""
import contextlib, json, os, runpy, sys, torch
det = sys.argv[1] == "1"
root = sys.argv[2]
sys.path.insert(0, root)
torch.use_deterministic_algorithms(det)
sys.argv = ["bench.py"] + sys.argv[3:]
prof_path = os.environ.get("EGOVLP_DET_PROFILE")
prof = (torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) if prof_path
        else contextlib.nullcontext())
try:
    with prof:
        runpy.run_path(root + "/bench.py", run_name="__main__")
finally:
    print(json.dumps({"peak_allocated_bytes": torch.cuda.max_memory_allocated()}), flush=True)
if prof_path:
    kern = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            k = kern.setdefault(e.name, [0.0, 0])
            k[0] += e.device_time_total / 1e3
            k[1] += 1
    json.dump(kern, open(prof_path, "w"))
"""

# kernel-name substrings -> the part of the step they belong to (for the --profile breakdown)
CATEGORIES = [("torch fill (NaN fill of torch.empty under the flag, zero fills)", ("fill", "Fill")),
              ("GEMM deterministic merge", ("gemm_det_merge",)),
              ("ordered merge of per-CTA partials", ("ordered_sum",)),
              ("GEMM", ("gemm_bf16_wgmma", "gemm_drop_wgmma")),
              ("attention", ("attn", "cls_grad", "cls_merge")),
              ("LayerNorm / column sums", ("layernorm", "colsum")),
              ("text embedding", ("text_embed",)),
              ("sort (text ids)", ("sort", "Sort", "radix", "Radix"))]


def categorise(kern):
    out = {}
    for name, (ms, n) in kern.items():
        cat = next((c for c, keys in CATEGORIES if any(k in name for k in keys)), "other")
        o = out.setdefault(cat, [0.0, 0])
        o[0] += ms
        o[1] += n
    return out


def profile(args, tmp):
    """One profiled cfg3 run with the flag off and one with it on (bench.py --steps 2 --warmup 1, all three steps in
    the trace): kernel time per category and the kernels whose time grew most, per step."""
    res = {}
    for det in (False, True):
        path = os.path.join(tmp, f"profile_{int(det)}.json")
        os.environ["EGOVLP_DET_PROFILE"] = path
        a = argparse.Namespace(steps=2, warmup=1)
        run(ROOT, det, "cfg3", a, os.path.join(tmp, f"profile_dump_{int(det)}"))
        res[det] = json.load(open(path))
    del os.environ["EGOVLP_DET_PROFILE"]
    steps = 3
    cat = {d: categorise(res[d]) for d in res}
    names = set(res[False]) | set(res[True])
    grew = sorted(((res[True].get(n, [0, 0])[0] - res[False].get(n, [0, 0])[0]) / steps, n) for n in names)[::-1][:12]
    return {"ms_per_step_by_category": {c: {"off": cat[False].get(c, [0, 0])[0] / steps,
                                            "det": cat[True].get(c, [0, 0])[0] / steps,
                                            "launches_det": cat[True].get(c, [0, 0])[1] / steps}
                                        for c in sorted(set(cat[False]) | set(cat[True]))},
            "kernel_ms_per_step": {"off": sum(v[0] for v in res[False].values()) / steps,
                                   "det": sum(v[0] for v in res[True].values()) / steps},
            "largest_increases_ms_per_step": [(n[:120], round(d, 3)) for d, n in grew]}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run(root, det, workload, args, dump):
    env = dict(os.environ)
    if det:
        env["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"
    cmd = [sys.executable, "-c", RUNNER, "1" if det else "0", root, "--gpus", "1", "--workload", workload,
           "--steps", str(args.steps), "--warmup", str(args.warmup), "--no-cpu-baseline", "--no-gpu-baseline",
           "--no-e2e", "--dump-outputs", dump]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=root)
    lines = [json.loads(s) for s in r.stdout.splitlines() if s.startswith("{")]
    if r.returncode or len(lines) < 2:
        raise RuntimeError(f"bench run failed ({root}, det={det}, {workload}):\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
    line, mem = lines[-2], lines[-1]
    clocks = line.get("clocks") or {}
    return {"det": det, "workload": workload, "root": root, "clips_per_s": line["value"],
            "peak_allocated_gb": mem["peak_allocated_bytes"] / 1e9, "loss": line.get("loss"),
            "sm_clock_median_mhz": clocks.get("sm_mhz"), "dump": dump}


def load(dump):
    return {f: np.load(os.path.join(dump, f)) for f in sorted(os.listdir(dump))}


def max_diff(a, b):
    return max(float(np.max(np.abs(a[k].astype(np.float64) - b[k].astype(np.float64)))) for k in a)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=2)
    ap.add_argument("--cfg2-pairs", type=int, default=1)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--parent", default=None, help="a built checkout of the revision to compare the default path with")
    ap.add_argument("--out", default=None, help="directory for the dumps (default: a temporary one)")
    ap.add_argument("--profile", action="store_true", help="only the kernel-time breakdown of one cfg3 step, off vs on")
    args = ap.parse_args()
    if args.parent:
        args.parent = os.path.abspath(args.parent)
    tmp = args.out or tempfile.mkdtemp(prefix="egovlp_det_bench_")
    if args.profile:
        print(json.dumps({"card": card(), "profile": profile(args, tmp)}), flush=True)
        return
    runs, checks = [], {}
    for workload, pairs in (("cfg3", args.pairs), ("cfg2", args.cfg2_pairs)):
        if pairs < 1:
            continue
        for i in range(pairs):
            for det in (False, True):
                runs.append(run(ROOT, det, workload, args, os.path.join(tmp, f"{workload}_{i}_{int(det)}")))
            if args.parent and workload == "cfg3":
                runs.append(dict(run(args.parent, False, workload, args, os.path.join(tmp, f"{workload}_{i}_parent")),
                                 parent=True))
        mine = [r for r in runs if r["workload"] == workload and not r.get("parent")]
        on = [load(r["dump"]) for r in mine if r["det"]]
        off = [load(r["dump"]) for r in mine if not r["det"]]
        same = all(all(np.array_equal(d[k], on[0][k]) and d[k].tobytes() == on[0][k].tobytes() for k in d)
                   for d in on[1:])
        off_spread = max([max_diff(a, b) for a in off for b in off if a is not b] or [0.0])
        off_vs_on = max(max_diff(a, on[0]) for a in off)
        checks[workload] = {"det_dumps_identical": same if len(on) > 1 else None, "default_vs_default_max_diff": off_spread,
                            "default_vs_det_max_diff": off_vs_on,
                            "default_vs_det_within_default_spread": off_vs_on <= off_spread if len(off) > 1 else None}
        rate = {k: [r["clips_per_s"] for r in runs if r["workload"] == workload and r["det"] == d
                    and bool(r.get("parent")) == p] for k, d, p in (("off", False, False), ("det", True, False),
                                                                    ("parent", False, True))}
        checks[workload]["clips_per_s"] = {k: v for k, v in rate.items() if v}
        checks[workload]["det_cost"] = 1 - statistics.median(rate["det"]) / statistics.median(rate["off"])
        if rate["parent"]:
            spread = max(rate["off"] + rate["parent"]) - min(rate["off"] + rate["parent"])
            gap = statistics.median(rate["parent"]) - statistics.median(rate["off"])
            checks[workload]["default_vs_parent"] = {"gap": gap, "spread": spread, "within_spread": gap <= spread}
    ok = all(c["det_dumps_identical"] is not False and c["default_vs_det_within_default_spread"] is not False
             and c.get("default_vs_parent", {}).get("within_spread", True) for c in checks.values())
    print(json.dumps({"card": card(), "runs": [{k: v for k, v in r.items() if k != "dump"} for r in runs],
                      "checks": checks, "ok": ok}), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
