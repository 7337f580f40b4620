"""A/B of the fused candidate round (PB_FUSED_AGG, DESIGN.md §9) on the bench.py workloads, in one session on one GPU.

Runs `bench.py --gpus 1 --steps K --warmup W --no-e2e --no-cpu-baseline` R times under PB_FUSED_AGG=0 (filter kernel +
pb_agg_rows_kernel) and R times under the default (fused), alternating, so that drift of the shared machine falls on both
sides alike.  Prints one JSON object: per side the median, min and max of the headline ms_per_step, of the 25 %
selectivity variant and of the strong-scaling curve, the kernel times, and the clocks, GPU name and power limit each run
recorded; then the headline's median gain and whether the slowest fused run beat the fastest unfused one.
`--out FILE` also writes every run's bench.py line there (JSON lines).  Nothing is written to the tree."""
import argparse
import json
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SIDES = (("unfused", "0"), ("fused", "1"))


def run_bench(fused: str, steps: int, warmup: int) -> dict:
    env = dict(os.environ, PB_FUSED_AGG=fused)
    cmd = [sys.executable, os.path.join(HERE, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
           "--no-e2e", "--no-cpu-baseline"]
    p = subprocess.run(cmd, cwd=HERE, env=env, capture_output=True, text=True, check=True)
    return json.loads([line for line in p.stdout.splitlines() if line.startswith("{")][-1])


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "all": [round(x, 4) for x in xs]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--out", help="JSON-lines file for every run's bench.py result")
    args = ap.parse_args()
    runs = {name: [] for name, _ in SIDES}
    for _ in range(args.repeats):
        for name, val in SIDES:
            r = run_bench(val, args.steps, args.warmup)
            runs[name].append(r)
            if args.out:
                with open(args.out, "a") as f:
                    f.write(json.dumps({"side": name, **r}) + "\n")
    summary = {}
    for name, rs in runs.items():
        summary[name] = {
            "ms_per_step": spread([r["ms_per_step"] for r in rs]),
            "filter_kernel_ms": spread([r["filter_kernel_ms"] for r in rs]),
            "agg_kernel_ms": spread([r["agg_kernel_ms"] for r in rs]),
            "selectivity_25pct_ms_per_step": spread([r["selectivity_25pct"]["ms_per_step"] for r in rs]),
            "strong_ms_per_step": spread([r["strong"]["ms_per_step"] for r in rs]),
            "clocks": [{k: r["clocks"].get(k) for k in ("gpu_name", "power_limit_w", "sm_mhz", "sm_max_mhz", "reasons")} for r in rs],
        }
    u, f = summary["unfused"], summary["fused"]
    summary["headline_gain"] = 1.0 - f["ms_per_step"]["median"] / u["ms_per_step"]["median"]
    summary["slowest_fused_beats_fastest_unfused"] = f["ms_per_step"]["max"] < u["ms_per_step"]["min"]
    summary["selectivity_25pct_ratio"] = f["selectivity_25pct_ms_per_step"]["median"] / u["selectivity_25pct_ms_per_step"]["median"]
    summary["strong_ratio"] = f["strong_ms_per_step"]["median"] / u["strong_ms_per_step"]["median"]
    print(json.dumps(summary, indent=1))


if __name__ == "__main__":
    main()
