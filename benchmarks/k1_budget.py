"""Price what a cfg2 confusion-matrix update (K1, `[65536, 1000]` bf16) loses above the HBM read stream.

Builds `metrics_b200/csrc/tools/k1_budget.cu` in a temporary directory, runs it on cuda:0 and splits the update's step
time into
  (a) the steady-state read of one 131 MB batch: slope of a read-only probe over 1, 2, 4 and 8 batches in one launch each;
  (b) the rest of one launch: drain, ramp-up and SM skew, of which the part the hardware block scheduler can remove is
      the gain of the best multi-wave grid (`k1_rpwN`, N rows per warp) over a one-wave grid-stride grid;
  (c) the `[C, C]` state's HBM round trips: the one-wave step minus the one-wave step whose REDs all land in 8 KB.
`k1` is the update as shipped, beside them.  `rows_C{C}_N{N}` price one resident wave against one row per warp for other row
sizes (the threshold of `vec_grid` in csrc/confmat.cu).
Variants alternate and repeat; min and median of each go to `<out>/k1_budget.json` with the card's name, power limit and
SM clock.

    python benchmarks/k1_budget.py --out DIR [--reps 7] [--steps 1000]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "metrics_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def card() -> dict:
    import pynvml as nv

    nv.nvmlInit()
    try:
        h = nv.nvmlDeviceGetHandleByIndex(0)
        name = nv.nvmlDeviceGetName(h)
        return {
            "name": name.decode() if isinstance(name, bytes) else name,
            "power_limit_w": nv.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0,
            "sm_clock_mhz": nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM),
            "max_sm_clock_mhz": nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM),
        }
    finally:
        nv.nvmlShutdown()


def build(tmp: str) -> str:
    exe = os.path.join(tmp, "k1_budget")
    cmd = [NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr",
           "-o", exe, os.path.join(CSRC, "tools", "k1_budget.cu"), os.path.join(CSRC, "core.cu")]
    subprocess.run(cmd, check=True)
    return exe


def fit(xs, ys):
    """least-squares line y = slope * x + intercept"""
    mx, my = statistics.fmean(xs), statistics.fmean(ys)
    slope = sum((x - mx) * (y - my) for x, y in zip(xs, ys)) / sum((x - mx) ** 2 for x in xs)
    return slope, my - slope * mx


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="directory for k1_budget.json")
    ap.add_argument("--reps", type=int, default=7, help="repetitions of every variant (alternating)")
    ap.add_argument("--steps", type=int, default=1000, help="back-to-back updates per K1 sample")
    args = ap.parse_args()

    with tempfile.TemporaryDirectory() as tmp:
        exe = build(tmp)
        before = card()
        proc = subprocess.run([exe, str(args.reps), str(args.steps)], check=True, capture_output=True, text=True)
        after = card()
    raw = json.loads(proc.stdout.strip().splitlines()[-1])
    stats = {k: {"min_us": min(v), "median_us": statistics.median(v), "samples_us": v} for k, v in raw["series"].items()}

    mults = [1, 2, 4, 8]
    slope, intercept = fit(mults, [stats[f"probe_x{m}"]["median_us"] for m in mults])
    wave = stats["k1_one_wave"]["median_us"]
    rpw = {k: s for k, s in stats.items() if k.startswith("k1_rpw")}
    best = min(rpw, key=lambda k: rpw[k]["median_us"])
    c = wave - stats["k1_state8k"]["median_us"]
    budget = {
        "a_read_us_per_batch": slope,
        "read_ceiling_tbs": raw["batch_bytes"] / slope / 1e6,
        "probe_launch_fixed_us": intercept,
        "one_wave_us_per_step": wave,
        "one_wave_above_read_us": wave - slope,
        "c_state_round_trips_us": c,
        "b_launch_fixed_us": wave - slope - c,
        "b_sm_skew_removed_us": wave - rpw[best]["median_us"],
        "best_multi_wave": best,
        "shipped_us_per_step": stats["k1"]["median_us"],
    }
    sweep = {k[: -len("_wave")]: {"wave_us": s["median_us"], "rpw1_us": stats[k[: -len("_wave")] + "_rpw1"]["median_us"]}
             for k, s in stats.items() if k.startswith("rows_") and k.endswith("_wave")}
    for v in sweep.values():
        v["rpw1_vs_wave"] = v["rpw1_us"] / v["wave_us"] - 1
    budget["row_sweep"] = sweep
    doc = {"card_before": before, "card_after": after, "tool": {k: v for k, v in raw.items() if k != "series"},
           "variants": stats, "budget": budget}
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "k1_budget.json")
    with open(path, "w") as f:
        json.dump(doc, f, indent=1)

    print(f"{before['name']}, power limit {before['power_limit_w']:.0f} W, SM clock {before['sm_clock_mhz']} -> "
          f"{after['sm_clock_mhz']} MHz (max {before['max_sm_clock_mhz']})")
    print(f"{'variant':<14} {'min us':>9} {'median us':>10}")
    for k, s in stats.items():
        if not k.startswith("rows_"):
            print(f"{k:<14} {s['min_us']:9.2f} {s['median_us']:10.2f}")
    for k, v in budget.items():
        if k != "row_sweep":
            print(f"{k:<26} {v:.3f}" if isinstance(v, float) else f"{k:<26} {v}")
    for k, v in sweep.items():
        print(f"{k:<22} one wave {v['wave_us']:9.2f} us  one row per warp {v['rpw1_us']:9.2f} us  {100 * v['rpw1_vs_wave']:+6.2f} %")
    print(f"wrote {path}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
