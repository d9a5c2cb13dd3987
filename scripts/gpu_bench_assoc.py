"""Pick association on the GPU (d4w_loc_associate through loc.associate_picks).

Workload: a 22.5 km straight cable of 11 020 channels at 2.04 m, 8 calls picked on every other channel (5 510 picks each)
plus 6 000 false picks at uniform channels and samples of a 60 s record: 50 080 picks, given as the pipelines' device CSR.
Grids of 161 x 161 x 1 and 81 x 81 x 8 nodes, tol = 0.5 s.  The time of associate_picks is the median over --reps calls of
CUDA events around each call, after two warm-up calls; the per-kernel split is a separate torch.profiler run.  Work counts
come from the shapes: tau evaluations per vote pass = nodes x picked channels, bin updates of the first pass = nodes x
picks (later passes skip the assigned picks).  The result is checked against the float64 oracle on the smaller grid before
timing.  Prints one JSON line, and also writes it to --out when given.

    python scripts/gpu_bench_assoc.py [--reps 20] [--out assoc_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NCH, DX, FS, C0, TOL = 11020, 2.0419046878814697, 200.0, 1500.0, 0.5
GRIDS = {"161x161x1": ((0.0, 22500.0, 161), (0.0, 8000.0, 161), (0.0, 0.0, 1)),
         "81x81x8": ((0.0, 22500.0, 81), (0.0, 8000.0, 81), (-700.0, 0.0, 8))}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception as e:                      # the measurement stands without it; say so in the record
        return [f"unknown ({e})", "unknown", "unknown"]


def workload():
    from oracle import assoc_oracle as A
    rng = np.random.default_rng(0)
    cable = A.straight_cable(NCH, DX)
    sources = [((rng.uniform(1000, 21500), rng.uniform(200, 7000), 0.0), 5.0 + 6.0 * k) for k in range(8)]
    ch, s, _ = A.synth_picks(cable, sources, FS, C0, rng, every=2, false_frac=0.0)
    fc, fsm = rng.integers(0, NCH, 6000), rng.integers(0, int(60 * FS), 6000)
    ch, s = np.r_[ch, fc], np.r_[s, fsm]
    o = np.lexsort((s, ch))
    return cable, ch[o], s[o]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from das4whales_b200 import loc
    from oracle import assoc_oracle as A

    name, plimit, clk = card()
    cable, ch, s = workload()
    off = np.zeros(NCH + 1, np.int32)
    off[1:] = np.cumsum(np.bincount(ch, minlength=NCH))
    picks = (torch.from_numpy(off).cuda(), torch.from_numpy(s.astype(np.int32)).cuda())
    picked = int(np.count_nonzero(np.diff(off)))
    rec = {"card": name, "power_limit": plimit, "max_sm_clock": clk, "channels": NCH, "picks": int(len(s)),
           "picked_channels": picked, "tol": TOL, "workloads": {}}

    # spot check against the oracle on a small grid before timing (the oracle is O(nodes x picks) in host memory)
    small = ((0.0, 22500.0, 21), (0.0, 8000.0, 9), (0.0, 0.0, 1))
    ref = A.associate(ch, s, FS, cable, C0, small, TOL, 1000)
    got = loc.associate_picks(picks, FS, cable, C0, small, TOL, 1000)
    rec["oracle_check_small_grid"] = all(np.array_equal(x.cpu().numpy(), y) for x, y in zip(got, ref))

    for label, grid in GRIDS.items():
        nodes = int(np.prod([g[2] for g in grid]))
        for _ in range(2):
            res = loc.associate_picks(picks, FS, cable, C0, grid, TOL, 1000)
        torch.cuda.synchronize()
        times = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            res = loc.associate_picks(picks, FS, cable, C0, grid, TOL, 1000)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        K = int(res.node.numel())
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            loc.associate_picks(picks, FS, cable, C0, grid, TOL, 1000)
            torch.cuda.synchronize()
        split = {}
        for ev in prof.key_averages():
            if ev.key.startswith(("void (anonymous namespace)::k_assoc", "k_assoc", "(anonymous namespace)::k_assoc")) \
                    or "k_assoc" in ev.key:
                short = ev.key.split("k_assoc")[1].split("(")[0]
                split["k_assoc" + short] = {"ms": round(ev.device_time_total / 1e3, 4), "calls": ev.count}
        rec["workloads"][label] = {
            "nodes": nodes, "calls_found": K, "counts": res.count.cpu().numpy().tolist(),
            "median_ms": round(float(np.median(times)), 4), "min_ms": round(float(np.min(times)), 4),
            "max_ms": round(float(np.max(times)), 4), "vote_passes": K + 1,
            "tau_evals_per_pass": nodes * picked, "bin_updates_first_pass": nodes * int(len(s)),
            "kernels": split}
    rec["reference_pipeline_ms_per_file"] = 134.0     # MfDetectPipeline on 11 020 x 12 000 (README), not measured here
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
