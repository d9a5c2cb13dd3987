"""Localisation on the GPU: the grid search (d4w_loc_grid) and the Gauss-Newton solve (d4w_loc_solve).

Workloads: the grid search for 100 calls x 3 000 observations on 161 x 161 x 1 nodes (fix_z) and on 81 x 81 x 9 nodes (free
z), and the solve alone (10 iterations) for 10 000 calls x 3 000 observations, each timed with CUDA events after a warm-up.
The grid's rate is distance evaluations (nodes x observations) per second; its FP64 share counts 14 operations per
evaluation (3 differences, 3 products and 2 sums for d^2, a square root counted as one, T - d / c0 as a multiply-add, the
shift, and the two sums) against the 34 TFLOP/s FP64 (non-tensor) figure of NVIDIA's H100 SXM data sheet.  A spot check
against the float64 oracle at small B comes first.  Prints one JSON line, and also writes it to --out when given.

    python scripts/gpu_bench_loc.py [--reps 20] [--out loc_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP64_PEAK = 34e12
FLOP_PER_EVAL = 14
C0 = 1490.0


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception as e:                      # the measurement stands without it; say so in the record
        return [f"unknown ({e})", "unknown", "unknown"]


def batch(ncalls, nobs, cable, seed, fix_z):
    from oracle import loc_oracle as O
    rng = np.random.default_rng(seed)
    T = np.empty(ncalls * nobs)
    for b in range(ncalls):
        w = (rng.uniform(0, 60000), rng.uniform(0, 60000), -50.0 if fix_z else rng.uniform(-1200, 0))
        T[b * nobs:(b + 1) * nobs] = O.arrivals(cable, w, rng.uniform(0, 100), C0, 2e-3, rng)
    P = np.tile(cable, (ncalls, 1))
    return T, P, np.arange(ncalls + 1, dtype=np.int64) * nobs


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    from das4whales_b200 import loc
    from oracle import loc_oracle as O
    name, power, maxclk = card()
    cable = O.bent_cable(3000)
    rec = dict(card=name, power_limit=power, max_sm_clock=maxclk, fp64_peak_tflops=FP64_PEAK / 1e12)

    # spot check against the oracle at small B
    T, P, off = batch(6, 3000, cable, 1, True)
    g = ((-10000, 70000, 41), (-10000, 70000, 41), (-50, -50, 1))
    res = loc.solve_lq_batch(T, P, off, C0, fix_z=True, grid=g)
    n, _, _ = O.solve_batch(T, P, off, C0, res.n0, 10, True)
    idx, score, _ = loc.grid_search(T, P, off, C0, g, fix_z=True)
    sc, _ = O.grid_scores(T[:3000], P[:3000], C0, O.grid_nodes(g), True)
    rec["spot_n_rel"] = float(np.max(np.abs(res.n - n) / np.abs(n)))
    rec["spot_score_rel"] = float(abs(score[0] - sc[idx[0]]) / sc[idx[0]])
    assert rec["spot_n_rel"] <= 1e-9 and rec["spot_score_rel"] <= 1e-9 and sc[idx[0]] <= (1 + 1e-9) * sc.min(), rec

    for tag, shape, fix_z in (("grid_161x161x1", (161, 161, 1), True), ("grid_81x81x9", (81, 81, 9), False)):
        T, P, off = batch(100, 3000, cable, 2, fix_z)
        grid = ((-10000, 70000, shape[0]), (-10000, 70000, shape[1]), (-50, -50, 1) if fix_z else (-1200, 0, shape[2]))
        Td, Pd = torch.from_numpy(T).cuda(), torch.from_numpy(P).cuda()
        ms = timed(lambda: loc.grid_search(Td, Pd, off, C0, grid, fix_z=fix_z), args.reps)
        evals = 100 * 3000 * shape[0] * shape[1] * shape[2]
        rec[tag] = dict(ms=ms, calls=100, nobs=3000, nodes=shape[0] * shape[1] * shape[2], evals_per_s=evals / (ms * 1e-3),
                        fp64_share=evals * FLOP_PER_EVAL / (ms * 1e-3) / FP64_PEAK)

    T, P, off = batch(10000, 3000, cable, 3, False)
    Td, Pd = torch.from_numpy(T).cuda(), torch.from_numpy(P).cuda()
    ms = timed(lambda: loc.solve_lq_batch(Td, Pd, off, C0), max(3, args.reps // 4))
    rec["solve_10000x3000"] = dict(ms=ms, calls=10000, nobs=3000, iterations=10, ms_per_call=ms / 10000)
    line = json.dumps(rec)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
