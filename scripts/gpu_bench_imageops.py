"""Time the image operators of improcess outside the Gabor path on the GPU: the Radon transform of the binned Gabor image
(1 102 x 1 200) and of the full trace2image image (11 020 x 12 000), both with skimage's default 180 angles, and the
float32 bilateral filter (d = 5 and 9) on the full image.  CUDA events around `--reps` calls after a warm-up call of every
shape.  Samples = the bilinear samples the clipped rays take (counted on the host from the same clipping rule), so
samples / s is the Radon kernel's own rate.  A sampled set of rays of the full-size transform is checked against the
float64 restatement first.  Prints one JSON line, and also writes it to --out when given.

    python scripts/gpu_bench_imageops.py [--reps 5] [--out imageops_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from das4whales_b200 import improcess  # noqa: E402
from oracle import radon_oracle as R  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception as e:                      # the measurement stands without it; say so in the record
        return [f"unknown ({e})", "unknown", "unknown"]


def ray_samples(h, w, theta):
    """rows each clipped ray visits, summed over bins and angles (the loop bounds of radon_ray, in float64 NumPy)"""
    n, pr, pc = improcess._radon_square(h, w)
    b = np.arange(n, dtype=np.float64)
    c = n // 2
    total = 0
    for t in np.deg2rad(theta):
        co, si = np.cos(t), np.sin(t)
        x0 = co * b - c * (co + si - 1) - pc
        y0 = -si * b - c * (co - si - 1) - pr
        lo, hi = np.zeros(n), np.full(n, n - 1.0)
        for k, x, e1 in ((si, x0, w), (co, y0, h)):
            if k == 0:
                bad = ~((x > -1) & (x < e1))
                lo[bad], hi[bad] = 1, 0
                continue
            a, bb = (-1 - x) / k, (e1 - x) / k
            lo, hi = np.maximum(lo, np.minimum(a, bb)), np.minimum(hi, np.maximum(a, bb))
        ok = lo <= hi
        r0 = np.maximum(np.floor(lo) - 1, 0)
        r1 = np.minimum(np.ceil(hi) + 1, n - 1)
        total += int(np.sum((r1 - r0 + 1)[ok]))
    return total


def timed(torch, f, reps):
    f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    name, power, maxclk = card()
    rec = dict(card=name, power_limit=power, max_sm_clock=maxclk, angles=180)
    g = torch.Generator(device="cuda").manual_seed(5)
    trace = torch.randn((11020, 12000), generator=g, device="cuda", dtype=torch.float32)
    image = improcess.trace2image(trace)
    binned = improcess.binning(image, 0.1, 0.1)
    theta = np.arange(180)

    # spot check of the full-size transform: 64 rays against the float64 restatement
    full = improcess.compute_radon_transform(image, theta)
    rng = np.random.default_rng(1)
    n = full.shape[0]
    bins, angles = rng.integers(n // 4, 3 * n // 4, 64), rng.integers(0, 180, 64)
    host = image.cpu().numpy()
    want = R.radon_bins(host, bins, angles)
    got = full[torch.from_numpy(bins).cuda(), torch.from_numpy(angles).cuda()].double().cpu().numpy()
    rec["fullsize_spot_check_rel_err"] = float(np.max(np.abs(got - want)) / np.abs(want).max())
    del full

    for label, img in (("radon_1102x1200", binned), ("radon_11020x12000", image)):
        ms = timed(torch, lambda: improcess.compute_radon_transform(img, theta), args.reps)
        s = ray_samples(img.shape[0], img.shape[1], theta)
        rec[label] = dict(ms=round(ms, 3), samples=s, gsamples_per_s=round(s / ms / 1e6, 2))
    for d in (5, 9):
        ms = timed(torch, lambda: improcess.bilateral_filter(image, d, 30.0, 30.0), args.reps)
        rec[f"bilateral_d{d}_11020x12000_ms"] = round(ms, 3)
        rec[f"bilateral_d{d}_gpix_per_s"] = round(image.numel() / ms / 1e6, 2)
    line = json.dumps(rec)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
