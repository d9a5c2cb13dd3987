"""Device time (CUDA events, after warm-up, alternated rounds) of the per-channel Welch PSD: tools.spec at 11 020 x 12 000
(4 chunks of 3 000 samples, nperseg 1 024) and whole-row dsp.welch(nperseg=1024) with the mean and the median at
11 020 x 12 000 and 10 000 x 120 000, plus nperseg 256 (92 segments, a median ranked in shared memory) at 11 020 x 12 000,
tensors resident on the device.  A separate torch.profiler pass per case gives the device time of each kernel (k_welch, and
k_row_median on the workspace route).  Prints one JSON line per measurement with the card's
name and power limit, and two floors computed from the shapes: HBM (4 B per input sample plus the float32 output at
3.35 TB/s) and FFT (5 n log2 n flops per complex nfft-point transform, two segments per transform, at the data-sheet 67
TFLOP/s fp32).
Usage: python scripts/gpu_bench_welch.py [reps]"""
import json, math, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from das4whales_b200 import dsp, tools
REPS = max(5, int(sys.argv[1]) if len(sys.argv) > 1 else 20)
WARMUP = 3
ROUNDS = 3
HBM_BPS, FP32_FLOPS = 3.35e12, 67e12


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:                     # noqa: BLE001
        return None


def timed(fn, reps=REPS):
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def floors(nx, ns, chunk, nperseg):
    lay = dsp.welch_layout(ns, nperseg, None, None, chunk)
    hbm = (4.0 * nx * ns + 4.0 * nx * lay.nchunks * lay.nbins) / HBM_BPS * 1e3
    ffts = nx * lay.nchunks * ((lay.nseg + 1) // 2)
    fft = ffts * 5.0 * lay.nfft * math.log2(lay.nfft) / FP32_FLOPS * 1e3
    return lay, hbm, fft


gpu, watts = torch.cuda.get_device_name(), power_limit_w()
cases = [(11020, 12000, 3000, 1024, "mean", "tools.spec"),
         (11020, 12000, None, 1024, "mean", "dsp.welch"), (11020, 12000, None, 1024, "median", "dsp.welch"),
         (11020, 12000, None, 256, "mean", "dsp.welch"), (11020, 12000, None, 256, "median", "dsp.welch"),
         (10000, 120000, None, 1024, "mean", "dsp.welch"), (10000, 120000, None, 1024, "median", "dsp.welch")]


def kernel_split(fn):
    """device time per kernel of one call (torch.profiler, run after the timed rounds)"""
    from torch.profiler import ProfilerActivity, profile
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(); torch.cuda.synchronize()
    split = {}
    for e in prof.key_averages():
        for k in ("k_welch", "k_row_median"):
            if k in e.key:
                us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                split[k] = round(split.get(k, 0.0) + us / 1e3, 3)
    return split


for shape in ((11020, 12000), (10000, 120000)):
    x = torch.randn(shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(shape[1])) * 1e-9
    todo = [c for c in cases if c[:2] == shape]
    fns = [(lambda: tools.spec(x)) if op == "tools.spec" else
           (lambda a=avg, n=npg: dsp.welch(x, fs=200., nperseg=n, average=a)) for _, _, _, npg, avg, op in todo]
    times = [[] for _ in todo]
    for _ in range(ROUNDS):                                   # alternated rounds: every case sees the same clocks
        for i, fn in enumerate(fns):
            times[i].append(timed(fn))
    for (nx, ns, chunk, npg, avg, op), t, fn in zip(todo, times, fns):
        lay, hbm, fft = floors(nx, ns, chunk or ns, npg)
        ms = float(np.median(t))
        print(json.dumps(dict(op=op, nx=nx, ns=ns, chunk=lay.chunk, nperseg=npg, nseg=lay.nseg, average=avg, ms=round(ms, 3),
                              ms_rounds=[round(v, 3) for v in t], hbm_floor_ms=round(hbm, 3), fft_floor_ms=round(fft, 3),
                              bound="HBM" if hbm >= fft else "FFT", share_of_floor=round(max(hbm, fft) / ms, 3), kernel_ms=kernel_split(fn),
                              reps=REPS, warmup=WARMUP, gpu=gpu, power_limit_w=watts)), flush=True)
    del x
    torch.cuda.empty_cache()
