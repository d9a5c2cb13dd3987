"""Device time (CUDA events, after warm-up, alternated rounds) of the cross-spectral density and coherence, tensors resident
on the device:
  - neighbour coherence, dsp.coherence(x[:-1], x[1:]), at 11 020 x 12 000 with nperseg 256 and 1 024;
  - dsp.csd of 10 000 x 120 000 against one reference row with nperseg 1 024, mean and median (233 segments: the
    workspace route and its signed selection);
  - dsp.welch on the same records, the yardstick: one spectrum per row, where a pair reads two rows.
A separate torch.profiler pass per case gives the device time of each kernel.  Prints one JSON line per measurement with
the card's name, power limit and maximum SM clock (and the SM clock read after each case), the algorithmic bytes (4 B per
sample of every input row read -- a neighbour pair reads both of its rows, a broadcast reference row is read once -- plus
the output) and their share of the data-sheet 3.35 TB/s.
Usage: python scripts/gpu_bench_csd.py [reps]"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from das4whales_b200 import dsp
REPS = max(20, int(sys.argv[1]) if len(sys.argv) > 1 else 20)
WARMUP = 3
ROUNDS = 3
HBM_BPS = 3.35e12
KERNELS = ("k_csd_median", "k_csd", "k_welch", "k_row_median")


def card_settings():
    """(power limit W, SM clock MHz, maximum SM clock MHz) from nvidia-smi, None where it cannot be read"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                              "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return tuple(float(v) for v in out.splitlines()[0].split(","))
    except Exception:                     # noqa: BLE001
        return None, None, None


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


def kernel_split(fn):
    """device time per kernel of one call (torch.profiler, run after the timed rounds)"""
    from torch.profiler import ProfilerActivity, profile
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(); torch.cuda.synchronize()
    split = {}
    for e in prof.key_averages():
        k = next((k for k in KERNELS if k + "(" in e.key), None)          # demangled: "...::k_csd(d4w::CsdParams, ..."
        if k:
            us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            split[k] = round(split.get(k, 0.0) + us / 1e3, 3)
    return split


gpu, (watts, _, sm_max_mhz) = torch.cuda.get_device_name(), card_settings()


def run(shape, cases):
    x = torch.randn(shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(shape[1])) * 1e-9
    ref = x[shape[0] // 2:shape[0] // 2 + 1].clone()              # the reference row (a co-located sensor)
    fns = []
    for op, npg, avg in cases:
        if op == "neighbour coherence":
            fns.append(lambda n=npg: dsp.coherence(x[:-1], x[1:], fs=200., nperseg=n))
        elif op == "csd vs reference row":
            fns.append(lambda n=npg, a=avg: dsp.csd(x, ref, fs=200., nperseg=n, average=a))
        else:
            fns.append(lambda n=npg, a=avg: dsp.welch(x, fs=200., nperseg=n, average=a))
    times = [[] for _ in cases]
    for _ in range(ROUNDS):                                       # alternated rounds: every case sees the same clocks
        for i, fn in enumerate(fns):
            times[i].append(timed(fn))
    nx, ns = shape
    for (op, npg, avg), t, fn in zip(cases, times, fns):
        lay = dsp.welch_layout(ns, npg)
        if op == "neighbour coherence":
            rows_out, rows_read, out_b = nx - 1, 2 * (nx - 1), 4
        elif op == "csd vs reference row":
            rows_out, rows_read, out_b = nx, nx + 1, 8
        else:
            rows_out, rows_read, out_b = nx, nx, 4
        nbytes = 4.0 * ns * rows_read + out_b * rows_out * lay.nbins
        ms = float(np.median(t))
        print(json.dumps(dict(op=op, nx=nx, ns=ns, nperseg=npg, nseg=lay.nseg, average=avg, ms=round(ms, 3),
                              ms_rounds=[round(v, 3) for v in t], bytes=int(nbytes), gb_per_s=round(nbytes / ms / 1e6, 1),
                              share_of_3_35_tb_s=round(nbytes / (ms * 1e-3) / HBM_BPS, 3), kernel_ms=kernel_split(fn),
                              reps=REPS, warmup=WARMUP, gpu=gpu, power_limit_w=watts, sm_max_mhz=sm_max_mhz,
                              sm_mhz_after=card_settings()[1])), flush=True)
    del x, ref
    torch.cuda.empty_cache()


run((11020, 12000), [("neighbour coherence", 256, "mean"), ("neighbour coherence", 1024, "mean"),
                     ("welch", 256, "mean"), ("welch", 1024, "mean")])
run((10000, 120000), [("csd vs reference row", 1024, "mean"), ("csd vs reference row", 1024, "median"),
                      ("welch", 1024, "mean"), ("welch", 1024, "median")])
