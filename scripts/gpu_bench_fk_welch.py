"""Device time of the f-k Welch spectrum (dsp.fk_welch on a CUDA tensor): CUDA events around each call, one warm-up call
first, the median of N calls.
  * 10 000 x 120 000, nperseg = 12 000 with 6 000 of overlap (19 segments, Hann windows, detrend 'constant'): the whole
    f >= 0 plane, and 0-50 Hz with |k| <= 0.02 1/m;
  * 11 020 x 12 000, nperseg = 1 200 and nperseg_x = 1 102 (19 x 19 half-overlapping segments, one f-k plane per
    channel segment).
The `object` rows time a reused FkWelch alone (no plan, support or window set-up); a torch.profiler run after the timings
splits its device time by kernel (stage, P1, P2, power).  Prints one JSON line per measurement with the card's name and
power limit read in the same run.  Usage: python scripts/gpu_bench_fk_welch.py [N]"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import scipy.signal as sps
import torch
from das4whales_b200 import dsp, fk
N = max(3, int(sys.argv[1]) if len(sys.argv) > 1 else 10)
DX, FS = 2.0419046878814697, 200.0


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:                     # noqa: BLE001
        return None


def kernel_ms(fn, reps=3):
    """Device time per call of each kernel fn launches (torch.profiler, after the timed runs)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    return {e.key.replace("(anonymous namespace)::", "").split("(")[0][:48]: round(e.device_time_total / 1000.0 / reps, 3) for e in prof.key_averages()
            if e.device_time_total > 0}


def median_ms(fn):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(N):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


gpu, watts = torch.cuda.get_device_name(), power_limit_w()
CASES = [((10000, 120000), "19 segments of 12000, whole plane (f >= 0, all k)", dict(nperseg=12000, noverlap=6000)),
         ((10000, 120000), "19 segments of 12000, 0-50 Hz, |k| <= 0.02",
          dict(nperseg=12000, noverlap=6000, f_range=(0., 50.), k_range=(-0.02, 0.02))),
         ((11020, 12000), "19 x 19 segments of 1102 x 1200, whole plane", dict(nperseg=1200, nperseg_x=1102))]
x = None
for (nx, ns), what, kw in CASES:
    if x is None or tuple(x.shape) != (nx, ns):
        x = None
        torch.cuda.empty_cache()
        x = torch.randn((nx, ns), device="cuda", generator=torch.Generator(device="cuda").manual_seed(ns))
    sel = [0, nx, 1]
    res = dsp.fk_welch(x, sel, DX, FS, **kw)
    p, f, k = res[:3]
    l, lx = kw["nperseg"], kw.get("nperseg_x", nx)
    lay = dsp.fk_welch_layout(nx, ns, l, kw.get("noverlap"), kw.get("nperseg_x"), None)
    k0 = int(np.searchsorted(np.fft.fftshift(np.fft.fftfreq(lx, DX)), k[0]))
    f0 = int(np.searchsorted(np.fft.fftshift(np.fft.fftfreq(l, 1 / FS)), f[0]))
    est = fk.FkWelch((nx, ns), (lx, l), (k0, k0 + len(k)), (f0, f0 + len(f)), sps.get_window("hann", l),
                     sps.get_window("hann", lx), True, 1.0, noverlap=lay.noverlap, noverlap_x=lay.noverlap_x)
    out = torch.empty(est.out_shape, dtype=torch.float32, device=x.device)
    call = median_ms(lambda: dsp.fk_welch(x, sel, DX, FS, **kw))
    obj = median_ms(lambda: est(x, out=out))
    print(json.dumps(dict(shape=[nx, ns], case=what, segment=[lx, l], nseg=lay.nseg, nseg_x=lay.nseg_x, batch=est.batch,
                          t1=est.plan.t1, col_scheme=est.plan.col_scheme, rows=est.spec.rows, out_shape=list(p.shape),
                          ms_dsp_call=round(call, 3), ms_object=round(obj, 3), n=N, gpu=gpu, power_limit_w=watts)), flush=True)
    print(json.dumps(dict(shape=[nx, ns], case=what, kernel_ms_per_call=kernel_ms(lambda: est(x, out=out)))), flush=True)
    del p, res, est, out
    fk.free_plans()
    torch.cuda.empty_cache()
