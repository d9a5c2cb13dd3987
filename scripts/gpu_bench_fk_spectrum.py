"""Device time of the f-k power spectrum (dsp.fk_spectrum on a CUDA tensor) against the f-k filter (dsp.fk_filter_filt
with the fan mask) at the same shape: CUDA events around each call, one warm-up call first, the median of N calls.
  * 10 000 x 120 000 (time split T1 = 12: the power pass stores columns T1 apart) and 11 020 x 12 000 (T1 = 1);
  * cases: the whole plane (f >= 0, every k), a 0-50 Hz band with |k| <= 0.02 1/m, nperseg = 12 000 over the large
    record (ten blocks), and the filter as the comparison row.
Each spectrum call includes making its FkSpectrum (support tables, a few host-to-device copies); the `object` rows time
a reused FkSpectrum alone, and a torch.profiler run after the timings splits its device time by kernel.  Prints one JSON line per measurement with the card's name and power limit read in the same
run.  Usage: python scripts/gpu_bench_fk_spectrum.py [N]"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from das4whales_b200 import dsp, fk
N = max(3, int(sys.argv[1]) if len(sys.argv) > 1 else 20)
DX, FS = 2.0419046878814697, 200.0


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:                     # noqa: BLE001
        return None


def kernel_ms(fn, reps=5):
    """Device time per call of each kernel fn launches (torch.profiler, after the timed runs)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    return {e.key.split("(")[0][:48]: round(e.device_time_total / 1000.0 / reps, 3) for e in prof.key_averages()
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
for nx, ns in ((10000, 120000), (11020, 12000)):
    sel = [0, nx, 1]
    x = torch.randn((nx, ns), device="cuda", generator=torch.Generator(device="cuda").manual_seed(ns))
    plan = fk.get_plan(nx, ns, torch.cuda.current_device())
    cases = {"whole plane (f >= 0, all k)": dict(),
             "0-50 Hz, |k| <= 0.02": dict(f_range=(0., 50.), k_range=(-0.02, 0.02))}
    if ns == 120000:
        cases["nperseg = 12000, whole plane"] = dict(nperseg=12000)
    for what, kw in cases.items():
        p, f, k = dsp.fk_spectrum(x, sel, DX, FS, **kw)
        n = kw.get("nperseg", ns)
        k0 = int(np.searchsorted(np.fft.fftshift(np.fft.fftfreq(nx, DX)), k[0]))
        f0 = int(np.searchsorted(np.fft.fftshift(np.fft.fftfreq(n, 1 / FS)), f[0]))
        spec = fk.FkSpectrum((nx, n), (k0, k0 + len(k)), (f0, f0 + len(f)))
        call = median_ms(lambda: dsp.fk_spectrum(x, sel, DX, FS, **kw))
        obj = median_ms(lambda: spec(x, out=p))
        print(json.dumps(dict(shape=[nx, ns], case=what, t1=spec.plan.t1, col_scheme=spec.plan.col_scheme, rows=spec.rows,
                              out_shape=list(p.shape), ms_dsp_call=round(call, 3), ms_object=round(obj, 3), n=N, gpu=gpu,
                              power_limit_w=watts)), flush=True)
        print(json.dumps(dict(shape=[nx, ns], case=what, kernel_ms_per_call=kernel_ms(lambda: spec(x, out=p)))), flush=True)
        del p, spec
        fk.free_plans()
        torch.cuda.empty_cache()
    fan = dsp.fk_filter_design((nx, ns), sel, DX, FS)
    flt = fk.FkFilter(fan)
    y = torch.empty_like(x)
    call = median_ms(lambda: dsp.fk_filter_filt(x, fan))
    obj = median_ms(lambda: flt(x, out=y))
    print(json.dumps(dict(shape=[nx, ns], case="fk_filter_filt, fan mask", t1=plan.t1, col_scheme=plan.col_scheme,
                          rows=flt.rows_kept, ms_dsp_call=round(call, 3), ms_object=round(obj, 3), n=N, gpu=gpu,
                          power_limit_w=watts)), flush=True)
    print(json.dumps(dict(shape=[nx, ns], case="fk_filter_filt, fan mask", kernel_ms_per_call=kernel_ms(lambda: flt(x, out=y)))),
          flush=True)
    del flt, y, x, fan
    fk.free_plans()
    torch.cuda.empty_cache()
