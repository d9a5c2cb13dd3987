"""Device time (CUDA events, after warm-up) of the tools-module f-k path on the GPU: the Gaussian-blurred fan designed on the
device (rows.blurred_fan, sigma 20 as dsp.fk_filt uses it, and sigma 40 as tools.fk_filt does) at 10 000 x 120 000 and
11 020 x 12 000; dsp.fk_filt end to end at those sizes; and tools.fk_filt with blocks of 3 000 samples (every channel per
block), tensors resident on the device.  For comparison, the host design the device one replaces (the float64 meshgrid +
scipy.ndimage.gaussian_filter of oracle.dsp_oracle.fk_filt_mask) at 2 000 x 12 000, timed on the host CPU.  Prints
one JSON line per measurement with the card's name and power limit, read in the same run.
Usage: python scripts/gpu_bench_tools.py [reps]"""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from das4whales_b200 import dsp, rows, tools
REPS = max(2, int(sys.argv[1]) if len(sys.argv) > 1 else 5)
WARMUP = 1
DX, FS = 2.0419046878814697, 200.0


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


gpu, watts = torch.cuda.get_device_name(), power_limit_w()


def emit(**kw):
    print(json.dumps(dict(kw, gpu=gpu, power_limit_w=watts)), flush=True)


for nx, ns in ((10000, 120000), (11020, 12000)):
    kval, fval = 1.0 / (nx * DX), 1.0 / (ns / FS)
    for sigma in (20, 40):
        ms = timed(lambda: rows.blurred_fan(nx, ns, kval, fval, 1450., 3400., sigma))
        emit(case="fan_design", nx=nx, ns=ns, sigma=sigma, ms=round(ms, 3))
    torch.cuda.empty_cache()
    x = torch.randn(nx, ns, device="cuda")
    ms = timed(lambda: dsp.fk_filt(x, 1, FS, 1, DX, 1450., 3400.))
    emit(case="dsp.fk_filt", nx=nx, ns=ns, ms=round(ms, 3))
    ms = timed(lambda: tools.fk_filt(x, 1, FS, 1, DX, 1450., 3400., chunks=(None, 3000)))
    emit(case="tools.fk_filt", nx=nx, ns=ns, chunks=[None, 3000], blocks=-(-ns // 3000), ms=round(ms, 3))
    del x
    torch.cuda.empty_cache()

from oracle import dsp_oracle as O                      # the host design dsp.fk_filt used to run
t0 = time.perf_counter()
O.fk_filt_mask((2000, 12000), 1, FS, 1, DX, 1450., 3400.)
emit(case="host_fan_design_cpu", nx=2000, ns=12000, sigma=20, ms=round((time.perf_counter() - t0) * 1e3, 1),
     cpu_threads=os.cpu_count())
