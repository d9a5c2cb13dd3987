"""Device time (CUDA events, after warm-up) of the Gabor detector's matched filter, detect.compute_cross_correlograms_same
(HF + LF notes of scripts/main_gabordetect.py, one pass), at 11 020 x 12 000 and 10 000 x 120 000 with 0 %, 90 % and 99 % of
the rows zeroed (as a Gabor mask leaves them), against the positive-lag detect.compute_cross_correlograms (HF + LF
fin-call templates zero-padded to ns) on the same matrix; and GaborDetectPipeline per file (int32 counts already on the
device -> picks) at 11 020 x 12 000.  One JSON line per measurement, with the card's name and power limit.
Usage: python scripts/gpu_bench_gabor_mf.py [reps]"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from das4whales_b200 import detect, pipeline
REPS = max(20, int(sys.argv[1]) if len(sys.argv) > 1 else 20)
WARMUP = 3
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


def hann_chirp(fmin, fmax, dur):
    c = detect.gen_hyperbolic_chirp(fmin, fmax, dur, FS)
    return np.hanning(len(c)) * c


gpu, watts = torch.cuda.get_device_name(), power_limit_w()
notes = [hann_chirp(17.8, 28.8, 0.68), hann_chirp(14.7, 21.8, 0.78)]
for nx, ns in ((11020, 12000), (10000, 120000)):
    x = torch.randn((nx, ns), device="cuda", generator=torch.Generator(device="cuda").manual_seed(ns))
    t = np.arange(ns) / FS
    padded = [detect.gen_template_fincall(t, FS, 17.8, 28.8, 0.68), detect.gen_template_fincall(t, FS, 14.7, 21.8, 0.78)]
    pos_ms = timed(lambda: detect.compute_cross_correlograms(x, padded))
    print(json.dumps({"nx": nx, "ns": ns, "op": "compute_cross_correlograms (positive lags, HF + LF)", "ms": round(pos_ms, 3),
                      "reps": REPS, "warmup": WARMUP, "gpu": gpu, "power_limit_w": watts}), flush=True)
    perm = torch.randperm(nx, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    for frac in (0.0, 0.9, 0.99):
        xm = x.clone()
        xm[perm[:int(round(frac * nx))]] = 0
        same_ms = timed(lambda: detect.compute_cross_correlograms_same(xm, notes))
        print(json.dumps({"nx": nx, "ns": ns, "op": "compute_cross_correlograms_same (HF + LF)", "rows_zeroed": frac,
                          "ms": round(same_ms, 3), "reps": REPS, "warmup": WARMUP, "gpu": gpu, "power_limit_w": watts}), flush=True)
        del xm
    del x
    torch.cuda.empty_cache()

nx, ns = 11020, 12000
rng = np.random.default_rng(0)
counts = torch.from_numpy(np.round(rng.standard_normal((nx, ns)) * 5.0e4).astype(np.int32)).cuda()
pipe = pipeline.GaborDetectPipeline(nx, ns, [0, nx, 1], DX, FS, 4.0838e-11 * 1550.0 / 2.0419)
file_ms = timed(lambda: pipe.process_device(counts))
print(json.dumps({"nx": nx, "ns": ns, "op": "GaborDetectPipeline.process_device per file (counts on the device -> picks)",
                  "ms": round(file_ms, 3), "reps": REPS, "warmup": WARMUP, "gpu": gpu, "power_limit_w": watts}), flush=True)
