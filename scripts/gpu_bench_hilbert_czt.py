"""Device time (CUDA events, after warm-up) of the envelope and the envelope SNR for chirp-z row lengths against their
neighbouring direct lengths: 10 000 x 1 501 (the 12 000-sample record's spectrogram-correlation correlogram) vs
10 000 x 1 500, and 10 000 x 15 001 vs 10 000 x 15 000.  One JSON line per shape, with the card's name and power limit.
Usage: python scripts/gpu_bench_hilbert_czt.py [reps]"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from das4whales_b200 import rows
REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
WARMUP = 3


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:                     # noqa: BLE001
        return None


def timed(fn):
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(REPS):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / REPS


gpu, watts = torch.cuda.get_device_name(), power_limit_w()
for nx, ns in ((10000, 1501), (10000, 1500), (10000, 15001), (10000, 15000)):
    x = torch.randn((nx, ns), device="cuda", generator=torch.Generator(device="cuda").manual_seed(ns))
    env_ms = timed(lambda: rows.envelope(x))
    snr_ms = timed(lambda: rows.snr(x, env=True))
    t1, t2, m = rows.row_plan(ns, x.device.index).info()
    print(json.dumps({"nx": nx, "ns": ns, "route": "chirp-z" if m else "direct", "t1": t1, "t2": t2, "czt_m": m,
                      "envelope_ms": round(env_ms, 3), "snr_env_ms": round(snr_ms, 3), "reps": REPS, "warmup": WARMUP,
                      "gpu": gpu, "power_limit_w": watts}), flush=True)
    del x
    torch.cuda.empty_cache()
