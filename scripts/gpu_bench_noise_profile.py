"""Device time (CUDA events, after warm-up) of the cable noise profile of scripts/main_bathynoise.py:183-259 at
11 020 x 12 000 and 10 000 x 120 000: rows.env_stats of the whole rows plus the 19-26 s noise window (1 400 samples)
against the calls d4w_env_stats makes, issued from Python (rows.row_stats, rows.envelope, rows.row_stats of the envelope for
its mean, rows.row_median; the window copied to a dense matrix first), in alternated rounds; and
NoiseProfilePipeline.process_device per 11 020 x 12 000 file (int32 counts on the device -> profile).  Checks that both give the same profile, and prints one JSON line per measurement with the card's
name and power limit.
Usage: python scripts/gpu_bench_noise_profile.py [reps]"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from das4whales_b200 import dsp, pipeline, rows
REPS = max(10, int(sys.argv[1]) if len(sys.argv) > 1 else 20)
WARMUP = 3
ROUNDS = 5
DX, FS = 2.0419046878814697, 200.0
I0, I1 = dsp.noise_window(12000, FS)


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


def env_stats(x):
    return rows.env_stats(x), rows.env_stats(x, I0, I1 - I0)


def composed_record(x):
    """the calls d4w_env_stats makes: row statistics of x, envelope, row statistics of the envelope (its
    mean, from the float32 envelope), median of the envelope"""
    st, _ = rows.row_stats(x)
    env = rows.envelope(x)
    ste, _ = rows.row_stats(env)
    med = rows.row_median(env).double()
    del env
    mean, var = st[:, 0], st[:, 2]
    return torch.stack([med, ste[:, 0], mean, var + mean * mean, var], dim=1)


def composed(x):
    # d4w_env_stats copies a strided window to a dense matrix first (cudaMemcpy2DAsync); so does .contiguous()
    return composed_record(x), composed_record(x[:, I0:I1].contiguous())


def line(**kw):
    print(json.dumps(dict(kw, reps=REPS, warmup=WARMUP, gpu=gpu, power_limit_w=watts)), flush=True)


gpu, watts = torch.cuda.get_device_name(), power_limit_w()
for nx, ns in ((11020, 12000), (10000, 120000)):
    x = torch.randn((nx, ns), device="cuda", generator=torch.Generator(device="cuda").manual_seed(ns)) * 1e-9
    a = dsp.noise_profile_from_stats(*env_stats(x))
    b = dsp.noise_profile_from_stats(*composed(x))
    dev = {k: float(((a[k] - b[k]).abs() / b[k].abs().clamp_min(1e-300)).max()) for k in ("med", "mean", "std", "noise_mean")}
    assert all(v <= 1e-4 for v in dev.values()), dev
    # ROUNDS alternated windows of REPS calls each, so that both sides see the same clocks and neighbours
    one, comp = [], []
    for _ in range(ROUNDS):
        one.append(timed(lambda: env_stats(x)))
        comp.append(timed(lambda: composed(x)))
    line(nx=nx, ns=ns, op=f"rows.env_stats, whole row + {I1 - I0}-sample window",
         ms=round(float(np.median(one)), 3), ms_rounds=[round(v, 3) for v in one])
    line(nx=nx, ns=ns, op="the same calls from Python (row_stats, envelope, row_stats of the envelope, row_median), "
         "whole row + copied window", ms=round(float(np.median(comp)), 3), ms_rounds=[round(v, 3) for v in comp],
         max_rel_diff_vs_env_stats={k: float(f"{v:.2e}") for k, v in dev.items()})
    del x
    torch.cuda.empty_cache()

nx, ns = 11020, 12000
rng = np.random.default_rng(0)
counts_h = np.round(rng.standard_normal((nx, ns)) * 5.0e4).astype(np.int32)
counts = torch.from_numpy(counts_h).cuda()
pipe = pipeline.NoiseProfilePipeline(nx, ns, [0, nx, 1], DX, FS, 4.0838e-11 * 1550.0 / 2.0419)
file_ms = timed(lambda: pipe.process_device(counts))
line(nx=nx, ns=ns, op="NoiseProfilePipeline.process_device per file (counts on the device -> profile)", ms=round(file_ms, 3))
pinned = torch.from_numpy(counts_h).pin_memory()
torch.cuda.synchronize()
stream_ms = timed(lambda: list(pipe.stream([pinned] * 4)), reps=max(3, REPS // 4)) / 4
line(nx=nx, ns=ns, op="NoiseProfilePipeline.stream per file (pinned host counts -> host profile)", ms=round(stream_ms, 3))
