"""Device time (CUDA events, after warm-up) of the spectrogram-correlation detector of scripts/main_spectrodetect.py:103-107
(HF + LF kernels, 0.8 s window, 95 % overlap, flims 14-30 Hz) at 10 000 x 12 000 and 10 000 x 120 000: two
detect.compute_cross_correlogram_spectrocorr calls (one STFT of each kernel's band) against one
detect.compute_cross_correlograms_spectrocorr call (one STFT of the union band), each with its split into STFT, medians
and correlation; and SpectroDetectPipeline.process_device per 11 020 x 12 000 file (int32 counts on the device -> picks).
One JSON line per measurement, with the card's name and power limit.
Usage: python scripts/gpu_bench_spectrocorr.py [reps]"""
import contextlib, io, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from das4whales_b200 import detect, pipeline, rows
REPS = max(20, int(sys.argv[1]) if len(sys.argv) > 1 else 20)
WARMUP = 3
DX, FS = 2.0419046878814697, 200.0
FLIMS, WIN, OV = (14., 30.), 0.8, 0.95
HF, LF = pipeline.KERNEL_HF, pipeline.KERNEL_LF


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


def stages(xd, kernels, reps=REPS):
    """ms per call of each stage of detect._spectrocorr_device's loop (the same calls, events between the stages)"""
    nx, ns = xd.shape
    nperseg, nhop, _, (b0, b1), per = detect.spectrocorr_layout(FS, FLIMS, kernels, WIN, OV, ns)
    nf, nt = b1 - b0 + 1, 1 + ns // nhop
    chunk = max(1, min(nx, rows._MAX_ROWS, (2 << 30) // max(1, nf * nt * 4)))
    outs = [torch.empty((nx, nt), dtype=torch.float32, device=xd.device) for _ in per]
    tot = np.zeros(3)
    for it in range(WARMUP + reps):
        for r0 in range(0, nx, chunk):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[0].record()
            S = rows.stft_mag(xd[r0:r0 + chunk], nperseg, nhop, b0, b1)
            ev[1].record()
            n = S.shape[0]
            meds = [rows.row_median_ld(S, n, k.shape[0] * nt, nf * nt, o * nt) for o, k, _ in per]
            ev[2].record()
            rows.spectro_correlate_multi(S, [k for _, k, _ in per], [o for o, _, _ in per], meds,
                                         outs=[o[r0:r0 + n] for o in outs])
            ev[3].record()
            torch.cuda.synchronize()
            if it >= WARMUP:
                tot += [ev[i].elapsed_time(ev[i + 1]) for i in range(3)]
            del S
    return tot / reps


def line(**kw):
    print(json.dumps(dict(kw, reps=REPS, warmup=WARMUP, gpu=gpu, power_limit_w=watts)), flush=True)


gpu, watts = torch.cuda.get_device_name(), power_limit_w()
quiet = io.StringIO()                     # compute_cross_correlogram_spectrocorr prints its STFT parameters, as the reference does
for nx, ns in ((10000, 12000), (10000, 120000)):
    x = torch.randn((nx, ns), device="cuda", generator=torch.Generator(device="cuda").manual_seed(ns))
    with contextlib.redirect_stdout(quiet):
        two_ms = timed(lambda: [detect.compute_cross_correlogram_spectrocorr(x, FS, FLIMS, k, WIN, OV) for k in (HF, LF)])
    one_ms = timed(lambda: detect.compute_cross_correlograms_spectrocorr(x, FS, FLIMS, [HF, LF], WIN, OV))
    split_two = stages(x, [HF]) + stages(x, [LF])
    split_one = stages(x, [HF, LF])
    for op, ms, split in (("compute_cross_correlogram_spectrocorr x 2 (HF, LF)", two_ms, split_two),
                          ("compute_cross_correlograms_spectrocorr (HF + LF, one STFT)", one_ms, split_one)):
        line(nx=nx, ns=ns, op=op, ms=round(ms, 3),
             stages_ms={k: round(float(v), 3) for k, v in zip(("stft", "medians", "correlation"), split)})
    del x
    torch.cuda.empty_cache()

nx, ns = 11020, 12000
rng = np.random.default_rng(0)
counts = torch.from_numpy(np.round(rng.standard_normal((nx, ns)) * 5.0e4).astype(np.int32)).cuda()
pipe = pipeline.SpectroDetectPipeline(nx, ns, [0, nx, 1], DX, FS, 4.0838e-11 * 1550.0 / 2.0419)
file_ms = timed(lambda: pipe.process_device(counts))
line(nx=nx, ns=ns, op="SpectroDetectPipeline.process_device per file (counts on the device -> picks)", ms=round(file_ms, 3))
