"""Sliding-DFT STFT (d4w_stft_slide) against the per-frame FFT path (d4w_stft_mag) and the fp64 oracle; timing of both."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import das4whales_b200 as dw
from das4whales_b200 import rows, synth
from oracle import detect_oracle as D, dsp_oracle as O

def timed(fn, reps=5):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps

rng = np.random.default_rng(5)
for (nfft, hop, b0, b1, ns) in [(160, 8, 2, 32, 9000), (160, 8, 0, 30, 9001), (160, 8, 50, 80, 12345), (128, 8, 5, 40, 6000),
                                (256, 16, 10, 50, 7000), (256, 16, 20, 27, 5000), (128, 8, 3, 18, 4000), (160, 8, 12, 24, 120000), (160, 8, 30, 30, 2000)]:
    x = rng.standard_normal((5, ns)).astype(np.float32)
    x[1] += 50 * np.sin(2 * np.pi * 0.7 * np.arange(ns) / 200).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    a = rows.stft_mag(xd, nfft, hop, b0, b1).cpu().numpy()
    b = rows._stft_frames(xd, nfft, hop, b0, b1).cpu().numpy()
    errs = []
    for i in range(5):
        ref = np.abs(O.stft_librosa(x[i].astype(np.float64), nfft, hop))[b0:b1 + 1]
        errs.append((np.abs(a[i] - ref).max() / ref.max(), np.abs(b[i] - ref).max() / ref.max()))
    print(f"nfft {nfft} hop {hop} bins {b0}..{b1} ns {ns}: slide err {max(e[0] for e in errs):.2e}  fft err {max(e[1] for e in errs):.2e}", flush=True)

nx, ns = 1000, 120000
xd = synth.synth_strain(nx, ns, seed=3) if hasattr(synth, "synth_strain") else torch.randn(nx, ns, device="cuda")
xd = xd.cuda() if not xd.is_cuda else xd
t_fft = timed(lambda: rows._stft_frames(xd, 160, 8, 11, 41))
print(f"fft path   {nx}x{ns} bins 11..41: {t_fft:.2f} ms -> {t_fft * 10:.1f} ms per 10 000 channels")
t = timed(lambda: rows.stft_mag(xd, 160, 8, 11, 41))
print(f"slide path {nx}x{ns} bins 11..41: {t:.2f} ms -> {t * 10:.1f} ms per 10 000 channels")
kern = {'f0': 27., 'f1': 17., 'dur': 0.8, 'bdwidth': 4.}
t = timed(lambda: dw.detect.compute_cross_correlogram_spectrocorr(xd, 200., [14., 30.], kern, 0.8, 0.95), reps=3)
print(f"spectrocorr detector {nx} rows: {t:.2f} ms -> {t * 10:.1f} ms per 10 000 channels")

# ---- median (sample-bracketed select) and spectrogram correlation
for name, a in [("rayleigh", np.abs(rng.standard_normal((7, 465031)) + 1j * rng.standard_normal((7, 465031)))),
                ("even", rng.random((5, 200000))), ("ties", np.floor(rng.random((5, 300001)) * 7)),
                ("half zeros", np.where(rng.random((4, 100001)) < 0.6, 0.0, rng.random((4, 100001)))),
                ("const", np.full((3, 50000), 2.5)), ("short", rng.random((6, 16384))), ("short odd", rng.random((6, 999))),
                ("just above cap", rng.random((6, 16385))), ("heavy tail", rng.standard_cauchy((4, 250000)) ** 2)]:
    a = a.astype(np.float32)
    got = rows.row_median(torch.from_numpy(a).cuda()).cpu().numpy()
    ref = np.median(a, axis=1)
    print(f"median {name:16s} n={a.shape[1]:7d}: exact={bool(np.array_equal(got, ref))}", flush=True)
Sx = rows.stft_mag(xd, 160, 8, 11, 41)
flat = Sx.reshape(nx, -1)
t_med = timed(lambda: rows.row_median(flat))
medv = rows.row_median(flat)
Kk = rng.standard_normal((31, 20))
t_sc = timed(lambda: rows.spectro_correlate(Sx, Kk, median=medv))
print(f"row_median {nx} rows x {flat.shape[1]}: {t_med:.2f} ms; speccorr {t_sc:.2f} ms")
t = timed(lambda: dw.detect.compute_cross_correlogram_spectrocorr(xd, 200., [14., 30.], kern, 0.8, 0.95), reps=3)
print(f"spectrocorr detector {nx} rows: {t:.2f} ms -> {t * 10:.1f} ms per 10 000 channels")
