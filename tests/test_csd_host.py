"""CPU: the cross-spectral density and coherence's host side -- dsp.csd / dsp.coherence signatures against SciPy and every
ValueError before any device work -- and the kernel bodies (csrc/csd_kernels.cuh csd_body and csd_median_body) run block
by block on the host (tests/host_emul/csd_emul.cu) against float64 scipy.signal.csd / coherence and np.median."""
import inspect
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest
import scipy.signal as sps

from conftest import ROOT
from das4whales_b200 import dsp

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
EMUL = os.path.join(ROOT, "tests", "host_emul")


@pytest.mark.parametrize("name", ["csd", "coherence"])
def test_signature_and_defaults_match_scipy(name):
    assert inspect.signature(getattr(dsp, name)) == inspect.signature(getattr(sps, name))


def test_value_errors_before_any_device_work():
    x, y = np.zeros((3, 512)), np.ones((3, 512))
    for fn in (dsp.csd, dsp.coherence):
        for kw in (dict(detrend="linear"), dict(detrend=lambda d: d), dict(axis=0), dict(window=np.ones(100), nperseg=64),
                   dict(window=np.ones((2, 64)))):
            with pytest.raises(ValueError):
                fn(x, y, **kw)
        with pytest.raises(ValueError, match="real"):
            fn(x + 1j, y, nperseg=64)
        with pytest.raises(ValueError, match="real"):
            fn(x, y + 1j, nperseg=64)
        with pytest.raises(ValueError, match="3-D"):
            fn(np.zeros((2, 2, 64)), np.zeros(64))
        with pytest.raises(ValueError, match="same length"):
            fn(x, np.ones((3, 500)), nperseg=64)
        with pytest.raises(ValueError, match="broadcast"):
            fn(x, np.ones((2, 512)), nperseg=64)
        with pytest.raises(ValueError, match="longer"):
            fn(np.zeros(50), np.ones(50), window=np.ones(64))
        with pytest.raises(ValueError, match="61"):
            fn(x, y, nperseg=64, nfft=71)
        with pytest.raises(ValueError, match="noverlap"):
            fn(x, y, nperseg=64, noverlap=64)
    for kw in (dict(return_onesided=False), dict(average="max"), dict(scaling="power")):
        with pytest.raises(ValueError):
            dsp.csd(x, y, **kw)


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError):
        dsp.csd(np.zeros((2, 512)), np.ones(512), nperseg=64)
    with pytest.raises(RuntimeError):
        dsp.coherence(np.zeros((2, 512)), np.ones((2, 512)), nperseg=64)


# ------------------------------------------------------------------------------ host emulation of the kernel bodies
@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    out = os.path.join(str(tmp_path_factory.mktemp("csd")), "csd_emul")
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "--expt-relaxed-constexpr", "-arch=sm_90a", "-o", out,
                        os.path.join(EMUL, "csd_emul.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    return out


def _emulate(exe, tmp, x, y, lay, win, detrend, scale, coherence, median):
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    (nx, ns), ny = x.shape, y.shape[0]
    with open(fin, "wb") as f:
        f.write(struct.pack("9i", nx, ny, ns, lay.nperseg, lay.step, lay.nfft, int(detrend), int(coherence), int(median)))
        f.write(struct.pack("d", scale))
        f.write(x.astype(np.float32).tobytes())
        f.write(y.astype(np.float32).tobytes())
        f.write(np.asarray(win, np.float32).tobytes())
    subprocess.run([exe, "csd", fin, fout], check=True)
    raw = open(fout, "rb").read()
    mode, frames, nseg, nbins = struct.unpack("4i", raw[:16])
    rows = max(nx, ny)
    out = np.frombuffer(raw, np.float32, rows * nbins * (1 if coherence else 2), 16)
    out = out.reshape(rows, nbins) if coherence else out.reshape(rows, nbins, 2).astype(np.float64).view(np.complex128)[..., 0]
    return mode, nseg, out


def _pairs(nx, ny, ns, seed):
    """rows that share a component and add independent noise, at amplitudes 1 ... 3e-12, with an all-zero row; an offset so
    that detrending matters"""
    rng = np.random.default_rng(seed)
    amps = np.array([1.0, 1e-9, 0.0, 3e-12])
    common = rng.standard_normal(ns)
    x = (0.6 * common + rng.standard_normal((nx, ns)) + 0.3) * np.resize(amps, nx)[:, None]
    y = (0.6 * common + rng.standard_normal((ny, ns)) - 0.2) * np.resize(amps[::-1], ny)[:, None]
    return x.astype(np.float32), y.astype(np.float32)


# (nx, ny, ns, nperseg, noverlap, nfft, window, detrend, scaling, average, route: 0 mean, 1 median in smem, 2 workspace)
EMUL_CASES = [
    (4, 4, 200, 32, 16, None, "hann_periodic", "constant", "density", "mean", 0),     # even nfft, 11 segments
    (4, 4, 200, 30, 10, 45, "hamming", False, "spectrum", "mean", 0),                 # odd nfft > nperseg
    (4, 1, 243, 27, 0, 35, ("tukey", 0.25), "constant", "density", "median", 1),      # generic radix 7, y broadcast
    (1, 4, 300, 20, 5, 40, "hann_periodic", "constant", "spectrum", "median", 1),     # even nfft > nperseg, x broadcast
    (4, 4, 600, 16, 8, None, "hann_periodic", "constant", "density", "median", 1),    # 74 segments, still in shared memory
    (4, 4, 1600, 16, 8, None, "hann_periodic", "constant", "density", "median", 2),   # 199 segments: workspace median
    (4, 1, 1608, 16, 8, 27, "hamming", False, "spectrum", "median", 2),               # 200 segments (even), odd nfft
    (4, 4, 5500, 2520, None, None, "hann_periodic", "constant", "density", "mean", 0),  # nfft 2520, 3 segments
    (4, 4, 130, 13, 6, None, "hann_periodic", False, "density", "median", 1),         # prime nfft 13, 17 segments
    (4, 4, 96, 24, 12, 24, "explicit", "constant", "density", "mean", 0),             # explicit array window
]


def _check_pxy(p, x, y, kw):
    _, ref = sps.csd(x.astype(np.float64), y.astype(np.float64), **kw)
    _, pxx = sps.welch(x.astype(np.float64), **kw)
    _, pyy = sps.welch(y.astype(np.float64), **kw)
    ref, pxx, pyy = np.atleast_2d(ref), np.atleast_2d(pxx), np.atleast_2d(pyy)
    pxx, pyy = np.broadcast_to(pxx, ref.shape), np.broadcast_to(pyy, ref.shape)
    worst = 0.0
    for r in range(ref.shape[0]):
        den = float(np.max(np.sqrt(pxx[r] * pyy[r])))
        if den == 0.0:
            assert np.all(p[r] == 0), r
            continue
        e = float(np.max(np.abs(p[r] - ref[r]))) / den
        worst = max(worst, e)
        assert e <= 1e-5, (r, e)
    return worst


@pytest.mark.parametrize("case", EMUL_CASES)
def test_csd_body_emulation_vs_float64_scipy(exe, tmp_path, case):
    nx, ny, ns, nperseg, noverlap, nfft, window, detrend, scaling, average, route = case
    x, y = _pairs(nx, ny, ns, ns * 7 + nperseg)
    if window == "explicit":
        window = np.random.default_rng(ns).uniform(0.2, 1.0, nperseg)
    win, nperseg = dsp.welch_window(window, nperseg, ns)
    lay = dsp.welch_layout(ns, nperseg, noverlap, nfft)
    scale = dsp.welch_scale(win, 200., scaling)
    mode, nseg, out = _emulate(exe, str(tmp_path), x, y, lay, win, detrend == "constant", scale, False, average == "median")
    assert (mode, nseg) == (route, lay.nseg)
    _check_pxy(out, x, y, dict(fs=200., window=win, nperseg=nperseg, noverlap=lay.noverlap, nfft=lay.nfft, detrend=detrend,
                              scaling=scaling, average=average))


# (nx, ny, ns, nperseg, noverlap, nfft, window, detrend)
COH_CASES = [
    (4, 4, 200, 32, 16, None, "hann_periodic", "constant"),
    (4, 1, 200, 30, 10, 45, "hamming", False),
    (1, 4, 243, 27, 0, 35, ("tukey", 0.25), "constant"),
    (4, 4, 130, 13, 6, None, "hann_periodic", False),
]


@pytest.mark.parametrize("case", COH_CASES)
def test_coherence_body_emulation_vs_float64_scipy(exe, tmp_path, case):
    nx, ny, ns, nperseg, noverlap, nfft, window, detrend = case
    x, y = _pairs(nx, ny, ns, ns + nperseg)
    win, nperseg = dsp.welch_window(window, nperseg, ns)
    lay = dsp.welch_layout(ns, nperseg, noverlap, nfft)
    mode, nseg, out = _emulate(exe, str(tmp_path), x, y, lay, win, detrend == "constant", 1.0, True, False)
    assert (mode, nseg) == (0, lay.nseg)
    with np.errstate(invalid="ignore"):
        _, ref = sps.coherence(x.astype(np.float64), y.astype(np.float64), fs=200., window=win, nperseg=nperseg,
                               noverlap=lay.noverlap, nfft=lay.nfft, detrend=detrend)
    ref = np.broadcast_to(np.atleast_2d(ref), out.shape)
    assert np.array_equal(np.isnan(out), np.isnan(ref))
    ok = ~np.isnan(ref)
    assert ok.any() and np.max(np.abs(out[ok] - ref[ok])) <= 1e-4


def _select(exe, tmp, v):
    fin, fout = os.path.join(tmp, "m.bin"), os.path.join(tmp, "m.out")
    with open(fin, "wb") as f:
        f.write(struct.pack("2i", *v.shape))
        f.write(v.astype(np.float32).tobytes())
    subprocess.run([exe, "median", fin, fout], check=True)
    return np.fromfile(fout, np.float32)


@pytest.mark.parametrize("n", [1, 2, 3, 8, 113, 200, 233, 1000])
def test_signed_selection_matches_np_median(exe, tmp_path, n):
    rng = np.random.default_rng(n)
    rows = [
        rng.standard_normal(n),                                      # mixed signs
        np.round(rng.standard_normal(n) * 2) / 2,                    # many ties, zeros among them
        np.where(rng.random(n) < 0.5, -0.0, 0.0),                   # only +0 and -0
        -np.abs(rng.standard_normal(n)) * 1e-30,                     # all negative, tiny
        rng.standard_normal(n) * np.exp(rng.uniform(-60, 60, n)),    # magnitudes 1e-26 ... 1e26
        np.full(n, 3.5),                                             # all equal
        np.r_[np.full(n // 2, -1.0), np.full(n - n // 2, 1.0)],      # the two middle values straddle 0
    ]
    v = np.stack(rows).astype(np.float32)
    got = _select(exe, str(tmp_path), v)
    assert np.array_equal(got, np.median(v, axis=1)), (got, np.median(v, axis=1))
