"""CPU: the Welch PSD's host side -- dsp.welch_layout / welch_window / welch_scale against SciPy, and every ValueError of
dsp.welch -- and the kernel body (csrc/welch_kernels.cuh welch_body) run block by block on the host
(tests/host_emul/welch_emul.cu) against float64 scipy.signal.welch."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest
import scipy.signal as sps
from scipy.signal import _spectral_py

from conftest import ROOT
from das4whales_b200 import dsp, tools

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
EMUL = os.path.join(ROOT, "tests", "host_emul")

LAYOUTS = [(ns, nperseg, noverlap, nfft, chunk)
           for ns, chunk in ((1000, None), (12000, 3000), (257, 100))
           for nperseg, noverlap, nfft in ((64, None, None), (100, 0, 125), (33, 24, 35), (100, 99, None), (7, 3, 7))
           if nperseg <= (chunk or ns)]


@pytest.mark.parametrize("ns,nperseg,noverlap,nfft,chunk", LAYOUTS)
def test_layout_matches_scipy(ns, nperseg, noverlap, nfft, chunk):
    lay = dsp.welch_layout(ns, nperseg, noverlap, nfft, chunk)
    c = ns if chunk is None else chunk
    assert lay.chunk == c and lay.nchunks == ns // c
    assert lay.nfft == (nperseg if nfft is None else nfft)
    assert lay.noverlap == (nperseg // 2 if noverlap is None else noverlap) and lay.step == nperseg - lay.noverlap
    _, t, s = sps.spectrogram(np.zeros(c), nperseg=nperseg, noverlap=lay.noverlap, nfft=lay.nfft)
    assert lay.nseg == t.size == s.shape[-1]
    assert lay.nbins == s.shape[0]
    f, _ = sps.welch(np.zeros(c), fs=200., nperseg=nperseg, noverlap=lay.noverlap, nfft=lay.nfft)
    assert np.array_equal(f, np.fft.rfftfreq(lay.nfft, 1 / 200.))
    assert lay.median_bias == pytest.approx(_spectral_py._median_bias(lay.nseg), rel=1e-15, abs=0)


@pytest.mark.parametrize("n", [1, 2, 3, 4, 9, 74, 233])
def test_median_bias(n):
    lay = dsp.welch_layout(n + 1, 2, 1)
    assert lay.nseg == n
    assert lay.median_bias == pytest.approx(_spectral_py._median_bias(n), rel=1e-15, abs=0)


@pytest.mark.parametrize("window", ["hann_periodic", "hamming", ("tukey", 0.25)])
@pytest.mark.parametrize("scaling", ["density", "spectrum"])
def test_window_and_scale_match_scipy(window, scaling):
    win, nperseg = dsp.welch_window(window, 100, 1000)
    assert nperseg == 100 and np.array_equal(win, sps.get_window(window, 100))
    # a flat input gives |X_0|^2 * scale at DC: recover SciPy's scale from its own output
    x = np.ones(100)
    _, p = sps.welch(x, fs=200., window=window, nperseg=100, detrend=False, scaling=scaling)
    assert dsp.welch_scale(win, 200., scaling) * np.sum(win) ** 2 == pytest.approx(p[0], rel=1e-12)
    win2, n2 = dsp.welch_window(np.arange(5.0), None, 10)
    assert n2 == 5 and np.array_equal(win2, np.arange(5.0))


def test_default_nperseg_and_cut_warn_as_scipy():
    win, nperseg = dsp.welch_window("hann_periodic", None, 1000)
    assert nperseg == 256 and np.array_equal(win, sps.get_window("hann_periodic", 256))
    with pytest.warns(UserWarning) as ours:
        win, nperseg = dsp.welch_window("hann_periodic", None, 200)
    with pytest.warns(UserWarning) as theirs:
        f, p = sps.welch(np.zeros(200))
    assert nperseg == 200 and p.shape == (101,) and np.array_equal(win, sps.get_window("hann_periodic", 200))
    assert str(ours[0].message) == str(theirs[0].message)
    with pytest.warns(UserWarning):
        _, nperseg = dsp.welch_window(("tukey", 0.25), 300, 120)
    assert nperseg == 120


@pytest.mark.parametrize("kw,match", [
    (dict(ns=100, nperseg=32, noverlap=32), "noverlap"),
    (dict(ns=100, nperseg=32, nfft=31), "nfft"),
    (dict(ns=1000, nperseg=64, nfft=67), "61"),
    (dict(ns=1000, nperseg=64, nfft=2 * 67), "61"),
    (dict(ns=100, nperseg=64, chunk=50), "chunk"),
    (dict(ns=100, nperseg=64, chunk=101), "chunk"),
    (dict(ns=100, nperseg=0), "positive"),
    (dict(ns=0, nperseg=1), "empty"),
])
def test_layout_errors(kw, match):
    with pytest.raises(ValueError, match=match):
        dsp.welch_layout(**kw)


def test_welch_value_errors_before_any_device_work():
    x = np.zeros((3, 512))
    for kw in (dict(detrend="linear"), dict(detrend=lambda d: d), dict(return_onesided=False), dict(axis=0),
               dict(window=np.ones(100), nperseg=64), dict(window=np.ones((2, 64))), dict(average="max"),
               dict(scaling="power")):
        with pytest.raises(ValueError):
            dsp.welch(x, **kw)
    with pytest.raises(ValueError, match="real"):
        dsp.welch(x + 1j, nperseg=64)
    with pytest.raises(ValueError, match="3-D"):
        dsp.welch(np.zeros((2, 2, 64)))
    with pytest.raises(ValueError, match="longer"):
        dsp.welch(np.zeros(50), window=np.ones(64))
    with pytest.raises(ValueError, match="61"):
        dsp.welch(x, nperseg=64, nfft=71)
    with pytest.raises(ValueError, match="whole chunk"):
        tools.spec(np.zeros((2, 2999)))


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError):
        dsp.welch(np.zeros((2, 512)), nperseg=64)
    with pytest.raises(RuntimeError):
        tools.spec(np.zeros((2, 6000)))


# ------------------------------------------------------------------------------ host emulation of the kernel body
@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    out = os.path.join(str(tmp_path_factory.mktemp("welch")), "welch_emul")
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "--expt-relaxed-constexpr", "-arch=sm_90a", "-o", out,
                        os.path.join(EMUL, "welch_emul.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    return out


def _emulate(exe, tmp, x, chunk, lay, win, detrend, scale, median):
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    nrows, ns = x.shape
    with open(fin, "wb") as f:
        f.write(struct.pack("8i", nrows, ns, chunk, lay.nperseg, lay.step, lay.nfft, int(detrend), int(median)))
        f.write(struct.pack("d", scale))
        f.write(x.astype(np.float32).tobytes())
        f.write(np.asarray(win, np.float32).tobytes())
    subprocess.run([exe, fin, fout], check=True)
    raw = open(fout, "rb").read()
    mode, pairs, nseg, nbins = struct.unpack("4i", raw[:16])
    out = np.frombuffer(raw, np.float32, nrows * (ns // chunk) * nbins, 16).reshape(nrows, ns // chunk, nbins)
    return mode, nseg, out


# (ns, chunk, nperseg, noverlap, nfft, window, detrend, scaling, average, route: 0 mean, 1 median in smem, 2 workspace)
EMUL_CASES = [
    (200, 200, 32, 16, None, "hann_periodic", "constant", "density", "mean", 0),     # even nfft, 11 segments (odd)
    (200, 100, 30, 10, 45, "hamming", False, "spectrum", "mean", 0),                 # odd nfft > nperseg, 2 chunks
    (243, 243, 27, 0, 35, ("tukey", 0.25), "constant", "density", "median", 1),      # generic radix 7, 9 segments
    (300, 150, 20, 5, 40, "hann_periodic", "constant", "spectrum", "median", 1),     # even nfft > nperseg, 2 chunks
    (600, 600, 16, 8, None, "hann_periodic", "constant", "density", "median", 1),    # 74 segments, still in shared memory
    (640, 640, 16, 8, 27, "hamming", False, "spectrum", "median", 1),                # 79 segments, odd nfft
    (1600, 1600, 16, 8, None, "hann_periodic", "constant", "density", "median", 2),  # 199 segments: workspace median
    (1700, 1700, 16, 8, 27, "hamming", False, "spectrum", "median", 2),              # 211 segments, odd nfft
    (5500, 5500, 2520, None, None, "hann_periodic", "constant", "density", "mean", 0),   # nfft 2520 (a prime-factor plan
    (5500, 2750, 2000, 1500, 2520, "hamming", False, "spectrum", "median", 1),           # on the GPU), 3 and 2 segments
    (130, 130, 13, 6, None, "hann_periodic", False, "density", "median", 1),         # prime nfft 13, 17 segments
    (96, 96, 24, 12, 24, "explicit", "constant", "density", "mean", 0),              # 7 segments, explicit array window
]


@pytest.mark.parametrize("case", EMUL_CASES)
def test_body_emulation_vs_float64_scipy(exe, tmp_path, case):
    ns, chunk, nperseg, noverlap, nfft, window, detrend, scaling, average, route = case
    rng = np.random.default_rng(ns * 7 + nperseg)
    amps = np.array([1.0, 1e-9, 0.0, 3e-12])[:, None]
    x = ((rng.standard_normal((4, ns)) + 0.3) * amps).astype(np.float32)     # an offset so that detrending matters
    if window == "explicit":
        window = rng.uniform(0.2, 1.0, nperseg)
    win, nperseg = dsp.welch_window(window, nperseg, chunk)
    lay = dsp.welch_layout(ns, nperseg, noverlap, nfft, chunk)
    scale = dsp.welch_scale(win, 200., scaling)
    mode, nseg, out = _emulate(exe, str(tmp_path), x, chunk, lay, win, detrend == "constant", scale, average == "median")
    assert (mode, nseg) == (route, lay.nseg)
    for c in range(lay.nchunks):
        _, ref = sps.welch(x[:, c * chunk:(c + 1) * chunk].astype(np.float64), fs=200., window=win, nperseg=nperseg,
                           noverlap=lay.noverlap, nfft=lay.nfft, detrend=detrend, scaling=scaling, average=average)
        for r in range(x.shape[0]):
            den = np.max(ref[r])
            if den == 0:
                assert np.all(out[r, c] == 0), (r, c)
                continue
            assert np.max(np.abs(out[r, c] - ref[r])) <= 1e-5 * den, (r, c, np.max(np.abs(out[r, c] - ref[r])) / den)
