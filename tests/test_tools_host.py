"""CPU: the tools module -- the float64 restatements against the reference's own chunk functions (fixture), the device fan
design's host emulation against scipy.ndimage, the filtfilt route in float64, and argument checks that raise before any
device work."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest
import scipy.signal as sps

from conftest import ROOT
from oracle import dsp_oracle as O, tools_oracle as T, tools_golden as G

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
DX, FS = G.DX, G.FS


def test_fk_filt_oracle_is_the_reference(golden):
    g = golden("tools")
    for i, (nx, ns, cmin, cmax) in enumerate(G.FK_CASES):
        y = T.fk_filt_chunk(g[f"fk_x_{i}"], 1, FS, 1, DX, cmin, cmax)
        ref = g[f"fk_y_{i}"]
        assert np.array_equal(np.isnan(y), np.isnan(ref)), (nx, ns)
        assert np.nanmax(np.abs(y - ref), initial=0.0) <= 1e-12, (nx, ns)
    assert np.isnan(g["fk_y_4"]).all()                       # the reference's 2 x 5 case


def test_energy_and_filtfilt_oracles_are_the_reference(golden):
    g = golden("tools")
    for chunk in (3001, 1000, 333):
        ref = g[f"energy_{chunk}"]
        assert ref.shape == (5, -(-3001 // chunk))
        assert np.max(np.abs(T.energy_time_domain(g["energy_x"], chunk) - ref) / ref) <= 1e-12
    for i in range(len(G.IIR_CASES)):
        for chunk in (2600, 1000):
            ref = g[f"iir_y_{i}_{chunk}"]
            y = T.filtfilt(g["iir_x"], g[f"iir_b_{i}"], g[f"iir_a_{i}"], chunk)
            assert np.max(np.abs(y - ref)) <= 1e-12 * np.max(np.abs(ref)), (i, chunk)


def test_filtfilt_route_in_float64(golden):
    """tools.filtfilt runs sosfiltfilt(tf2sos(b, a), padlen = 3 max(len(a), len(b))): in float64 that route is filtfilt(b, a)
    to far inside the GPU tolerance (the order-8 band-pass in (b, a) form is the worst conditioned)."""
    g = golden("tools")
    x = g["iir_x"]
    for i in range(len(G.IIR_CASES)):
        b, a = g[f"iir_b_{i}"], g[f"iir_a_{i}"]
        y = sps.sosfiltfilt(sps.tf2sos(b, a), x, padlen=3 * max(len(a), len(b)))
        ref = g[f"iir_y_{i}_2600"]
        assert np.max(np.abs(y - ref)) <= 1e-5 * np.max(np.abs(ref)), i


def test_oracle_fan_is_dsp_fk_filt_mask_at_sigma_20():
    for shape in ((40, 240), (41, 239), (7, 3)):
        a = T.fan_mask(shape, 1, FS, 1, DX, 1450., 3400., sigma=20)
        b = O.fk_filt_mask(shape, 1, FS, 1, DX, 1450., 3400.)
        assert np.array_equal(a, b, equal_nan=True)


# (nx, ns, sigma, c_min, c_max): odd / even on both axes, a radius beyond one or both axes (with repeated reflection), and
# fans that blur to a constant (NaN everywhere)
EMUL_CASES = [(40, 240, 20, 1450., 3400.), (41, 239, 40, 1400., 3500.), (120, 33, 20, 1450., 3400.), (300, 600, 40, 1400., 3500.),
              (7, 3, 40, 10., 3500.), (6, 40, 20, 300., 3500.), (3, 70, 20, 300., 3400.), (51, 100, 5, 1400., 3400.),
              (2, 5, 20, 1400., 3500.), (3, 7, 40, 1400., 3500.)]


@pytest.fixture(scope="module")
def fan_exe(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("fan") / "fan_blur_emul")
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "--expt-relaxed-constexpr", "-arch=sm_90a", "-o", exe,
                        os.path.join(ROOT, "tests", "host_emul", "fan_blur_emul.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    return exe


@pytest.mark.parametrize("nx,ns,sigma,cmin,cmax", EMUL_CASES)
def test_fan_emulation_vs_scipy(fan_exe, tmp_path, nx, ns, sigma, cmin, cmax):
    """the device fan design's bodies (tools_kernels.cuh), CTA by CTA on the host, against scipy.ndimage in float64"""
    kval, fval = 1.0 / (nx * (1 * DX)), 1.0 / (ns * (1 / FS))
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("2i", nx, ns) + struct.pack("5d", kval, fval, cmin, cmax, sigma))
    r = subprocess.run([fan_exe, fin, fout], capture_output=True, text=True)
    assert r.returncode == 0 and "OK" in r.stdout, r.stderr
    y = np.fromfile(fout, dtype=np.float32).reshape(nx, ns)
    ref = O.fk_filt_mask((nx, ns), 1, FS, 1, DX, cmin, cmax) if sigma == 20 else \
        T.fan_mask((nx, ns), 1, FS, 1, DX, cmin, cmax, sigma=sigma)
    assert np.array_equal(np.isnan(y), np.isnan(ref))
    if not np.isnan(ref).all():
        assert np.max(np.abs(y - ref)) <= 2e-7


@pytest.fixture
def no_device(monkeypatch):
    from das4whales_b200 import dsp

    def refuse(*a, **k):
        raise AssertionError("device work before argument checks")
    monkeypatch.setattr(dsp, "_to_device", refuse)


def test_value_errors_before_any_device_work(no_device):
    from das4whales_b200 import tools
    x = np.zeros((4, 3000))
    b, a = sps.butter(4, 0.1)
    with pytest.raises(ValueError, match="padtype"):
        tools.filtfilt(x, b, a, padtype="even")
    with pytest.raises(ValueError, match="padlen"):
        tools.filtfilt(x, b, a, chunk=15)                    # padlen = 15
    with pytest.raises(ValueError, match="padlen"):
        tools.filtfilt(x, b, a, chunk=1000, padlen=1000)
    with pytest.raises(ValueError, match="padlen"):
        tools.filtfilt(x, b, a, chunk=2990)                  # the ragged last chunk of 10 samples
    bb, aa = sps.butter(34, 0.1)
    with pytest.raises(ValueError, match="second-order sections"):
        tools.filtfilt(x, bb, aa)
    with pytest.raises(ValueError, match="chunk"):
        tools.filtfilt(x, b, a, chunk=0)
    with pytest.raises(ValueError, match="chunk"):
        tools.energy_TimeDomain(x, chunk=-3)
    with pytest.raises(ValueError, match="real"):
        tools.energy_TimeDomain(x + 1j)
    with pytest.raises(ValueError, match="3-D"):
        tools.energy_TimeDomain(np.zeros((2, 2, 2)))
    with pytest.raises(ValueError, match="1-D"):
        tools.fk_filt(np.zeros(100), 1, FS, 1, DX, 1400., 3500.)
    with pytest.raises(ValueError, match="chunks"):
        tools.fk_filt(x, 1, FS, 1, DX, 1400., 3500., chunks=(2, 0))
    with pytest.raises(ValueError, match="chunks"):
        tools.fk_filt(x, 1, FS, 1, DX, 1400., 3500., chunks=(2.5, None))
