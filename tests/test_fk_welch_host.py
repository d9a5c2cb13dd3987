"""CPU: the f-k Welch spectrum's segment geometry (dsp.fk_welch_layout) against a direct enumeration of the segments, the
ValueErrors dsp.fk_welch raises before any device work, and the staging body (csrc/fk_welch.cuh, k_fk_segment_stage) run
on the host against NumPy float64: per-(channel, segment) mean removal, both windows, channel and time offsets, both
row routes (shared memory and re-read), on data with a large DC offset."""
import os
import struct
import subprocess

import numpy as np
import pytest
import scipy.signal as sps

import das4whales_b200 as dw
from test_hilbert_czt_host import NVCC, _compile

DX, FS = 2.0419046878814697, 200.0


def _enumerate(n, nper, nover):
    """Starts of every whole segment, found by walking the axis."""
    step, starts, s = nper - nover, [], 0
    while s + nper <= n:
        starts.append(s)
        s += step
    return starts


@pytest.mark.parametrize("ns,nperseg,noverlap", [(1000, 100, 50), (1000, 100, 0), (1000, 1000, None), (1000, 1000, 999),
                                                 (1037, 100, 30), (1099, 100, None), (120000, 12000, 6000),
                                                 (12000, 1200, None), (10, 1, 0), (257, 256, 255), (999, 333, 1),
                                                 (500, 128, -22)])
def test_layout_matches_enumeration(ns, nperseg, noverlap):
    lay = dw.dsp.fk_welch_layout(40, ns, nperseg, noverlap, None, None)
    nover = nperseg // 2 if noverlap is None else noverlap
    starts = _enumerate(ns, nperseg, nover)
    assert (lay.nperseg, lay.noverlap, lay.step) == (nperseg, nover, nperseg - nover)
    assert lay.nseg == len(starts) and list(lay.starts) == starts
    assert lay.starts[-1] + nperseg <= ns < lay.starts[-1] + lay.step + nperseg     # a trailing partial segment is dropped
    assert (lay.nperseg_x, lay.nseg_x, lay.starts_x) == (40, 1, (0,))               # one segment spans every channel
    # the channel axis follows the same rules
    lay = dw.dsp.fk_welch_layout(ns, 64, 16, None, nperseg, noverlap)
    assert (lay.nperseg_x, lay.noverlap_x, lay.step_x) == (nperseg, nover, nperseg - nover)
    assert lay.nseg_x == len(starts) and list(lay.starts_x) == starts
    assert (lay.nperseg, lay.noverlap, lay.nseg) == (16, 8, (64 - 16) // 8 + 1)


def test_layout_defaults():
    lay = dw.dsp.fk_welch_layout(100, 1000, None, None, None, 7)           # noverlap_x is ignored without nperseg_x
    assert (lay.nperseg, lay.noverlap, lay.step, lay.nseg) == (256, 128, 128, (1000 - 256) // 128 + 1)
    assert (lay.nperseg_x, lay.noverlap_x, lay.nseg_x) == (100, 0, 1)
    lay = dw.dsp.fk_welch_layout(11020, 12000, 1200, None, 1102, None)
    assert (lay.nseg, lay.step, lay.nseg_x, lay.step_x) == (19, 600, 19, 551) and lay.starts_x[-1] == 18 * 551


@pytest.mark.parametrize("args,match", [((40, 1000, 0, None, None, None), "nperseg"), ((40, 1000, 1001, None, None, None), "nperseg"),
                                        ((40, 1000, 100, 100, None, None), "overlap"), ((40, 1000, 100, 150, None, None), "overlap"),
                                        ((40, 1000, 100, None, 41, None), "nperseg_x"), ((40, 1000, 100, None, 0, None), "nperseg_x"),
                                        ((40, 1000, 100, None, 20, 20), "overlap"), ((0, 1000, 100, None, None, None), "empty"),
                                        ((40, 0, 100, None, None, None), "empty"), ((40, 100, None, None, None, None), "nperseg")])
def test_layout_value_errors(args, match):
    with pytest.raises(ValueError, match=match):
        dw.dsp.fk_welch_layout(*args)


def test_fk_welch_value_errors_before_any_device_work():
    x = np.zeros((40, 1000), dtype=np.float32)
    sel = [0, 40, 1]
    for bad in (x[0], x[None], x.astype(np.complex64)):
        with pytest.raises(ValueError, match="real 2-D"):
            dw.dsp.fk_welch(bad, sel, DX, FS)
    with pytest.raises(ValueError, match="detrend"):
        dw.dsp.fk_welch(x, sel, DX, FS, detrend="linear")
    with pytest.raises(ValueError, match="scaling"):
        dw.dsp.fk_welch(x, sel, DX, FS, scaling="psd")
    for kw, match in ((dict(nperseg=0), "nperseg"), (dict(nperseg=1001), "nperseg"), (dict(nperseg_x=41), "nperseg_x"),
                      (dict(nperseg_x=-1), "nperseg_x"), (dict(nperseg=100, noverlap=100), "overlap"),
                      (dict(nperseg_x=20, noverlap_x=25), "overlap"), (dict(nperseg=100, window=np.ones(99)), "len"),
                      (dict(window=np.ones(1001)), "longer"), (dict(window_x=np.ones(39)), "len"),
                      (dict(nperseg_x=20, window_x=np.ones(40)), "len"), (dict(window=np.ones((2, 50))), "1-D"),
                      (dict(f_range=(150., 200.)), "selects no"), (dict(k_range=(1.0, 2.0)), "selects no")):
        with pytest.raises(ValueError, match=match):
            dw.dsp.fk_welch(x, sel, DX, FS, **kw)


# ---- the staging body on the host -------------------------------------------------------------------------------------
needs_nvcc = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return _compile(tmp_path_factory, "fk_welch_emul")


def _stage(exe, tmp, x, c0, lx, t0, l, step, nseg, wx, wt, detrend, smem_row, pad):
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("11i", *x.shape, c0, lx, t0, l, step, nseg, int(detrend), int(smem_row), pad))
        for a in (x, wx, wt):
            f.write(np.ascontiguousarray(a, dtype=np.float32).tobytes())
    subprocess.run([exe, fin, fout], check=True)
    return np.fromfile(fout, dtype=np.float32).reshape(nseg, lx * l + pad)


@needs_nvcc
@pytest.mark.parametrize("nx,ns,c0,lx,t0,l,step,nseg,pad", [(12, 1000, 0, 12, 0, 100, 50, 19, 0),
                                                             (30, 777, 5, 11, 13, 120, 120, 5, 4),
                                                             (9, 4099, 2, 7, 1, 1200, 600, 5, 8),
                                                             (7, 1000, 1, 5, 3, 99, 45, 7, 3),
                                                             (5, 300, 4, 1, 299, 1, 1, 1, 0)])
def test_stage_body_against_float64(exe, tmp_path, nx, ns, c0, lx, t0, l, step, nseg, pad):
    rng = np.random.default_rng(nx * 31 + l)
    x = (1000.0 + rng.standard_normal((nx, ns)) + 50.0 * rng.standard_normal((nx, 1))).astype(np.float32)
    wt = sps.get_window("hann", l) if l > 1 else np.ones(1)
    wx = sps.get_window(("tukey", 0.3), lx) + 0.25
    for detrend in (True, False):
        outs = []
        for smem_row in (1, 0):
            got = _stage(exe, str(tmp_path), x, c0, lx, t0, l, step, nseg, wx, wt, detrend, smem_row, pad)
            assert np.all(got[:, lx * l:] == -7.0), "a write outside its segment"
            outs.append(got[:, :lx * l].reshape(nseg, lx, l))
        assert np.array_equal(outs[0], outs[1]), "the shared-memory and re-read routes differ"
        x64 = x.astype(np.float64)
        wx32, wt32 = wx.astype(np.float32).astype(np.float64), wt.astype(np.float32).astype(np.float64)
        for s in range(nseg):
            seg = x64[c0:c0 + lx, t0 + s * step:t0 + s * step + l]
            if detrend:
                seg = seg - seg.mean(axis=1, keepdims=True)
            ref = seg * wx32[:, None] * wt32[None, :]
            err = np.max(np.abs(outs[0][s] - ref)) / max(np.max(np.abs(ref)), 1e-30)
            assert err <= 1e-6, (detrend, s, err)
