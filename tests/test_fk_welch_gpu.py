"""GPU: the f-k Welch spectrum (dsp.fk_welch, fk.FkWelch) against a float64 oracle computed on the device: detrend, then
window, then |fftshift(fft2)|^2 per segment, then the mean over time segments, then the density or spectrum scaling.

Segment shapes of each column route (single-level, two-level, pipelined two-level, chirp-z) with T1 = 1 and T1 = 3 time
splits, noverlap 0 and nperseg // 2, on data with a per-channel DC offset; Hann and boxcar windows with detrend 'constant'
and False; channel segments with overlap; a band; ndarray and tensor input.  Then three invariants: boxcar, no overlap,
no detrend and 'spectrum' scaling give fk_spectrum(nperseg=L) / (Lx L)^2; the density of white noise integrates to its
variance; the input is never modified.  The 10 000 x 120 000 case (19 overlapping segments of 12 000 samples) is compared
with the oracle run one segment at a time, when enough device memory is free."""
import os

import numpy as np
import pytest
import scipy.signal as sps

pytestmark = pytest.mark.gpu
DX, FS = 2.0419046878814697, 200.0
MAX_TOL, L2_TOL = 1e-4, 1e-5


@pytest.fixture(scope="module")
def fk():
    """The routes shapes pick by themselves: no D4W_* variable, and no plan cached under another environment."""
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from das4whales_b200 import _lib, fk
    _lib.lib()
    with pytest.MonkeyPatch.context() as mp:
        for k in [k for k in os.environ if k.startswith("D4W_")]:
            mp.delenv(k)
        fk.free_plans()
        yield fk
        fk.free_plans()
    torch.cuda.empty_cache()


def _window(w, n):
    return np.asarray(sps.get_window(w, n), dtype=np.float64) if isinstance(w, (str, tuple)) else np.asarray(w, np.float64)


def _scale(wt, wx, scaling, dxc=DX):
    if scaling == "density":
        return 1.0 / (FS * (1.0 / dxc) * np.sum(wt * wt) * np.sum(wx * wx))
    return 1.0 / (np.sum(wt) ** 2 * np.sum(wx) ** 2)


def _oracle(x, lay, wt, wx, detrend, scale, k_idx=None, f_idx=None):
    """float64 [nseg_x, k, f]: per channel segment, the mean over time segments of |fftshift(fft2(w * detrend(seg)))|^2,
    times scale, cut to the band (half-open index ranges; None is the whole axis)."""
    import torch
    x = torch.as_tensor(x).cuda()
    lx, l = lay.nperseg_x, lay.nperseg
    k_idx, f_idx = k_idx or (0, lx), f_idx or (0, l)
    wt64 = torch.as_tensor(wt, dtype=torch.float64, device=x.device)
    wx64 = torch.as_tensor(wx, dtype=torch.float64, device=x.device)
    out = []
    for c0 in lay.starts_x:
        acc = None
        for t0 in lay.starts:
            seg = x[c0:c0 + lx, t0:t0 + l].to(torch.float64)
            if detrend:
                seg = seg - seg.mean(dim=1, keepdim=True)
            p = (torch.fft.fftshift(torch.fft.fft2(seg * wx64[:, None] * wt64[None, :])).abs() ** 2)
            p = p[k_idx[0]:k_idx[1], f_idx[0]:f_idx[1]]
            acc = p if acc is None else acc + p
        out.append(acc * (scale / lay.nseg))
    return torch.stack(out)


def _check(p, ref, what):
    import torch
    p = torch.as_tensor(p, device=ref.device).to(torch.float64).reshape(ref.shape)
    d = p - ref
    emax = float(d.abs().max() / ref.abs().max())
    el2 = float(torch.linalg.vector_norm(d) / torch.linalg.vector_norm(ref))
    print(f"{what}: max-norm {emax:.2e}, l2 {el2:.2e}")
    assert emax <= MAX_TOL and el2 <= L2_TOL, (what, emax, el2)


def _data(nx, ns, seed):
    """standard normal noise on a per-channel DC offset of about 20 standard deviations (float32 CUDA)"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((nx, ns), device="cuda", generator=g)
    return x + 20.0 + 3.0 * torch.randn((nx, 1), device="cuda", generator=g)


def _idx(axis, vals):
    i0 = int(np.flatnonzero(axis == vals[0])[0])
    return i0, i0 + len(vals)


# (segment shape, record length, column scheme, T1): one segment shape per column route and time split
ROUTE_CASES = [((5510, 1200), 3000, 0, 1),      # single-level, dual cp.async
               ((64, 24000), 60000, 0, 3),      # single-level, time split T1 = 3
               ((6000, 1200), 3000, 2, 1),      # two-level, shared-memory level B
               ((400, 24000), 60000, 2, 3),     # two-level, T1 = 3
               ((10000, 2480), 6200, 3, 1),     # pipelined two-level
               ((4897, 1200), 3000, 4, 1)]      # chirp-z


@pytest.mark.parametrize("seg,ns,scheme,t1", ROUTE_CASES)
@pytest.mark.parametrize("half_overlap", [False, True])
def test_route_vs_float64(fk, seg, ns, scheme, t1, half_overlap):
    import torch
    import das4whales_b200 as dw
    lx, l = seg
    plan = fk.get_plan(lx, l, torch.cuda.current_device())
    assert (plan.col_scheme, plan.t1) == (scheme, t1), seg
    x = _data(lx, ns, lx + l + int(half_overlap))
    noverlap = l // 2 if half_overlap else 0
    lay = dw.dsp.fk_welch_layout(lx, ns, l, noverlap, None, None)
    wt, wx = _window("hann", l), _window("hann", lx)
    # half overlap: the default band (f >= 0, every k); no overlap: 0-50 Hz and a third of the wavenumber range
    kmax = 1.0 / (2 * DX) / 3
    kw = dict(k_range=(-kmax, kmax), f_range=(0., 50.)) if not half_overlap else {}
    p, f, k = dw.dsp.fk_welch(x, [0, lx, 1], DX, FS, nperseg=l, noverlap=noverlap, **kw)
    assert isinstance(p, torch.Tensor) and p.dtype == torch.float32 and p.shape == (len(k), len(f))
    freq, knum = np.fft.fftshift(np.fft.fftfreq(l, 1 / FS)), np.fft.fftshift(np.fft.fftfreq(lx, DX))
    ref = _oracle(x, lay, wt, wx, True, _scale(wt, wx, "density"), _idx(knum, k), _idx(freq, f))[0]
    _check(p, ref, f"{lx} x {l} (scheme {scheme}, T1 {t1}), {lay.nseg} segments, noverlap {noverlap}, "
                   f"{'f >= 0' if half_overlap else '0-50 Hz, |k| <= %.3f' % kmax}")
    del p, ref, x
    fk.free_plans()
    torch.cuda.empty_cache()


NX, NS, L = 120, 4000, 1200        # five half-overlapping segments; the last 400 samples are not used


@pytest.mark.parametrize("window", ["hann", "boxcar"])
@pytest.mark.parametrize("detrend", ["constant", False])
@pytest.mark.parametrize("scaling", ["density", "spectrum"])
def test_windows_detrend_and_scaling(fk, window, detrend, scaling):
    import das4whales_b200 as dw
    x = _data(NX, NS, 5).cpu().numpy()
    keep = x.copy()
    p, f, k = dw.dsp.fk_welch(x, [0, NX, 1], DX, FS, nperseg=L, window=window, window_x=window, detrend=detrend,
                              scaling=scaling, f_range=(-np.inf, np.inf))
    assert np.array_equal(x, keep)
    assert isinstance(p, np.ndarray) and p.dtype == np.float64 and p.shape == (NX, L)
    assert np.array_equal(f, np.fft.fftshift(np.fft.fftfreq(L, 1 / FS))) and np.array_equal(k, np.fft.fftshift(np.fft.fftfreq(NX, DX)))
    lay = dw.dsp.fk_welch_layout(NX, NS, L, None, None, None)
    assert lay.nseg == 5
    wt, wx = _window(window, L), _window(window, NX)
    _check(p, _oracle(x, lay, wt, wx, detrend == "constant", _scale(wt, wx, scaling))[0],
           f"{window}, detrend {detrend!r}, {scaling}")


def test_channel_segments_with_overlap(fk):
    """nperseg_x = 120 with 60 channels of overlap over 330 channels: four channel segments (the last 30 channels are not
    used), each its own f-k plane; a channel-spacing step of 2 and an array time window; ndarray and tensor input."""
    import torch
    import das4whales_b200 as dw
    nx, ns, lx = 330, 4000, 120
    xt = _data(nx, ns, 7)
    keep = xt.clone()
    wt = sps.windows.tukey(L, 0.25)
    sel = [0, nx * 2, 2]
    kw = dict(nperseg=L, noverlap=300, window=wt, nperseg_x=lx, noverlap_x=60, window_x=("tukey", 0.5), f_range=(10., 60.))
    pt, f, k, c0 = dw.dsp.fk_welch(xt, sel, DX, FS, **kw)
    assert torch.equal(xt, keep)
    assert list(c0) == [0, 60, 120, 180]
    assert pt.shape == (4, lx, len(f)) and pt.dtype == torch.float32 and pt.is_cuda
    lay = dw.dsp.fk_welch_layout(nx, ns, L, 300, lx, 60)
    wx = _window(("tukey", 0.5), lx)
    freq = np.fft.fftshift(np.fft.fftfreq(L, 1 / FS))
    assert np.array_equal(k, np.fft.fftshift(np.fft.fftfreq(lx, 2 * DX)))
    ref = _oracle(xt, lay, wt, wx, True, _scale(wt, wx, "density", 2 * DX), None, _idx(freq, f))
    _check(pt, ref, "4 channel segments, noverlap_x 60, 10-60 Hz")
    x = xt.cpu().numpy()
    p, f2, k2, c02 = dw.dsp.fk_welch(x, sel, DX, FS, **kw)
    assert isinstance(p, np.ndarray) and p.dtype == np.float64 and np.array_equal(c02, c0)
    assert np.array_equal(p, pt.cpu().numpy().astype(np.float64))
    # the segments really differ along the cable: a signal on the last channels only shows in the last segment
    x[-100:] += 5.0 * np.sin(2 * np.pi * 30.0 * np.arange(ns) / FS)
    p2 = dw.dsp.fk_welch(x, sel, DX, FS, **kw)[0]
    assert np.array_equal(p2[:2], p[:2]) and not np.array_equal(p2[3], p[3])


def test_boxcar_spectrum_is_fk_spectrum_over_blocks(fk):
    import das4whales_b200 as dw
    x = _data(NX, NS, 9)
    p = dw.dsp.fk_welch(x, [0, NX, 1], DX, FS, nperseg=L, noverlap=0, window="boxcar", window_x="boxcar", detrend=False,
                        scaling="spectrum")[0]
    q = dw.dsp.fk_spectrum(x, [0, NX, 1], DX, FS, nperseg=L)[0] / float(NX * L) ** 2
    d = float((p - q).abs().max() / q.abs().max())
    print(f"boxcar / no overlap / no detrend / spectrum against fk_spectrum(nperseg): max-norm {d:.2e}")
    assert d <= 1e-6


def test_white_noise_density_integrates_to_its_variance(fk):
    import torch
    import das4whales_b200 as dw
    nx, ns, sigma = 256, 12000, 0.37
    x = sigma * torch.randn((nx, ns), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    p, f, k = dw.dsp.fk_welch(x, [0, nx, 1], DX, FS, nperseg=L, f_range=(-np.inf, np.inf))
    total = float(p.to(torch.float64).sum()) * (FS / L) * (1.0 / DX / nx)
    print(f"white noise of variance {sigma ** 2:.4f}: integrated density {total:.4f}")
    assert abs(total / sigma ** 2 - 1.0) < 0.02


def test_object_reuse_and_planner_errors(fk):
    import torch
    import das4whales_b200 as dw
    x = _data(NX, NS, 13)
    wt, wx = _window("hann", L), _window("hann", NX)
    est = fk.FkWelch((NX, NS), (NX, L), (0, NX), (0, L), wt, wx, True, 1.0)
    assert est.out_shape == (1, NX, L) and est.layout.nseg == 5
    p = est(x)
    out = torch.empty_like(p)
    assert est(x, out=out) is out and torch.equal(out, p), "two runs differ"
    with pytest.raises(ValueError, match="records of"):
        est(x[:, :L].contiguous())
    with pytest.raises(ValueError, match="supported_shape"):          # 67 samples: a prime factor above 61
        dw.dsp.fk_welch(x, [0, NX, 1], DX, FS, nperseg=67)
    with pytest.raises(ValueError, match="window"):
        fk.FkWelch((NX, NS), (NX, L), (0, NX), (0, L), wt[:-1], wx, True, 1.0)


# ---- full size -------------------------------------------------------------------------------------------------------
FX, FNS, FL = 10000, 120000, 12000


def test_fullsize_vs_float64(fk):
    """10 000 x 120 000, nperseg 12 000 with 6 000 of overlap (19 segments), Hann windows, detrend 'constant', the default
    band, against the float64 oracle run one segment at a time on the same GPU."""
    import torch
    import das4whales_b200 as dw
    need = FX * FNS * 4 + FX * FL * (4 + 8 + 16 * 3) + FX * (FL // 2) * 12
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 1e9:.1f} GB of free device memory; {free / 1e9:.1f} GB are free")
    x = _data(FX, FNS, 99)
    p, f, k = dw.dsp.fk_welch(x, [0, FX, 1], DX, FS, nperseg=FL, noverlap=FL // 2)
    assert p.shape == (FX, FL // 2) and f[0] == 0.0
    fk.free_plans()
    torch.cuda.empty_cache()
    lay = dw.dsp.fk_welch_layout(FX, FNS, FL, FL // 2, None, None)
    assert lay.nseg == 19
    wt, wx = _window("hann", FL), _window("hann", FX)
    ref = _oracle(x, lay, wt, wx, True, _scale(wt, wx, "density"), None, (FL // 2, FL))[0]
    _check(p, ref, f"full size {FX} x {FNS}, 19 segments of {FL}, default band")
    del x, p, ref
    torch.cuda.empty_cache()
