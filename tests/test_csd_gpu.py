"""GPU: cross-spectral density and coherence (d4w_csd through rows.csd, dsp.csd and dsp.coherence) against float64 SciPy on
the same fp32-rounded input.  Rows mix a shared component with independent noise at amplitudes 1 ... 1e-12, plus an
all-zero row.  Tolerances per row: max |Pxy - Pxy_ref| <= 1e-5 max_k sqrt(Pxx_ref Pyy_ref), exact zeros for a zero row;
|Cxy - Cxy_ref| <= 1e-4 with NaN exactly where SciPy has NaN."""
import numpy as np
import pytest
import scipy.signal as sps

pytestmark = pytest.mark.gpu

AMPS = np.array([1.0, 1e-3, 1e-6, 1e-9, 1e-12, 0.0])
ODD_NFFT = {256: 275, 1000: 1125, 1024: 1215, 4096: 4725}        # odd lengths above nperseg, prime factors <= 61
WINDOWS = ["hann_periodic", "hamming", ("tukey", 0.25), "array"]
PAIRINGS = ["pairwise", "y broadcast", "x broadcast"]
WORST = {}


def _pairs(nx, ny, ns, seed):
    rng = np.random.default_rng(seed)
    common = rng.standard_normal(ns)
    x = (0.7 * common + rng.standard_normal((nx, ns)) + 0.25) * np.resize(AMPS, nx)[:, None]
    ya = np.resize(AMPS[::-1], ny) if ny > 1 else np.ones(1)            # a single (reference) row is live
    y = (0.7 * common + rng.standard_normal((ny, ns)) - 0.1) * ya[:, None]
    return x.astype(np.float32), y.astype(np.float32)


def _host(p):
    import torch
    return p.cpu().numpy() if isinstance(p, torch.Tensor) else p


def _check_pxy(p, x, y, what, **kw):
    x64, y64 = x.astype(np.float64), y.astype(np.float64)
    _, ref = sps.csd(x64, y64, **kw)
    _, pxx = sps.welch(x64, **kw)
    _, pyy = sps.welch(y64, **kw)
    p = _host(p)
    assert p.shape == ref.shape, (what, p.shape, ref.shape)
    ref2 = np.atleast_2d(ref)
    pxx, pyy = np.broadcast_to(np.atleast_2d(pxx), ref2.shape), np.broadcast_to(np.atleast_2d(pyy), ref2.shape)
    worst = 0.0
    for r, (a, b) in enumerate(zip(np.atleast_2d(p), ref2)):
        den = float(np.max(np.sqrt(pxx[r] * pyy[r])))
        if den == 0.0:
            assert np.all(a == 0), (what, r)
            continue
        e = float(np.max(np.abs(a - b))) / den
        worst = max(worst, e)
        assert e <= 1e-5, (what, r, e)
    WORST["csd " + what] = worst
    return worst


def _check_coh(c, x, y, what, **kw):
    with np.errstate(invalid="ignore"):
        _, ref = sps.coherence(x.astype(np.float64), y.astype(np.float64), **kw)
    c = _host(c)
    assert c.shape == ref.shape, (what, c.shape, ref.shape)
    assert np.array_equal(np.isnan(c), np.isnan(ref)), what
    ok = ~np.isnan(ref)
    worst = float(np.max(np.abs(c[ok] - ref[ok]))) if ok.any() else 0.0
    assert worst <= 1e-4, (what, worst)
    WORST["coherence " + what] = worst
    return worst


def _pair_shapes(pairing, nrows):
    return {"pairwise": (nrows, nrows), "y broadcast": (nrows, 1), "x broadcast": (1, nrows)}[pairing]


@pytest.mark.parametrize("nperseg", [256, 1000, 1024, 4096])
@pytest.mark.parametrize("noverlap", ["default", 0, "3/4"])
@pytest.mark.parametrize("odd_nfft", [False, True])
@pytest.mark.parametrize("window", WINDOWS, ids=lambda w: w if isinstance(w, str) else "tukey")
def test_csd_and_coherence_vs_scipy(nperseg, noverlap, odd_nfft, window):
    import torch
    import das4whales_b200 as dw
    nov = None if noverlap == "default" else 0 if noverlap == 0 else 3 * nperseg // 4
    nfft = ODD_NFFT[nperseg] if odd_nfft else None
    ns = 7 * nperseg + 37
    win = np.random.default_rng(nperseg).uniform(0.1, 1.0, nperseg) if window == "array" else window
    case = 0
    for scaling in ("density", "spectrum"):
        for average in ("mean", "median"):
            pairing = PAIRINGS[case % 3]
            tensor = case % 2 == 1
            case += 1
            nx, ny = _pair_shapes(pairing, 6)
            x, y = _pairs(nx, ny, ns, nperseg + 7 * (nov or 1) + case)
            if pairing == "y broadcast" and odd_nfft:
                y = y[0]                                                  # a 1-D row broadcasts like [1, ns]
            kw = dict(fs=200., window=win, nperseg=nperseg, noverlap=nov, nfft=nfft, scaling=scaling, average=average)
            args = (torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()) if tensor else (x, y)
            f, p = dw.dsp.csd(*args, **kw)
            assert isinstance(f, np.ndarray) and f.dtype == np.float64
            assert np.array_equal(f, np.fft.rfftfreq(nfft or nperseg, 1 / 200.))
            if tensor:
                assert isinstance(p, torch.Tensor) and p.is_cuda and p.dtype == torch.complex64
            else:
                assert isinstance(p, np.ndarray) and p.dtype == np.complex128
            _check_pxy(p, x, y, f"nperseg={nperseg} noverlap={nov} nfft={nfft} window={window} {scaling} {average} {pairing}",
                       **kw)
    nx, ny = _pair_shapes(PAIRINGS[nperseg % 3], 6)
    x, y = _pairs(nx, ny, ns, nperseg + 1)
    kw = dict(fs=200., window=win, nperseg=nperseg, noverlap=nov, nfft=nfft)
    f, c = dw.dsp.coherence(x, y, **kw)
    assert isinstance(c, np.ndarray) and c.dtype == np.float64
    _check_coh(c, x, y, f"nperseg={nperseg} noverlap={nov} nfft={nfft} window={window}", **kw)
    _, ct = dw.dsp.coherence(torch.from_numpy(x).cuda(), y, **kw)                   # one tensor: both go to the device
    assert isinstance(ct, torch.Tensor) and ct.is_cuda and ct.dtype == torch.float32
    assert np.array_equal(ct.cpu().numpy(), c.astype(np.float32), equal_nan=True)


def test_one_d_and_detrend_false():
    import torch
    import das4whales_b200 as dw
    x, y = _pairs(1, 1, 9000, 3)
    for detrend in ("constant", False):
        kw = dict(fs=200., nperseg=512, detrend=detrend)
        f, p = dw.dsp.csd(x[0], y[0], **kw)
        assert p.shape == (257,) and p.dtype == np.complex128
        _check_pxy(p, x[0], y[0], f"1-D detrend={detrend}", **kw)
        f, c = dw.dsp.coherence(torch.from_numpy(x[0]).cuda(), torch.from_numpy(y[0]).cuda(), **kw)
        assert tuple(c.shape) == (257,)
        _check_coh(c, x[0], y[0], f"1-D detrend={detrend}", **kw)
    _, p = dw.dsp.csd(x, y, nperseg=512)                                          # [1, ns] with [1, ns]: [1, nbins]
    assert p.shape == (1, 257)


def test_neighbour_coherence_synthetic_record():
    """coherence(x[:-1], x[1:]) at 11 020 x 12 000 (synth.synth_strain), every row: the two row ranges of one contiguous
    tensor are passed without a copy"""
    import das4whales_b200 as dw
    from das4whales_b200 import synth
    nx, ns = 11020, 12000
    xt = synth.synth_strain(nx, ns, seed=7)
    x = xt.cpu().numpy()
    for nperseg in (256, 1024):
        f, c = dw.dsp.coherence(xt[:-1], xt[1:], fs=200., nperseg=nperseg)
        assert tuple(c.shape) == (nx - 1, nperseg // 2 + 1)
        w = _check_coh(c, x[:-1], x[1:], f"neighbours 11020x12000 nperseg={nperseg}", fs=200., nperseg=nperseg)
        print(f"neighbour coherence 11020x12000 nperseg={nperseg}: worst |dC| {w:.2e}")
    kw = dict(fs=200., nperseg=1024)
    f, p = dw.dsp.csd(xt[:-1], xt[1:], **kw)
    sample = np.r_[0:4, 5000:5004, nx - 5:nx - 1]
    _check_pxy(p[sample], x[sample], x[sample + 1], "neighbours 11020x12000 sample", **kw)


def test_workspace_median_reference_row():
    """csd of 64 rows of 120 000 samples against one reference row, nperseg 1024: 233 segments, so the median goes through
    the workspace and the signed selection; and 240 segments (an even count)"""
    import torch
    import das4whales_b200 as dw
    x, y = _pairs(64, 1, 120000, 233)
    assert dw.dsp.welch_layout(120000, 1024).nseg == 233
    xt, yt = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    for ns, scaling in ((120000, "density"), (123392, "spectrum")):
        if ns != 120000:
            x, y = _pairs(64, 1, ns, 240)
            assert dw.dsp.welch_layout(ns, 1024).nseg == 240
            xt, yt = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
        kw = dict(fs=200., nperseg=1024, average="median", scaling=scaling)
        f, p = dw.dsp.csd(xt, yt, **kw)
        w = _check_pxy(p, x, y, f"workspace median {ns} samples {scaling}", **kw)
        print(f"csd workspace median, {ns} samples: worst {w:.2e}")


def test_nfft_2520():
    import torch
    import das4whales_b200 as dw
    x, y = _pairs(6, 6, 8000, 2520)
    t = np.arange(8000)
    tone = np.cos(2 * np.pi * 100 * t / 2520).astype(np.float32)
    x[:5] += tone * AMPS[:5, None].astype(np.float32)
    y[:5] += tone * AMPS[:5, None].astype(np.float32)
    for nperseg, nfft in ((2520, None), (2000, 2520)):
        for average in ("mean", "median"):
            kw = dict(fs=200., nperseg=nperseg, nfft=nfft, average=average)
            f, p = dw.dsp.csd(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), **kw)
            assert np.all(np.argmax(np.abs(p[:3].cpu().numpy()), axis=1) == 100)        # the tone dominates x and y
            _check_pxy(p, x, y, f"nfft=2520 nperseg={nperseg} {average}", **kw)
        # the coherence on the noise pairs: away from the tone, a row that is nearly a pure periodic tone has a spectrum of
        # float32 rounding noise, where Cxy is a ratio of noise in any float32 computation
        xc, yc = _pairs(6, 6, 8000, 2521)
        kw = dict(fs=200., nperseg=nperseg, nfft=nfft)
        _check_coh(dw.dsp.coherence(xc, yc, **kw)[1], xc, yc, f"nfft=2520 nperseg={nperseg}", **kw)


def test_nfft_8192():
    import das4whales_b200 as dw
    x, y = _pairs(6, 6, 30000, 8192)
    kw = dict(fs=200., nperseg=8192)
    _check_coh(dw.dsp.coherence(x, y, **kw)[1], x, y, "nfft=8192", **kw)
    _check_pxy(dw.dsp.csd(x, y, **kw)[1], x, y, "nfft=8192", **kw)


def test_nfft_limit_is_a_value_error():
    import das4whales_b200 as dw
    x = np.ones((2, 20000), np.float32)
    with pytest.raises(ValueError, match=r"nfft <= \d+ for the coherence"):
        dw.dsp.coherence(x, x + 1, nperseg=1024, nfft=12000)
    with pytest.raises(ValueError, match=r"nfft <= \d+ for the mean cross spectrum"):
        dw.dsp.csd(x, x + 1, nperseg=1024, nfft=16384)


def test_median_nfft_limit_is_its_own():
    """the workspace median keeps no bin sums: nfft 16 384, past the mean route's limit, works there, and its own limit is
    the one named when it is exceeded"""
    import re
    import das4whales_b200 as dw
    x, y = _pairs(6, 6, 20000, 16384)
    kw = dict(fs=200., nperseg=1024, nfft=16384, average="median")
    _check_pxy(dw.dsp.csd(x, y, **kw)[1], x, y, "median nfft=16384", **kw)
    with pytest.raises(ValueError, match=r"nfft <= \d+ for the median cross spectrum") as err:
        dw.dsp.csd(x, y, nperseg=1024, nfft=32768, average="median")
    assert int(re.search(r"nfft <= (\d+)", str(err.value)).group(1)) > 16384


def test_zero_rows():
    """a matrix of 0 rows against one row broadcasts to 0 rows, as NumPy broadcasts (0,) with (1,)"""
    import torch
    import das4whales_b200 as dw
    f, p = dw.dsp.csd(np.zeros((0, 512), np.float32), np.ones(512, np.float32), nperseg=64)
    assert p.shape == (0, 33) and p.dtype == np.complex128 and np.array_equal(f, np.fft.rfftfreq(64))
    f, c = dw.dsp.coherence(np.ones((1, 512), np.float32), torch.zeros((0, 512), device="cuda"), nperseg=64)
    assert tuple(c.shape) == (0, 33) and c.dtype == torch.float32


def test_y_is_x_is_real_and_equals_welch():
    import torch
    import das4whales_b200 as dw
    x, _ = _pairs(6, 1, 6000, 11)
    for arg in (x, torch.from_numpy(x).cuda()):
        for average in ("mean", "median"):
            f, p = dw.dsp.csd(arg, arg, fs=200., nperseg=512, average=average)
            fw, pw = dw.dsp.welch(arg, fs=200., nperseg=512, average=average)
            p, pw = _host(p), _host(pw)
            assert not np.iscomplexobj(p) and np.array_equal(p, pw) and np.array_equal(f, fw)
            x64 = x.astype(np.float64)
            assert not np.iscomplexobj(sps.csd(x64, x64, fs=200., nperseg=512, average=average)[1])
    with np.errstate(invalid="ignore"):
        f, c = dw.dsp.coherence(x, x, fs=200., nperseg=512)
    live = np.max(np.abs(x), axis=1) > 0
    assert np.all(np.isnan(c[~live])) and np.max(np.abs(c[live] - 1.0)) <= 1e-6
    _check_coh(c, x, x, "coherence(x, x)", fs=200., nperseg=512)


def test_rows_csd_strides_without_copies():
    """rows.csd on neighbour row ranges of one tensor, and on a broadcast row, against dsp.csd of copies"""
    import torch
    from das4whales_b200 import dsp, rows
    x, y = _pairs(6, 1, 4096, 5)
    xt, yt = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    win, _ = dsp.welch_window("hann_periodic", 256, 4096)
    scale = dsp.welch_scale(win, 1.0, "density")
    a = rows.csd(xt[:-1], xt[1:], 256, 128, 256, win, True, scale, "mean")
    b = rows.csd(xt[:-1].clone(), xt[1:].clone(), 256, 128, 256, win, True, scale, "mean")
    assert torch.equal(a, b)
    c = rows.csd(yt, xt, 256, 128, 256, win, True, scale, "mean", coherence=True)
    d = rows.csd(yt.expand(6, -1).contiguous(), xt, 256, 128, 256, win, True, scale, "mean", coherence=True)
    assert tuple(c.shape) == (6, 129) and torch.equal(torch.nan_to_num(c, 7.0), torch.nan_to_num(d, 7.0))


def test_report_worst_errors():
    """prints the worst error of every case above (run with -s)"""
    for kind in ("csd", "coherence"):
        ks = [k for k in WORST if k.startswith(kind)]
        if ks:
            k = max(ks, key=WORST.get)
            print(f"{kind} worst over {len(ks)} cases: {WORST[k]:.2e} ({k})")
