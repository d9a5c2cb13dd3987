"""GPU: per-channel Welch PSD (d4w_welch through rows.welch, dsp.welch and tools.spec) against float64 SciPy on the same
fp32-rounded input.  Rows span amplitudes 1 ... 1e-12 plus an all-zero row, whose PSD must be exactly 0.  Tolerance per
(row, chunk): max |P - P_ref| <= 1e-5 max(P_ref of that row); over the whole array the parity contract of conftest.rel_err
(max-norm <= 1e-4, l2 <= 1e-5)."""
import numpy as np
import pytest
import scipy.signal as sps

from conftest import rel_err
from oracle import welch_oracle as O

pytestmark = pytest.mark.gpu

AMPS = np.array([1.0, 1e-3, 1e-6, 1e-9, 1e-12, 0.0])
ODD_NFFT = {256: 275, 1000: 1125, 1024: 1215, 4096: 4725}        # odd lengths above nperseg, prime factors <= 61
WINDOWS = ["hann_periodic", "hamming", ("tukey", 0.25), "array"]
WORST = {}


def _rows(nrows, ns, seed):
    rng = np.random.default_rng(seed)
    a = np.resize(AMPS, nrows)[:, None]
    return ((rng.standard_normal((nrows, ns)) + 0.25) * a).astype(np.float32)


def _check(p, ref, what):
    p = np.asarray(p, dtype=np.float64).reshape(ref.shape)
    rows_ = p.reshape(-1, p.shape[-1]) if p.ndim > 1 else p[None]
    refs = ref.reshape(-1, ref.shape[-1]) if ref.ndim > 1 else ref[None]
    worst = 0.0
    for i, (a, b) in enumerate(zip(rows_, refs)):
        den = float(np.max(b))
        if den == 0.0:
            assert np.all(a == 0.0), (what, i)
            continue
        e = float(np.max(np.abs(a - b))) / den
        worst = max(worst, e)
        assert e <= 1e-5, (what, i, e)
    mx, l2 = rel_err(p, ref)
    assert mx <= 1e-4 and l2 <= 1e-5, (what, mx, l2)
    WORST[what] = worst
    return worst


@pytest.mark.parametrize("nperseg", [256, 1000, 1024, 4096])
@pytest.mark.parametrize("noverlap", ["default", 0, "3/4"])
@pytest.mark.parametrize("odd_nfft", [False, True])
@pytest.mark.parametrize("window", WINDOWS, ids=lambda w: w if isinstance(w, str) else "tukey")
def test_welch_vs_scipy(nperseg, noverlap, odd_nfft, window):
    import torch
    import das4whales_b200 as dw
    nov = None if noverlap == "default" else 0 if noverlap == 0 else 3 * nperseg // 4
    nfft = ODD_NFFT[nperseg] if odd_nfft else None
    ns = 7 * nperseg + 37
    x = _rows(6, ns, nperseg + 7 * (nov or 1))
    win = np.random.default_rng(nperseg).uniform(0.1, 1.0, nperseg) if window == "array" else window
    xt = torch.from_numpy(x).cuda()
    case = 0
    for scaling in ("density", "spectrum"):
        for average in ("mean", "median"):
            kw = dict(fs=200., window=win, nperseg=nperseg, noverlap=nov, nfft=nfft, scaling=scaling, average=average)
            tensor, one_d = case % 2 == 1, case // 2 == 1
            case += 1
            arg = (xt if tensor else x)[case % 6] if one_d else (xt if tensor else x)
            f, p = dw.dsp.welch(arg, **kw)
            fr, ref = O.welch(x[case % 6] if one_d else x, **kw)
            assert isinstance(f, np.ndarray) and f.dtype == np.float64 and np.array_equal(f, fr)
            if tensor:
                assert isinstance(p, torch.Tensor) and p.is_cuda and p.dtype == torch.float32
                p = p.cpu().numpy()
            else:
                assert isinstance(p, np.ndarray) and p.dtype == np.float64
            assert p.shape == ref.shape
            _check(p, ref, f"welch nperseg={nperseg} noverlap={nov} nfft={nfft} window={window} {scaling} {average}")


def test_detrend_false_and_rows_welch_chunks():
    import torch
    from das4whales_b200 import dsp, rows
    x = _rows(6, 9000, 3)
    f, p = dsp.welch(x, nperseg=512, detrend=False, average="median")
    _check(p, O.welch(x, nperseg=512, detrend=False, average="median")[1], "welch detrend=False median")
    win, _ = dsp.welch_window("hamming", 500, 3000)
    lay = dsp.welch_layout(9000, 500, 100, 625, 3000)
    out = rows.welch(torch.from_numpy(x).cuda(), 500, lay.step, 625, win, True, dsp.welch_scale(win, 1.0, "spectrum"), "mean",
                     chunk=3000)
    assert tuple(out.shape) == (6, 3, 313)
    for c in range(3):
        ref = sps.welch(x[:, c * 3000:(c + 1) * 3000].astype(np.float64), window=win, nperseg=500, noverlap=100, nfft=625,
                        scaling="spectrum")[1]
        _check(out[:, c].cpu().numpy(), ref, f"rows.welch chunk {c}")


def test_tools_spec_reference_shape():
    """tools.spec at 11 020 x 12 000: 4 chunks of 3 000 samples, 4 segments of 1 024 each, every chunk of every channel"""
    import torch
    import das4whales_b200 as dw
    nx, ns = 11020, 12000
    x = _rows(nx, ns, 11)
    fr, ref = O.spec(x)
    f, p = dw.tools.spec(torch.from_numpy(x).cuda())
    assert tuple(p.shape) == (nx, 4, 513) and np.array_equal(f, fr)
    w = _check(p.cpu().numpy(), ref, "tools.spec 11020x12000")
    print(f"tools.spec 11020x12000: worst per-(row, chunk) error {w:.2e} of the row max")
    f1, p1 = dw.tools.spec(x[7])                                          # 1-D ndarray in, float64 out
    assert p1.shape == (4, 513) and p1.dtype == np.float64
    _check(p1, ref[7], "tools.spec 1-D")


def test_whole_row_median_workspace_route():
    """10 000 x 120 000, nperseg 1024: 233 segments per row, so the median goes through the workspace and d4w_row_median"""
    import torch
    import das4whales_b200 as dw
    nx, ns = 10000, 120000
    assert dw.dsp.welch_layout(ns, 1024).nseg == 233
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn((nx, ns), device="cuda", generator=g)
    x *= torch.from_numpy(np.resize(AMPS, nx).astype(np.float32)).cuda()[:, None]
    f, p = dw.dsp.welch(x, fs=200., nperseg=1024, average="median")
    assert tuple(p.shape) == (nx, 513)
    sample = np.r_[0:6, 1997, 4242, 6001:6007, nx - 6:nx]
    xs = x[torch.from_numpy(sample).cuda()].cpu().numpy()
    ref = O.welch(xs, fs=200., nperseg=1024, average="median")[1]
    w = _check(p[torch.from_numpy(sample).cuda()].cpu().numpy(), ref, "welch median 10000x120000")
    print(f"welch median 10000x120000: worst per-row error {w:.2e} of the row max")


@pytest.mark.parametrize("nperseg,nfft", [(2520, None), (2000, 2520), (1260, 2520)])
def test_nfft_2520_prime_factor_plan(nperseg, nfft):
    """2520 is the length whose fft plan carries the matched filter's prime-factor position table; the Welch kernel reads
    bins at the positions of the plan's own mixed-radix stages.  A tone at bin 100 must peak there, and every spectrum must
    match SciPy."""
    import torch
    import das4whales_b200 as dw
    ns = 8000
    t = np.arange(ns)
    x = _rows(6, ns, 2520)
    x[:5] += (np.cos(2 * np.pi * 100 * t / 2520) * AMPS[:5, None]).astype(np.float32)
    for average in ("mean", "median"):
        kw = dict(fs=200., nperseg=nperseg, nfft=nfft, average=average)
        f, p = dw.dsp.welch(torch.from_numpy(x).cuda(), **kw)
        p = p.cpu().numpy()
        assert np.all(np.argmax(p[:5], axis=1) == 100), np.argmax(p[:5], axis=1)
        _check(p, O.welch(x, **kw)[1], f"welch nfft=2520 nperseg={nperseg} {average}")


def test_median_in_shared_memory_past_64_segments():
    """nperseg 256 over 12 000 samples: 92 segments, ranked in shared memory"""
    import das4whales_b200 as dw
    x = _rows(6, 12000, 92)
    assert dw.dsp.welch_layout(12000, 256).nseg == 92
    for scaling in ("density", "spectrum"):
        f, p = dw.dsp.welch(x, fs=200., nperseg=256, average="median", scaling=scaling)
        _check(p, O.welch(x, fs=200., nperseg=256, average="median", scaling=scaling)[1], f"welch median 92 segments {scaling}")


def test_nfft_limit_is_a_value_error():
    import das4whales_b200 as dw
    x = np.zeros((2, 4096), np.float32)
    with pytest.raises(ValueError, match=r"nfft <= \d+"):
        dw.dsp.welch(x, nperseg=1024, nfft=32768)


def test_report_worst_errors():
    """prints the worst per-(row, chunk) error of every case above (run with -s)"""
    if WORST:
        k = max(WORST, key=WORST.get)
        print(f"welch worst over {len(WORST)} cases: {WORST[k]:.2e} ({k})")
