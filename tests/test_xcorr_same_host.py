"""CPU: the host layout of the "same"-mode matched filter (rows.same_mode_layout: prepended taps, lag offset, block length,
kept outputs per block and template spectra) drives a NumPy overlap-save that follows d4w_xcorr_same step by step -- block s
reads samples s * valid - lag0 .. (zero outside the row), one forward FFT per block serves every template, the first
`valid` outputs of each inverse are kept -- and must reproduce scipy.signal.correlate(x / max(x), c, mode='same') of
scripts/main_gabordetect.py:245, with all-zero output for rows whose maximum is <= 0."""
import numpy as np
import pytest
import scipy.signal as sp

from das4whales_b200.rows import same_mode_layout

FS = 200.0


def _hann_chirp(fmin, fmax, dur):
    t = np.arange(0, dur, 1 / FS)
    c = sp.chirp(t, f0=fmax, f1=fmin, t1=dur, method="hyperbolic")
    return np.hanning(len(c)) * c


def _overlap_save_same(x, templates):
    ns = x.shape[-1]
    taps, lag0, nb, valid, spec = same_mode_layout(templates, ns)
    out = np.zeros((len(templates), ns))
    m = np.max(x)
    if not m > 0:
        return out, (taps, lag0, nb, valid)
    xs = x / m
    for t0 in range(0, ns, valid):
        idx = t0 - lag0 + np.arange(nb)
        blk = np.where((idx >= 0) & (idx < ns), xs[np.clip(idx, 0, ns - 1)], 0.0)
        X = np.fft.fft(blk)
        keep = min(valid, ns - t0)
        for t in range(len(templates)):
            y = nb * np.fft.ifft(X * spec[t])              # the kernels' inverse transform is unnormalised
            out[t, t0:t0 + keep] = y.real[:keep]
    return out, (taps, lag0, nb, valid)


def _check(x, templates, tol=1e-12):
    got, (taps, lag0, nb, valid) = _overlap_save_same(x, templates)
    m = np.max(x)
    for t, c in enumerate(templates):
        ref = sp.correlate(x / m, c, mode="same", method="direct") if m > 0 else np.zeros_like(x)
        den = max(np.max(np.abs(ref)), 1e-300)
        assert np.max(np.abs(got[t] - ref)) <= tol * den, (len(c), len(x), t)
    return taps, lag0, nb, valid


HF = _hann_chirp(17.8, 28.8, 0.68)          # 136 taps
LF = _hann_chirp(14.7, 21.8, 0.78)          # 156 taps


def test_script_templates_and_layout():
    assert (len(HF), len(LF)) == (136, 156)
    rng = np.random.default_rng(0)
    x = rng.standard_normal(12000)
    taps, lag0, nb, valid = _check(x, [HF, LF])
    assert lag0 == 78 and len(taps[0]) == 78 - 68 + 136 and len(taps[1]) == 156
    assert np.all(taps[0][:10] == 0) and np.array_equal(taps[0][10:], HF)
    assert nb == 2520 and valid == nb - 156 + 1                     # prime-factor blocks for the script's notes


@pytest.mark.parametrize("L", [1, 2, 7, 136, 155, 156, 400, 401, 2500])
def test_odd_and_even_lengths(L):
    rng = np.random.default_rng(L)
    c = rng.standard_normal(L)
    for ns in (1200, 12001):
        _check(rng.standard_normal(ns) + 0.5, [c])


def test_two_lengths_one_table_set():
    rng = np.random.default_rng(1)
    a, b = rng.standard_normal(137), rng.standard_normal(400)        # odd + even, different lag offsets
    taps, lag0, nb, valid = _check(rng.standard_normal(5003), [a, b])
    assert lag0 == 200 and len(taps[0]) == 200 - 68 + 137 and len(taps[1]) == 400
    assert nb in (1250, 2500, 5000)                                   # Cooley-Tukey blocks above 315 taps


@pytest.mark.parametrize("ns", [2519, 2521, 4729, 4731, 7097])
def test_row_length_not_a_multiple_of_valid(ns):
    rng = np.random.default_rng(ns)
    _, _, nb, valid = _check(rng.standard_normal(ns), [HF, LF])
    assert ns % valid != 0


@pytest.mark.parametrize("ns", [1, 5, 77, 100, 155])
def test_row_shorter_than_template(ns):
    rng = np.random.default_rng(ns)
    _check(rng.standard_normal(ns) + 1.0, [HF, LF])


def test_rows_with_max_not_positive_are_zero():
    rng = np.random.default_rng(2)
    for x in (np.zeros(3000), -np.abs(rng.standard_normal(3000)) - 1e-3):
        got, _ = _overlap_save_same(x, [HF, LF])
        assert np.array_equal(got, np.zeros_like(got))
    x = np.zeros(3000)
    x[1234] = 2.5                                                     # a single positive sample is enough
    _check(x, [HF, LF])


def test_layout_rejects_what_one_pass_cannot_take():
    with pytest.raises(ValueError):
        same_mode_layout([np.ones(2501)], 10000)
    with pytest.raises(ValueError):
        same_mode_layout([], 10000)
