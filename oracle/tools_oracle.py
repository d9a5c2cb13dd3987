"""Float64 restatements of the reference's tools module chunk functions (das4whales/tools.py), on plain
ndarrays with time on the last axis (no xarray / dask).

    fan_mask             tools.py:30-48   the Gaussian-blurred speed fan (sigma = 40 there; dsp.fk_filt's is sigma = 20)
    fk_filt_chunk        tools.py:8-58    detrend, fft2, x float32(fan), ifft2, real
    energy_chunk         tools.py:84-101  sum of x^2 over the chunk
    filtfilt_chunk       tools.py:190-209 scipy.signal.filtfilt(b, a) along time
and the block maps tools.fk_filt / energy_TimeDomain / filtfilt apply with dask-style uniform chunks (the last one ragged).
"""
import numpy as np
from scipy import ndimage, signal


def fan_mask(shape, tint, fs, xint, dx, c_min, c_max, sigma=40):
    """(g - min g) / (max g - min g) of g = gaussian_filter(fan + fliplr(fan) - fan2 - fliplr(fan2), sigma), float64; NaN
    everywhere when g is constant (NumPy's 0 / 0)."""
    nx, ns = shape
    f = np.fft.fftshift(np.fft.fftfreq(ns, d=tint / fs))
    k = np.fft.fftshift(np.fft.fftfreq(nx, d=xint * dx))
    ff, kk = np.meshgrid(f, k)
    g = 1.0 * ((ff < kk * c_min) & (ff < -kk * c_min))
    g2 = 1.0 * ((ff < kk * c_max) & (ff < -kk * c_max))
    g = (g + np.fliplr(g)) - (g2 + np.fliplr(g2))
    g = ndimage.gaussian_filter(g, sigma)
    with np.errstate(invalid="ignore", divide="ignore"):
        return (g - np.min(g)) / (np.max(g) - np.min(g))


def fk_filt_chunk(data, tint, fs, xint, dx, c_min, c_max):
    """tools.fk_filt_chunk on an [nx, ns] ndarray: the mask is cast to float32 as the reference does (g.astype('f'))."""
    data = np.asarray(data, dtype=np.float64)
    spec = np.fft.fft2(signal.detrend(data))
    g = fan_mask(data.shape, tint, fs, xint, dx, c_min, c_max).astype(np.float32)
    return np.fft.ifft2(np.fft.ifftshift(np.fft.fftshift(spec) * g)).real


def energy_chunk(x):
    """tools._energy_TimeDomain_chunk: sum of x^2 along time, keeping the axis."""
    x = np.asarray(x, dtype=np.float64)
    return (x ** 2).sum(axis=-1, keepdims=True)


def filtfilt_chunk(x, b, a, **kwargs):
    """tools.filtfilt_chunk: scipy.signal.filtfilt(b, a, x) along time."""
    return signal.filtfilt(b, a, np.asarray(x, dtype=np.float64), axis=-1, **kwargs)


def blocks(n, c):
    """dask-style uniform blocks of an axis of n: [(start, stop)], the last one ragged; c = None is one block."""
    c = n if c is None else int(c)
    return [(s, min(s + c, n)) for s in range(0, n, c)]


def fk_filt(data, tint, fs, xint, dx, c_min, c_max, chunks=None):
    """tools.fk_filt: fk_filt_chunk mapped over the blocks of `chunks` = (cx, ct) (None: one block)."""
    data = np.asarray(data, dtype=np.float64)
    cx, ct = (None, None) if chunks is None else chunks
    out = np.empty_like(data)
    for r0, r1 in blocks(data.shape[0], cx):
        for t0, t1 in blocks(data.shape[1], ct):
            out[r0:r1, t0:t1] = fk_filt_chunk(data[r0:r1, t0:t1], tint, fs, xint, dx, c_min, c_max)
    return out


def energy_time_domain(x, chunk=None):
    """tools.energy_TimeDomain: [..., ceil(ns / chunk)], sum of x^2 over every time chunk."""
    x = np.asarray(x, dtype=np.float64)
    return np.concatenate([energy_chunk(x[..., t0:t1]) for t0, t1 in blocks(x.shape[-1], chunk)], axis=-1)


def filtfilt(x, b, a, chunk=None, **kwargs):
    """tools.filtfilt: filtfilt_chunk of every time chunk."""
    x = np.asarray(x, dtype=np.float64)
    return np.concatenate([filtfilt_chunk(x[..., t0:t1], b, a, **kwargs) for t0, t1 in blocks(x.shape[-1], chunk)], axis=-1)
