"""das4whales_b200.dsp -- drop-in for the hot-path functions of `das4whales.dsp`
(/root/reference/src/das4whales/dsp.py), same names / positional order / defaults, running
on hand-written sm_90a CUDA kernels (libd4w.so) instead of NumPy/SciPy.

Accepted data: `numpy.ndarray` (any float dtype; the result is a new float64 ndarray, as the
reference returns) or a CUDA `torch.Tensor` (float32; the result stays on the device).
"""
import numpy as np
import scipy.signal as sp

from . import _lib, fk as _fk
from . import rows as _rows


def _is_tensor(x):
    try:
        import torch
        return isinstance(x, torch.Tensor)
    except Exception:
        return False


def _to_device(x):
    """ndarray / tensor -> contiguous float32 CUDA tensor (chunked H2D, conversion on the GPU)."""
    torch = _fk._torch()
    if _is_tensor(x):
        if not x.is_cuda:
            x = x.cuda()
        return x.to(torch.float32).contiguous()
    a = np.asarray(x)
    if a.ndim == 1:
        a = a[None, :]
    dev = torch.cuda.current_device()
    out = torch.empty(a.shape, dtype=torch.float32, device=f"cuda:{dev}")
    step = max(1, (128 << 20) // max(1, a.shape[1] * a.dtype.itemsize))
    for r0 in range(0, a.shape[0], step):
        chunk = np.ascontiguousarray(a[r0:r0 + step])
        out[r0:r0 + step] = torch.from_numpy(chunk).to(out.device, non_blocking=False).to(torch.float32)
    return out


def _to_host64(y):
    """float32 CUDA tensor -> float64 ndarray (widened on the GPU, one D2H pass)."""
    torch = _fk._torch()
    out = np.empty(tuple(y.shape), dtype=np.float64)
    step = max(1, (128 << 20) // max(1, y.shape[-1] * 8)) if y.ndim == 2 else y.shape[0]
    if y.ndim != 2:
        return y.to(torch.float64).cpu().numpy()
    for r0 in range(0, y.shape[0], step):
        out[r0:r0 + step] = y[r0:r0 + step].to(torch.float64).cpu().numpy()
    return out


# ------------------------------------------------------------------------------ mask design
def _fftfreq_steps(trace_shape, selected_channels, dx, fs):
    nnx, nns = trace_shape
    # numpy.fft.fftfreq(n, d) multiplies integers by val = 1.0 / (n * d)  (dsp.py:129-130)
    fval = 1.0 / (nns * (1 / fs))
    kval = 1.0 / (nnx * (selected_channels[2] * dx))
    return kval, fval


def fk_filter_design(trace_shape, selected_channels, dx, fs, cs_min=1400, cp_min=1450, cp_max=3400, cs_max=3500):
    """Speed-fan f-k mask (reference: dsp.py:85-171).  Returns a lazy `FkMask`; `np.asarray`
    of it is the reference's Fortran-ordered float64 [channel x time sample] matrix."""
    kval, fval = _fftfreq_steps(trace_shape, selected_channels, dx, fs)
    np.seterr(invalid="ignore")      # side effect of the reference (dsp.py:133)
    return _fk.FkMask("fan", trace_shape, dict(kval=kval, fval=fval, cs_min=float(cs_min), cp_min=float(cp_min),
                                              cp_max=float(cp_max), cs_max=float(cs_max)), order="F")


def hybrid_ninf_filter_design(trace_shape, selected_channels, dx, fs, cs_min=1400., cp_min=1450., cp_max=3400,
                              cs_max=3500, fmin=15., fmax=25., display_filter=False):
    """Butterworth-in-frequency x speed-band hybrid mask (reference: dsp.py:308-454; the mask
    every reference script uses).  Returns a lazy `FkMask` (has `.todense()` like sparse.COO)."""
    nnx, nns = trace_shape
    if nns % 2:
        # the reference builds H with 2*(nns//2) entries (dsp.py:349) and fails to broadcast
        raise ValueError(f"operands could not be broadcast together with shapes ({nnx},{nns}) ({2 * (nns // 2)},)")
    kval, fval = _fftfreq_steps(trace_shape, selected_channels, dx, fs)
    freq = np.fft.fftshift(np.fft.fftfreq(nns, d=1 / fs))
    b, a = sp.butter(8, [fmin / (fs / 2), fmax / (fs / 2)], "bp")
    H = np.concatenate((np.zeros(len(freq) // 2), np.abs(sp.freqz(b, a, worN=len(freq) // 2)[1]) ** 2))
    df_taper = 14
    col_lo = int(np.argmax(freq >= fmin - df_taper))
    col_hi = int(np.argmax(freq >= fmax + df_taper))
    mask = _fk.FkMask("hybrid_ninf", trace_shape,
                      dict(kval=kval, fval=fval, cs_min=float(cs_min), cp_min=float(cp_min), cp_max=float(cp_max),
                           cs_max=float(cs_max), H=H, col_lo=col_lo, col_hi=col_hi), order="C")
    if display_filter:
        _display_mask(mask, freq, np.fft.fftshift(np.fft.fftfreq(nnx, d=selected_channels[2] * dx)))
    return mask



def _shifted_axes(trace_shape, selected_channels, dx, fs):
    nnx, nns = trace_shape
    freq = np.fft.fftshift(np.fft.fftfreq(nns, d=1 / fs))
    knum = np.fft.fftshift(np.fft.fftfreq(nnx, d=selected_channels[2] * dx))
    return freq, knum


def hybrid_filter_design(trace_shape, selected_channels, dx, fs, cs_min=1400., cp_min=1450., fmin=15., fmax=25.,
                         display_filter=False):
    """Infinite-speed hybrid mask, sine tapers in f and k (reference: dsp.py:174-305).  Built on the
    host at design time (vectorised) and applied through the dense-mask GPU path."""
    freq, knum = _shifted_axes(trace_shape, selected_channels, dx, fs)
    fpmin, fpmax = fmin - 4, fmax + 4                          # df_taper = 4 Hz (dsp.py:216)
    H = np.zeros_like(freq)
    up = (freq >= fpmin) & (freq <= fmin)
    H[up] = np.sin(0.5 * np.pi * (freq[up] - fpmin) / (fmin - fpmin))
    H[(freq >= fmin) & (freq <= fmax)] = 1
    dn = (freq >= fmax) & (freq <= fpmax)
    H[dn] = np.cos(0.5 * np.pi * (freq[dn] - fmax) / (fmax - fpmax))
    lo, hi = int(np.argmax(freq >= fpmin)), int(np.argmax(freq >= fpmax))
    f = freq[lo:hi][None, :]
    k = knum[:, None]
    ks, kp = f / cs_min, f / cp_min
    col = np.zeros((len(knum), hi - lo))
    with np.errstate(divide="ignore", invalid="ignore"):
        neg = (k >= -ks) & (k <= -kp) & (ks != kp)
        col = np.where(neg, -np.sin(0.5 * np.pi * (k + ks) / (kp - ks)), col)
        pos = (-k >= -ks) & (-k <= -kp) & (ks != kp)
        col = np.where(pos, np.sin(0.5 * np.pi * (k - ks) / (kp - ks)), col)
    col = np.where((k < kp) & (k > -kp), 1.0, col)
    M = np.tile(H, (len(knum), 1))
    M[:, lo:hi] *= col
    M = M + M[:, ::-1]                                         # np.fliplr symmetrisation (dsp.py:264)
    mask = _fk.FkMask.from_dense(M)
    if display_filter:
        _display_mask(mask, freq, knum)
    return mask


def _gs_start(trace_shape, selected_channels, dx, fs, fmin, fmax):
    freq, knum = _shifted_axes(trace_shape, selected_channels, dx, fs)
    H = np.zeros_like(freq)
    H[(freq >= fmin) & (freq <= fmax)] = 1
    lo, hi = int(np.argmax(freq >= fmin - 4)), int(np.argmax(freq >= fmax + 4))
    return freq, knum, np.tile(H, (len(knum), 1)), lo, hi


def hybrid_gs_filter_design(trace_shape, selected_channels, dx, fs, cs_min=1400., cp_min=1450., fmin=15., fmax=25.,
                            display_filter=False):
    """Infinite-speed hybrid mask with Gaussian (sigma = 20 bins) tapers (reference: dsp.py:457-579)."""
    from scipy import ndimage
    freq, knum, M, lo, hi = _gs_start(trace_shape, selected_channels, dx, fs, fmin, fmax)
    kp = freq[lo:hi][None, :] / cp_min
    M[:, lo:hi] *= ((knum[:, None] < kp) & (knum[:, None] > -kp))
    M = ndimage.gaussian_filter(M + M[:, ::-1], 20)            # dsp.py:539-540
    mask = _fk.FkMask.from_dense(M)
    if display_filter:
        _display_mask(mask, freq, knum)
    return mask


def hybrid_ninf_gs_filter_design(trace_shape, selected_channels, dx, fs, cs_min=1400., cp_min=1450., cp_max=3400,
                                 cs_max=3500, fmin=15., fmax=25., display_filter=False):
    """Finite-speed hybrid mask with Gaussian tapers (reference: dsp.py:582-702)."""
    from scipy import ndimage
    freq, knum, M, lo, hi = _gs_start(trace_shape, selected_channels, dx, fs, fmin, fmax)
    f = freq[lo:hi][None, :]
    M[:, lo:hi] *= ((knum[:, None] > -f / cp_min) & (knum[:, None] < -f / cp_max))
    M = ndimage.gaussian_filter(M, 20)                         # dsp.py:659
    M = M + M[:, ::-1]
    M = M + M[::-1, :]
    mask = _fk.FkMask.from_dense(M)
    if display_filter:
        _display_mask(mask, freq, knum)
    return mask


def fk_filt(data, tint, fs, xint, dx, c_min, c_max):
    """Legacy one-call f-k filter: Gaussian-blurred boolean fan built and applied in one go
    (reference: dsp.py:883-953).  The fan is built on the host, the 2-D filtering runs on the GPU."""
    from scipy import ndimage
    shape = tuple(data.shape)
    f = np.fft.fftshift(np.fft.fftfreq(shape[1], d=tint / fs))
    k = np.fft.fftshift(np.fft.fftfreq(shape[0], d=xint * dx))
    ff, kk = np.meshgrid(f, k)
    g = 1.0 * ((ff < kk * c_min) & (ff < -kk * c_min))
    g2 = 1.0 * ((ff < kk * c_max) & (ff < -kk * c_max))
    g = g + g[:, ::-1] - (g2 + g2[:, ::-1])
    g = ndimage.gaussian_filter(g, 20)
    g = (g - np.min(g)) / (np.max(g) - np.min(g))
    return fk_filter_filt(data, _fk.FkMask.from_dense(g))


def _display_mask(mask, freq, knum):
    import matplotlib.pyplot as plt
    m = np.asarray(mask)
    plt.figure(figsize=(12, 6))
    plt.imshow(m, extent=[min(freq), max(freq), min(knum), max(knum)], aspect="auto", origin="lower")
    plt.xlabel("f [Hz]")
    plt.ylabel("k [m$^{-1}$]")
    plt.show()


# ------------------------------------------------------------------------------ f-k apply
def taper_data(trace):
    """In-place Tukey(alpha=0.03) taper along time (reference: dsp.py:705-722)."""
    nt = trace.shape[1]
    if _is_tensor(trace):
        torch = _fk._torch()
        win = torch.from_numpy(sp.windows.tukey(nt, alpha=0.03)).to(trace.device, trace.dtype)
        trace *= win[None, :]
        return trace
    trace *= sp.windows.tukey(nt, alpha=0.03)[np.newaxis, :]
    return trace


def _taper_edges_inplace(trace):
    """Same mutation as taper_data but touching only the samples where the window != 1."""
    nt = trace.shape[1]
    win = sp.windows.tukey(nt, alpha=0.03)
    width = int(np.floor(0.03 * (nt - 1) / 2.0)) + 1
    width = min(width, nt)
    if _is_tensor(trace):
        import torch
        win = torch.from_numpy(win).to(trace.device, trace.dtype)
    trace[:, :width] *= win[np.newaxis, :width]
    if nt - width >= width:
        trace[:, nt - width:] *= win[np.newaxis, nt - width:]
    else:
        trace[:, width:] *= win[np.newaxis, width:]


def fk_filter_filt(trace, fk_filter_matrix, tapering=False):
    """Apply a pre-computed f-k mask: real(ifft2(ifftshift(fftshift(fft2(trace)) * mask)))
    (reference: dsp.py:725-756).  `fk_filter_matrix` may be an `FkMask`, a dense ndarray in the
    reference's shifted layout (any memory order), a sparse.COO, or a CUDA tensor.

    Like the reference, `tapering=True` tapers the caller's array in place before filtering."""
    torch = _fk._torch()
    if _is_tensor(trace):
        x = _to_device(trace)
        flt = _fk.FkFilter(fk_filter_matrix, shape=tuple(x.shape), device=x.device.index)
        y = flt(x, tapering=tapering)
        if tapering:
            _taper_edges_inplace(trace)          # the reference's side effect; the window is exactly 1 between the edges
        return y
    arr = np.asarray(trace)
    x = _to_device(arr)
    flt = _fk.FkFilter(fk_filter_matrix, shape=tuple(x.shape))
    y = flt(x, out=x, tapering=tapering)
    if tapering and isinstance(trace, np.ndarray) and trace.flags.writeable and np.issubdtype(trace.dtype, np.floating):
        _taper_edges_inplace(trace)
    return _to_host64(y)


def fk_filter_sparsefilt(trace, fk_filter_matrix, tapering=False):
    """Same arithmetic as fk_filter_filt for a sparse mask (reference: dsp.py:759-786)."""
    return fk_filter_filt(trace, fk_filter_matrix, tapering=tapering)


# ------------------------------------------------------------------------------ IIR
def butterworth_filter(filterspec, fs):
    """SOS Butterworth design (reference: dsp.py:789-827) -- design only, host side."""
    filter_order, filter_critical_freq, filter_type_str = filterspec
    wn = np.array(filter_critical_freq) / (fs / 2)
    return sp.butter(filter_order, wn, btype=filter_type_str, output="sos")


def sosfiltfilt(sos, x, axis=1):
    """GPU replacement for the caller-side `scipy.signal.sosfiltfilt(sos, trace, axis=1)` the
    reference's notebook / Example.py:55 applies after `butterworth_filter`."""
    if axis not in (1, -1):
        raise ValueError("das4whales_b200.dsp.sosfiltfilt filters along the time axis (axis=1)")
    xd = _to_device(x)
    y = _rows.sosfiltfilt(np.asarray(sos, dtype=np.float64), xd)
    return y if _is_tensor(x) else _to_host64(y)


def bp_filt(data, fs, fmin, fmax):
    """Order-8 Butterworth band-pass, zero-phase (reference: dsp.py:859-880 =
    scipy.signal.filtfilt(b, a, data, axis=1) with default odd padding of 3*17 samples)."""
    sos = sp.butter(8, [fmin / (fs / 2), fmax / (fs / 2)], "bp", output="sos")
    xd = _to_device(data)
    y = _rows.sosfiltfilt(sos, xd, padlen=3 * 17)
    return y if _is_tensor(data) else _to_host64(y)


# ------------------------------------------------------------------------------ spectra
def get_spectrogram(waveform, fs, nfft=128, overlap_pct=0.8):
    """Single-channel spectrogram in dB re max (reference: dsp.py:41-78, librosa.stft with
    a periodic Hann window, centred frames, hop = floor(nfft * (1 - overlap)))."""
    hop = int(np.floor(nfft * (1 - overlap_pct)))
    xd = _to_device(np.asarray(waveform)[None, :] if not _is_tensor(waveform) else waveform.reshape(1, -1))
    mag = _rows.stft_mag(xd, nfft, hop)[0]             # [1 + nfft/2, frames]
    torch = _fk._torch()
    p = torch.empty_like(mag)
    ws = torch.empty(2, dtype=torch.int32, device=mag.device)
    with torch.cuda.device(mag.device.index):          # 20 log10(S / max S) on the device (d4w_db_re_max)
        _lib.check(_lib.lib().d4w_db_re_max(_lib.ptr(mag, "float*"), _lib.ptr(p, "float*"), mag.numel(), _lib.ptr(ws), _lib.stream_ptr()),
                   "get_spectrogram")
    height, width = p.shape
    tt = np.linspace(0, xd.shape[1] / fs, num=width)
    ff = np.linspace(0, fs / 2, num=height)
    if _is_tensor(waveform):
        return p, tt, ff
    return p.to(torch.float64).cpu().numpy(), tt, ff


def get_fx(trace, nfft):
    """Per-channel FFT magnitude in nano-strain, fftshift-ed along frequency (reference: dsp.py:18-38):
    2 |fft(trace, nfft)| / nfft * 1e9 -- one shared-memory FFT per channel on the GPU (d4w_row_fft_mag)."""
    xd = _to_device(trace)
    fx = _rows.row_fft_mag(xd, int(nfft), 2.0e9 / int(nfft))
    return fx if _is_tensor(trace) else _to_host64(fx)


def instant_freq(channel, fs):
    """Instantaneous frequency of one channel, diff(unwrap(angle(hilbert(x)))) / 2 pi * fs (reference: dsp.py:830-856):
    Hilbert transform on the row engine (d4w_hilbert mode 2), phase difference + numpy.unwrap's wrapping on the device."""
    torch = _fk._torch()
    xd = _to_device(channel.reshape(1, -1) if _is_tensor(channel) else np.asarray(channel).reshape(1, -1))
    fi = _rows.inst_freq(xd[0], float(fs))
    return fi if _is_tensor(channel) else fi.to(torch.float64).cpu().numpy()


def snr_tr_array(trace, env=False):
    """10*log10(x^2 / var_row(x)) or, with env=True, of the squared Hilbert envelope
    (reference: dsp.py:956-976)."""
    xd = _to_device(trace)
    y = _rows.snr(xd, env=bool(env))
    return y if _is_tensor(trace) else _to_host64(y)


# ------------------------------------------------------------------------------ cable noise profile
NOISE_PROFILE_KEYS = ("med", "mean", "std", "std_med_diff", "SNR_1d", "noise_power", "noise_power_db", "noise_mean")


def noise_window(ns, fs, tnoise=(19., 26.)):
    """Sample range [i0, i1) of the noise window, int(t * fs) for each end (scripts/main_bathynoise.py:251).
    Raises ValueError for an empty window or one outside [0, ns]."""
    i0, i1 = (int(t * fs) for t in tnoise)
    if not 0 <= i0 < i1 <= int(ns):
        raise ValueError(f"noise window {tuple(tnoise)} s -> samples [{i0}, {i1}) is empty or outside [0, {int(ns)}]")
    return i0, i1


def noise_profile_from_stats(full, win, p_ref=1e-11):
    """The profile of scripts/main_bathynoise.py:183-194, :257-259 from two rows.env_stats records ([nx, 5] float64,
    ndarrays or tensors): `full` of the whole rows, `win` of the noise window.  Division and log follow IEEE, as NumPy: a
    zero channel gives SNR_1d = nan and noise_power_db = -inf."""
    if _is_tensor(full):
        import torch
        sqrt, log10, col = torch.sqrt, torch.log10, (lambda a, j: a[:, j].contiguous())
    else:
        sqrt, log10, col = np.sqrt, np.log10, (lambda a, j: np.ascontiguousarray(a[:, j], dtype=np.float64))
    med, std = col(full, 0), sqrt(col(full, 4))
    noise_power = col(win, 3)
    with np.errstate(divide="ignore", invalid="ignore"):
        return {"med": med, "mean": col(full, 1), "std": std, "std_med_diff": std - med, "SNR_1d": 20 * log10(std / med),
                "noise_power": noise_power, "noise_power_db": 10 * log10(noise_power / p_ref ** 2),
                "noise_mean": col(win, 1)}


def cable_noise_profile(trace, fs, tnoise=(19., 26.), p_ref=1e-11):
    """Per-channel noise floor of scripts/main_bathynoise.py:183-194, :248-259 for the f-k filtered strain `trace`
    [nx, ns]: median and mean of the Hilbert envelope (med, mean), the population std, std_med_diff = std - med,
    SNR_1d = 20 log10(std / med), and over the window tnoise (seconds, int(t * fs) samples) noise_power = mean(x^2),
    noise_power_db = 10 log10(noise_power / p_ref^2) and noise_mean = the mean envelope of the window alone.
    Returns a dict of NOISE_PROFILE_KEYS: float64 ndarrays for an ndarray in, float64 CUDA tensors for a tensor in.
    Only [nx]-long vectors leave the GPU."""
    i0, i1 = noise_window(np.shape(trace)[-1], fs, tnoise)
    xd = _to_device(trace)
    full = _rows.env_stats(xd)
    win = _rows.env_stats(xd, i0, i1 - i0)
    if _is_tensor(trace):
        return noise_profile_from_stats(full, win, p_ref)
    return noise_profile_from_stats(full.cpu().numpy(), win.cpu().numpy(), p_ref)


# Channel counts with a prime factor > 61 go through the chirp-z column transform of length M = the smallest 2^a 3^b 5^c
# >= 2 nx - 1, and one M-point complex column must fit the 200 KB column budget: M <= 25 600, so nx <= 12 800
# (csrc/fk_hostplan.hpp, czt_max_channels).
CZT_MAX_CHANNELS = 12800


def supported_shape(nx, ns):
    """Largest (nx', ns') <= (nx, ns) the f-k filter's planner accepts.  The f-k filter takes any channel count up to
    12 800; above that the channel count must have no prime factor > 61 and one channel column must fit an SM's shared
    memory (about 28 000 channels).  Its time axis is mixed-radix: every prime factor must be <= 61 and it must split as
    ns = T1 * T2 with T1 <= 25 and T2 <= 10 240.  numpy.fft takes any length; crop (or pad the record before loading) to the
    suggested shape when `fk_filter_filt` raises ValueError for an unsupported length.
    The Hilbert family (`envelope`, `pick_times_env`, `snr_tr_array(env=True)`, `instant_freq`, `trace2image`) is not bound
    by the time-axis rule: a row length without such a split runs through a chirp-z transform up to
    rows.HILBERT_MAX_SAMPLES = 128 000 samples."""
    def smooth(n):
        for p in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37, 41, 43, 47, 53, 59, 61):
            while n % p == 0:
                n //= p
        return n == 1

    def time_ok(n):
        if not smooth(n):
            return False
        return any(n % t1 == 0 and n // t1 <= (16384 if t1 == 1 else 10240) for t1 in (1, 2, 3, 4, 5, 6, 8, 10, 12, 15, 16, 20, 25))
    nx2 = min(int(nx), 28000)
    while nx2 > CZT_MAX_CHANNELS and not smooth(nx2):
        nx2 -= 1
    ns2 = int(ns)
    while ns2 > 1 and not time_ok(ns2):
        ns2 -= 1
    return nx2, ns2


# north-star aliases
bandpass = bp_filt
compute_spectrogram = get_spectrogram
