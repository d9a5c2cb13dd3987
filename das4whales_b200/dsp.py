"""das4whales_b200.dsp -- drop-in for the hot-path functions of `das4whales.dsp`
(/root/reference/src/das4whales/dsp.py), same names / positional order / defaults, running
on hand-written sm_90a CUDA kernels (libd4w.so) instead of NumPy/SciPy.

Accepted data: `numpy.ndarray` (any float dtype; the result is a new float64 ndarray, as the
reference returns) or a CUDA `torch.Tensor` (float32; the result stays on the device).
"""
import warnings
from collections import namedtuple

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


def _design_steps(trace_shape, selected_channels, dx, fs, speeds, fmin, fmax):
    """(kval, fval) when the device design covers the arguments, else None: positive finite speeds, finite fmin < fmax,
    numpy's fftfreq steps finite with fval > 0 (the shifted frequency axis then increases, which the interval argument of
    csrc/tools_kernels.cuh needs) and at most 65 535 channels."""
    try:
        kval, fval = _fftfreq_steps(trace_shape, selected_channels, dx, fs)
        vals = np.array([float(v) for v in speeds] + [float(fmin), float(fmax), kval, fval])
        nx, ns = (int(n) for n in trace_shape)
    except (ZeroDivisionError, TypeError, ValueError, OverflowError):
        return None
    if not (np.isfinite(vals).all() and (vals[:len(speeds)] > 0).all() and fmin < fmax and fval > 0 and 1 <= nx <= 65535
            and ns >= 1):
        return None
    return kval, fval


def _designed_mask(kind, host, trace_shape, selected_channels, dx, fs, speeds, fmin, fmax, H, col_lo, col_hi):
    """The lazy mask designed on the device (fk.DESIGN_KINDS), or FkMask.from_dense(host()) for arguments outside its domain.
    speeds = (cs_min, cp_min, cp_max): the ones the design function takes, cp_max = None when it takes none."""
    steps = _design_steps(trace_shape, selected_channels, dx, fs, [c for c in speeds if c is not None], fmin, fmax)
    if steps is None or (kind == "hybrid" and col_hi < col_lo):
        return _fk.FkMask.from_dense(host())
    cs_min, cp_min, cp_max = speeds
    return _fk.FkMask(kind, trace_shape, dict(kval=steps[0], fval=steps[1], cs_min=float(cs_min), cp_min=float(cp_min),
                                              cp_max=float(cp_min if cp_max is None else cp_max), fmin=float(fmin),
                                              fmax=float(fmax), H=H, col_lo=int(col_lo), col_hi=int(col_hi)),
                      order="C", host=host)


def _hybrid_H(freq, fmin, fmax):
    fpmin, fpmax = fmin - 4, fmax + 4                          # df_taper = 4 Hz (dsp.py:216)
    H = np.zeros_like(freq)
    up = (freq >= fpmin) & (freq <= fmin)
    H[up] = np.sin(0.5 * np.pi * (freq[up] - fpmin) / (fmin - fpmin))
    H[(freq >= fmin) & (freq <= fmax)] = 1
    dn = (freq >= fmax) & (freq <= fpmax)
    H[dn] = np.cos(0.5 * np.pi * (freq[dn] - fmax) / (fmax - fpmax))
    return H, int(np.argmax(freq >= fpmin)), int(np.argmax(freq >= fpmax))


def _hybrid_host(trace_shape, selected_channels, dx, fs, cs_min, cp_min, fmin, fmax):
    freq, knum = _shifted_axes(trace_shape, selected_channels, dx, fs)
    H, lo, hi = _hybrid_H(freq, fmin, fmax)
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
    return M + M[:, ::-1]                                      # np.fliplr symmetrisation (dsp.py:264)


def hybrid_filter_design(trace_shape, selected_channels, dx, fs, cs_min=1400., cp_min=1450., fmin=15., fmax=25.,
                         display_filter=False):
    """Infinite-speed hybrid mask, sine tapers in f and k (reference: dsp.py:174-305).  Returns a lazy `FkMask` at once:
    the filter designs it on the device (d4w_mask_design), `np.asarray` / `todense()` build the float64 matrix on the host."""
    freq, knum = _shifted_axes(trace_shape, selected_channels, dx, fs)
    H, lo, hi = _hybrid_H(freq, fmin, fmax)
    mask = _designed_mask("hybrid", lambda: _hybrid_host(trace_shape, selected_channels, dx, fs, cs_min, cp_min, fmin, fmax),
                          trace_shape, selected_channels, dx, fs, (cs_min, cp_min, None), fmin, fmax, H, lo, hi)
    if display_filter:
        _display_mask(mask, freq, knum)
    return mask


def _gs_H(freq, fmin, fmax):
    H = np.zeros_like(freq)
    H[(freq >= fmin) & (freq <= fmax)] = 1
    return H, int(np.argmax(freq >= fmin - 4)), int(np.argmax(freq >= fmax + 4))


def _gs_start(trace_shape, selected_channels, dx, fs, fmin, fmax):
    freq, knum = _shifted_axes(trace_shape, selected_channels, dx, fs)
    H, lo, hi = _gs_H(freq, fmin, fmax)
    return freq, knum, np.tile(H, (len(knum), 1)), lo, hi


def _hybrid_gs_host(trace_shape, selected_channels, dx, fs, fmin, fmax, cp_min):
    from scipy import ndimage
    freq, knum, M, lo, hi = _gs_start(trace_shape, selected_channels, dx, fs, fmin, fmax)
    kp = freq[lo:hi][None, :] / cp_min
    M[:, lo:hi] *= ((knum[:, None] < kp) & (knum[:, None] > -kp))
    return ndimage.gaussian_filter(M + M[:, ::-1], 20)         # dsp.py:539-540


def hybrid_gs_filter_design(trace_shape, selected_channels, dx, fs, cs_min=1400., cp_min=1450., fmin=15., fmax=25.,
                            display_filter=False):
    """Infinite-speed hybrid mask with Gaussian (sigma = 20 bins) tapers (reference: dsp.py:457-579).  Returns a lazy
    `FkMask` at once: designed on the device for the filter, on the host (scipy.ndimage) for `np.asarray` / `todense()`."""
    freq, knum = _shifted_axes(trace_shape, selected_channels, dx, fs)
    H, lo, hi = _gs_H(freq, fmin, fmax)
    mask = _designed_mask("hybrid_gs", lambda: _hybrid_gs_host(trace_shape, selected_channels, dx, fs, fmin, fmax, cp_min),
                          trace_shape, selected_channels, dx, fs, (cs_min, cp_min, None), fmin, fmax, H, lo, hi)
    if display_filter:
        _display_mask(mask, freq, knum)
    return mask


def _hybrid_ninf_gs_host(trace_shape, selected_channels, dx, fs, fmin, fmax, cp_min, cp_max):
    from scipy import ndimage
    freq, knum, M, lo, hi = _gs_start(trace_shape, selected_channels, dx, fs, fmin, fmax)
    f = freq[lo:hi][None, :]
    M[:, lo:hi] *= ((knum[:, None] > -f / cp_min) & (knum[:, None] < -f / cp_max))
    M = ndimage.gaussian_filter(M, 20)                         # dsp.py:659
    M = M + M[:, ::-1]
    return M + M[::-1, :]


def hybrid_ninf_gs_filter_design(trace_shape, selected_channels, dx, fs, cs_min=1400., cp_min=1450., cp_max=3400,
                                 cs_max=3500, fmin=15., fmax=25., display_filter=False):
    """Finite-speed hybrid mask with Gaussian tapers (reference: dsp.py:582-702).  Returns a lazy `FkMask` at once:
    designed on the device for the filter, on the host (scipy.ndimage) for `np.asarray` / `todense()`."""
    freq, knum = _shifted_axes(trace_shape, selected_channels, dx, fs)
    H, lo, hi = _gs_H(freq, fmin, fmax)
    mask = _designed_mask("hybrid_ninf_gs",
                          lambda: _hybrid_ninf_gs_host(trace_shape, selected_channels, dx, fs, fmin, fmax, cp_min, cp_max),
                          trace_shape, selected_channels, dx, fs, (cs_min, cp_min, cp_max), fmin, fmax, H, lo, hi)
    if display_filter:
        _display_mask(mask, freq, knum)
    return mask


def fk_filt(data, tint, fs, xint, dx, c_min, c_max):
    """Legacy one-call f-k filter: Gaussian-blurred boolean fan built and applied in one go
    (reference: dsp.py:883-953).  The fan (sigma = 20) is designed on the GPU (rows.blurred_fan) and goes to the filter as
    a device tensor: the [nx, ns] plane never exists on the host."""
    nx, ns = (int(n) for n in data.shape)
    # numpy.fft.fftfreq(n, d) steps 1 / (n * d), d = tint / fs and xint * dx (dsp.py:931-932)
    kval, fval = 1.0 / (nx * (xint * dx)), 1.0 / (ns * (tint / fs))
    dev = data.device.index if _is_tensor(data) and data.is_cuda else None
    return fk_filter_filt(data, _rows.blurred_fan(nx, ns, kval, fval, c_min, c_max, 20, device=dev))


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


def fk_filter_filts(trace, fk_filter_matrices, tapering=False):
    """fk_filter_filt of one trace with several masks (what scripts/main_fkcomp.py:73-95 does with four
    fk_filter_sparsefilt calls), through one forward transform (fk.FkFilterBank).  Each output equals
    fk_filter_filt(trace, mask_i, tapering).  An ndarray goes up once and gives a list of float64 ndarrays; a CUDA
    tensor gives a list of float32 tensors.  `tapering=True` tapers the caller's array once, in place."""
    if _is_tensor(trace):
        x = _to_device(trace)
        bank = _fk.FkFilterBank(fk_filter_matrices, shape=tuple(x.shape), device=x.device.index)
        ys = bank(x, tapering=tapering)
        if tapering:
            _taper_edges_inplace(trace)
        return ys
    arr = np.asarray(trace)
    x = _to_device(arr)
    bank = _fk.FkFilterBank(fk_filter_matrices, shape=tuple(x.shape))
    ys = bank(x, outs=[x] + [_fk._torch().empty_like(x) for _ in range(len(bank) - 1)], tapering=tapering)
    if tapering and isinstance(trace, np.ndarray) and trace.flags.writeable and np.issubdtype(trace.dtype, np.floating):
        _taper_edges_inplace(trace)
    return [_to_host64(y) for y in ys]


def _band(axis, lo, hi, what, who="fk_spectrum"):
    """Half-open index range of {i : lo <= axis[i] <= hi} (a contiguous run: the shifted axes are monotonic)."""
    idx = np.flatnonzero((axis >= lo) & (axis <= hi))
    if idx.size == 0:
        raise ValueError(f"{who}: {what} selects no bin of the axis [{axis[0]}, {axis[-1]}]")
    return int(idx[0]), int(idx[-1]) + 1


def fk_spectrum(trace, selected_channels, dx, fs, f_range=(0., np.inf), k_range=(-np.inf, np.inf), nperseg=None,
                tapering=False):
    """f-k power spectrum P = |fftshift(fft2(trace))|^2 over a frequency and wavenumber band, unnormalised, on the
    axes the mask designs use: knum = fftshift(fftfreq(nx, selected_channels[2] * dx)) and
    freq = fftshift(fftfreq(n, 1 / fs)), n the record length or `nperseg`.  Returns (P, f, k): P [len(k), len(f)],
    f = freq[f_range[0] <= freq <= f_range[1]] and k = knum[k_range[0] <= knum <= k_range[1]] (float64 ndarrays).

    The default band is numpy's non-negative frequencies (for even n the Nyquist bin sits at -fs/2 and is left out;
    a negative f_range[0] takes it) and every wavenumber.  nperseg=L: the mean of the spectra of the ns // L whole
    blocks trace[:, b*L:(b+1)*L] (a trailing partial block is not used).  tapering=True multiplies each block by
    Tukey(n, alpha=0.03) along time, as taper_data does, but never modifies the caller's array.  An ndarray gives a
    float64 P, a CUDA tensor a float32 CUDA tensor.  Shapes ([nx, ns], or [nx, nperseg]) follow the f-k filter's rules
    (supported_shape); an unsupported one raises ValueError."""
    if _is_tensor(trace):
        if trace.dim() != 2 or trace.is_complex():
            raise ValueError(f"fk_spectrum: expected a real 2-D [channel x time] array, got {tuple(trace.shape)} {trace.dtype}")
        x = _to_device(trace)
    else:
        arr = np.asarray(trace)
        if arr.ndim != 2 or np.iscomplexobj(arr):
            raise ValueError(f"fk_spectrum: expected a real 2-D [channel x time] array, got {arr.shape} {arr.dtype}")
        x = None
    nx, ns = (int(v) for v in trace.shape)
    n = ns
    if nperseg is not None:
        n = int(nperseg)
        if n < 1 or n > ns:
            raise ValueError(f"fk_spectrum: nperseg = {nperseg} must lie in [1, {ns}]")
    knum = np.fft.fftshift(np.fft.fftfreq(nx, selected_channels[2] * dx))
    freq = np.fft.fftshift(np.fft.fftfreq(n, 1 / fs))
    f_idx = _band(freq, f_range[0], f_range[1], f"f_range {tuple(f_range)}")
    k_idx = _band(knum, k_range[0], k_range[1], f"k_range {tuple(k_range)}")
    device = x.device.index if x is not None else _fk._torch().cuda.current_device()
    spec = _fk.FkSpectrum((nx, n), k_idx, f_idx, device=device)
    if x is None:
        x = _to_device(arr)
    p = spec(x, tapering=tapering)
    f, k = freq[f_idx[0]:f_idx[1]], knum[k_idx[0]:k_idx[1]]
    return (p if _is_tensor(trace) else _to_host64(p)), f, k


fk_welch_layout = _fk.fk_welch_layout


def fk_welch(trace, selected_channels, dx, fs, nperseg=None, noverlap=None, window="hann", nperseg_x=None, noverlap_x=None,
             window_x="hann", detrend="constant", scaling="density", f_range=(0., np.inf), k_range=(-np.inf, np.inf)):
    """f-k power spectral density by Welch's method, the 2-D (channel x time) counterpart of `welch`.

    Time segments follow welch_layout (nperseg=None is 256, noverlap=None is nperseg // 2, a trailing partial segment is
    dropped) and their spectra are averaged (mean).  Channel segments follow the same rules but are not averaged:
    nperseg_x=None is one segment spanning every channel; with nperseg_x the result has a leading channel-segment axis.
    window / window_x are resolved like welch_window (a string or tuple through scipy.signal.get_window, a 1-D array as
    given, of length nperseg and nperseg_x or nx) and the 2-D window is their outer product.  detrend='constant' subtracts
    each channel's mean over each segment before windowing; detrend=False does not.  The plane is two-sided, with
    fsx = 1 / (selected_channels[2] * dx):  'density' is P / (fs fsx sum(wt^2) sum(wx^2)) in units^2 / Hz / (1/m),
    'spectrum' is P / ((sum wt)^2 (sum wx)^2), P the mean of |fftshift(fft2(segment))|^2.  The axes are those of
    fk_spectrum for the segment shape (freq = fftshift(fftfreq(nperseg, 1 / fs)), knum = fftshift(fftfreq(nperseg_x,
    selected_channels[2] * dx))), cut to f_range and k_range with fk_spectrum's rules.

    Returns (P, f, k) with P [len(k), len(f)], or (P, f, k, c0) with P [nseg_x, len(k), len(f)] and c0 the first channel
    of each channel segment when nperseg_x is given.  An ndarray gives float64 ndarrays, a CUDA tensor a float32 CUDA P;
    the caller's array is never modified.  ValueError for complex or non-2-D input, an empty or out-of-range segment
    geometry, noverlap >= nperseg, a window of the wrong length, another detrend or scaling, and a segment shape the f-k
    planner rejects (see supported_shape)."""
    if _is_tensor(trace):
        if trace.dim() != 2 or trace.is_complex():
            raise ValueError(f"fk_welch: expected a real 2-D [channel x time] array, got {tuple(trace.shape)} {trace.dtype}")
    else:
        trace = np.asarray(trace)
        if trace.ndim != 2 or np.iscomplexobj(trace):
            raise ValueError(f"fk_welch: expected a real 2-D [channel x time] array, got {trace.shape} {trace.dtype}")
    if detrend is not False and detrend != "constant":
        raise ValueError(f"detrend={detrend!r}: only 'constant' and False are computed")
    if scaling not in ("density", "spectrum"):
        raise ValueError(f"Parameter scaling={scaling!r} not in {{'spectrum': 'magnitude', 'density': 'psd'}}!")
    nx, ns = (int(v) for v in trace.shape)
    if nx < 1 or ns < 1:
        raise ValueError(f"fk_welch: empty record of shape {(nx, ns)}")
    for what, n, lim in (("nperseg", nperseg, ns), ("nperseg_x", nperseg_x, nx)):
        if n is not None and not 1 <= int(n) <= lim:
            raise ValueError(f"fk_welch: {what} = {n} must lie in [1, {lim}]")
    wt, lt = welch_window(window, nperseg, ns)
    wx, lx = welch_window(window_x, nx if nperseg_x is None else nperseg_x, nx)
    lay = fk_welch_layout(nx, ns, lt, noverlap, None if nperseg_x is None else lx, noverlap_x)
    dxc = selected_channels[2] * dx
    if scaling == "density":
        scale = 1.0 / (fs * (1.0 / dxc) * float(np.sum(wt * wt)) * float(np.sum(wx * wx)))
    else:
        scale = 1.0 / (float(np.sum(wt)) ** 2 * float(np.sum(wx)) ** 2)
    freq = np.fft.fftshift(np.fft.fftfreq(lt, 1 / fs))
    knum = np.fft.fftshift(np.fft.fftfreq(lx, dxc))
    f_idx = _band(freq, f_range[0], f_range[1], f"f_range {tuple(f_range)}", "fk_welch")
    k_idx = _band(knum, k_range[0], k_range[1], f"k_range {tuple(k_range)}", "fk_welch")
    x = _to_device(trace) if _is_tensor(trace) else None
    device = x.device.index if x is not None else _fk._torch().cuda.current_device()
    est = _fk.FkWelch((nx, ns), (lx, lt), k_idx, f_idx, wt, wx, detrend == "constant", scale, device=device,
                      noverlap=lay.noverlap, noverlap_x=lay.noverlap_x)
    if x is None:
        x = _to_device(trace)
    p = est(x)
    f, k = freq[f_idx[0]:f_idx[1]], knum[k_idx[0]:k_idx[1]]
    if not _is_tensor(trace):
        p = _to_host64(p.reshape(-1, p.shape[-1])).reshape(tuple(p.shape))
    if nperseg_x is None:
        return p[0], f, k
    return p, f, k, np.asarray(lay.starts_x, dtype=np.int64)


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


# ------------------------------------------------------------------------------ Welch power spectral density
WelchLayout = namedtuple("WelchLayout", "nperseg noverlap step nfft chunk nchunks nseg nbins median_bias")


def _largest_prime_factor(n):
    p, big = 2, 1
    while p * p <= n:
        while n % p == 0:
            big, n = p, n // p
        p += 1
    return max(big, n)


def welch_layout(ns, nperseg, noverlap=None, nfft=None, chunk=None):
    """Segments and bins of scipy.signal.welch over whole chunks of ns-sample rows, pure Python (d4w_welch's geometry).
    noverlap=None is nperseg // 2, nfft=None is nperseg, chunk=None is the whole row.  Segment s of a chunk covers samples
    [s * step, s * step + nperseg), step = nperseg - noverlap, nseg = (chunk - nperseg) // step + 1 (no padding; a
    trailing partial segment is dropped).  median_bias = SciPy's _median_bias(nseg).  ValueError for inconsistent sizes
    and for an nfft with a prime factor above 61, which the shared-memory FFT does not take."""
    ns, nperseg = int(ns), int(nperseg)
    chunk = ns if chunk is None else int(chunk)
    if ns < 1:
        raise ValueError("welch: empty input")
    if not 1 <= chunk <= ns:
        raise ValueError(f"chunk = {chunk} must be in [1, {ns}]")
    if nperseg < 1:
        raise ValueError(f"nperseg = {nperseg} is not a positive integer")
    if nperseg > chunk:
        raise ValueError(f"nperseg = {nperseg} is longer than the chunk of {chunk} samples")
    nfft = nperseg if nfft is None else int(nfft)
    if nfft < nperseg:
        raise ValueError(f"nfft = {nfft} must be greater than or equal to nperseg = {nperseg}")
    noverlap = nperseg // 2 if noverlap is None else int(noverlap)
    if noverlap >= nperseg:
        raise ValueError(f"noverlap = {noverlap} must be less than nperseg = {nperseg}")
    if nfft < 2 or _largest_prime_factor(nfft) > 61:
        raise ValueError(f"nfft = {nfft}: the shared-memory FFT takes lengths >= 2 whose prime factors are all <= 61")
    step = nperseg - noverlap
    nseg = (chunk - nperseg) // step + 1
    ii = 2.0 * np.arange(1.0, (nseg - 1) // 2 + 1)
    bias = float(1.0 + np.sum(1.0 / (ii + 1) - 1.0 / ii))
    return WelchLayout(nperseg, noverlap, step, nfft, chunk, ns // chunk, nseg, nfft // 2 + 1, bias)


def welch_window(window, nperseg, ns):
    """(window values float64 [nperseg], nperseg) by scipy.signal.welch's rules: a string or tuple is
    scipy.signal.get_window(window, nperseg) with nperseg=None meaning 256, cut to ns with SciPy's warning when longer than
    the input; an array gives nperseg = its length and must match nperseg when both are given."""
    if isinstance(window, (str, tuple)):
        nperseg = 256 if nperseg is None else int(nperseg)
        if nperseg < 1:
            raise ValueError(f"nperseg = {nperseg} is not a positive integer")
        if ns < nperseg:
            warnings.warn(f"nperseg={nperseg} is greater than signal length max(len(x), len(y)) = {ns}, using nperseg = {ns}",
                          stacklevel=3)
            nperseg = ns
        return np.asarray(sp.get_window(window, nperseg), dtype=np.float64), nperseg
    win = np.asarray(window)
    if win.ndim != 1 or np.iscomplexobj(win):
        raise ValueError("an array window must be real and 1-D")
    nperseg = len(win) if nperseg is None else int(nperseg)
    if nperseg != len(win):
        raise ValueError(f"nperseg={nperseg} does not equal len(win)={len(win)}")
    if nperseg > ns:
        raise ValueError(f"window of {nperseg} samples is longer than the input of {ns}")
    return win.astype(np.float64), nperseg


def welch_scale(win, fs, scaling):
    """SciPy's periodogram scale: 1 / (fs sum w^2) for 'density', 1 / (sum w)^2 for 'spectrum'"""
    win = np.asarray(win, dtype=np.float64)
    if scaling == "density":
        return 1.0 / (fs * float(np.sum(win * win)))
    if scaling == "spectrum":
        return 1.0 / float(np.sum(win)) ** 2
    raise ValueError(f"Parameter scaling={scaling!r} not in {{'spectrum': 'magnitude', 'density': 'psd'}}!")


def welch(x, fs=1.0, window="hann_periodic", nperseg=None, noverlap=None, nfft=None, detrend="constant",
          return_onesided=True, scaling="density", axis=-1, average="mean"):
    """scipy.signal.welch (SciPy 1.18 defaults) of 1-D or 2-D real input along the last axis, every row in one d4w_welch
    call.  Returns (f, Pxx): f = rfftfreq(nfft, 1 / fs) as a float64 ndarray; Pxx [nbins] or [nrows, nbins], a float64
    ndarray for an ndarray in and a float32 CUDA tensor for a tensor in.  ValueError, with no fall-back to SciPy, for what
    the kernel does not compute: detrend other than 'constant' or False, return_onesided=False, another axis, complex input."""
    tensor = _is_tensor(x)
    a = x if tensor else np.asarray(x)
    if a.ndim not in (1, 2):
        raise ValueError(f"welch takes 1-D or 2-D input, not {a.ndim}-D")
    if int(axis) not in (-1, a.ndim - 1):
        raise ValueError("welch computes along the last axis only (axis=-1)")
    if (a.is_complex() if tensor else np.iscomplexobj(a)):
        raise ValueError("welch takes real input only")
    if not return_onesided:
        raise ValueError("welch computes one-sided spectra only (return_onesided=True)")
    if detrend is not False and detrend != "constant":
        raise ValueError(f"detrend={detrend!r}: only 'constant' and False are computed")
    if average not in ("mean", "median"):
        raise ValueError(f"Parameter average={average!r} must be 'median' or 'mean'!")
    ns = int(a.shape[-1])
    win, nperseg = welch_window(window, nperseg, ns)
    lay = welch_layout(ns, nperseg, noverlap, nfft)
    scale = welch_scale(win, fs, scaling)
    xd = _to_device(a)
    if xd.ndim == 1:
        xd = xd.reshape(1, -1)
    p = _rows.welch(xd, lay.nperseg, lay.step, lay.nfft, win, detrend == "constant", scale, average)[:, 0, :]
    f = np.fft.rfftfreq(lay.nfft, 1 / fs)
    if a.ndim == 1:
        p = p[0]
    return f, (p if tensor else _to_host64(p))


def _cross_spectrum(name, x, y, fs, window, nperseg, noverlap, nfft, detrend, return_onesided, scaling, axis, average,
                    coherence):
    """csd / coherence: every check before any device work, then one rows.csd over all row pairs"""
    tensor = _is_tensor(x) or _is_tensor(y)
    a = x if _is_tensor(x) else np.asarray(x)
    b = y if _is_tensor(y) else np.asarray(y)
    for v in (a, b):
        if v.ndim not in (1, 2):
            raise ValueError(f"{name} takes 1-D or 2-D input, not {v.ndim}-D")
        if int(axis) not in (-1, v.ndim - 1):
            raise ValueError(f"{name} computes along the last axis only (axis=-1)")
        if (v.is_complex() if _is_tensor(v) else np.iscomplexobj(v)):
            raise ValueError(f"{name} takes real input only")
    ns = int(a.shape[-1])
    if int(b.shape[-1]) != ns:
        raise ValueError(f"{name}: x and y must have the same length, not {ns} and {int(b.shape[-1])} (zero-padding the "
                         "shorter one is not computed)")
    nx, ny = (int(v.shape[0]) if v.ndim == 2 else 1 for v in (a, b))
    if nx != ny and 1 not in (nx, ny):
        raise ValueError(f"{name}: x and y cannot be broadcast together ({nx} and {ny} rows)")
    if not return_onesided:
        raise ValueError(f"{name} computes one-sided spectra only (return_onesided=True)")
    if detrend is not False and detrend != "constant":
        raise ValueError(f"detrend={detrend!r}: only 'constant' and False are computed")
    if average not in ("mean", "median"):
        raise ValueError(f"Parameter average={average!r} must be 'median' or 'mean'!")
    win, nperseg = welch_window(window, nperseg, ns)
    lay = welch_layout(ns, nperseg, noverlap, nfft)
    scale = welch_scale(win, fs, scaling)
    cuda = [v.device for v in (a, b) if _is_tensor(v) and v.is_cuda]
    with _fk._torch().cuda.device(cuda[0] if cuda else None):        # an ndarray joins the tensor on its device
        xd = _to_device(a)
        yd = xd if y is x else _to_device(b)
    xd, yd = xd.reshape(-1, ns), yd.reshape(-1, ns)
    p = _rows.csd(xd, yd, lay.nperseg, lay.step, lay.nfft, win, detrend == "constant", scale, average, coherence)
    f = np.fft.rfftfreq(lay.nfft, 1 / fs)
    if a.ndim == 1 and b.ndim == 1:
        p = p[0]
    if tensor:
        return f, p
    if coherence:
        return f, _to_host64(p)
    h = np.ascontiguousarray(_to_host64(_fk._torch().view_as_real(p)))
    return f, h.view(np.complex128)[..., 0]


def csd(x, y, fs=1.0, window="hann_periodic", nperseg=None, noverlap=None, nfft=None, detrend="constant",
        return_onesided=True, scaling="density", axis=-1, average="mean"):
    """scipy.signal.csd (SciPy 1.18 defaults) of 1-D or 2-D real input along the last axis, every row pair in one d4w_csd
    call.  x and y have the same length and the same number of rows, or one of them is a single row (1-D or [1, ns]) that
    is paired with every row of the other; x[:-1], x[1:] are the neighbour pairs.  Returns (f, Pxy): f = rfftfreq(nfft,
    1 / fs) as a float64 ndarray; Pxy [nbins] (both 1-D) or [max(rows), nbins], Pxy = conj(X) Y averaged over the segments,
    a complex128 ndarray for ndarrays in and a complex64 CUDA tensor when either input is a tensor.  y is x gives the real
    dsp.welch(x), as SciPy returns the real part.  ValueError, with no fall-back to SciPy, for what the kernel does not
    compute: unequal lengths, detrend other than 'constant' or False, return_onesided=False, another axis, complex input."""
    if y is x:
        return welch(x, fs, window, nperseg, noverlap, nfft, detrend, return_onesided, scaling, axis, average)
    return _cross_spectrum("csd", x, y, fs, window, nperseg, noverlap, nfft, detrend, return_onesided, scaling, axis, average,
                           False)


def coherence(x, y, fs=1.0, window="hann_periodic", nperseg=None, noverlap=None, nfft=None, detrend="constant", axis=-1):
    """scipy.signal.coherence (SciPy 1.18 defaults): Cxy = |Pxy|^2 / (Pxx Pyy) of the mean Welch spectra, with csd's
    shapes, pairing and errors; one d4w_csd call computes all three spectra of every row pair.  Returns (f, Cxy): Cxy a
    float64 ndarray for ndarrays in and a float32 CUDA tensor when either input is a tensor.  A row of zeros gives NaN, as
    0 / 0 does in NumPy.  coherence(trace[:-1], trace[1:]) is the neighbour-channel coherence along a cable."""
    return _cross_spectrum("coherence", x, y, fs, window, nperseg, noverlap, nfft, detrend, True, "density", axis, "mean",
                           True)


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
