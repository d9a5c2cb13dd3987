"""Per-channel (row) operators on the GPU: row statistics, overlap-save matched filter, Hilbert
envelope / SNR, forward-backward SOS IIR, batched STFT.  Thin host wrappers over libd4w.so
(csrc/rows_kernels.cuh); inputs are contiguous float32 CUDA tensors [nx, ns]."""
import os as _os

import numpy as np
import scipy.signal as sp

from . import _lib

_fft_plans = {}
_row_plans = {}
_tab_cache = {}


def _torch():
    import torch
    if not torch.cuda.is_available():
        raise _lib.D4WError("das4whales_b200 needs a CUDA device (no CPU fallback)")
    return torch


def _check_input(x):
    torch = _torch()
    if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.ndim == 2):
        raise ValueError("expected a contiguous float32 CUDA tensor [channels, samples]")
    return x.device.index


class _FftPlan:
    def __init__(self, n, device):
        L = _lib.lib()
        out = _lib.ffi.new("d4w_fft_plan**")
        _lib.check(L.d4w_fft_plan_create(out, int(n), int(device)), f"fft plan n={n}")
        self.ptr, self.n = out[0], int(n)
        order = np.empty(n, dtype=np.int32)
        _lib.check(L.d4w_fft_plan_order(self.ptr, _lib.ffi.cast("int*", order.ctypes.data)), "fft order")
        self.pos2freq = order
        tab = np.empty(n, dtype=np.int32)
        _lib.check(L.d4w_fft_plan_table_order(self.ptr, _lib.ffi.cast("int*", tab.ctypes.data)), "fft table order")
        self.tab2freq = tab                      # order of the multiplier tables d4w_xcorr reads


def fft_plan(n, device):
    key = (int(n), int(device))
    if key not in _fft_plans:
        _fft_plans[key] = _FftPlan(*key)
    return _fft_plans[key]


# Longest row the Hilbert family takes when the length has no T1 x T2 split: its chirp-z convolution (>= 2 ns - 1 points)
# must split as T1 x T2 <= 25 x 10 240 (csrc/fk_hostplan.hpp, kHilbertMaxSamples).  Lengths with a split have no limit here.
HILBERT_MAX_SAMPLES = 128000


class _RowPlan:
    def __init__(self, ns, device):
        L = _lib.lib()
        out = _lib.ffi.new("d4w_row_plan**")
        _lib.check(L.d4w_row_plan_create(out, int(ns), int(device)), f"row plan ns={ns}")
        self.ptr, self.ns, self.device = out[0], int(ns), int(device)
        t1, t2, m = _lib.ffi.new("int*"), _lib.ffi.new("int*"), _lib.ffi.new("int*")
        _lib.check(L.d4w_row_plan_info(self.ptr, t1, t2, m), "row plan info")
        self.t1, self.t2, self.czt_m = int(t1[0]), int(t2[0]), int(m[0])     # czt_m = 0: direct transform

    def info(self):
        """(T1, T2, czt_m): the time split of the transform, and the chirp-z convolution length (0 for a direct plan)"""
        return self.t1, self.t2, self.czt_m


def row_plan(ns, device):
    key = (int(ns), int(device))
    if key not in _row_plans:
        _row_plans[key] = _RowPlan(*key)
    return _row_plans[key]


# ------------------------------------------------------------------------------ statistics
def row_stats(x, seglen=0):
    """-> (stats [nx,4] float64 = mean, absmax, var, 0 ; segpre [nx,nseg] float64 or None)"""
    torch = _torch()
    dev = _check_input(x)
    nx, ns = x.shape
    stats = torch.empty((nx, 4), dtype=torch.float64, device=x.device)
    segpre = None
    if seglen:
        nseg = (ns + seglen - 1) // seglen
        segpre = torch.empty((nx, nseg), dtype=torch.float64, device=x.device)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().d4w_row_stats(_lib.ptr(x, "float*"), nx, ns, int(seglen), _lib.ptr(stats, "double*"),
                                            _lib.ptr(segpre, "double*") if segpre is not None else _lib.ffi.NULL,
                                            _lib.stream_ptr()), "row_stats")
    return stats, segpre


# ------------------------------------------------------------------------------ matched filter
def _pick_block(L, ns=0):
    """Overlap-save block length for templates of L taps.  2520 = 5 * 7 * 8 * 9: prime-factor blocks (no twiddles,
    csrc/fft_pfa.cuh), the default up to 315 taps (>= 87 % of each block valid); longer templates use Cooley-Tukey blocks of
    2500 / 5000 samples (three float2 buffers of a block must fit one SM's shared memory, so 5000 is the largest block and
    2500 taps the longest template one pass can take -- detect.shift_xcorr cuts longer ones into pieces)."""
    def nseg(nb):
        return (ns + (nb - L)) // (nb - L + 1) if ns else 0
    if L <= 2520 // 8 and nseg(2520) <= 512 and _os.environ.get("D4W_XCORR_PFA", "1") != "0":
        return 2520
    for nb, lmax in ((1250, 156), (2500, 312), (5000, 2500)):
        if L <= lmax and (nseg(nb) <= 512 or nb == 5000):   # row statistics keep at most 512 segment prefixes per row
            return nb
    raise ValueError(f"template with {L} taps is too long for one pass of the overlap-save matched filter (max 2500 taps)")


def cross_correlogram(x, templates, normalize=True):
    """Positive-lag correlation of every row with each template (detect.py:96-166).
    templates: list of 1-D float64 arrays (zero-padded to ns, as gen_template_fincall returns).
    Returns a list of float32 CUDA tensors [nx, ns]."""
    torch = _torch()
    dev = _check_input(x)
    nx, ns = x.shape
    taps, mus, ms = [], [], []
    for t in templates:
        t = np.asarray(t, dtype=np.float64).ravel()
        if len(t) != ns and normalize:
            raise ValueError(f"template length {len(t)} != number of samples {ns}")
        nz = np.nonzero(t)[0]
        L = int(nz[-1]) + 1 if len(nz) else 1
        c = t[:L]
        if normalize:
            m = float(np.max(np.abs(t)))              # detect.py:158: abs-max of the un-demeaned template
            mu = float(np.sum(c) / len(t))            # mean of the PADDED template
            taps.append(c - mu)                       # taps of (template - mean) inside the support ...
            mus.append(mu / m)                        # ... and -mu/m outside it (handled as a prefix-sum term)
            ms.append(m)
        else:
            taps.append(c); mus.append(0.0); ms.append(1.0)
    Lmax = max(len(c) for c in taps)
    nb = _pick_block(Lmax, ns)
    valid = nb - Lmax + 1
    plan = fft_plan(nb, dev)
    tabs = np.empty((len(taps), nb), dtype=np.complex64)
    for i, (c, m) in enumerate(zip(taps, ms)):
        spec = np.fft.fft(c, nb)
        tabs[i] = (np.conj(spec) / (nb * m))[plan.tab2freq]
    out = torch.empty((len(taps), nx, ns), dtype=torch.float32, device=x.device)
    with torch.cuda.device(dev):
        tabs_d = torch.from_numpy(tabs.view(np.float32).reshape(len(taps), nb, 2)).to(x.device)
        null = _lib.ffi.NULL
        if normalize:
            stats, segpre = row_stats(x, seglen=valid)
            mu_d = torch.tensor(mus, dtype=torch.float64, device=x.device)
            a_mu, a_st, a_sp = _lib.ptr(mu_d, "double*"), _lib.ptr(stats, "double*"), _lib.ptr(segpre, "double*")
        else:
            a_mu = a_st = a_sp = null
        _lib.check(_lib.lib().d4w_xcorr(plan.ptr, _lib.ptr(x, "float*"), nx, ns, valid, len(taps), _lib.ptr(tabs_d),
                                        a_mu, a_st, a_sp, _lib.ptr(out, "float*"), _lib.stream_ptr()), "xcorr")
    return [out[i] for i in range(len(taps))]


_MAX_ROWS = 65535       # gridDim.y limit of the row kernels


def _row_chunked(corr, x, ntpl):
    """corr(rows) -> ntpl float32 tensors [len(rows), ns], for any number of rows: corr is called on slices of <= 65535 rows
    (the kernels' launch limit) and the parts are copied into whole-matrix outputs."""
    torch = _torch()
    nx = x.shape[0]
    if nx <= _MAX_ROWS:
        return corr(slice(0, nx))
    outs = [torch.empty_like(x) for _ in range(ntpl)]
    for r0 in range(0, nx, _MAX_ROWS):
        part = corr(slice(r0, r0 + _MAX_ROWS))
        for o, p in zip(outs, part):
            o[r0:r0 + _MAX_ROWS] = p
    return outs


def cross_correlogram_chunked(x, templates, normalize=True):
    """cross_correlogram for any number of rows (the kernels take <= 65535 rows per launch)."""
    return _row_chunked(lambda rs: cross_correlogram(x[rs], templates, normalize), x, len(templates))


def same_mode_layout(templates, ns):
    """Host side of the "same"-mode correlation (d4w_xcorr_same), pure NumPy.
    templates: 1-D tap arrays c_t (un-padded, any lengths).  Template t gets D - floor(L_t / 2) zeros prepended, D = max_t
    floor(L_t / 2), so every template has the same lag offset lag0 = D and one forward transform per block serves all of
    them.  Returns (taps, lag0, nb, valid, spec): the prepended taps, the block length (_pick_block of the longest prepended
    template), the outputs kept per block and spec[t] = conj(FFT_nb(taps[t])) / nb in natural frequency order."""
    cs = [np.asarray(c, dtype=np.float64).ravel() for c in templates]
    if not cs or any(len(c) == 0 for c in cs):
        raise ValueError("same-mode correlation needs at least one non-empty template")
    lag0 = max(len(c) // 2 for c in cs)
    taps = [np.concatenate((np.zeros(lag0 - len(c) // 2), c)) for c in cs]
    lmax = max(len(c) for c in taps)
    nb = _pick_block(lmax, ns)
    valid = nb - lmax + 1
    spec = np.stack([np.conj(np.fft.fft(c, nb)) / nb for c in taps])
    return taps, lag0, nb, valid, spec


def cross_correlogram_same(x, templates):
    """scipy.signal.correlate(row / max(row), c, mode='same') of every row with each template, in one pass over the data
    (scripts/main_gabordetect.py:243-246): un-padded templates, no demeaning; a row whose maximum is <= 0 is all zeros (the
    script skips it).  templates: list of 1-D tap arrays (up to 2 500 taps).  Any number of rows.
    Returns a list of float32 CUDA tensors [nx, ns]."""
    torch = _torch()
    dev = _check_input(x)
    nx, ns = x.shape
    _, lag0, nb, valid, spec = same_mode_layout(templates, ns)
    plan = fft_plan(nb, dev)
    tabs = np.ascontiguousarray(spec[:, plan.tab2freq], dtype=np.complex64)
    ntpl = len(templates)
    with torch.cuda.device(dev):
        tabs_d = torch.from_numpy(tabs.view(np.float32).reshape(ntpl, nb, 2)).to(x.device)
        rowmax = row_max(x)                                   # clamped at 0: "> 0" is the script's test, the value its max

        def corr(rs):
            xs = x[rs]
            out = torch.empty((ntpl,) + tuple(xs.shape), dtype=torch.float32, device=x.device)
            _lib.check(_lib.lib().d4w_xcorr_same(plan.ptr, _lib.ptr(xs, "float*"), xs.shape[0], ns, valid, lag0, ntpl,
                                                 _lib.ptr(tabs_d), _lib.ptr(rowmax[rs], "float*"), _lib.ptr(out, "float*"),
                                                 _lib.stream_ptr()), "xcorr_same")
            return [out[i] for i in range(ntpl)]
        return _row_chunked(corr, x, ntpl)


# ------------------------------------------------------------------------------ Hilbert envelope / SNR
def _hilbert(x, mode, stats=None):
    torch = _torch()
    dev = _check_input(x)
    nx, ns = x.shape
    plan = row_plan(ns, dev)
    out = torch.empty_like(x)
    L = _lib.lib()
    with torch.cuda.device(dev):
        # rows are independent: chunk so the complex workspace stays bounded (and gridDim.y <= 65535); a workspace row is
        # ns complex samples on the direct route and czt_m ~ 2 ns on the chirp-z route
        max_rows = max(1, min(65535, (8 << 30) // max(1, int(L.d4w_row_workspace_bytes(plan.ptr, 1)))))
        wsb = L.d4w_row_workspace_bytes(plan.ptr, min(nx, max_rows))
        ws = torch.empty(int(wsb), dtype=torch.uint8, device=x.device)
        for r0 in range(0, nx, max_rows):
            r1 = min(nx, r0 + max_rows)
            st = _lib.ptr(stats[r0:r1], "double*") if stats is not None else _lib.ffi.NULL
            _lib.check(L.d4w_hilbert(plan.ptr, _lib.ptr(x[r0:r1], "float*"), _lib.ptr(out[r0:r1], "float*"), r1 - r0,
                                     _lib.ptr(ws), int(mode), st, _lib.stream_ptr()), "hilbert")
    return out


def envelope(x):
    """|scipy.signal.hilbert(x, axis=1)|"""
    return _hilbert(x, 0)


def hilbert_imag(x):
    """imag(scipy.signal.hilbert(x, axis=1)) = the Hilbert transform H(x) of every row"""
    return _hilbert(x, 2)


def envelope_over_std(x):
    """|hilbert(x)| / std_row(x)  (improcess.trace2image before the pixel scaling, improcess.py:61)"""
    stats, _ = row_stats(x)
    return _hilbert(x, 3, stats)


ENV_STATS_FIELDS = ("median_env", "mean_env", "mean", "mean_sq", "var")


def env_stats(x, t0=0, n=None):
    """Envelope and moment statistics of the window x[:, t0:t0 + n] of every row (scripts/main_bathynoise.py:183-189,
    :257-259), read in place.  x: contiguous float32 CUDA tensor [nx, ns]; n defaults to ns - t0.  Returns a float64 CUDA
    tensor [nx, 5] with the columns ENV_STATS_FIELDS: median and mean of |scipy.signal.hilbert(window)|, and the mean, mean
    square and population variance of the window.  The Hilbert transform is that of the window alone."""
    torch = _torch()
    dev = _check_input(x)
    nx, ns = x.shape
    t0 = int(t0)
    n = ns - t0 if n is None else int(n)
    if t0 < 0 or n < 1 or t0 + n > ns:
        raise ValueError(f"env_stats: window [{t0}, {t0 + n}) is empty or outside the {ns} samples of a row")
    plan = row_plan(n, dev)
    out = torch.empty((nx, 5), dtype=torch.float64, device=x.device)
    L = _lib.lib()
    with torch.cuda.device(dev):
        # the workspace holds the envelope and the Hilbert workspace of a chunk of rows: chunk so that it stays bounded, as _hilbert
        per_row = max(1, int(L.d4w_env_stats_workspace_bytes(plan.ptr, 1, ns)))
        max_rows = max(1, min(nx, (8 << 30) // per_row))
        ws = torch.empty(int(L.d4w_env_stats_workspace_bytes(plan.ptr, max_rows, ns)), dtype=torch.uint8, device=x.device)
        base = x.data_ptr() + 4 * t0
        for r0 in range(0, nx, max_rows):
            r1 = min(nx, r0 + max_rows)
            _lib.check(L.d4w_env_stats(plan.ptr, _lib.ffi.cast("float*", base + 4 * r0 * ns), r1 - r0, ns,
                                       _lib.ptr(out[r0:r1], "double*"), _lib.ptr(ws), _lib.stream_ptr()), "env_stats")
    return out


def row_fft_mag(x, nfft, scale):
    """|numpy.fft.fft(x, nfft)| * scale in fftshift order for every row (dsp.get_fx, dsp.py:35-37)."""
    torch = _torch()
    dev = _check_input(x)
    nx, ns = x.shape
    plan = fft_plan(int(nfft), dev)
    out = torch.empty((nx, int(nfft)), dtype=torch.float32, device=x.device)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().d4w_row_fft_mag(plan.ptr, _lib.ptr(x, "float*"), nx, ns, min(ns, int(nfft)), float(scale),
                                              _lib.ptr(out, "float*"), _lib.stream_ptr()), "row_fft_mag")
    return out


def inst_freq(x1d, fs):
    """dsp.instant_freq for one channel: float32 CUDA tensor [n] -> [n - 1]"""
    torch = _torch()
    x = x1d.reshape(1, -1).contiguous()
    hx = hilbert_imag(x)
    n = x.shape[1]
    out = torch.empty(n - 1, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device.index):
        _lib.check(_lib.lib().d4w_inst_freq(_lib.ptr(x, "float*"), _lib.ptr(hx, "float*"), n, float(fs), _lib.ptr(out, "float*"),
                                            _lib.stream_ptr()), "inst_freq")
    return out


def snr(x, env=False):
    """dsp.snr_tr_array (dsp.py:956-976)"""
    torch = _torch()
    dev = _check_input(x)
    stats, _ = row_stats(x)
    if env:
        return _hilbert(x, 1, stats)
    out = torch.empty_like(x)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().d4w_snr(_lib.ptr(x, "float*"), _lib.ptr(out, "float*"), x.shape[0], x.shape[1],
                                      _lib.ptr(stats, "double*"), _lib.stream_ptr()), "snr")
    return out


# ------------------------------------------------------------------------------ zero-phase SOS IIR
def sosfiltfilt(sos, x, padlen=None):
    """scipy.signal.sosfiltfilt(sos, x, axis=1) semantics (odd extension, sosfilt_zi initial
    state); padlen=None uses SciPy's default, bp_filt passes filtfilt's 3*max(len(a),len(b))."""
    torch = _torch()
    dev = _check_input(x)
    sos = np.ascontiguousarray(sos, dtype=np.float64)
    if sos.ndim != 2 or sos.shape[1] != 6:
        raise ValueError("sos must have shape (n_sections, 6)")
    nsec = sos.shape[0]
    if padlen is None:
        ntaps = 2 * nsec + 1
        ntaps -= min((sos[:, 2] == 0).sum(), (sos[:, 5] == 0).sum())
        padlen = 3 * ntaps
    nx, ns = x.shape
    if ns <= padlen:
        raise ValueError(f"The length of the input vector x must be greater than padlen, which is {padlen}.")
    zi = np.ascontiguousarray(sp.sosfilt_zi(sos), dtype=np.float64)
    y = torch.empty_like(x)
    tmp = torch.empty((nx, ns + 2 * padlen), dtype=torch.float32, device=x.device)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().d4w_sosfiltfilt(_lib.ptr(x, "float*"), _lib.ptr(y, "float*"), _lib.ptr(tmp, "float*"), nx, ns,
                                              _lib.ffi.cast("double*", sos.ctypes.data), _lib.ffi.cast("double*", zi.ctypes.data),
                                              nsec, int(padlen), _lib.stream_ptr()), "sosfiltfilt")
    return y


# ------------------------------------------------------------------------------ STFT magnitude
def stft_mag(x, nfft, hop, bin_lo=0, bin_hi=None):
    """|librosa.stft(y, n_fft=nfft, hop_length=hop)| for every row, DFT bins bin_lo..bin_hi
    -> [nx, bin_hi-bin_lo+1, 1+ns//hop]"""
    torch = _torch()
    dev = _check_input(x)
    nx, ns = x.shape
    plan = fft_plan(nfft, dev)
    nframes = 1 + ns // hop
    bin_hi = nfft // 2 if bin_hi is None else int(bin_hi)
    out = torch.empty((nx, bin_hi - bin_lo + 1, nframes), dtype=torch.float32, device=x.device)
    key = ("hann", nfft, dev)
    if key not in _tab_cache:
        _tab_cache[key] = torch.from_numpy(sp.get_window("hann", nfft, fftbins=True).astype(np.float32)).to(x.device)
    win = _tab_cache[key]
    L = _lib.lib()
    slide = bool(L.d4w_stft_slide_supported(int(nfft), int(hop), bin_hi - bin_lo + 1))    # band of bins, hop | n_fft
    with torch.cuda.device(dev):
        for r0 in range(0, nx, 65535):
            r1 = min(nx, r0 + 65535)
            if slide:
                _lib.check(L.d4w_stft_slide(plan.ptr, _lib.ptr(x[r0:r1], "float*"), _lib.ptr(out[r0:r1], "float*"), r1 - r0, ns,
                                            int(hop), int(bin_lo), bin_hi, _lib.stream_ptr()), "stft_slide")
                continue
            _lib.check(L.d4w_stft_mag(plan.ptr, _lib.ptr(x[r0:r1], "float*"), _lib.ptr(out[r0:r1], "float*"), r1 - r0, ns,
                                      int(hop), _lib.ptr(win, "float*"), int(bin_lo), bin_hi, _lib.stream_ptr()), "stft_mag")
    return out


# ------------------------------------------------------------------------------ spectrogram correlation
def row_max(x2d):
    """max over the last axis of a [rows, n] float32 CUDA tensor"""
    torch = _torch()
    rows_, n = x2d.shape
    out = torch.empty(rows_, dtype=torch.float32, device=x2d.device)
    with torch.cuda.device(x2d.device.index):
        _lib.check(_lib.lib().d4w_row_max(_lib.ptr(x2d, "float*"), rows_, n, _lib.ptr(out, "float*"), _lib.stream_ptr()), "row_max")
    return out


def row_median(x2d):
    """np.median over the last axis of a non-negative [rows, n] float32 CUDA tensor"""
    torch = _torch()
    rows_, n = x2d.shape
    out = torch.empty(rows_, dtype=torch.float32, device=x2d.device)
    with torch.cuda.device(x2d.device.index):
        _lib.check(_lib.lib().d4w_row_median(_lib.ptr(x2d, "float*"), rows_, n, _lib.ptr(out, "float*"), _lib.stream_ptr()), "row_median")
    return out


def row_median_ld(x, nrows, n, ld, offset=0):
    """np.median of x.flat[offset + r * ld : offset + r * ld + n] for r < nrows, x a contiguous non-negative float32 CUDA
    tensor.  For the band of rows f0 .. f0 + m - 1 of every channel of a spectrogram [nx, nf, nt]: nrows = nx, n = m * nt,
    ld = nf * nt, offset = f0 * nt.  Returns [nrows] float32."""
    torch = _torch()
    if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()):
        raise ValueError("expected a contiguous float32 CUDA tensor")
    nrows, n, ld, offset = int(nrows), int(n), int(ld), int(offset)
    if nrows < 1 or n < 1 or ld < n or offset < 0 or offset + (nrows - 1) * ld + n > x.numel():
        raise ValueError(f"row_median_ld: {nrows} rows of {n} values at stride {ld} from {offset} do not fit {x.numel()} values")
    out = torch.empty(nrows, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device.index):
        _lib.check(_lib.lib().d4w_row_median_ld(_lib.ffi.cast("float*", x.data_ptr() + 4 * offset), nrows, n, ld,
                                                _lib.ptr(out, "float*"), _lib.stream_ptr()), "row_median_ld")
    return out


SPECCORR_MAX_KERNELS = 8        # kernels per d4w_speccorr_multi call (csrc/rows_kernels.cuh, kScMaxKernels)


def spectro_correlate_multi(S, kernels, offsets, medians, outs=None):
    """spectro_correlate of several kernels against one band spectrogram S [nx, nf, nt] (float32 CUDA), S read once per
    group of up to 8 kernels: kernel k ([nf_k, kw_k]) covers the rows offsets[k] .. offsets[k] + nf_k - 1 of S and is
    normalised by medians[k] ([nx] float32 CUDA).  Output k is bit-equal to spectro_correlate(S[:, o:o + nf_k], kernel,
    median).  outs: optional contiguous [nx, nt] float32 tensors to write.  Any number of rows.  Returns the list of outputs."""
    torch = _torch()
    if not (isinstance(S, torch.Tensor) and S.is_cuda and S.dtype == torch.float32 and S.is_contiguous() and S.ndim == 3):
        raise ValueError("expected a contiguous float32 CUDA tensor [channels, bins, frames]")
    nx, nf, nt = S.shape
    Ks = [torch.from_numpy(np.ascontiguousarray(k, dtype=np.float32)).to(S.device) for k in kernels]
    if len(Ks) == 0 or len(Ks) != len(offsets) or len(Ks) != len(medians):
        raise ValueError("spectro_correlate_multi: one offset and one median per kernel")
    for K, o in zip(Ks, offsets):
        if K.ndim != 2 or K.shape[1] < 1 or o < 0 or o + K.shape[0] > nf:
            raise ValueError(f"kernel of shape {tuple(K.shape)} at bin offset {o} does not fit a band of {nf} bins")
    if any(m.dtype != torch.float32 or not m.is_cuda or tuple(m.shape) != (nx,) for m in medians):
        raise ValueError(f"medians must be float32 CUDA tensors of {nx} values")
    if outs is None:
        outs = [torch.empty((nx, nt), dtype=torch.float32, device=S.device) for _ in Ks]
    if len(outs) != len(Ks) or any(o.dtype != torch.float32 or tuple(o.shape) != (nx, nt) or not o.is_contiguous() for o in outs):
        raise ValueError(f"outs must be contiguous float32 CUDA tensors [{nx}, {nt}]")
    ffi, L = _lib.ffi, _lib.lib()
    with torch.cuda.device(S.device.index):
        for g0 in range(0, len(Ks), SPECCORR_MAX_KERNELS):
            g = range(g0, min(len(Ks), g0 + SPECCORR_MAX_KERNELS))
            f0 = ffi.new("int[]", [int(offsets[k]) for k in g])
            nfk = ffi.new("int[]", [Ks[k].shape[0] for k in g])
            kw = ffi.new("int[]", [Ks[k].shape[1] for k in g])
            kp = ffi.new("float*[]", [_lib.ptr(Ks[k], "float*") for k in g])
            for r0 in range(0, nx, _MAX_ROWS):
                r1 = min(nx, r0 + _MAX_ROWS)
                mp = ffi.new("float*[]", [_lib.ptr(medians[k][r0:r1], "float*") for k in g])
                op = ffi.new("float*[]", [_lib.ptr(outs[k][r0:r1], "float*") for k in g])
                _lib.check(L.d4w_speccorr_multi(_lib.ptr(S[r0:r1], "float*"), r1 - r0, nf, nt, len(g), f0, nfk, kp, kw, mp, op,
                                                _lib.stream_ptr()), "speccorr_multi")
    return outs


def spectro_correlate(S, kernel, median=None):
    """detect.xcorr2d for a batch: S [nx, nf, nt] float32 CUDA (un-normalised magnitudes are fine:
    the max-normalisation of get_sliced_nspectrogram cancels against the median), kernel [nf, kw]."""
    torch = _torch()
    nx, nf, nt = S.shape
    K = torch.from_numpy(np.ascontiguousarray(kernel, dtype=np.float32)).to(S.device)
    if K.shape[0] != nf:
        raise ValueError(f"kernel has {K.shape[0]} frequency rows, spectrogram slice has {nf}")
    kw = K.shape[1]
    if median is None:
        median = row_median(S.reshape(nx, nf * nt))
    out = torch.empty((nx, nt), dtype=torch.float32, device=S.device)
    with torch.cuda.device(S.device.index):
        _lib.check(_lib.lib().d4w_speccorr(_lib.ptr(S, "float*"), nx, nf, nt, _lib.ptr(K, "float*"), kw, _lib.ptr(median, "float*"),
                                           _lib.ptr(out, "float*"), _lib.stream_ptr()), "speccorr")
    return out


def find_peaks_flags(x2d, prominence):
    """scipy.signal.find_peaks(row, prominence=prominence) on every row of a [rows, n] float32 CUDA tensor;
    returns a uint8 [rows, n] tensor with 1 at every accepted peak (reference call sites: detect.py:192, :271)."""
    torch = _torch()
    rows_, n = x2d.shape
    L = _lib.lib()
    flags = torch.empty((rows_, n), dtype=torch.uint8, device=x2d.device)
    with torch.cuda.device(x2d.device.index):
        ws = torch.empty(int(L.d4w_find_peaks_workspace_bytes(min(rows_, 65535), n)), dtype=torch.uint8, device=x2d.device)
        for r0 in range(0, rows_, 65535):
            r1 = min(rows_, r0 + 65535)
            _lib.check(L.d4w_find_peaks(_lib.ptr(x2d[r0:r1], "float*"), r1 - r0, n, float(prominence),
                                        _lib.ffi.cast("unsigned char*", flags[r0:r1].data_ptr()), _lib.ptr(ws, "void*"),
                                        _lib.stream_ptr()), "find_peaks")
    return flags


def compact_picks(flags):
    """flags uint8 [rows, n] -> (offsets int32 [rows + 1], idx int32 [total]) on the device: ascending sample indices of
    every row, rows concatenated (d4w_peaks_offsets / d4w_peaks_fill).  One 4-byte D2H read (the total) in between."""
    torch = _torch()
    rows_, n = flags.shape
    L = _lib.lib()
    counts = torch.empty(rows_, dtype=torch.int32, device=flags.device)
    offsets = torch.empty(rows_ + 1, dtype=torch.int32, device=flags.device)
    u8 = lambda t: _lib.ffi.cast("unsigned char*", t.data_ptr())
    with torch.cuda.device(flags.device.index):
        _lib.check(L.d4w_peaks_offsets(u8(flags), rows_, n, _lib.ptr(counts, "int*"), _lib.ptr(offsets, "int*"), _lib.stream_ptr()),
                   "peaks_offsets")
        total = int(offsets[-1].item())
        idx = torch.empty(max(total, 1), dtype=torch.int32, device=flags.device)
        if total:
            _lib.check(L.d4w_peaks_fill(u8(flags), rows_, n, _lib.ptr(offsets, "int*"), _lib.ptr(idx, "int*"), _lib.stream_ptr()),
                       "peaks_fill")
    return offsets, idx[:total]


def find_peaks_device(x2d, prominence):
    """(offsets, idx) of compact_picks for scipy.signal.find_peaks(row, prominence=...) on every row; stays on the GPU."""
    return compact_picks(find_peaks_flags(x2d, prominence))


def find_peaks(x2d, prominence):
    """Per-row peak indices (list of int64 ndarrays, ascending) -- only the picks leave the GPU."""
    offsets, idx = find_peaks_device(x2d, prominence)
    off = offsets.cpu().numpy().astype(np.int64)
    ii = idx.cpu().numpy().astype(np.int64)
    return [ii[off[r]:off[r + 1]] for r in range(x2d.shape[0])]


def raw2strain(raw2d, scale_factor):
    """(raw - mean_row) * scale_factor from int32 / float32 counts to float32 strain (data_handle.py:157-177)."""
    torch = _torch()
    if raw2d.dtype not in (torch.int32, torch.float32):
        raise ValueError("raw2strain: raw data must be int32 or float32")
    rows_, n = raw2d.shape
    out = torch.empty((rows_, n), dtype=torch.float32, device=raw2d.device)
    with torch.cuda.device(raw2d.device.index):
        _lib.check(_lib.lib().d4w_raw2strain(_lib.ffi.cast("void*", raw2d.data_ptr()), 1 if raw2d.dtype == torch.int32 else 0,
                                             rows_, n, float(scale_factor), _lib.ptr(out, "float*"), _lib.stream_ptr()), "raw2strain")
    return out
