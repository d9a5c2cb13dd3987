"""das4whales_b200.detect -- drop-in for the hot-path functions of `das4whales.detect`
(/root/reference/src/das4whales/detect.py): same names, positional order and defaults.
"""
import numpy as np
import scipy.signal as sp

from . import rows as _rows
from .dsp import _is_tensor, _to_device, _to_host64


# ---- templates (host side: tiny, keeps SciPy's chirp formula -- detect.py:20-93) --------
def gen_linear_chirp(fmin, fmax, duration, sampling_rate):
    """Linear down-sweep fmax -> fmin (reference: detect.py:20-41)."""
    t = np.arange(0, duration, 1 / sampling_rate)
    return sp.chirp(t, f0=fmax, f1=fmin, t1=duration, method="linear")


def gen_hyperbolic_chirp(fmin, fmax, duration, sampling_rate):
    """Hyperbolic down-sweep fmax -> fmin (reference: detect.py:44-65)."""
    t = np.arange(0, duration, 1 / sampling_rate)
    return sp.chirp(t, f0=fmax, f1=fmin, t1=duration, method="hyperbolic")


def gen_template_fincall(time, fs, fmin=15., fmax=25., duration=1., window=True):
    """Fin-whale call template, zero-padded to len(time) (reference: detect.py:68-93)."""
    chirp_signal = gen_hyperbolic_chirp(fmin, fmax, duration, fs)
    template = np.zeros(np.shape(time))
    n = len(chirp_signal)
    template[:n] = chirp_signal * np.hanning(n) if window else chirp_signal
    return template


def _host1d(a):
    if _is_tensor(a):
        return a.detach().to("cpu").numpy().astype(np.float64).ravel()
    return np.asarray(a, dtype=np.float64).ravel()


_MAX_TAPS = 2400        # one pass of the overlap-save correlator takes templates of up to 2 500 taps; longer ones are cut into pieces


def _lags_on_device(x_dev, y_host):
    """z[tau] = sum_n x[n + tau] y[n] for tau = 0 .. len(x) - 1 (float32 CUDA tensor), y = FIR taps on the host.
    Long tap vectors are split into pieces of <= 2 400 taps: the correlation with piece p (taps p*B ...) is the piece's own
    correlogram read p*B lags later, so the pieces' shifted correlograms add up to the full one."""
    import torch
    y = np.asarray(y_host, dtype=np.float64).ravel()
    nz = np.nonzero(y)[0]
    L = int(nz[-1]) + 1 if len(nz) else 1
    if L <= _MAX_TAPS:
        return _rows.cross_correlogram(x_dev, [y], normalize=False)[0][0]
    n = x_dev.shape[1]
    out = torch.zeros(n, dtype=torch.float32, device=x_dev.device)
    for p0 in range(0, min(L, n), _MAX_TAPS):
        piece = y[p0:min(L, p0 + _MAX_TAPS)]
        if not np.any(piece):
            continue
        z = _rows.cross_correlogram(x_dev, [piece], normalize=False)[0][0]          # lags of the piece alone
        out[: n - p0] += z[p0:]
    return out


def shift_xcorr(x, y):
    """`scipy.signal.correlate(x, y, 'full', 'fft')[len(x) - 1:]` (reference: detect.py:96-112): len(y) values, lag
    tau_j = len(x) - len(y) + j.  For equal lengths (the reference's use) these are the positive lags 0 .. len(x) - 1;
    for unequal lengths the same slice of the full correlation is returned, negative lags included.
    ndarray in -> float64 ndarray out; CUDA tensor in -> float32 CUDA tensor out."""
    import torch
    tens = _is_tensor(x)
    xh = None if tens else np.asarray(x, dtype=np.float64).ravel()
    xd = (x.reshape(1, -1).to(torch.float32).contiguous() if tens else _to_device(xh[None, :]))
    yh = _host1d(y)
    nx_, ny_ = xd.shape[1], len(yh)
    zpos = _lags_on_device(xd, yh)                                 # lags 0 .. nx_-1
    first = nx_ - ny_                                              # lag of the first returned sample
    if first >= 0:
        out = zpos[first:first + ny_]
    else:
        # negative lags: z_xy[-m] = z_yx[m] -- correlate y (as the signal) against x (as the taps)
        yd = torch.from_numpy(yh.astype(np.float32))[None, :].to(xd.device)
        xtaps = _host1d(x)
        zneg = _lags_on_device(yd, xtaps)                          # z_yx[m], m = 0 .. ny_-1
        out = torch.cat((torch.flip(zneg[1:-first + 1], dims=(0,)), zpos))[:ny_]
    return out if tens else out.to(torch.float64).cpu().numpy()


def shift_nxcorr(x, y):
    """Std-normalised cross-correlation, same lags as shift_xcorr (reference: detect.py:115-137)."""
    xh, yh = _host1d(x), _host1d(y)
    return shift_xcorr(x, y) / (np.std(xh) * np.std(yh) * len(xh))


def compute_cross_correlogram(data, template):
    """Matched filter of every channel against `template` (reference: detect.py:140-166):
    rows demeaned and divided by their raw abs-max, template (zero-padded to ns) demeaned and
    divided by its abs-max, positive lags of the full correlation."""
    xd = _to_device(data)
    out = _rows.cross_correlogram_chunked(xd, [np.asarray(template, dtype=np.float64)], normalize=True)[0]
    return out if _is_tensor(data) else _to_host64(out)


def compute_cross_correlograms(data, templates):
    """Several templates in ONE pass over the data (HF + LF notes of scripts/main_mfdetect.py:79-80)."""
    xd = _to_device(data)
    outs = _rows.cross_correlogram_chunked(xd, [np.asarray(t, dtype=np.float64) for t in templates], normalize=True)
    return outs if _is_tensor(data) else [_to_host64(o) for o in outs]


def compute_cross_correlogram_same(data, template):
    """Matched filter of scripts/main_gabordetect.py:238-246 (there is no library function for it): for every channel,
    `scipy.signal.correlate(row / max(row), template, mode='same')` with the un-padded template (the script's Hann-windowed
    hyperbolic chirp), no demeaning.  Channels whose maximum is <= 0 -- the ones a Gabor mask zeroes -- come back as zeros
    (the script skips them and leaves np.empty_like values).  ndarray in -> float64 ndarray out; CUDA tensor in -> float32
    CUDA tensor out."""
    return compute_cross_correlograms_same(data, [template])[0]


def compute_cross_correlograms_same(data, templates):
    """compute_cross_correlogram_same for several templates in ONE pass over the data (the HF and LF notes of
    scripts/main_gabordetect.py:223-246).  Returns a list with one correlogram per template."""
    xd = _to_device(data)
    outs = _rows.cross_correlogram_same(xd, [_host1d(t) for t in templates])
    return outs if _is_tensor(data) else [_to_host64(o) for o in outs]


def envelope(corr_m):
    """|hilbert(row)| for every row -- the quantity pick_times_env thresholds (detect.py:192)."""
    y = _rows.envelope(_to_device(corr_m))
    return y if _is_tensor(corr_m) else _to_host64(y)


def pick_times_env(corr_m, threshold):
    """Peaks of the Hilbert envelope with prominence >= threshold (reference: detect.py:169-195).
    Envelope and scipy.signal.find_peaks' prominence search both run on the GPU (d4w_hilbert, d4w_find_peaks);
    only the picks are copied back: list with one int64 index array per channel, like the reference."""
    return _rows.find_peaks(_rows.envelope(_to_device(corr_m)), float(threshold))


def pick_times(corr_m, threshold):
    """Peaks of the raw correlogram with prominence >= threshold (reference: detect.py:249-274)."""
    return _rows.find_peaks(_to_device(corr_m), float(threshold))


def process_corr(corr, threshold):
    """Peak indexes of ONE correlation series: find_peaks(|hilbert(corr)|, prominence=threshold)[0]
    (reference: detect.py:198-218, the per-channel kernel of pick_times_par)."""
    c = corr.reshape(1, -1) if _is_tensor(corr) else np.asarray(corr)[None, :]
    return pick_times_env(c, threshold)[0]


def pick_times_par(corr_m, threshold):
    """Reference: detect.py:221-246 (a thread pool over process_corr whose results arrive in completion order).  All
    channels are picked in one batched GPU pass; the list is returned in channel order, like pick_times_env."""
    return pick_times_env(corr_m, threshold)


def convert_pick_times(peaks_indexes_m):
    """list of per-channel index arrays -> array([[channel...],[time...]]) (detect.py:277-303)."""
    counts = [len(p) for p in peaks_indexes_m]
    ch = np.repeat(np.arange(len(counts), dtype=np.int64), counts)
    tt = np.concatenate([np.asarray(p, dtype=np.int64) for p in peaks_indexes_m]) if counts else np.empty(0, dtype=np.int64)
    return np.asarray((ch, tt))


def select_picked_times(idx_tp, tstart, tend, fs):
    """Keep picks with tstart <= t <= tend (reference: detect.py:306-330)."""
    keep = (idx_tp[1] >= tstart * fs) & (idx_tp[1] <= tend * fs)
    return (idx_tp[0][keep], idx_tp[1][keep])


# north-star aliases
matched_filter = compute_cross_correlogram
xcorr_templates = compute_cross_correlograms


# ---- spectrogram-correlation detector (reference: detect.py:334-708) -----------------------
def _band_bins(nfft, fs, fmin, fmax):
    ff = np.linspace(0, fs / 2, num=nfft // 2 + 1)
    sel = np.where((ff >= fmin) & (ff <= fmax))[0]
    if len(sel) == 0:
        raise ValueError("no STFT bin inside [fmin, fmax]")
    return ff, int(sel[0]), int(sel[-1])


def get_sliced_nspectrogram(trace, fs, fmin, fmax, nperseg, nhop, plotflag=False):
    """|STFT| / max, rows with fmin <= f <= fmax (reference: detect.py:334-408)."""
    import torch
    xd = _to_device(np.asarray(trace)[None, :] if not _is_tensor(trace) else trace.reshape(1, -1))
    ff, b0, b1 = _band_bins(nperseg, fs, fmin, fmax)
    full = _rows.stft_mag(xd, nperseg, nhop)                       # max is taken over ALL bins (detect.py:387)
    mx = _rows.row_max(full.reshape(1, -1))
    p = full[0, b0:b1 + 1] / mx
    nt = p.shape[1]
    tt = np.linspace(0, xd.shape[1] / fs, num=nt)
    if plotflag:
        import matplotlib.pyplot as plt
        plt.pcolormesh(tt, ff[b0:b1 + 1], 20 * np.log10(p.cpu().numpy() / float(p.max())))
        plt.show()
    return (p if _is_tensor(trace) else p.to(torch.float64).cpu().numpy()), ff[b0:b1 + 1], tt


def buildkernel(f0, f1, bdwdth, dur, f, t, samp, fmin, fmax, plotflag=False):
    """Hat-function hyperbolic-sweep kernel x Hann in time (reference: detect.py:411-492).
    Host side: the kernel is a few hundred values."""
    tvec = np.linspace(0, dur, np.size(np.nonzero((t < dur * 8) & (t > dur * 7))))
    fvec = np.asarray(f)
    x = fvec[:, None] - (f0 * f1 * dur / ((f0 - f1) * tvec[None, :] + f1 * dur))
    kdist = (1 - np.square(x) / (bdwdth * bdwdth)) * np.exp(-np.square(x) / (2 * (bdwdth * bdwdth)))
    return tvec, fvec, kdist * np.hanning(len(tvec))[np.newaxis, :]


def buildkernel_from_template(fmin, fmax, dur, fs, nperseg, nhop, plotflag=False):
    """Spectrogram of the windowed template as a kernel (reference: detect.py:495-541)."""
    template = gen_hyperbolic_chirp(fmin, fmax, dur, fs)
    template *= np.hanning(len(template))
    spectro, _, _ = get_sliced_nspectrogram(template, fs, fmin, fmax, nperseg, nhop, plotflag=False)
    return spectro


def xcorr2d(spectro, kernel):
    """Sum over frequency of the time-correlation of spectrogram and kernel, clipped at zero and
    divided by median(spectro) * kernel width (reference: detect.py:579-602)."""
    import torch
    if _is_tensor(spectro):
        S = spectro.to(torch.float32).contiguous()[None]
    else:
        S = torch.from_numpy(np.ascontiguousarray(spectro, dtype=np.float32)).cuda()[None]
    out = _rows.spectro_correlate(S, kernel)[0]
    return out if _is_tensor(spectro) else out.to(torch.float64).cpu().numpy()


def nxcorr2d(spectro, kernel):
    """max over frequency lags of the normalised 2-D cross-correlation (reference: detect.py:544-576):
    scipy.signal.correlate(spectro, kernel, 'same') / (std(spectro) std(kernel) n_time) -> max over axis 0."""
    import torch
    from . import improcess as _imp
    tens = _is_tensor(spectro)
    S = spectro.to(torch.float32).contiguous() if tens else torch.from_numpy(np.ascontiguousarray(spectro, dtype=np.float32)).cuda()
    K = np.ascontiguousarray(_host2d(kernel), dtype=np.float64)
    corr = _imp.filter2D(S, None, K, border="zeros")
    s_std = float(_rows.row_stats(S.reshape(1, -1))[0][0, 2].sqrt().item())      # population std of the whole spectrogram
    out = _rows.row_max(corr.t().contiguous()) / (s_std * float(np.std(K)) * S.shape[1])      # max over the frequency lags
    return out if tens else out.to(torch.float64).cpu().numpy()


def _host2d(a):
    if _is_tensor(a):
        return a.detach().to("cpu").numpy()
    return np.asarray(a)


def xcorr(t, f, Sxx, tvec, fvec, BlueKernel):
    """Sliding dot product of a kernel with a spectrogram ('valid' lags), normalised by median(Sxx) * len(tvec), first and
    last value zeroed, negatives clipped (reference: detect.py:605-647).  Returns [t_scale, CorrVal]."""
    import torch
    tvec_size, fvec_size = int(np.size(tvec)), int(np.size(fvec))
    tens = _is_tensor(Sxx)
    S = Sxx.to(torch.float32).contiguous() if tens else torch.from_numpy(np.ascontiguousarray(Sxx, dtype=np.float32)).cuda()
    nt = S.shape[1]
    nval = nt - (tvec_size - 1)
    med = _rows.row_median(S.reshape(1, -1))                       # median over the WHOLE spectrogram (detect.py:642)
    same = _rows.spectro_correlate(S[:fvec_size][None].contiguous(), _host2d(BlueKernel), median=med)[0]
    corr = same[tvec_size // 2: tvec_size // 2 + nval].clone()     # 'valid' lags of the 'same'-mode correlation
    corr[0] = 0
    corr[-1] = 0
    t = np.asarray(t)
    t_scale = t[int(tvec_size / 2) - 1:-int(np.ceil(tvec_size / 2))]
    return [t_scale, corr if tens else corr.to(torch.float64).cpu().numpy()]


def spectrocorr_layout(fs, flims, kernels, win_size, overlap_pct, ns):
    """Host side of the spectrogram-correlation detector for several kernels sharing one STFT, pure NumPy.
    kernels: dicts {f0, f1, dur, bdwidth} (scripts/main_spectrodetect.py:103-104).  Each kernel widens flims as
    detect.py:693-696 does (fmax -> f1 + 3 bdwidth when fmax - f1 < 2 bdwidth, fmin -> f0 - 3 bdwidth when
    f0 - fmin < 2 bdwidth) and gets its buildkernel matrix on its own bins and the ns-sample record's frame times.
    Returns (nperseg, nhop, bands, (b0, b1), per_kernel): bands[k] = the widened (fmin, fmax); b0 .. b1 the union of the
    kernels' STFT bins (inclusive); per_kernel[k] = (offset of the kernel's first bin from b0, kernel [nf_k, kw_k], kw_k)."""
    nperseg = int(win_size * fs)
    nhop = int(np.floor(nperseg * (1 - overlap_pct)))
    if nperseg < 1 or nhop < 1:
        raise ValueError(f"window of {nperseg} samples with a hop of {nhop}: both must be >= 1")
    nt = 1 + int(ns) // nhop
    tt = np.linspace(0, int(ns) / fs, num=nt)
    bands, bins, kers = [], [], []
    for kernel in kernels:
        fmin, fmax = flims
        f1, f0, duration, bandwidth = kernel["f1"], kernel["f0"], kernel["dur"], kernel["bdwidth"]
        if fmax - f1 < 2 * bandwidth:
            fmax = f1 + 3 * bandwidth
        if f0 - fmin < 2 * bandwidth:
            fmin = f0 - 3 * bandwidth
        ff, b0, b1 = _band_bins(nperseg, fs, fmin, fmax)
        _, _, ker = buildkernel(f0, f1, bandwidth, duration, ff[b0:b1 + 1], tt, fs, fmin, fmax, plotflag=False)
        if ker.shape[1] == 0:
            raise ValueError(f"a kernel of {duration} s has no frames in a {int(ns) / fs:g} s record: buildkernel takes "
                             f"its width from the frames with {7 * duration:g} s < t < {8 * duration:g} s")
        bands.append((fmin, fmax))
        bins.append((b0, b1))
        kers.append(ker)
    if not kers:
        raise ValueError("spectrogram correlation needs at least one kernel")
    u0, u1 = min(b[0] for b in bins), max(b[1] for b in bins)
    return nperseg, nhop, bands, (u0, u1), [(b[0] - u0, k, k.shape[1]) for b, k in zip(bins, kers)]


def _spectrocorr_device(xd, nperseg, nhop, union, per_kernel):
    """The multi-kernel pass of spectrocorr_layout's layout on a float32 CUDA tensor [nx, ns], in channel chunks: one STFT
    of the union band, one median per kernel over its slice of the band, one d4w_speccorr_multi.  -> list of [nx, nt]."""
    import torch
    nx, ns = xd.shape
    b0, b1 = union
    nf, nt = b1 - b0 + 1, 1 + ns // nhop
    outs = [torch.empty((nx, nt), dtype=torch.float32, device=xd.device) for _ in per_kernel]
    chunk = max(1, min(nx, _rows._MAX_ROWS, (2 << 30) // max(1, nf * nt * 4)))
    for r0 in range(0, nx, chunk):
        S = _rows.stft_mag(xd[r0:r0 + chunk], nperseg, nhop, b0, b1)
        n = S.shape[0]
        meds = [_rows.row_median_ld(S, n, ker.shape[0] * nt, nf * nt, off * nt) for off, ker, _ in per_kernel]
        _rows.spectro_correlate_multi(S, [k for _, k, _ in per_kernel], [off for off, _, _ in per_kernel], meds,
                                      outs=[o[r0:r0 + n] for o in outs])
        del S
    return outs


def compute_cross_correlograms_spectrocorr(data, fs, flims, kernels, win_size, overlap_pct):
    """compute_cross_correlogram_spectrocorr for several kernels (the HF and LF notes of scripts/main_spectrodetect.py:103-107)
    from ONE STFT per channel: the STFT covers the union of the kernels' (widened) bands, each kernel is correlated with its
    slice of it and normalised by the median of that slice, as its own call would do.  Returns a list with one correlogram
    per kernel dict.  ndarray in -> float64 ndarrays out; CUDA tensor in -> float32 CUDA tensors out."""
    xd = _to_device(data)
    nperseg, nhop, _, union, per_kernel = spectrocorr_layout(fs, flims, kernels, win_size, overlap_pct, xd.shape[1])
    outs = _spectrocorr_device(xd, nperseg, nhop, union, per_kernel)
    return outs if _is_tensor(data) else [_to_host64(o) for o in outs]


def compute_cross_correlogram_spectrocorr(data, fs, flims, kernel, win_size, overlap_pct):
    """Spectrogram-correlation detector over all channels (reference: detect.py:650-708): batched
    STFT of the band of interest, kernel correlation + frequency sum, median normalisation, all
    on the GPU in channel chunks (the one-kernel case of compute_cross_correlograms_spectrocorr)."""
    nperseg = int(win_size * fs)
    nhop = int(np.floor(nperseg * (1 - overlap_pct)))
    noverlap = nperseg - nhop
    print(f'nperseg: {nperseg}, noverlap: {noverlap}, hop_length: {nhop}')
    return compute_cross_correlograms_spectrocorr(data, fs, flims, [kernel], win_size, overlap_pct)[0]
