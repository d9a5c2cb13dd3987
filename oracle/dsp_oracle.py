"""oracle/dsp_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Float64 NumPy/SciPy restatement of the DAS4Whales `dsp` hot-path functions, written
from the reference's behaviour (file:line cited per function, all relative to
/root/reference/src/das4whales/dsp.py).  Only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs may import it; it is the checker,
never the thing shipped.  das4whales_b200/ never imports anything from oracle/.

Pinning: oracle/make_golden.py runs the *unmodified* reference (oracle/ref_loader.py)
and this restatement on the same seeded inputs, asserts agreement (<= 1e-12 relative)
and writes tests/golden/*.npz; tests/test_oracle_vs_golden.py re-checks the
restatement against those committed vectors on every run, and -- when /root/reference
is present -- against the live reference as well.  The two known-answer tests of the
reference (tests/test_dsp.py:85-88 taper_data, :136-141 snr_tr_array) are included.

The reference functions that call librosa.stft (get_spectrogram) cannot be executed
here (librosa is not installed): `stft_librosa` restates librosa 0.10.1's documented
defaults (SURVEY.md App. A.6) and is pinned only against scipy.signal.stft
(independent implementation) -- flagged "restated, cross-checked against SciPy".
"""
import numpy as np
import scipy.signal as sps


# ----------------------------------------------------------------------------- masks
def _axes(trace_shape, selected_channels, dx, fs):
    """fftshift-ed frequency / wavenumber axes (dsp.py:129-130)."""
    nx, ns = trace_shape
    freq = np.fft.fftshift(np.fft.fftfreq(ns, d=1.0 / fs))
    knum = np.fft.fftshift(np.fft.fftfreq(nx, d=selected_channels[2] * dx))
    return freq, knum


def fk_filter_design(trace_shape, selected_channels, dx, fs,
                     cs_min=1400, cp_min=1450, cp_max=3400, cs_max=3500):
    """Speed-fan mask in the shifted (k, f) layout -- dsp.py:85-171.

    Row is zero where |k| < 0.005 (dsp.py:142); else with v = |f / k| (dsp.py:146):
    sine ramp up on [cs_min, cp_min] (:149-151), 1 inside, 1 - sine ramp on
    [cp_max, cs_max] (:153-155), 0 for v >= cs_max or v < cs_min (:157-158).
    Returned Fortran-ordered float64 like the reference (:137).
    """
    freq, knum = _axes(trace_shape, selected_channels, dx, fs)
    k = knum[:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        v = np.abs(freq[None, :] / k)
        m = np.ones(v.shape)
        up = (v >= cs_min) & (v <= cp_min)
        m[up] = np.sin(0.5 * np.pi * (v[up] - cs_min) / (cp_min - cs_min))
        dn = (v >= cp_max) & (v <= cs_max)
        m[dn] = 1.0 - np.sin(0.5 * np.pi * (v[dn] - cp_max) / (cs_max - cp_max))
        m[v >= cs_max] = 0.0
        m[v < cs_min] = 0.0
    m[np.abs(knum) < 0.005, :] = 0.0
    return np.asfortranarray(m)


def hybrid_ninf_filter_design(trace_shape, selected_channels, dx, fs, cs_min=1400., cp_min=1450.,
                              cp_max=3400, cs_max=3500, fmin=15., fmax=25.):
    """Butterworth-in-f x speed band mask -- dsp.py:308-454 (dense; the reference wraps
    the same array in sparse.COO at :454).

    H(f) = |freqz(butter(8,[fmin,fmax]/(fs/2)), worN=ns//2)|^2 on the upper half of the
    shifted axis, zeros on the lower half (:348-349); tiled over k (:372); columns with
    fmin-14 <= f < fmax+14 (:354-360, :376) are multiplied by a k-band with sine ramps
    (:381-402); then `+= fliplr`, `+= flipud` (:405-406).
    """
    nx, ns = trace_shape
    freq, knum = _axes(trace_shape, selected_channels, dx, fs)
    b, a = sps.butter(8, [fmin / (fs / 2), fmax / (fs / 2)], "bp")
    H = np.concatenate((np.zeros(ns // 2), np.abs(sps.freqz(b, a, worN=ns // 2)[1]) ** 2))
    M = np.tile(H, (nx, 1))
    i0 = int(np.argmax(freq >= fmin - 14))
    i1 = int(np.argmax(freq >= fmax + 14))
    for i in range(i0, i1):
        f = freq[i]
        ks_lo, kp_lo = f / cs_max, f / cp_max
        ks_hi, kp_hi = f / cs_min, f / cp_min
        col = np.zeros(nx)
        if ks_lo != kp_lo:
            s = (knum >= ks_lo) & (knum <= kp_lo)
            col[s] = np.sin(0.5 * np.pi * (knum[s] - ks_lo) / (kp_lo - ks_lo))
        if ks_hi != kp_hi:
            s = (knum >= kp_hi) & (knum <= ks_hi)
            col[s] = -np.sin(0.5 * np.pi * (knum[s] - ks_hi) / (ks_hi - kp_hi))
        col[(knum > kp_lo) & (knum < kp_hi)] = 1.0
        M[:, i] *= col
    M = M + M[:, ::-1]
    M = M + M[::-1, :]
    return M


def hybrid_filter_design(trace_shape, selected_channels, dx, fs, cs_min=1400., cp_min=1450.,
                         fmin=15., fmax=25.):
    """Infinite-speed hybrid mask with sine tapers -- dsp.py:174-305 (dense)."""
    nx, ns = trace_shape
    freq, knum = _axes(trace_shape, selected_channels, dx, fs)
    fpmin, fpmax = fmin - 4, fmax + 4
    H = np.zeros_like(freq)
    r = (freq >= fpmin) & (freq <= fmin)
    H[r] = np.sin(0.5 * np.pi * (freq[r] - fpmin) / (fmin - fpmin))
    H[(freq >= fmin) & (freq <= fmax)] = 1
    r = (freq >= fmax) & (freq <= fpmax)
    H[r] = np.cos(0.5 * np.pi * (freq[r] - fmax) / (fmax - fpmax))
    M = np.tile(H, (nx, 1))
    i0 = int(np.argmax(freq >= fpmin))
    i1 = int(np.argmax(freq >= fpmax))
    for i in range(i0, i1):
        ks, kp = freq[i] / cs_min, freq[i] / cp_min
        col = np.zeros(nx)
        if ks != kp:
            s = (knum >= -ks) & (knum <= -kp)
            col[s] = -np.sin(0.5 * np.pi * (knum[s] + ks) / (kp - ks))
            s = (-knum >= -ks) & (-knum <= -kp)
            col[s] = np.sin(0.5 * np.pi * (knum[s] - ks) / (kp - ks))
        col[(knum < kp) & (knum > -kp)] = 1
        M[:, i] *= col
    return M + M[:, ::-1]



def _gs_band(trace_shape, selected_channels, dx, fs, fmin, fmax):
    nx, ns = trace_shape
    freq, knum = _axes(trace_shape, selected_channels, dx, fs)
    H = np.zeros_like(freq)
    H[(freq >= fmin) & (freq <= fmax)] = 1
    i0 = int(np.argmax(freq >= fmin - 4))
    i1 = int(np.argmax(freq >= fmax + 4))
    return freq, knum, np.tile(H, (nx, 1)), i0, i1


def hybrid_gs_filter_design(trace_shape, selected_channels, dx, fs, cs_min=1400., cp_min=1450., fmin=15., fmax=25.):
    """Boolean band (|k| < f/cp_min) blurred with a sigma=20 Gaussian -- dsp.py:457-579 (dense)."""
    from scipy import ndimage
    freq, knum, M, i0, i1 = _gs_band(trace_shape, selected_channels, dx, fs, fmin, fmax)
    for i in range(i0, i1):
        kp = freq[i] / cp_min
        M[:, i] *= ((knum < kp) & (knum > -kp)).astype(float)
    M = M + M[:, ::-1]
    return ndimage.gaussian_filter(M, 20)


def hybrid_ninf_gs_filter_design(trace_shape, selected_channels, dx, fs, cs_min=1400., cp_min=1450., cp_max=3400,
                                 cs_max=3500, fmin=15., fmax=25.):
    """Boolean band (-f/cp_min < k < -f/cp_max), Gaussian sigma=20, then fliplr / flipud sums
    -- dsp.py:582-702 (dense)."""
    from scipy import ndimage
    freq, knum, M, i0, i1 = _gs_band(trace_shape, selected_channels, dx, fs, fmin, fmax)
    for i in range(i0, i1):
        M[:, i] *= ((knum > -freq[i] / cp_min) & (knum < -freq[i] / cp_max)).astype(float)
    M = ndimage.gaussian_filter(M, 20)
    M = M + M[:, ::-1]
    return M + M[::-1, :]


def fk_filt_mask(shape, tint, fs, xint, dx, c_min, c_max):
    """The Gaussian-blurred fan the legacy dsp.fk_filt builds and applies -- dsp.py:883-953."""
    from scipy import ndimage
    nx, ns = shape
    f = np.fft.fftshift(np.fft.fftfreq(ns, d=tint / fs))
    k = np.fft.fftshift(np.fft.fftfreq(nx, d=xint * dx))
    ff, kk = np.meshgrid(f, k)
    g = 1.0 * ((ff < kk * c_min) & (ff < -kk * c_min))
    g2 = 1.0 * ((ff < kk * c_max) & (ff < -kk * c_max))
    g = g + g[:, ::-1]
    g = g - (g2 + g2[:, ::-1])
    g = ndimage.gaussian_filter(g, 20)
    return (g - np.min(g)) / (np.max(g) - np.min(g))


def fk_filt(data, tint, fs, xint, dx, c_min, c_max):
    """Legacy one-call f-k filter -- dsp.py:883-953."""
    data = np.asarray(data, dtype=np.float64)
    g = fk_filt_mask(data.shape, tint, fs, xint, dx, c_min, c_max)
    return np.fft.ifft2(np.fft.ifftshift(np.fft.fftshift(np.fft.fft2(data)) * g)).real


def fold_mask(mask_shifted):
    """Hermitian fold of a shifted-layout mask (SURVEY.md App. A.1).

    `real(ifft2(ifftshift(fftshift(fft2(x)) * M)))` (dsp.py:748-756) equals filtering
    with M_sym[k,f] = (Mu[k,f] + Mu[-k,-f]) / 2, Mu = ifftshift(M).  Returns M_sym in
    the *un-shifted* DFT layout.
    """
    mu = np.fft.ifftshift(np.asarray(mask_shifted, dtype=np.float64))
    partner = np.roll(mu[::-1, ::-1], (1, 1), axis=(0, 1))
    return 0.5 * (mu + partner)


# ----------------------------------------------------------------------------- f-k apply
def tukey_window(ns, alpha=0.03):
    """scipy.signal.windows.tukey(ns, alpha) as used at dsp.py:721."""
    return sps.windows.tukey(ns, alpha=alpha)


def taper_data(trace):
    """In-place Tukey(alpha=0.03) taper along time -- dsp.py:705-722."""
    trace *= tukey_window(trace.shape[1])[None, :]
    return trace


def fk_filter_filt(trace, fk_filter_matrix, tapering=False, workers=None):
    """fft2 -> shift -> x mask -> unshift -> ifft2 -> real  -- dsp.py:725-756.
    (fk_filter_sparsefilt, :759-786, is the same arithmetic with a COO mask.)

    workers=None: numpy.fft, single-threaded, exactly the reference's calls.  workers=N: the same statements with
    scipy.fft (the same pocketfft algorithm, N threads) -- bench.py's all-host-cores CPU arm; pinned equal to the
    numpy.fft route by tests/test_oracle_golden.py."""
    trace = np.asarray(trace, dtype=np.float64)
    if tapering:
        trace = taper_data(trace)
    if workers is None:
        spec = np.fft.fftshift(np.fft.fft2(trace))
        spec = spec * np.asarray(fk_filter_matrix)
        return np.fft.ifft2(np.fft.ifftshift(spec)).real
    import scipy.fft as sfft
    spec = sfft.fftshift(sfft.fft2(trace, workers=workers))
    spec *= np.asarray(fk_filter_matrix)
    return sfft.ifft2(sfft.ifftshift(spec), workers=workers, overwrite_x=True).real


def fold_rowmax(mask_shifted):
    """rowmax[k] = max_f float32(|M_sym[k, f]|) for 0 <= k <= nx/2: the support scan of the opt-in eps pruning."""
    msym = fold_mask(mask_shifted)
    return np.abs(msym[: msym.shape[0] // 2 + 1]).astype(np.float32).max(axis=1)


def fk_filter_filt_pruned(x, mask_shifted, eps):
    """The f-k filter with support pruning at threshold eps (FkFilter(mask, eps=eps)): wavenumber row k of the folded
    mask is kept iff rowmax[k] > float32(eps); otherwise rows k and nx - k of M_sym are zeroed.  Returns
    (real(ifft2(fft2(x) * M_sym_pruned)), number of kept rows among 0 <= k <= nx/2).  Pruning removes at most eps of
    every spectral coefficient, so ||y_eps - y||_2 <= eps ||x||_2 (Parseval)."""
    msym = fold_mask(mask_shifted)
    nx = msym.shape[0]
    keep = fold_rowmax(mask_shifted) > np.float32(eps)
    for k in np.nonzero(~keep)[0]:
        msym[k] = 0.0
        msym[(nx - k) % nx] = 0.0
    y = np.fft.ifft2(np.fft.fft2(np.asarray(x, dtype=np.float64)) * msym).real
    return y, int(np.count_nonzero(keep))


def fk_filter_filt_rows(trace, fk_filter_matrix, rows, cols=None, tapering=False):
    """Same result as fk_filter_filt restricted to output `rows` (all columns) -- used at
    sizes where the full float64 fft2 does not fit in host RAM (SURVEY.md 8d).  Uses the
    folded-mask identity and separable 1-D FFTs; memory ~ 2 complex128 half-spectra."""
    x = np.asarray(trace, dtype=np.float64)
    if tapering:
        x = x * tukey_window(x.shape[1])[None, :]
    nx, ns = x.shape
    msym = fold_mask(fk_filter_matrix)[:, : ns // 2 + 1]
    spec = np.fft.rfft(x, axis=1)
    spec = np.fft.fft(spec, axis=0)
    spec *= msym
    # inverse DFT along channels, evaluated only at the requested rows
    k = np.arange(nx)
    w = np.exp(2j * np.pi * np.outer(np.asarray(rows), k) / nx) / nx
    part = w @ spec
    return np.fft.irfft(part, n=ns, axis=1)


# ----------------------------------------------------------------------------- IIR
def butterworth_filter(filterspec, fs):
    """SOS Butterworth design -- dsp.py:789-827."""
    order, fc, kind = filterspec
    return sps.butter(order, np.array(fc) / (fs / 2), btype=kind, output="sos")


def bp_filt(data, fs, fmin, fmax):
    """Order-8 Butterworth band-pass, zero-phase filtfilt along time -- dsp.py:859-880."""
    b, a = sps.butter(8, [fmin / (fs / 2), fmax / (fs / 2)], "bp")
    return sps.filtfilt(b, a, np.asarray(data, dtype=np.float64), axis=1)


def sosfiltfilt(sos, data):
    """Caller-side application used by the notebook / Example.py:55."""
    return sps.sosfiltfilt(sos, np.asarray(data, dtype=np.float64), axis=1)


# ----------------------------------------------------------------------------- spectra
def stft_librosa(y, n_fft, hop_length):
    """librosa.stft(y, n_fft, hop_length) with 0.10.1 defaults (SURVEY.md App. A.6):
    periodic Hann of length n_fft, center=True with zero ('constant') padding of
    n_fft//2 each side, frames 0..len(y)//hop, no normalisation."""
    y = np.asarray(y, dtype=np.float64)
    win = sps.get_window("hann", n_fft, fftbins=True)
    ypad = np.concatenate((np.zeros(n_fft // 2), y, np.zeros(n_fft // 2)))
    nfr = 1 + len(y) // hop_length
    idx = np.arange(n_fft)[None, :] + hop_length * np.arange(nfr)[:, None]
    frames = ypad[idx] * win[None, :]
    return np.fft.rfft(frames, axis=1).T


def stft_sliding_band(y, n_fft, hop, bin_lo, bin_hi, run=160, dtype=np.float32):
    """The algorithm of the CUDA kernel k_stft_slide restated with NumPy in the kernel's precision (test infrastructure: it
    pins the numerics of the recursion on the CPU; the kernel itself is checked against stft_librosa on the GPU).
    |librosa.stft| for bins bin_lo..bin_hi when n_fft = hop * P:  block sums B_b[k] = sum_t x[b*hop + t] W^{tk},
    Y_{m+1} = (Y_m - B_m + B_{m+P}) W^{-hop k}, re-anchored every `run` frames (Horner over the P blocks),
    S[k] = Y[k]/2 - (Y[k-1] + Y[k+1])/4 for the periodic Hann window."""
    assert n_fft % hop == 0
    P = n_fft // hop
    cdt = np.complex64 if dtype == np.float32 else np.complex128
    y = np.asarray(y, dtype=dtype)
    nfr = 1 + len(y) // hop
    ypad = np.concatenate((np.zeros(n_fft // 2, dtype), y, np.zeros(n_fft + (run + P) * hop, dtype)))
    ks = np.arange(bin_lo - 1, bin_hi + 2)
    T = np.exp(-2j * np.pi * np.outer(ks, np.arange(hop)) / n_fft).astype(cdt)        # W^{tk}
    w = np.exp(-2j * np.pi * hop * ks / n_fft).astype(cdt)                             # W^{hop k}
    nblk = len(ypad) // hop
    B = (ypad[:nblk * hop].reshape(nblk, 1, hop).astype(cdt) * T[None]).sum(-1).astype(cdt)
    Y = np.zeros((nfr + run, len(ks)), cdt)
    for m0 in range(0, nfr, run):
        acc = np.zeros(len(ks), cdt)
        for p in range(P - 1, -1, -1):
            acc = (acc * w + B[m0 + p]).astype(cdt)
        for f in range(run):
            Y[m0 + f] = acc
            acc = ((acc - B[m0 + f] + B[m0 + f + P]) * np.conj(w)).astype(cdt)
    Y = Y[:nfr]
    S = dtype(0.5) * Y[:, 1:-1] - dtype(0.25) * (Y[:, :-2] + Y[:, 2:])
    return np.abs(S).T


def get_spectrogram(waveform, fs, nfft=128, overlap_pct=0.8):
    """|STFT| in dB re max, with linspace axes -- dsp.py:41-78."""
    hop = int(np.floor(nfft * (1 - overlap_pct)))
    s = np.abs(stft_librosa(waveform, nfft, hop))
    tt = np.linspace(0, len(waveform) / fs, num=s.shape[1])
    ff = np.linspace(0, fs / 2, num=s.shape[0])
    with np.errstate(divide="ignore"):
        p = 20 * np.log10(s / np.max(s))
    return p, tt, ff


def get_fx(trace, nfft):
    """Per-channel FFT magnitude view -- dsp.py:18-38."""
    fx = 2 * np.abs(np.fft.fftshift(np.fft.fft(np.asarray(trace, dtype=np.float64), nfft), axes=1))
    return fx / nfft * 1e9


def hilbert_envelope(x):
    """|scipy.signal.hilbert(x, axis=1)| (used at dsp.py:975, detect.py:192)."""
    return np.abs(sps.hilbert(np.asarray(x, dtype=np.float64), axis=1))


def snr_tr_array(trace, env=False):
    """10 log10(x^2 / var_row) or with the Hilbert envelope -- dsp.py:956-976."""
    trace = np.asarray(trace, dtype=np.float64)
    var = np.std(trace, axis=1, keepdims=True) ** 2
    num = hilbert_envelope(trace) ** 2 if env else trace ** 2
    with np.errstate(divide="ignore"):
        return 10 * np.log10(num / var)


def get_fx(trace, nfft):
    """dsp.py:18-38 -- per-channel FFT magnitude, fftshift-ed, in nano-strain"""
    fx = 2 * (abs(np.fft.fftshift(np.fft.fft(np.asarray(trace, dtype=np.float64), nfft), axes=1)))
    fx /= nfft
    fx *= 10 ** 9
    return fx


def instant_freq(channel, fs):
    """dsp.py:830-856"""
    import scipy.signal as sps
    return np.diff(np.unwrap(np.angle(sps.hilbert(np.asarray(channel, dtype=np.float64))))) / (2.0 * np.pi) * fs
