"""oracle/torch_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Second oracle for BASELINE-size parity: the reference's f-k masks and `fk_filter_filt` restated with float64 torch
tensor operations, so that the whole-matrix float64 answer can be computed on the test GPU (cuFFT through
torch.fft, test-only, SURVEY.md 7) where a 10 000 x 120 000 complex128 transform does not fit host memory.
Device-agnostic: tests/test_oracle_golden.py pins these functions against oracle/dsp_oracle.py (itself pinned against
the unmodified reference) on the CPU at small shapes; tests/test_fullsize_gpu.py runs the streaming comparison
`fk_filter_errors` at config-2 size.
File:line citations are to /root/reference/src/das4whales/dsp.py.
"""
import collections
import math

import numpy as np
import scipy.signal as sps
import torch


def _axes(trace_shape, selected_channels, dx, fs, device):
    nx, ns = trace_shape
    freq = torch.from_numpy(np.fft.fftshift(np.fft.fftfreq(ns, d=1 / fs))).to(device)                      # :129
    knum = torch.from_numpy(np.fft.fftshift(np.fft.fftfreq(nx, d=selected_channels[2] * dx))).to(device)   # :130
    return freq, knum


def fk_filter_design(trace_shape, selected_channels, dx, fs, cs_min=1400, cp_min=1450, cp_max=3400, cs_max=3500, device="cpu",
                     rows_per_chunk=512):
    """dsp.py:85-171, float64 [nx, ns] in the shifted layout (C order)."""
    nx, ns = trace_shape
    freq, knum = _axes(trace_shape, selected_channels, dx, fs, device)
    out = torch.empty((nx, ns), dtype=torch.float64, device=device)
    hp = 0.5 * math.pi
    for r0 in range(0, nx, rows_per_chunk):
        k = knum[r0:r0 + rows_per_chunk, None]
        v = (freq[None, :] / k).abs()                                                      # :146
        m = torch.ones_like(v)
        m = torch.where((v >= cs_min) & (v <= cp_min), torch.sin(hp * (v - cs_min) / (cp_min - cs_min)), m)       # :149-151
        m = torch.where((v >= cp_max) & (v <= cs_max), 1.0 - torch.sin(hp * (v - cp_max) / (cs_max - cp_max)), m)   # :153-155
        m = torch.where(v >= cs_max, torch.zeros_like(m), m)                              # :157
        m = torch.where(v < cs_min, torch.zeros_like(m), m)                               # :158
        m = torch.where(k.abs() < 0.005, torch.zeros_like(m), m)                          # :142 (also removes the NaNs of k = 0)
        out[r0:r0 + rows_per_chunk] = m
    return out


def hybrid_ninf_filter_design(trace_shape, selected_channels, dx, fs, cs_min=1400., cp_min=1450., cp_max=3400, cs_max=3500,
                              fmin=15., fmax=25., device="cpu", cols_per_chunk=2048):
    """dsp.py:308-454, dense float64 [nx, ns] (the reference wraps the same array in sparse.COO at :454)."""
    nx, ns = trace_shape
    freq, knum = _axes(trace_shape, selected_channels, dx, fs, device)
    b, a = sps.butter(8, [fmin / (fs / 2), fmax / (fs / 2)], "bp")
    H = np.concatenate((np.zeros(ns // 2), np.abs(sps.freqz(b, a, worN=ns // 2)[1]) ** 2))     # :348-349
    M = torch.from_numpy(H).to(device)[None, :].repeat(nx, 1)                                    # :372
    fnp = freq.cpu().numpy()
    i0 = int(np.argmax(fnp >= fmin - 14))                                                        # :354-360
    i1 = int(np.argmax(fnp >= fmax + 14))
    hp = 0.5 * math.pi
    k = knum[:, None]
    for c0 in range(i0, i1, cols_per_chunk):
        c1 = min(i1, c0 + cols_per_chunk)
        f = freq[None, c0:c1]
        ks_lo, kp_lo = f / cs_max, f / cp_max                                                    # :381-382
        ks_hi, kp_hi = f / cs_min, f / cp_min                                                    # :384-385
        col = torch.zeros((nx, c1 - c0), dtype=torch.float64, device=device)
        s = (ks_lo != kp_lo) & (k >= ks_lo) & (k <= kp_lo)
        col = torch.where(s, torch.sin(hp * (k - ks_lo) / (kp_lo - ks_lo)), col)                 # :388-391
        s = (ks_hi != kp_hi) & (k >= kp_hi) & (k <= ks_hi)
        col = torch.where(s, -torch.sin(hp * (k - ks_hi) / (ks_hi - kp_hi)), col)                # :392-395
        col = torch.where((k > kp_lo) & (k < kp_hi), torch.ones_like(col), col)                  # :399
        M[:, c0:c1] *= col                                                                       # :402
    M = M + M.flip(1)                                                                            # :405
    M = M + M.flip(0)                                                                            # :406
    return M


def fk_filter_filt(x64, mask_shifted):
    """dsp.py:725-756: real(ifft2(ifftshift(fftshift(fft2(x)) * M))) == real(ifft2(fft2(x) * ifftshift(M))), float64."""
    assert x64.dtype == torch.float64 and mask_shifted.dtype == torch.float64
    mu = torch.fft.ifftshift(mask_shifted)
    spec = torch.fft.fft2(x64)
    spec.mul_(mu)
    del mu
    return torch.fft.ifft2(spec).real


# ----------------------------------------------------------------------------- streaming whole-matrix comparison
# At 10 000 x 120 000 the dense float64 mask (9.6 GB) and fft2's temporaries do not fit beside the filter under test on an
# 80 GB card.  The functions below produce the same float64 answer one slab at a time: a mask is a function
# `cols(j) -> float64 [nx, len(j)]` returning the shifted-layout columns j, and `fk_filter_errors` compares y with
# real(ifft2(fft2(x) * ifftshift(M))) without ever holding the dense mask or the output matrix.

def fan_columns(trace_shape, selected_channels, dx, fs, cs_min=1400, cp_min=1450, cp_max=3400, cs_max=3500, device="cpu"):
    """Columns of fk_filter_design (dsp.py:85-171), elementwise in (k, f): same statements, any column subset."""
    freq, knum = _axes(trace_shape, selected_channels, dx, fs, device)
    hp = 0.5 * math.pi
    k = knum[:, None]

    def cols(j):
        v = (freq[None, j] / k).abs()                                                      # :146
        m = torch.ones_like(v)
        m = torch.where((v >= cs_min) & (v <= cp_min), torch.sin(hp * (v - cs_min) / (cp_min - cs_min)), m)       # :149-151
        m = torch.where((v >= cp_max) & (v <= cs_max), 1.0 - torch.sin(hp * (v - cp_max) / (cs_max - cp_max)), m)   # :153-155
        m = torch.where(v >= cs_max, torch.zeros_like(m), m)                              # :157
        m = torch.where(v < cs_min, torch.zeros_like(m), m)                               # :158
        return torch.where(k.abs() < 0.005, torch.zeros_like(m), m)                      # :142
    return cols


def hybrid_ninf_columns(trace_shape, selected_channels, dx, fs, cs_min=1400., cp_min=1450., cp_max=3400, cs_max=3500,
                        fmin=15., fmax=25., device="cpu"):
    """Columns of hybrid_ninf_filter_design (dsp.py:308-454).  Before the flips (:405-406) the mask A is H(f) times a
    k-band in the speed-filtered columns; column j of the result is A[:, j] + A[:, ns-1-j] (fliplr first), then that
    column plus itself flipped along k (flipud) -- the reference's order of additions."""
    nx, ns = trace_shape
    freq, knum = _axes(trace_shape, selected_channels, dx, fs, device)
    b, a = sps.butter(8, [fmin / (fs / 2), fmax / (fs / 2)], "bp")
    H = torch.from_numpy(np.concatenate((np.zeros(ns // 2), np.abs(sps.freqz(b, a, worN=ns // 2)[1]) ** 2))).to(device)
    fnp = freq.cpu().numpy()
    i0 = int(np.argmax(fnp >= fmin - 14))                                                        # :354-360
    i1 = int(np.argmax(fnp >= fmax + 14))
    hp = 0.5 * math.pi
    k = knum[:, None]

    def a_cols(j):
        out = H[None, j].repeat(nx, 1)                                                           # :372
        band = (j >= i0) & (j < i1)
        if bool(band.any()):
            jb = j[band]
            f = freq[None, jb]
            ks_lo, kp_lo = f / cs_max, f / cp_max                                                # :381-382
            ks_hi, kp_hi = f / cs_min, f / cp_min                                                # :384-385
            col = torch.zeros((nx, jb.numel()), dtype=torch.float64, device=device)
            s = (ks_lo != kp_lo) & (k >= ks_lo) & (k <= kp_lo)
            col = torch.where(s, torch.sin(hp * (k - ks_lo) / (kp_lo - ks_lo)), col)             # :388-391
            s = (ks_hi != kp_hi) & (k >= kp_hi) & (k <= ks_hi)
            col = torch.where(s, -torch.sin(hp * (k - ks_hi) / (ks_hi - kp_hi)), col)            # :392-395
            col = torch.where((k > kp_lo) & (k < kp_hi), torch.ones_like(col), col)              # :399
            out[:, band] *= col                                                                  # :402
        return out

    def cols(j):
        m = a_cols(j) + a_cols(ns - 1 - j)                                                       # :405
        return m + m.flip(0)                                                                     # :406
    return cols


def dense_columns(mask):
    """Columns of a caller-supplied [nx, ns] mask (any float dtype, any device), as float64."""
    return lambda j: mask[:, j.to(mask.device)].to(torch.float64)


# max_norm = max|y - ref| / max|ref|, l2 = ||y - ref||_2 / ||ref||_2; ref_max and ref_l2 are max|ref| and ||ref||_2
FkErrors = collections.namedtuple("FkErrors", "max_norm l2 ref_max ref_l2")


def fk_filter_errors(x, y, mask_cols, tapering=False, rows_per_slab=256, cols_per_slab=1024):
    """Errors of y against the float64 f-k filter of x (dsp.py:725-756) with the mask given by `mask_cols`.

    The literal fft2 -> x ifftshift(M) -> ifft2 -> real, with the full complex spectrum (no Hermitian fold, which is the
    identity the CUDA filter is built on), computed in slabs: time FFT of row slabs, then per column slab the channel
    FFT, the mask columns, the inverse channel FFT; finally the inverse time FFT of row slabs, compared with the same
    rows of y.  Device memory: the complex128 spectrum (16 nx ns bytes) plus slab temporaries.  x and y are [nx, ns]
    real tensors on one device, any float dtype; x is not modified."""
    nx, ns = x.shape
    assert tuple(y.shape) == (nx, ns)
    dev = x.device
    spec = torch.empty((nx, ns), dtype=torch.complex128, device=dev)
    win = torch.from_numpy(sps.windows.tukey(ns, alpha=0.03)).to(dev)[None, :] if tapering else None   # dsp.py:721
    for r0 in range(0, nx, rows_per_slab):
        xs = x[r0:r0 + rows_per_slab].to(torch.float64)
        if win is not None:
            xs = xs * win
        spec[r0:r0 + rows_per_slab] = torch.fft.fft(xs, dim=1)
    del xs
    rows_shift = (torch.arange(nx, device=dev) + nx // 2) % nx          # ifftshift along k
    for c0 in range(0, ns, cols_per_slab):
        c = torch.arange(c0, min(ns, c0 + cols_per_slab), device=dev)
        s = torch.fft.fft(spec[:, c0:c0 + cols_per_slab], dim=0)
        s *= mask_cols((c + ns // 2) % ns)[rows_shift]                  # ifftshift along f, then along k
        spec[:, c0:c0 + cols_per_slab] = torch.fft.ifft(s, dim=0)
        del s
    emax = rmax = 0.0
    e2 = torch.zeros((), dtype=torch.float64, device=dev)
    r2 = torch.zeros((), dtype=torch.float64, device=dev)
    for r0 in range(0, nx, rows_per_slab):
        ref = torch.fft.ifft(spec[r0:r0 + rows_per_slab], dim=1).real
        d = y[r0:r0 + rows_per_slab].to(torch.float64) - ref
        emax = max(emax, float(d.abs().max()))
        rmax = max(rmax, float(ref.abs().max()))
        e2 += (d * d).sum()
        r2 += (ref * ref).sum()
        del ref, d
    del spec
    e_l2, r_l2 = math.sqrt(float(e2)), math.sqrt(float(r2))
    return FkErrors(emax / max(rmax, 1e-300), e_l2 / max(r_l2, 1e-300), rmax, r_l2)
