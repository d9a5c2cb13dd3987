"""CPU: the host layout of the multi-kernel spectrogram correlation (detect.spectrocorr_layout: STFT framing, each kernel's
widened band and buildkernel matrix, the union of their bins and each kernel's offset in it) against the oracle's
parameter derivation, and a float64 NumPy restatement of the pass the GPU runs with that layout -- one STFT of the union
band, the median of each kernel's slice of it, every kernel zero-padded on the left to the common centre max kw // 2 --
which must reproduce detect_oracle.compute_cross_correlogram_spectrocorr (one STFT per kernel) for every kernel."""
import numpy as np
import pytest

from das4whales_b200.detect import spectrocorr_layout
from oracle import detect_oracle as D, dsp_oracle as O

FS = 200.0
HF = {'f0': 27., 'f1': 17., 'dur': 0.8, 'bdwidth': 4.}          # scripts/main_spectrodetect.py:103-104
LF = {'f0': 20., 'f1': 14., 'dur': 1.2, 'bdwidth': 4.}
FMAX_ONLY = {'f0': 28., 'f1': 25., 'dur': 0.8, 'bdwidth': 4.}   # fmax - f1 < 2 bdwidth: fmax -> f1 + 3 bdwidth
NEITHER = {'f0': 20.5, 'f1': 19.5, 'dur': 1.0, 'bdwidth': .5}   # 2 bdwidth inside 18-22 Hz at both ends: no widening
# (flims, kernels, win_size, overlap_pct)
CASES = {
    "script_pair": ((14., 30.), [HF, LF], 0.8, 0.95),
    "three_kernels": ((14., 30.), [HF, LF, FMAX_ONLY], 0.8, 0.95),
    # widening only moves fmax up and fmin down, so bands are disjoint only when fmin > fmax: 8-26 Hz and 40-82 Hz
    "disjoint_bands": ((40., 20.), [LF, {'f0': 80., 'f1': 70., 'dur': 0.9, 'bdwidth': 4.}], 0.8, 0.95),
    # fmax only, fmin only (LF), both and neither; 90 % overlap
    "each_widening_rule": ((18., 22.), [FMAX_ONLY, LF, {'f0': 20., 'f1': 19., 'dur': 0.8, 'bdwidth': 2.}, NEITHER], 0.8, 0.90),
}


def _oracle_kernel(kernel, flims, win, ov, ns):
    nperseg, nhop, fmin, fmax = D.spectrocorr_params(FS, flims, kernel, win, ov)
    _, ff, tt = D.get_sliced_nspectrogram(np.ones(ns), FS, fmin, fmax, nperseg, nhop)
    _, _, ker = D.buildkernel(kernel["f0"], kernel["f1"], kernel["bdwidth"], kernel["dur"], ff, tt, FS, fmin, fmax)
    return nperseg, nhop, (fmin, fmax), ff, ker


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("ns", [9000, 12001])
def test_layout_matches_oracle_parameters(case, ns):
    flims, kernels, win, ov = CASES[case]
    nperseg, nhop, bands, (u0, u1), per = spectrocorr_layout(FS, flims, kernels, win, ov, ns)
    ff_all = np.linspace(0, FS / 2, nperseg // 2 + 1)
    lo, hi = [], []
    for kernel, band, (off, ker, kw) in zip(kernels, bands, per):
        np_, nh_, band_ref, ff, ker_ref = _oracle_kernel(kernel, flims, win, ov, ns)
        assert (nperseg, nhop) == (np_, nh_) and band == band_ref
        assert ker.shape == ker_ref.shape and kw == ker.shape[1] >= 1
        assert np.max(np.abs(ker - ker_ref)) <= 1e-14 * np.max(np.abs(ker_ref))
        assert np.array_equal(ff_all[u0 + off:u0 + off + ker.shape[0]], ff)          # the kernel's bins inside the union
        lo.append(u0 + off); hi.append(u0 + off + ker.shape[0] - 1)
    assert (u0, u1) == (min(lo), max(hi))
    if case == "disjoint_bands":
        assert hi[0] < lo[1]
    if case == "each_widening_rule":
        assert [b != flims for b in bands] == [True, True, True, False]
        assert bands[0][0] == flims[0] and bands[1][1] == flims[1]


def multi_pass(x, flims, kernels, win, ov):
    """The GPU pass in float64 on spectrocorr_layout's layout: union-band STFT, slice medians, common centre."""
    nx, ns = x.shape
    nperseg, nhop, _, (u0, u1), per = spectrocorr_layout(FS, flims, kernels, win, ov, ns)
    c0 = max(kw // 2 for _, _, kw in per)
    outs = [np.empty((nx, 1 + ns // nhop)) for _ in per]
    for i in range(nx):
        S = np.abs(O.stft_librosa(x[i], nperseg, nhop))[u0:u1 + 1]
        nt = S.shape[1]
        for out, (off, ker, kw) in zip(outs, per):
            sl = S[off:off + ker.shape[0]]
            kp = np.concatenate((np.zeros((ker.shape[0], c0 - kw // 2)), ker), axis=1)       # left zeros up to the centre
            sp = np.concatenate((np.zeros((ker.shape[0], c0)), sl, np.zeros((ker.shape[0], kp.shape[1]))), axis=1)
            acc = np.zeros(nt)
            for j in range(kp.shape[1]):                       # window t - c0 + j, the same for every kernel
                acc += kp[:, j] @ sp[:, j:j + nt]
            out[i] = np.maximum(acc, 0.0) / (np.median(sl) * kw)
    return outs


@pytest.mark.parametrize("case", sorted(CASES))
def test_multi_pass_restatement_matches_oracle(case):
    flims, kernels, win, ov = CASES[case]
    rng = np.random.default_rng(len(case))
    x = rng.standard_normal((3, 4001))
    x[1] += 3 * np.sin(2 * np.pi * 21.0 * np.arange(4001) / FS)
    outs = multi_pass(x, flims, kernels, win, ov)
    for out, kernel in zip(outs, kernels):
        ref = D.compute_cross_correlogram_spectrocorr(x, FS, flims, kernel, win, ov)
        assert out.shape == ref.shape
        assert np.max(np.abs(out - ref)) <= 1e-12 * np.max(np.abs(ref)), kernel


def test_record_too_short_for_a_kernel():
    # LF takes its width from the frames with 8.4 s < t < 9.6 s: an 8 s record has none
    with pytest.raises(ValueError, match="no frames"):
        spectrocorr_layout(FS, (14., 30.), [HF, LF], 0.8, 0.95, 1600)
    nperseg, nhop, _, _, per = spectrocorr_layout(FS, (14., 30.), [HF], 0.8, 0.95, 1600)
    assert per[0][2] >= 1
    with pytest.raises(ValueError):
        spectrocorr_layout(FS, (14., 30.), [], 0.8, 0.95, 12000)
