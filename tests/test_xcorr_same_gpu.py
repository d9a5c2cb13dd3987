"""GPU tests of the "same"-mode matched filter (d4w_xcorr_same, rows.cross_correlogram_same,
detect.compute_cross_correlogram(s)_same) and of pipeline.GaborDetectPipeline.

The reference is the loop of scripts/main_gabordetect.py:243-246 restated here in float64 -- there is no library function to
pin it against: every channel with max > 0 is `scipy.signal.correlate(row / max(row), note, mode='same')`, and the channels
the script skips (max <= 0, left as np.empty_like values there) are zeros.  The file-level oracle chain is
scripts/main_gabordetect.py:58-266 on the float64 oracles of raw2strain, bp_filt, the hybrid_ninf f-k filter and the Gabor
mask (oracle/improcess_oracle.py), then this loop, threshold thres_frac * max (HF at 0.9 of it) and pick_times_env."""
import numpy as np
import pytest
import scipy.signal as sp

from conftest import rel_err

pytestmark = pytest.mark.gpu
DX, FS = 2.0419046878814697, 200.0


@pytest.fixture(scope="module")
def dw():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import das4whales_b200 as dw
    from das4whales_b200 import _lib
    _lib.lib()
    return dw


def _hann_chirp(fmin, fmax, dur):
    t = np.arange(0, dur, 1 / FS)
    c = sp.chirp(t, f0=fmax, f1=fmin, t1=dur, method="hyperbolic")
    return np.hanning(len(c)) * c


HF = _hann_chirp(17.8, 28.8, 0.68)          # 136 taps (scripts/main_gabordetect.py:223-224)
LF = _hann_chirp(14.7, 21.8, 0.78)          # 156 taps (:226-227)


def script_loop(masked_tr, note):
    """scripts/main_gabordetect.py:243-246 in float64, np.zeros_like for the skipped channels."""
    x = np.asarray(masked_tr, dtype=np.float64)
    out = np.zeros_like(x)
    for i in range(x.shape[0]):
        if np.max(x[i, :]) > 0:
            out[i, :] = sp.correlate(x[i, :] / np.max(x[i, :]), note, mode="same", method="fft")
    return out


def same_ref(x, note):
    """script_loop for many rows at once (one 2-D FFT correlation with a one-row kernel)."""
    x = np.asarray(x, dtype=np.float64)
    m = np.max(x, axis=1)
    keep = m > 0
    out = np.zeros_like(x)
    if keep.any():
        out[keep] = sp.correlate(x[keep] / m[keep, None], np.asarray(note, dtype=np.float64)[None, :], mode="same", method="fft")
    return out


def _rows(nx, ns, seed):
    """fp32 rows of mixed character: noise, positive-offset noise, a single spike, plus rows the script skips
    (all zero, all negative) at fixed places."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((nx, ns))
    x[1::5] += 0.7
    x[2, :] = 0.0
    x[2, ns // 3] = 1.5
    x[3, :] = 0.0
    x[4, :] = -np.abs(x[4, :]) - 1e-3
    return x.astype(np.float32)


def _check(got, ref):
    e_max, e_l2 = rel_err(got, ref)
    assert e_max <= 1e-4 and e_l2 <= 1e-5, (e_max, e_l2)


def _tpl(L, seed):
    rng = np.random.default_rng(seed)
    return np.hanning(L) * rng.standard_normal(L)


@pytest.mark.parametrize("ns", [1200, 12000, 12001])
def test_script_notes_match_scipy(dw, ns):
    x = _rows(48, ns, ns)
    outs = dw.detect.compute_cross_correlograms_same(x, [HF, LF])
    assert len(outs) == 2 and all(o.dtype == np.float64 and o.shape == x.shape for o in outs)
    for o, note in zip(outs, (HF, LF)):
        _check(o, same_ref(x, note))
        assert np.array_equal(o[3], np.zeros(ns)) and np.array_equal(o[4], np.zeros(ns))


@pytest.mark.parametrize("L", [137, 400, 401, 2500])
@pytest.mark.parametrize("ns", [1200, 12000, 12001])
def test_long_and_odd_templates_match_scipy(dw, L, ns):
    """400 / 401 taps run on 1 250- or 2 500-sample Cooley-Tukey blocks, 2 500 taps on 5 000-sample blocks."""
    x = _rows(24, ns, L + ns)
    c = _tpl(L, L)
    _check(dw.detect.compute_cross_correlogram_same(x, c), same_ref(x, c))


def test_rows_of_120000_samples(dw):
    x = _rows(6, 120000, 7)
    for o, note in zip(dw.detect.compute_cross_correlograms_same(x, [HF, LF]), (HF, LF)):
        _check(o, same_ref(x, note))
    c = _tpl(2500, 3)
    _check(dw.detect.compute_cross_correlogram_same(x, c), same_ref(x, c))


def test_rows_shorter_than_the_template(dw):
    x = _rows(8, 100, 11)
    for o, note in zip(dw.detect.compute_cross_correlograms_same(x, [HF, LF]), (HF, LF)):
        _check(o, same_ref(x, note))


@pytest.mark.parametrize("pair", [(HF, LF), (_tpl(137, 1), _tpl(400, 2))])
def test_one_pass_equals_single_template_calls(dw, pair):
    """Several templates share one forward transform; each gets zeros prepended up to the common lag offset, so the
    results differ from single-template calls only by rounding."""
    x = _rows(32, 12000, 5)
    both = dw.detect.compute_cross_correlograms_same(x, list(pair))
    for o, c in zip(both, pair):
        single = dw.detect.compute_cross_correlogram_same(x, c)
        assert np.max(np.abs(o - single)) <= 1e-6 * np.max(np.abs(single))


def test_skipped_rows_are_exact_zeros_and_tensor_io(dw):
    import torch
    x = _rows(40, 12000, 9)
    x[10:20] = 0.0
    x[20:30] = -np.abs(x[20:30]) - 1e-6
    xt = torch.from_numpy(x).cuda()
    outs_t = dw.detect.compute_cross_correlograms_same(xt, [HF, LF])
    one_t = dw.detect.compute_cross_correlogram_same(xt, LF)
    assert all(isinstance(o, torch.Tensor) and o.is_cuda and o.dtype == torch.float32 and tuple(o.shape) == x.shape for o in outs_t)
    assert isinstance(one_t, torch.Tensor) and one_t.dtype == torch.float32 and tuple(one_t.shape) == x.shape
    outs_h = dw.detect.compute_cross_correlograms_same(x, [HF, LF])
    for ot, oh, note in zip(outs_t, outs_h, (HF, LF)):
        o = ot.cpu().numpy()
        assert np.array_equal(o.astype(np.float64), oh)                      # same kernels, ndarray or tensor
        assert not np.any(o[10:30]) and np.any(o[:10]) and np.any(o[30:])
        _check(o, same_ref(x, note))


def test_more_than_65535_rows(dw):
    nx, ns = 70001, 200
    rng = np.random.default_rng(4)
    x = rng.standard_normal((nx, ns)).astype(np.float32)
    x[65530:65540] = 0.0                                                     # skipped rows on both sides of the chunk edge
    outs = dw.detect.compute_cross_correlograms_same(x, [HF, LF])
    for o, note in zip(outs, (HF, LF)):
        _check(o, same_ref(x, note))
        assert not np.any(o[65530:65540])


# ---------------------------------------------------------------------------------------------------- file pipeline
GABOR_THR, GABOR_THR2 = 42000., 100.       # the mask keeps 29 of the 40 binned channel rows of the synthetic record
FRAC = 0.2


def _oracle_chain(raw, scale, sel):
    from oracle import dsp_oracle as O, detect_oracle as D, data_oracle as DH, improcess_oracle as IO
    nx, ns = raw.shape
    x = DH.raw2strain(raw, {"scale_factor": scale})
    x = O.bp_filt(x, FS, 14., 30.)
    m = O.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, 1350., 1450., 3300, 3450, 14., 30.)
    y = O.fk_filter_filt(x, m)
    masked, _ = IO.gabor_detect(y, FS, DX, sel, c0=1500., bin_factor=10, threshold=GABOR_THR, threshold2=GABOR_THR2)
    chf, clf = script_loop(masked, HF), script_loop(masked, LF)
    maxv = max(chf.max(), clf.max())
    thr = FRAC * maxv
    return maxv, D.convert_pick_times(D.pick_times_env(chf, thr * 0.9)), D.convert_pick_times(D.pick_times_env(clf, thr)), masked


def test_gabor_pipeline_matches_oracle_chain(dw):
    from das4whales_b200 import pipeline
    from oracle.make_golden import synth
    nx, ns, sel = 400, 6000, [0, 400, 1]
    x = synth(nx, ns, seed=9, ncalls=3)
    counts = np.round(x * 5.0e4).astype(np.int32) + 1234
    scale = 4.0838e-11 * 1550.0 / 2.0419
    pipe = pipeline.GaborDetectPipeline(nx, ns, sel, DX, FS, scale, thres_frac=FRAC, threshold=GABOR_THR, threshold2=GABOR_THR2)
    import torch
    dev = pipe.process_device(torch.from_numpy(counts).cuda(), with_intermediates=True)
    masked = dev["masked"].cpu().numpy()
    kept = np.any(masked != 0, axis=1)
    assert kept.any() and not kept.all(), int(kept.sum())                   # both the skip and the correlation path run
    # the correlograms against the float64 loop on the device's own masked trace (a mask pixel flipping at a threshold
    # cannot hide a correlation error)
    for c, note in zip(dev["corr"], (HF, LF)):
        c = c.cpu().numpy()
        _check(c, script_loop(masked, note))
        assert not np.any(c[~kept])
    res = pipe.process_file(counts)
    maxv, phf, plf, _ = _oracle_chain(counts, scale, sel)
    assert abs(res["maxv"] - maxv) <= 1e-4 * maxv
    for got, ref in ((res["picks_hf"], phf), (res["picks_lf"], plf)):
        a = set(zip(got[0].tolist(), got[1].tolist()))
        b = set(zip(ref[0].tolist(), ref[1].tolist()))
        assert len(a ^ b) <= max(2, len(b) // 100), (len(a), len(b), len(a ^ b))
        assert len(b) > 0
    outs = list(pipe.stream([counts, counts.astype(np.float32), counts]))
    assert len(outs) == 3
    for o in outs:
        assert np.array_equal(o["picks_hf"], res["picks_hf"]) and np.array_equal(o["picks_lf"], res["picks_lf"])
    one = pipeline.process_file_gabor(counts, {"dx": DX, "fs": FS, "scale_factor": scale}, sel, thres_frac=FRAC,
                                      threshold=GABOR_THR, threshold2=GABOR_THR2)
    assert np.array_equal(one["picks_hf"], res["picks_hf"]) and np.array_equal(one["picks_lf"], res["picks_lf"])
