"""GPU tests of the multi-kernel spectrogram correlation (d4w_speccorr_multi, d4w_row_median_ld,
detect.compute_cross_correlograms_spectrocorr) and of pipeline.SpectroDetectPipeline.

The kernels are pinned bit for bit to the one-kernel path (rows.spectro_correlate on the same slice with the same median)
and to np.median; the correlograms to the float64 oracle at the detector's 1e-4 tolerance on both STFT routes; the
pipeline to scripts/main_spectrodetect.py:39-123 restated on the float64 oracles: raw2strain, bp_filt, the hybrid_ninf
f-k filter, one spectrogram-correlation correlogram per kernel and pick_times (find_peaks, absolute prominence)."""
import numpy as np
import pytest
import scipy.signal as sps

from conftest import rel_err
from oracle import dsp_oracle as O, detect_oracle as D

pytestmark = pytest.mark.gpu
DX, FS = 2.0419046878814697, 200.0
TOL = 1e-4
HF = {'f0': 27., 'f1': 17., 'dur': 0.8, 'bdwidth': 4.}          # scripts/main_spectrodetect.py:103-104
LF = {'f0': 20., 'f1': 14., 'dur': 1.2, 'bdwidth': 4.}
FLIMS = (14., 30.)


@pytest.fixture(scope="module")
def dw():
    import torch
    assert torch.cuda.is_available()
    import das4whales_b200 as dw
    from das4whales_b200 import _lib
    _lib.lib()
    return dw


def _spectrogram(nx, nf, nt, seed):
    """non-negative fp32 [nx, nf, nt], Rayleigh like |STFT| of noise, a few exact zeros and ties"""
    rng = np.random.default_rng(seed)
    S = np.abs(rng.standard_normal((nx, nf, nt)) + 1j * rng.standard_normal((nx, nf, nt)))
    S[0, :, :7] = 0.0
    S[1, 3] = 0.5
    return S.astype(np.float32)


def _kernel(nf, kw, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((nf, kw)) * np.hanning(kw + 2)[1:-1]


# (offset, rows, width) per kernel in a 30-bin band: odd and even widths, kernels of the script's shapes, overlapping and
# disjoint slices; 900 frames is too wide for the tiled kernel's shared memory and runs on the untiled one from a copy
SETS = {
    "script": [(5, 13, 20), (0, 18, 30)],
    "odd_even": [(0, 30, 7), (2, 9, 8), (20, 10, 33), (11, 1, 1)],
    "with_untiled": [(4, 20, 900), (0, 13, 21), (17, 13, 44)],
    "untiled_whole_band": [(0, 30, 600)],
}


@pytest.mark.parametrize("nt", [1501, 512, 2049, 300])
@pytest.mark.parametrize("name", sorted(SETS))
def test_speccorr_multi_bit_equal_to_single_kernel(dw, name, nt):
    import torch
    from das4whales_b200 import rows
    nx, nf = 5, 30
    S = torch.from_numpy(_spectrogram(nx, nf, nt, nt + len(name))).cuda()
    spec = SETS[name]
    kers = [_kernel(m, kw, i) for i, (_, m, kw) in enumerate(spec)]
    meds = [rows.row_median_ld(S, nx, m * nt, nf * nt, o * nt) for o, m, _ in spec]
    outs = rows.spectro_correlate_multi(S, kers, [o for o, _, _ in spec], meds)
    for (o, m, kw), K, med, out in zip(spec, kers, meds, outs):
        single = rows.spectro_correlate(S[:, o:o + m].contiguous(), K, median=med)
        assert torch.equal(out, single), (name, o, m, kw)
        assert torch.equal(med, rows.row_median(S[:, o:o + m].reshape(nx, -1).contiguous()))
        Sh = S[:, o:o + m].cpu().numpy().astype(np.float64)
        ref = np.stack([D.xcorr2d(Sh[i], K) for i in range(nx)])
        assert rel_err(out.cpu().numpy(), ref)[0] <= TOL


def test_speccorr_multi_more_than_eight_kernels_and_rows(dw):
    """Kernels go in groups of eight per call, rows in chunks of 65 535 per launch."""
    import torch
    from das4whales_b200 import rows
    nx, nf, nt = 65600, 12, 40
    S = torch.from_numpy(_spectrogram(nx, nf, nt, 3)).cuda()
    spec = [(i % 5, 7, 3 + i) for i in range(10)]
    kers = [_kernel(m, kw, i) for i, (_, m, kw) in enumerate(spec)]
    meds = [rows.row_median_ld(S, nx, m * nt, nf * nt, o * nt) for o, m, _ in spec]
    outs = rows.spectro_correlate_multi(S, kers, [o for o, _, _ in spec], meds)
    for (o, m, kw), K, med, out in zip(spec, kers, meds, outs):
        for r0 in (0, 65535):
            single = rows.spectro_correlate(S[r0:r0 + 65].contiguous()[:, o:o + m].contiguous(), K, median=med[r0:r0 + 65])
            assert torch.equal(out[r0:r0 + 65], single)


def test_speccorr_multi_rejects_bad_layouts(dw):
    import torch
    from das4whales_b200 import rows
    S = torch.zeros((2, 10, 50), dtype=torch.float32, device="cuda")
    med = torch.ones(2, dtype=torch.float32, device="cuda")
    with pytest.raises(ValueError):
        rows.spectro_correlate_multi(S, [np.ones((5, 3))], [6], [med])            # rows 6 .. 10 of a 10-bin band
    with pytest.raises(ValueError):
        rows.row_median_ld(S, 2, 600, 500)                                        # runs past the end
    with pytest.raises(ValueError):
        rows.row_median_ld(S, 2, 501, 500)                                        # ld < n


@pytest.mark.parametrize("nt,m,nf", [(300, 13, 30), (1501, 18, 19), (1501, 13, 30), (15001, 13, 18)])
def test_row_median_ld_exact(dw, nt, m, nf):
    """In-buffer (n <= 16 384) and bracketed lengths, ties, medians inside a block of zeros."""
    import torch
    from das4whales_b200 import rows
    nx = 6
    rng = np.random.default_rng(nt + m)
    S = _spectrogram(nx, nf, nt, nt)
    S[2] = np.floor(rng.random((nf, nt)) * 4)                                    # four distinct values: ties everywhere
    S[3] = np.where(rng.random((nf, nt)) < 0.6, 0.0, S[3])
    S[4] = 2.5
    St = torch.from_numpy(S).cuda()
    for o in sorted({0, nf - m, (nf - m) // 2}):
        med = rows.row_median_ld(St, nx, m * nt, nf * nt, o * nt).cpu().numpy()
        ref = np.median(S[:, o:o + m].reshape(nx, -1), axis=1).astype(np.float32)
        assert np.array_equal(med, ref), (o, med, ref)


def _strain(nx, ns, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((nx, ns))
    t = np.arange(ns) / FS
    for i in range(0, nx, 2):                                 # a hyperbolic 25 -> 16 Hz sweep in every other channel
        t0 = 1.0 + (i * 0.37) % max(1.0, t[-1] - 3.0)
        m = (t >= t0) & (t < t0 + 1.0)
        x[i, m] += 4 * sps.chirp(t[m] - t0, f0=25, f1=16, t1=1.0, method="hyperbolic") * np.hanning(m.sum())
    return x.astype(np.float32)


@pytest.mark.parametrize("ov,slide", [(0.95, True), (0.90, False)])
@pytest.mark.parametrize("nx,ns", [(6, 9000), (6, 12000), (6, 12001), (2, 120000)])
def test_correlograms_match_oracle(dw, nx, ns, ov, slide):
    from das4whales_b200 import _lib
    from das4whales_b200.detect import spectrocorr_layout
    nperseg, nhop, _, (u0, u1), _ = spectrocorr_layout(FS, FLIMS, [HF, LF], 0.8, ov, ns)
    assert bool(_lib.lib().d4w_stft_slide_supported(nperseg, nhop, u1 - u0 + 1)) == slide
    x = _strain(nx, ns, ns)
    outs = dw.detect.compute_cross_correlograms_spectrocorr(x, FS, FLIMS, [HF, LF], 0.8, ov)
    assert len(outs) == 2
    for out, kern in zip(outs, (HF, LF)):
        ref = D.compute_cross_correlogram_spectrocorr(x.astype(np.float64), FS, FLIMS, kern, 0.8, ov)
        assert out.dtype == np.float64 and out.shape == ref.shape
        e = rel_err(out, ref)
        assert e[0] <= TOL and e[1] <= TOL, (kern, e)


def test_one_kernel_equals_the_single_call_and_tensor_io(dw, capsys):
    import torch
    x = _strain(20, 12000, 1)
    both = dw.detect.compute_cross_correlograms_spectrocorr(x, FS, FLIMS, [HF, LF], 0.8, 0.95)
    for out, kern in zip(both, (HF, LF)):
        one = dw.detect.compute_cross_correlograms_spectrocorr(x, FS, FLIMS, [kern], 0.8, 0.95)[0]
        single = dw.detect.compute_cross_correlogram_spectrocorr(x, FS, FLIMS, kern, 0.8, 0.95)
        assert np.array_equal(one, single)
        # the pair reads the kernel's bins from the union band's STFT: the same values up to the STFT's rounding
        assert rel_err(out, single)[0] <= 1e-5
    assert "nperseg: 160, noverlap: 152, hop_length: 8" in capsys.readouterr().out
    xt = torch.from_numpy(x).cuda()
    outs_t = dw.detect.compute_cross_correlograms_spectrocorr(xt, FS, FLIMS, [HF, LF], 0.8, 0.95)
    for ot, oh in zip(outs_t, both):
        assert isinstance(ot, torch.Tensor) and ot.is_cuda and ot.dtype == torch.float32 and tuple(ot.shape) == oh.shape
        assert np.array_equal(ot.cpu().numpy().astype(np.float64), oh)


def test_more_than_65535_short_records(dw):
    nx, ns = 70001, 1800                                      # 9 s: LF takes its 15 frames from 8.4 s < t < 9 s
    rng = np.random.default_rng(5)
    x = rng.standard_normal((nx, ns)).astype(np.float32)
    outs = dw.detect.compute_cross_correlograms_spectrocorr(x, FS, FLIMS, [HF, LF], 0.8, 0.95)
    part = dw.detect.compute_cross_correlograms_spectrocorr(x[65530:65540], FS, FLIMS, [HF, LF], 0.8, 0.95)
    for out, p, kern in zip(outs, part, (HF, LF)):
        assert out.shape == (nx, 226)
        assert np.array_equal(out[65530:65540], p)                                # rows on both sides of the launch edge
        rows_ = [0, 65534, 65535, nx - 1]
        ref = D.compute_cross_correlogram_spectrocorr(x[rows_].astype(np.float64), FS, FLIMS, kern, 0.8, 0.95)
        e = rel_err(out[rows_], ref)
        assert e[0] <= TOL and e[1] <= TOL, e


# ---------------------------------------------------------------------------------------------------- file pipeline
def _marginal(row, t, thr, tol):
    """True when sample t of the float64 correlogram is a peak whose prominence lies within tol of the threshold"""
    peaks, props = sps.find_peaks(row, prominence=0)
    hit = np.nonzero(peaks == t)[0]
    return len(hit) == 1 and abs(props["prominences"][hit[0]] - thr) <= tol


def _oracle_chain(raw, scale, sel):
    from oracle import data_oracle as DH
    nx, ns = raw.shape
    x = DH.raw2strain(raw, {"scale_factor": scale})
    x = O.bp_filt(x, FS, 14., 30.)
    m = O.hybrid_ninf_filter_design((nx, ns), sel, DX, FS, 1350., 1450., 3300, 3450, 14., 30.)
    y = O.fk_filter_filt(x, m)
    return [D.compute_cross_correlogram_spectrocorr(y, FS, list(FLIMS), k, 0.8, 0.95) for k in (HF, LF)]


def test_spectro_pipeline_matches_oracle_chain(dw):
    import torch
    from das4whales_b200 import pipeline
    from oracle.make_golden import synth
    nx, ns, sel = 200, 6000, [0, 200, 1]
    x = synth(nx, ns, seed=9, ncalls=3)
    counts = np.round(x * 5.0e4).astype(np.int32) + 1234
    scale = 4.0838e-11 * 1550.0 / 2.0419
    refs = _oracle_chain(counts, scale, sel)
    maxv = max(r.max() for r in refs)
    # a threshold that keeps some peaks and rejects others in both correlograms: half the smaller of their top prominences
    proms = [np.concatenate([sps.find_peaks(row, prominence=0)[1]["prominences"] for row in r]) for r in refs]
    thr = 0.5 * min(float(p.max()) for p in proms)
    assert all((p >= thr).any() and (p < thr).any() for p in proms)
    pipe = pipeline.SpectroDetectPipeline(nx, ns, sel, DX, FS, scale, threshold=thr)
    assert pipe.nt == 751 and pipe.spectro_fs == 751 / ((ns - 1) / FS)
    dev = pipe.process_device(torch.from_numpy(counts).cuda(), with_snr=True, with_intermediates=True)
    assert abs(float(dev["maxv"].item()) - maxv) <= 1e-4 * maxv
    for name, c, ref in zip(("hf", "lf"), dev["corr"], refs):
        c64 = c.cpu().numpy().astype(np.float64)
        err = float(np.max(np.abs(c64 - ref)))
        assert err <= TOL * maxv, (name, err / maxv)
        snr = dev["snr_" + name].cpu().numpy()
        assert rel_err(10 ** (snr / 10), 10 ** (O.snr_tr_array(c64, env=True) / 10))[0] <= TOL
        got = pipe.picks_to_host(dev["picks_" + name])
        want = D.convert_pick_times(D.pick_times(ref, thr))
        assert want.shape[1] > 0
        gs, ws = set(map(tuple, got.T.tolist())), set(map(tuple, want.T.tolist()))
        for ch, t in gs ^ ws:                                 # a flip needs a prominence within 2 x the error of thr
            assert _marginal(ref[ch], t, thr, 2 * err + 1e-12 * maxv), (name, ch, t)
    res = pipe.process_file(counts)
    assert abs(res["maxv"] - maxv) <= 1e-4 * maxv and res["threshold"] == thr
    for name in ("hf", "lf"):
        assert np.array_equal(res["picks_" + name], pipe.picks_to_host(dev["picks_" + name]))
    outs = list(pipe.stream([counts, counts.astype(np.float32), counts]))
    assert len(outs) == 3
    for o in outs:
        assert np.array_equal(o["picks_hf"], res["picks_hf"]) and np.array_equal(o["picks_lf"], res["picks_lf"])
    one = pipeline.process_file_spectro(counts, {"dx": DX, "fs": FS, "scale_factor": scale}, sel, threshold=thr)
    assert np.array_equal(one["picks_hf"], res["picks_hf"]) and np.array_equal(one["picks_lf"], res["picks_lf"])
