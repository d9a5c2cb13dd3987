"""GPU parity of the Hilbert family for row lengths with no T1 x T2 split (chirp-z rows, csrc/hilbert_czt.cuh): envelope,
H(x), envelope / std, envelope SNR and instant_freq against the float64 oracle on every route (whole row in one CTA below
16 384 convolution points, five split launches on two real rows per transform above; either middle-pass kernel), the
spectrogram-correlation flow of scripts/main_spectrodetect.py on 1 501-frame correlograms, and the 128 000-sample limit."""
import numpy as np
import pytest
import scipy.signal as sps

from conftest import rel_err
from oracle import dsp_oracle as O, detect_oracle as D
from test_rows_gpu import HILBERT_ROUTES

pytestmark = pytest.mark.gpu
FS = 200.0
TOL = 1e-4
# every one of these lengths has a prime factor > 61 (no direct plan); 8 191 / 8 193 sit on either side of the
# whole-row (convolution <= 16 384 points) / split boundary; from 16 933 on, one length per further split radix
LENGTHS = [751, 1126, 1501, 4099, 8191, 8193, 15001, 127997,
           16933, 16399, 19573, 30723, 31161, 39083, 41877, 61854, 62234, 8443]
# T1 of the split lengths (convolution length M = T1 x T2 in the comments); every other length is a whole row (T1 = 1)
SPLIT_T1 = {
    8193: 3,        # 16 875
    15001: 3,       # 30 375
    127997: 25,     # 256 000
    16933: 4,       # 34 560
    16399: 5,       # 32 805
    19573: 6,       # 39 366
    30723: 8,       # 62 208
    31161: 10,      # 62 500
    39083: 12,      # 78 732
    41877: 15,      # 84 375
    61854: 16,      # 124 416
    62234: 20,      # 125 000
    8443: 2,        # 17 280
}


@pytest.fixture(scope="module")
def dw():
    import torch
    assert torch.cuda.is_available()
    import das4whales_b200 as dw
    from das4whales_b200 import _lib
    _lib.lib()
    return dw


@pytest.fixture
def fresh_plans(monkeypatch):
    """Plans read D4W_ROW_FUSED when they are created: start from an empty cache, free what was made."""
    from das4whales_b200 import _lib, rows
    monkeypatch.setattr(rows, "_row_plans", {})
    yield rows
    for p in rows._row_plans.values():
        _lib.lib().d4w_row_plan_destroy(p.ptr)


def _chirp_rows(nx, n, seed):
    """smooth-envelope chirps (well-defined instantaneous frequency) plus a little noise"""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / FS
    rows = []
    for i in range(nx):
        f0, f1 = 8.0 + 3 * i, 30.0 + 5 * i
        c = sps.chirp(t, f0=f0, f1=f1, t1=t[-1], method="linear") * (1.0 + 0.3 * np.sin(2 * np.pi * 0.7 * t + i))
        rows.append(c + 0.01 * rng.standard_normal(n))
    return np.asarray(rows, dtype=np.float32)


@pytest.mark.parametrize("env", HILBERT_ROUTES)
def test_hilbert_family_czt_lengths(dw, fresh_plans, monkeypatch, env):
    from das4whales_b200 import _lib
    rows = fresh_plans
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    import torch
    for i, n in enumerate(LENGTHS):
        nx = (1, 2, 3)[i % 3]
        x = _chirp_rows(nx, n, seed=n)
        x64 = x.astype(np.float64)
        a = sps.hilbert(x64, axis=1)
        env_ = dw.detect.envelope(x)
        assert rel_err(env_, np.abs(a))[0] <= 2e-5, (n, nx)
        xd = torch.from_numpy(x).cuda()
        hx = rows.hilbert_imag(xd).cpu().numpy()
        assert rel_err(hx, a.imag)[0] <= 2e-5, (n, nx)
        eos = rows.envelope_over_std(xd).cpu().numpy()
        assert rel_err(eos, np.abs(a) / x64.std(axis=1, keepdims=True))[0] <= 2e-5, (n, nx)
        snr = dw.dsp.snr_tr_array(x, env=True)
        ref = O.snr_tr_array(x64, env=True)
        assert rel_err(10 ** (snr / 10), 10 ** (ref / 10))[0] <= TOL, (n, nx)
        fi = dw.dsp.instant_freq(x[0], FS)
        fref = O.instant_freq(x64[0], FS)
        assert fi.shape == fref.shape == (n - 1,)
        assert np.max(np.abs(fi - fref)) <= 2e-4 * FS, n
        assert np.max(np.abs(fi[50:-50] - fref[50:-50])) <= 2e-5 * FS, n
        plan = rows.row_plan(n, 0)
        t1, t2, m = plan.info()
        assert m >= 2 * n - 1 and t1 * t2 == m, (n, t1, t2, m)
        assert (t1 == 1) == (m <= 16384), (n, t1, m)
        assert t1 == SPLIT_T1.get(n, 1), (n, t1)
        ws = _lib.lib().d4w_row_workspace_bytes(plan.ptr, nx)
        assert ws == (16 if t1 == 1 else (nx + 1) // 2 * m * 8), (n, ws)


def test_plan_info_direct_lengths_unchanged(dw, fresh_plans):
    """Lengths with a T1 x T2 split keep the direct plan (czt_m = 0) and its workspace of ns complex samples per row."""
    from das4whales_b200 import _lib
    rows = fresh_plans
    for n, split in ((600, (1, 600)), (12000, (1, 12000)), (36000, (4, 9000)), (120000, (12, 10000)), (240000, (25, 9600))):
        plan = rows.row_plan(n, 0)
        assert plan.info() == split + (0,), n
        if split[0] > 1:
            assert _lib.lib().d4w_row_workspace_bytes(plan.ptr, 3) == 2 * n * 8
    assert rows.HILBERT_MAX_SAMPLES == 128000


def test_length_limit(dw, fresh_plans):
    x = np.random.default_rng(1).standard_normal((1, 128001)).astype(np.float32)      # 3 x 42 667 (prime)
    with pytest.raises(ValueError, match="128000"):
        dw.detect.envelope(x)
    x = np.random.default_rng(2).standard_normal((2, 240000)).astype(np.float32)      # direct plan, no limit
    assert rel_err(dw.detect.envelope(x), D.envelope(x.astype(np.float64)))[0] <= 2e-5


def _marginal(env_row, t, thr, tol):
    """True when sample t of the float64 envelope is a peak whose prominence lies within tol of the threshold"""
    peaks, props = sps.find_peaks(env_row, prominence=0)
    hit = np.nonzero(peaks == t)[0]
    return len(hit) == 1 and abs(props["prominences"][hit[0]] - thr) <= tol


def test_spectrodetect_correlogram_flow(dw):
    """scripts/main_spectrodetect.py:106-119 on synthetic strain (64 x 12 000): 1 501-frame correlograms (19 x 79) through
    snr_tr_array(env=True), envelope and pick_times_env, against the float64 oracle applied to the device's own correlogram.
    Picks may differ only at peaks whose prominence sits at the threshold."""
    from das4whales_b200 import synth
    x = synth.synth_strain(64, 12000, seed=7).cpu().numpy()
    flims = [14., 30.]
    for kern in ({'f0': 27., 'f1': 17., 'dur': 0.8, 'bdwidth': 4.}, {'f0': 20., 'f1': 14., 'dur': 1.2, 'bdwidth': 4.}):
        corr = dw.detect.compute_cross_correlogram_spectrocorr(x, FS, flims, kern, 0.8, 0.95)
        assert corr.shape == (64, 1501)
        c64 = np.asarray(corr, dtype=np.float64)
        snr = dw.dsp.snr_tr_array(corr, env=True)
        ref = O.snr_tr_array(c64, env=True)
        assert rel_err(10 ** (snr / 10), 10 ** (ref / 10))[0] <= TOL
        env_ref = D.envelope(c64)
        assert rel_err(dw.detect.envelope(corr), env_ref)[0] <= 2e-5
        thr = 0.25 * float(np.max(env_ref))
        got = dw.detect.convert_pick_times(dw.detect.pick_times_env(corr, thr))
        want = D.convert_pick_times(D.pick_times_env(c64, thr))
        assert want.shape[1] >= 1
        gs, ws = set(map(tuple, got.T.tolist())), set(map(tuple, want.T.tolist()))
        tol = 1e-4 * float(np.max(env_ref))
        for ch, t in gs ^ ws:
            assert _marginal(env_ref[ch], t, thr, tol), (ch, t)
