"""CPU: the route map of the overlap-save matched filter (rows._pick_block) and the float64 references that
test_xcorr_routes_gpu.py checks every kernel route against.

_pick_block only ever returns 2 520-sample prime-factor blocks (k_xcorr_pfa) or 5 000-sample Cooley-Tukey blocks
(k_xcorr_fused); the GPU file forces 1 250 / 2 500 (k_xcorr_dual) and 1 274 (k_xcorr) itself.  If a test here fails because
_pick_block changed, the GPU cases that rely on the real route map (REAL_ROUTE_CASES, the 315 / 316-tap and
1 221 120 / 1 221 121-sample boundaries, the 512-segment limit) no longer reach the kernel their names say.

The positive-lag reference is the closed form of oracle.detect_oracle.compute_cross_correlogram_direct for a 2-D block of
rows: out[t] = (sum_{n<L} x~[t+n] c[n] - mu * sum_{j>=t} x~[j]) / m, x~ = (x - mean) / max|x| per row, c the template's
taps up to its last non-zero, mu = sum(c) / ns the mean of the zero-padded template and m = max|c|.  The last term is the
"mu term": the kernels add it as (mu / m) * (exclusive prefix of x~).  With the script's Hann-windowed chirps it is below
the suite's 2e-5 regression level, so only templates with a visible mean (Hann pulses) can tell whether it is right."""
import numpy as np
import pytest
import scipy.signal as sp

from conftest import rel_err
from oracle import detect_oracle as D
from das4whales_b200.rows import _pick_block
from test_xcorr_same_gpu import HF, LF, same_ref

MAX_SEGMENTS = 512          # segment prefixes k_row_stats keeps per row (rows_kernels.cuh, kMaxSeg)


def pulse(L):
    """Hann pulse of L taps: mean L / (2 ns) of the padded template, so the mu term is large."""
    return np.hanning(L + 2)[1:-1]


NEG = -np.hanning(92)[1:-1] * (1.0 + 0.5 * np.sin(0.2 * np.arange(90)))      # negative mean
ONE = np.array([0.7])                                                        # out = (x~ - mu * suffix) / m, mu / m = 1 / ns
GAPPY = pulse(200) * np.where((np.arange(200) // 25) % 3 == 1, 0.0, 1.0)      # interior zero runs
GAPPY[-30:] = 0.0                                                            # ... and trailing ones


def padded(c, ns):
    t = np.zeros(ns)
    t[:len(c)] = c
    return t


def trimmed(t):
    nz = np.nonzero(t)[0]
    return np.asarray(t[:nz[-1] + 1], dtype=np.float64)


def _normalised(x):
    x = np.asarray(x, dtype=np.float64)
    return (x - x.mean(axis=1, keepdims=True)) / np.abs(x).max(axis=1, keepdims=True)


def lags_ref(x, c):
    """sum_n x[t + n] c[n] for t = 0 .. ns - 1 of every row, zero past the row end: the correlation of a 2-D block of rows
    with a [1, L] kernel, as a convolution with the reversed taps along the rows only (no transform across rows, so that
    70 001 rows cost no more than 70 001 one-row correlations)."""
    x = np.asarray(x, dtype=np.float64)
    c = np.asarray(c, dtype=np.float64)
    L, ns = len(c), x.shape[1]
    return sp.fftconvolve(x, c[None, ::-1], mode="full", axes=1)[:, L - 1:L - 1 + ns]


def mu_term(x, c):
    """The part of pos_ref that comes from the padded template's mean: -mu / m * sum_{j>=t} x~[j]."""
    xt = _normalised(x)
    c = trimmed(c)
    mu, m = c.sum() / xt.shape[1], np.max(np.abs(c))
    return -mu / m * np.cumsum(xt[:, ::-1], axis=1)[:, ::-1]


def pos_ref(x, t, normalize=True):
    """rows.cross_correlogram(x, [t], normalize) in float64.  t: template zero-padded to ns (normalize=True) or taps."""
    if not normalize:
        return lags_ref(x, t)
    c = trimmed(t)
    return lags_ref(_normalised(x), c) / np.max(np.abs(c)) + mu_term(x, c)


def mu_visibility(x, t):
    """max-norm error of a kernel that left the mu term out, relative to the reference."""
    ref = pos_ref(x, t)
    return rel_err(ref - mu_term(x, trimmed(t)), ref)[0]


def _rows(nx, ns, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((nx, ns)) + 0.3
    x[1] += 1e3
    return x


# ---------------------------------------------------------------------------------------------------- route map
def test_pick_block_returns_only_pfa_or_5000_blocks():
    seen = set()
    for ns in (1, 100, 400, 1500, 2520, 12000, 120000, 1221120, 1221121, 2490881):
        for L in (1, 2, 50, 136, 156, 157, 300, 312, 313, 315, 316, 600, 1250, 2500):
            if L <= ns or ns == 1:
                seen.add(_pick_block(L, ns))
    assert seen == {2520, 5000}
    with pytest.raises(ValueError):
        _pick_block(2501, 12000)


def test_template_length_boundary_315_316():
    for ns in (400, 1500, 12000, 120000):
        assert _pick_block(315, ns) == 2520 and _pick_block(316, ns) == 5000
    assert _pick_block(2500, 12000) == 5000


def test_segment_count_boundaries():
    def nseg(ns, nb, L):
        return -(-ns // (nb - L + 1))
    L = 136
    assert nseg(1221120, 2520, L) == MAX_SEGMENTS and _pick_block(L, 1221120) == 2520
    assert nseg(1221121, 2520, L) == MAX_SEGMENTS + 1 and _pick_block(L, 1221121) == 5000
    # 1 250 / 2 500 blocks would need even more segments, so they are never the fallback
    assert nseg(1221121, 1250, L) > MAX_SEGMENTS and nseg(1221121, 2500, L) > MAX_SEGMENTS
    # 5 000 blocks are returned whatever the count; the normalised pass fails in d4w_row_stats above 512
    assert nseg(2490880, 5000, L) == MAX_SEGMENTS and nseg(2490881, 5000, L) == MAX_SEGMENTS + 1
    assert _pick_block(L, 2490881) == 5000


# ---------------------------------------------------------------------------------------------------- references
@pytest.mark.parametrize("c", [HF, pulse(50), NEG, ONE, GAPPY], ids=["hf", "pulse50", "neg", "one", "gappy"])
@pytest.mark.parametrize("ns", [203, 1500])
def test_pos_ref_matches_oracle(c, ns):
    x = _rows(3, ns, ns)
    t = padded(c, ns)
    ref = pos_ref(x, t)
    assert rel_err(ref, D.compute_cross_correlogram(x, t))[0] <= 1e-12
    assert rel_err(ref, D.compute_cross_correlogram_direct(x, t))[0] <= 1e-12
    raw = pos_ref(x, c, normalize=False)
    loop = np.stack([np.correlate(np.concatenate((r, np.zeros(len(c) - 1))), c, mode="valid") for r in x])
    assert rel_err(raw, loop)[0] <= 1e-12


def test_same_ref_matches_per_row_loop():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((4, 777))
    x[1] += 1e3
    x[2] = -np.abs(x[2]) - 1e-3                                     # max <= 0: zeros
    for c in (HF, pulse(300), ONE):
        ref = same_ref(x, c)
        for i in range(4):
            want = sp.correlate(x[i] / x[i].max(), c, mode="same", method="direct") if x[i].max() > 0 else np.zeros(777)
            assert np.max(np.abs(ref[i] - want)) <= 1e-12 * max(1.0, np.max(np.abs(want)))


def test_raw_taps_plus_prefix_term_is_the_reference():
    """What the kernels compute: the raw taps c (rows.cross_correlogram's tables) plus (mu / m) * exclusive prefix of x~.
    Demeaning the taps inside the support as well counts mu * sum_{n<L} x~[t+n] twice: 15 % off with a Hann pulse."""
    ns = 1500
    x = _rows(3, ns, 4)
    c = pulse(300)
    t = padded(c, ns)
    xt = _normalised(x)
    mu, m = c.sum() / ns, np.max(np.abs(c))
    prefix = np.concatenate((np.zeros((3, 1)), np.cumsum(xt, axis=1)[:, :-1]), axis=1)
    ref = pos_ref(x, t)
    assert rel_err(lags_ref(xt, c) / m + mu / m * prefix, ref)[0] <= 1e-12
    assert rel_err(lags_ref(xt, c - mu) / m + mu / m * prefix, ref)[0] > 0.1


def test_constant_row_reference_is_zero():
    x = np.full((1, 1500), 0.37)
    assert not np.any(pos_ref(x, padded(pulse(300), 1500)))


# ---------------------------------------------------------------------------------------------------- sensitivity
@pytest.mark.parametrize("ns", [1500, 12000, 120000])
def test_mu_term_is_invisible_with_the_script_chirps(ns):
    """Why the chirp tests cannot see the mu term: leaving it out stays below their 2e-5 bound."""
    x = _rows(4, ns, 1)
    for c in (HF, LF):
        assert mu_visibility(x, padded(c, ns)) < 2e-5


@pytest.mark.parametrize("c", [pulse(50), pulse(300), pulse(600), NEG], ids=["pulse50", "pulse300", "pulse600", "neg"])
@pytest.mark.parametrize("ns", [600, 1500, 12000])
def test_mu_term_is_visible_with_pulses(c, ns):
    """Leaving the mu term out costs >= 100 x the 1e-4 contract bound with these templates up to 12 000 samples."""
    if len(c) > ns:
        pytest.skip("template longer than the row")
    assert mu_visibility(_rows(4, ns, 2), padded(c, ns)) >= 1e-2
