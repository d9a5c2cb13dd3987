"""GPU: every kernel route of the overlap-save matched filter (rows.cross_correlogram: positive lags, normalised and
normalize=False; rows.cross_correlogram_same) against float64, with templates whose mean the correlation can see.

Each route is forced by replacing rows._pick_block, which cross_correlogram and same_mode_layout look up by global name,
so the whole host path (tables in the plan's order, row_stats and its segment prefixes, mu) runs unchanged.  The
float64 references and the template set are in test_xcorr_routes_host.py, which also pins them against
oracle.detect_oracle and checks the route map these cases rely on.

Which kernel a block length reaches (csrc/xcorr_launch.cuh):
  2520 = 5 * 7 * 8 * 9   the prime-factor plan                                                        -> k_xcorr_pfa
  1250 = 10.5.5.5,       fused plans (in-register first and last radix, so the tables are regrouped),
  2500 = 10.10.5.5       every radix <= 10 and 32 nb + 16 ceil(V / 8) + 16 <= 85 024 B <= 110 KB      -> k_xcorr_dual
  5000 = 10.10.10.5      fused, but 32 nb = 160 000 B > 110 KB                                         -> k_xcorr_fused
  1274 = 2 * 7^2 * 13    every plan has 7, 13 or 14 at one end: not fused, tables in plan order     -> k_xcorr
each as <false> (positive lags) and <true> ("same" mode)."""
import numpy as np
import pytest

from conftest import rel_err
from test_xcorr_same_gpu import HF, LF, same_ref
from test_xcorr_routes_host import GAPPY, NEG, ONE, mu_term, padded, pos_ref, pulse, trimmed

pytestmark = pytest.mark.gpu

ROUTES = [2520, 1250, 2500, 5000, 1274]
CHIRP_TOL = (2e-5, 2e-5)            # max-norm, l2: the suite's regression level
MEAN_TOL = (1e-4, 1e-5)             # templates with a visible mean: the 1e-4 contract bound, l2 at 1e-5
TEMPLATES = {"hf": HF, "lf": LF, "pulse50": pulse(50), "pulse300": pulse(300), "pulse600": pulse(600), "neg": NEG,
             "one": ONE, "gappy": GAPPY}
CHIRPS = ("hf", "lf")
MU_VISIBLE = ("pulse50", "pulse300", "pulse600", "neg", "gappy")      # leaving the mu term out costs >= 100 x MEAN_TOL
CASES = [(nb, name) for nb in ROUTES for name in TEMPLATES if name != "pulse600" or nb in (2520, 2500, 5000)]


@pytest.fixture(scope="module")
def dw():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import das4whales_b200 as dw
    from das4whales_b200 import _lib
    _lib.lib()
    return dw


@pytest.fixture
def force_block(dw, monkeypatch):
    from das4whales_b200 import rows

    def force(nb):
        plan = rows.fft_plan(nb, 0)
        assert sorted(plan.pos2freq) == list(range(nb))
        if nb == 2520:                  # table order of the radix-9 last dimension: [m * 280 + j] <- position j * 9 + m
            assert np.array_equal(plan.tab2freq, plan.pos2freq.reshape(280, 9).T.ravel())
        elif nb == 1274:
            assert np.array_equal(plan.tab2freq, plan.pos2freq)
        else:
            assert not np.array_equal(plan.tab2freq, plan.pos2freq)
        monkeypatch.setattr(rows, "_pick_block", lambda L, ns=0: nb)
    return force


def _rows(nx, ns, seed):
    """fp32 rows: noise, noise + 1e3 (the kernels subtract a float-rounded mean), a single spike, a constant non-zero row
    (exactly zero out of the normalised pass) and noise on a slow drift (large suffix sums, so a large mu term)."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((nx, ns))
    x[1] += 1e3
    x[2] = 0.0
    x[2, (2 * ns) // 3] = 1.5
    x[3] = 0.37
    x[4] += 0.3 + 2.0 * np.sin(2 * np.pi * np.arange(ns) / ns)
    return x.astype(np.float32)


def _lengths(nb, L):
    """Row lengths around the kept outputs per block V = nb - L + 1: shorter than V (and than nb), V, V + 1, the ragged
    2- and 4-segment CTAs 4V + 1 and 5V + 3, and the script's 12 000 / 120 000 samples."""
    V = nb - L + 1
    short = max(L, (V // 3) | 1)
    return [short if short < V else L, V, V + 1, 4 * V + 1, 5 * V + 3, 12000, 120000]


def _run(x, templates, normalize=True, same=False):
    import torch
    from das4whales_b200 import rows
    xd = torch.from_numpy(x).cuda()
    outs = rows.cross_correlogram_same(xd, templates) if same else rows.cross_correlogram(xd, templates, normalize)
    return [o.cpu().numpy().astype(np.float64) for o in outs]


def _check(got, ref, tol, what):
    e = rel_err(got, ref)
    assert e[0] <= tol[0] and e[1] <= tol[1], (what, e)
    return e


def _check_rows(got, ref, what):
    """Row by row at CHIRP_TOL (row 1's 1e3 offset would otherwise set the scale of the whole matrix).  Without
    normalisation the DC of rows 1 (offset 1e3) and 3 (constant) reaches the transform: a zero-mean chirp's output cancels
    it, and the fp32 rounding of the DC leaves up to 3e-5 l2 error on those rows (max-norm stays near 1e-6), so their l2
    is held at 1e-4."""
    errs = []
    for i in range(got.shape[0]):
        e = rel_err(got[i], ref[i])
        assert e[0] <= CHIRP_TOL[0] and e[1] <= (1e-4 if i in (1, 3) else CHIRP_TOL[1]), (what, i, e)
        errs.append(e)
    return errs


def _report(mode, nb, name, errs):
    print(f"xcorr route {mode} nb={nb} {name}: max {max(e[0] for e in errs):.2e} l2 {max(e[1] for e in errs):.2e}")


# ---------------------------------------------------------------------------------------------------- every route
@pytest.mark.parametrize("nb,name", CASES)
def test_normalised_positive_lags(force_block, nb, name):
    c = TEMPLATES[name]
    force_block(nb)
    tol = CHIRP_TOL if name in CHIRPS else MEAN_TOL
    errs = []
    for ns in _lengths(nb, len(trimmed(c))):
        x = _rows(5, ns, nb + ns)
        t = padded(c, ns)
        got = _run(x, [t])[0]
        ref = pos_ref(x, t)
        errs.append(_check(got, ref, tol, ns))
        assert not np.any(got[3]), ns                                       # constant row
        if name in MU_VISIBLE and ns <= 12000:
            assert rel_err(ref - mu_term(x, t), ref)[0] >= 100 * tol[0], ns
    _report("normalised", nb, name, errs)


@pytest.mark.parametrize("nb,name", CASES)
def test_unnormalised_positive_lags(force_block, nb, name):
    """normalize=False (detect.shift_xcorr): plain lags of the raw taps; trailing zeros are dropped from the taps."""
    c = TEMPLATES[name]
    force_block(nb)
    errs = []
    for ns in _lengths(nb, len(trimmed(c))):
        x = _rows(5, ns, nb + ns + 1)
        got = _run(x, [c], normalize=False)[0]
        ref = pos_ref(x, c, normalize=False)
        errs.extend(_check_rows(got, ref, ns))
    _report("raw", nb, name, errs)


@pytest.mark.parametrize("nb,name", CASES)
def test_same_mode(force_block, nb, name):
    c = TEMPLATES[name]
    force_block(nb)
    errs = []
    for ns in _lengths(nb, len(c)):
        x = _rows(5, ns, nb + ns + 2)
        got = _run(x, [c], same=True)[0]
        ref = same_ref(x, c)
        errs.extend(_check_rows(got, ref, ns))
    _report("same", nb, name, errs)


# ---------------------------------------------------------------------------------------------------- the real route map
@pytest.mark.parametrize("L,nb", [(315, 2520), (316, 5000), (2500, 5000)])
@pytest.mark.parametrize("ns", [2600, 12000, 120000])
def test_block_boundaries_of_the_real_route(dw, L, nb, ns):
    from das4whales_b200 import rows
    assert rows._pick_block(L, ns) == nb
    c = pulse(L)
    x = _rows(5, ns, L + ns)
    t = padded(c, ns)
    ref = pos_ref(x, t)
    _check(_run(x, [t])[0], ref, MEAN_TOL, "normalised")
    if ns <= 12000:
        assert rel_err(ref - mu_term(x, t), ref)[0] >= 100 * MEAN_TOL[0]
    _check_rows(_run(x, [c], same=True)[0], same_ref(x, c), "same")


def test_template_longer_than_one_pass_is_refused(dw):
    x = _rows(5, 12000, 1)
    with pytest.raises(ValueError):
        _run(x, [padded(pulse(2501), 12000)])


@pytest.mark.parametrize("lengths", [(1, 136, 300, 315), (136, 600)])
def test_one_pass_equals_single_template_calls(dw, lengths):
    """Several templates share one forward transform and one block length (that of the longest), so each result must
    equal its single-template call, which may run on another block length, up to rounding.  {1, 136, 300, 315} stay on
    2 520-sample blocks with fewer kept outputs per block; {136, 600} move the 136-tap chirp to 5 000-sample blocks."""
    from das4whales_b200 import rows
    ns = 12000
    shapes = {1: ONE, 136: HF, 300: pulse(300), 315: pulse(315) * np.cos(0.02 * np.arange(315)), 600: pulse(600)}
    cs = [shapes[L] for L in lengths]
    assert rows._pick_block(max(lengths), ns) == (2520 if max(lengths) <= 315 else 5000)
    x = _rows(8, ns, 5)
    for same in (False, True):
        tpls = cs if same else [padded(c, ns) for c in cs]
        together = _run(x, tpls, same=same)
        for t, o in zip(tpls, together):
            single = _run(x, [t], same=same)[0]
            assert np.max(np.abs(o - single)) <= 1e-6 * np.max(np.abs(single)), (same, len(trimmed(t)))
            if not same:
                _check(o, pos_ref(x, t), MEAN_TOL, len(trimmed(t)))


def test_more_than_65535_rows_normalised(dw):
    nx, ns = 70001, 400
    rng = np.random.default_rng(8)
    x = (rng.standard_normal((nx, ns)) + rng.standard_normal((nx, 1))).astype(np.float32)
    t = padded(pulse(300), ns)
    got = dw.detect.compute_cross_correlogram(x, t)
    ref = pos_ref(x, t)
    _check(got, ref, MEAN_TOL, "all rows")
    _check(got[65530:65540], ref[65530:65540], MEAN_TOL, "chunk edge")
    assert rel_err(ref - mu_term(x, t), ref)[0] >= 100 * MEAN_TOL[0]


# ---------------------------------------------------------------------------------------------------- segment limits
@pytest.mark.parametrize("ns,nb", [(1221120, 2520), (1221121, 5000)])
def test_512_segments(dw, ns, nb):
    """136 taps: 1 221 120 samples are 512 segments of 2 520-sample blocks, the most k_row_stats keeps; one more sample
    moves the row to 5 000-sample blocks."""
    from das4whales_b200 import rows
    assert rows._pick_block(136, ns) == nb
    x = _rows(5, ns, 9)[[0, 4]]
    t = padded(pulse(136), ns)
    ref = pos_ref(x, t)
    _check(_run(x, [t])[0], ref, MEAN_TOL, ns)
    assert rel_err(ref - mu_term(x, t), ref)[0] >= 100 * MEAN_TOL[0]


def test_more_than_512_segments_raise(dw):
    """513 segments of 5 000-sample blocks with 136 taps: d4w_row_stats refuses them (D4W_ERR_UNSUPPORTED, raised as
    ValueError), so the normalised pass returns nothing rather than a correlogram without its mu term."""
    import torch
    from das4whales_b200 import rows
    ns = 2490881
    xd = torch.zeros((2, ns), dtype=torch.float32, device="cuda")
    xd[:, ::7] = 1.0
    with pytest.raises(ValueError, match="more than 512 segments"):
        rows.cross_correlogram(xd, [padded(pulse(136), ns)])


def test_10000_sample_blocks_are_unsupported(dw):
    """d4w_fft_plan_create prefers 10.10.10.10 for 10 000 samples, but three float2 buffers (240 000 B) exceed the opt-in
    shared memory: d4w_xcorr must refuse it with D4W_ERR_UNSUPPORTED instead of launching."""
    import torch
    from das4whales_b200 import _lib, rows
    nb, ns, L = 10000, 20000, 136
    plan = rows.fft_plan(nb, 0)
    xd = torch.zeros((1, ns), dtype=torch.float32, device="cuda")
    tabs = torch.zeros((1, nb, 2), dtype=torch.float32, device="cuda")
    out = torch.full((1, 1, ns), 7.0, dtype=torch.float32, device="cuda")
    null = _lib.ffi.NULL
    rc = _lib.lib().d4w_xcorr(plan.ptr, _lib.ptr(xd, "float*"), 1, ns, nb - L + 1, 1, _lib.ptr(tabs), null, null, null,
                              _lib.ptr(out, "float*"), _lib.stream_ptr())
    assert rc == 2                                  # D4W_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert bool(torch.all(out == 7.0))              # nothing was launched
