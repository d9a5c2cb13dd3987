"""GPU: localisation (d4w_loc_solve / d4w_loc_grid through das4whales_b200.loc) against the reference's outputs
(tests/golden/loc.npz) and the float64 oracle.  Tolerances are those of the host emulation of the same kernel bodies
(tests/test_loc_host.py): positions and variances within 1e-9 relative, uncertainties within 1e-6."""
import re

import numpy as np
import pytest

from das4whales_b200 import detect, loc
from oracle import loc_oracle as O
from test_loc_host import C0, TOL_N, TOL_UNC, TOL_VAR, ragged_batch, rel

pytestmark = pytest.mark.gpu
NUM = re.compile(r"-?\d+\.\d+")


def test_solve_lq_and_covariance_match_reference(golden, capsys):
    g = golden("loc")
    cable = g["cable"]
    for k, (_, _, _, fz) in enumerate(g["cases"]):
        fz = bool(fz)
        T = g[f"T{k}"]
        capsys.readouterr()
        n = loc.solve_lq(T, cable, C0, fix_z=fz)
        out = capsys.readouterr().out.splitlines()
        ref = g[f"stdout{k}"].item().splitlines()
        assert len(out) == len(ref) == 10
        for a, b in zip(out, ref):
            assert NUM.sub("#", a) == NUM.sub("#", b)                  # same text around the numbers
            va, vb = np.array(NUM.findall(a), float), np.array(NUM.findall(b), float)
            assert np.all(np.abs(va - vb) <= 1e-4 + TOL_N * np.abs(vb)), (a, b)
        assert isinstance(n, np.ndarray) and n.shape == (4,)
        assert rel(n, g[f"n{k}"]) <= TOL_N
        var = loc.cal_variance_residuals(T, loc.calc_arrival_times(n[-1], cable, n[:3], C0), fz)
        assert rel(var, g[f"var{k}"]) <= TOL_VAR
        cov = loc.calc_covariance_matrix(cable, n, C0, var, fz)
        assert rel(cov, g[f"cov{k}"]) <= TOL_UNC
        assert rel(loc.calc_uncertainty_position(cable, n, C0, var, fz), g[f"unc{k}"]) <= TOL_UNC
        assert capsys.readouterr().out == ""
    cov = loc.calc_covariance_matrix(g["flat_cable"], g["flat_whale"], C0, float(g["flat_var"]))
    unc = loc.calc_uncertainty_position(g["flat_cable"], g["flat_whale"], C0, float(g["flat_var"]))
    assert capsys.readouterr().out == g["flat_covout"].item() == "Matrix is singular\nMatrix is singular\n"
    assert rel(cov, g["flat_cov"]) <= TOL_UNC and rel(unc, g["flat_unc"]) <= TOL_UNC


@pytest.mark.parametrize("fix_z", [False, True])
def test_batch_vs_oracle_ragged(fix_z):
    import torch
    cable = O.bent_cable(3000)
    rng = np.random.default_rng(21 + fix_z)
    counts = np.r_[[0, 1, 2, 3, 4, 5, 3000, 0], rng.integers(0, 3001, 1992)]
    T, P, off = ragged_batch(31 + fix_z, counts, cable, fix_z)
    p = 3 if fix_z else 4
    n0 = None if not fix_z else rng.uniform([0, 0, -800, 0], [60000, 60000, -10, 50], (len(counts), 4))
    res = loc.solve_lq_batch(T, P, off, C0, fix_z=fix_z, n0=n0)
    assert all(isinstance(a, np.ndarray) for a in res)
    assert res.n.shape == (len(counts), 4) and res.unc.shape == (len(counts), p)
    assert np.array_equal(res.nobs, counts)
    n, var, unc = O.solve_batch(T, P, off, C0, n0, 10, fix_z)
    assert rel(res.n, n) <= TOL_N and rel(res.var, var) <= TOL_VAR and rel(res.unc, unc) <= TOL_UNC
    assert np.all(np.isnan(res.var[counts <= p])) and np.all(np.isnan(res.unc[counts <= p]))
    assert np.all(np.isnan(res.n[counts == 0])) and np.all(np.isnan(res.n0[counts == 0]))
    if n0 is None:
        b = np.flatnonzero(counts > 0)
        assert np.array_equal(res.n0[b, :3], np.tile(O.REF_GUESS, (len(b), 1)))
        assert np.array_equal(res.n0[b, 3], [T[off[i]:off[i + 1]].min() for i in b])
    else:                                                       # an empty call's first guess is NaN like the rest of its row
        assert np.array_equal(res.n0[counts > 0], n0[counts > 0])
    # the tensor path: same numbers, tensors out, on the current stream
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        rt = loc.solve_lq_batch(torch.from_numpy(T).cuda(), torch.from_numpy(P).cuda(), off, C0, fix_z=fix_z, n0=n0)
    s.synchronize()
    assert all(isinstance(a, torch.Tensor) and a.is_cuda for a in rt)
    for a, b in zip(rt, res):
        assert np.array_equal(a.cpu().numpy(), b, equal_nan=True)


@pytest.mark.parametrize("fix_z,shape", [(True, (41, 37, 1)), (False, (21, 19, 5))])
def test_grid_vs_oracle(fix_z, shape):
    import torch
    cable = O.bent_cable(3000)
    counts = np.r_[[0, 3, 4, 5], np.random.default_rng(4).integers(6, 3001, 40)]
    T, P, off = ragged_batch(17, counts, cable, fix_z)
    grid = ((-10000, 70000, shape[0]), (-10000, 70000, shape[1]), (-50, -50, 1) if fix_z else (-1200, 0, shape[2]))
    index, score, n0 = loc.grid_search(T, P, off, C0, grid, fix_z=fix_z)
    nodes = O.grid_nodes(grid)
    p = 3 if fix_z else 4
    assert index[0] == -1 and np.isnan(score[0]) and np.all(np.isnan(n0[0]))
    for b in range(1, len(counts)):
        s = slice(off[b], off[b + 1])
        i = index[b]
        assert np.array_equal(n0[b, :3], nodes[i])
        if counts[b] <= p:
            assert np.isnan(score[b])
            continue
        sc, t0 = O.grid_scores(T[s], P[s], C0, nodes, fix_z)
        assert abs(score[b] - sc[i]) <= 1e-9 * sc[i], b
        assert sc[i] <= (1 + 1e-9) * sc.min(), b
        assert abs(n0[b, 3] - t0[i]) <= 1e-12 * abs(t0[i]), b
    it, st, nt = loc.grid_search(torch.from_numpy(T).cuda(), torch.from_numpy(P).cuda(), off, C0, grid, fix_z=fix_z)
    assert np.array_equal(it.cpu().numpy(), index) and np.array_equal(nt.cpu().numpy(), n0, equal_nan=True)
    # the batch solve starts from exactly these guesses
    res = loc.solve_lq_batch(T, P, off, C0, fix_z=fix_z, grid=grid)
    assert np.array_equal(res.n0, n0, equal_nan=True)
    n, var, unc = O.solve_batch(T, P, off, C0, np.where(np.isnan(n0), 0.0, n0), 10, fix_z)
    live = counts > 0
    assert rel(res.n[live], n[live]) <= TOL_N and rel(res.var[live], var[live]) <= TOL_VAR


def test_grid_recovers_whales_where_the_fixed_guess_diverges():
    cable = O.bent_cable(3000)
    rng = np.random.default_rng(0)
    whales = np.array([(40000., 23000.), (12000., 30000.), (30000., 45000.), (55000., 10000.), (5000., 20000.),
                       (23456., 31234.), (61234., 2345.)])
    T = np.concatenate([O.arrivals(cable, (x, y, -50.), 3.0, C0, 2e-3, rng) for x, y in whales])
    P = np.tile(cable, (len(whales), 1))
    off = np.arange(len(whales) + 1) * len(cable)
    grid = ((-10000, 70000, 161), (-10000, 70000, 161), (-50, -50, 1))
    ref = loc.solve_lq_batch(T, P, off, C0, fix_z=True)
    res = loc.solve_lq_batch(T, P, off, C0, fix_z=True, grid=grid)
    err_ref = np.hypot(*(ref.n[:, :2] - whales).T)
    err = np.hypot(*(res.n[:, :2] - whales).T)
    assert np.all(err_ref[[1, 2, 4]] > 10000), err_ref          # the reference's first guess diverges there
    assert np.all(err <= 50), err
    assert np.all(np.abs(res.n[:, 2] + 50) == 0)


def test_localize_picks_is_solve_lq_batch_of_select_picked_times():
    rng = np.random.default_rng(12)
    nch, fs = 2000, 200.0
    cable = O.bent_cable(nch)
    calls = [((20000., 25000., -50.), 30.0), ((45000., 15000., -50.), 95.0), ((10000., 40000., -50.), 160.0)]
    picks = [[] for _ in range(nch)]
    for w, t0 in calls:
        tt = O.arrivals(cable, w, t0, C0, 2e-3, rng)
        for c in range(0, nch, 3):
            picks[c].append(int(round(tt[c] * fs)))
    for c in range(0, nch, 7):
        picks[c].append(int(rng.integers(0, 200 * fs)))            # spurious picks
    idx_tp = detect.convert_pick_times([np.sort(p) for p in picks])
    windows = [(25.0, 75.0), (90.0, 140.0), (155.0, 205.0), (300.0, 301.0)]
    grid = ((-10000, 70000, 81), (-10000, 70000, 81), (-50, -50, 1))
    res = loc.localize_picks(idx_tp, fs, windows, cable, C0, fix_z=True, grid=grid)
    T, P = [], []
    for a, b in windows:
        ch, tt = detect.select_picked_times(idx_tp, a, b, fs)
        T.append(tt / fs)
        P.append(cable[ch])
    off = np.concatenate([[0], np.cumsum([len(t) for t in T])])
    want = loc.solve_lq_batch(np.concatenate(T), np.concatenate(P), off, C0, fix_z=True, grid=grid)
    for a, b in zip(res, want):
        assert np.array_equal(a, b, equal_nan=True)
    assert np.all(np.isnan(res.n[3]))


def test_two_runs_bit_identical():
    cable = O.bent_cable(3000)
    counts = np.random.default_rng(8).integers(0, 3001, 300)
    T, P, off = ragged_batch(41, counts, cable)
    grid = ((-10000, 70000, 41), (-10000, 70000, 41), (-1200, 0, 4))
    a = loc.solve_lq_batch(T, P, off, C0, grid=grid)
    b = loc.solve_lq_batch(T, P, off, C0, grid=grid)
    for x, y in zip(a, b):
        assert np.array_equal(x, y, equal_nan=True)
