"""CPU: localisation.  The float64 oracle (oracle/loc_oracle.py) against the reference's loc module and its fixture; the
kernel bodies of csrc/loc_kernels.cuh run block by block on the host (tests/host_emul/loc_emul.cu) against the oracle;
the window bookkeeping of loc.localize_picks against detect.select_picked_times; and every ValueError before device work.

Emulated against the oracle, positions agree to about 1e-12 relative (also on trajectories that diverge from the
reference's fixed first guess) and variances to 1e-13: both are held to 1e-9.  Uncertainties come from C = (G^T G)^-1,
which scales last-bit differences of G^T G by its condition number; that is large for free-z calls of few observations
(3.7e-8 was the worst of 2 000 ragged calls on an H100), so they are held to 1e-6.  The GPU tests use the same bounds."""
import contextlib
import io
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from das4whales_b200 import detect, loc
from oracle import loc_golden, loc_oracle as O, ref_loader

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
EMUL = os.path.join(ROOT, "tests", "host_emul")
C0 = 1490.0
TOL_N, TOL_VAR, TOL_UNC = 1e-9, 1e-9, 1e-6


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(b))
    m = ~np.isnan(b)
    return float(np.max(np.abs(a[m] - b[m]) / np.maximum(np.abs(b[m]), 1e-300), initial=0.0))


def ragged_batch(seed, counts, cable, fix_z=False):
    """calls at random whales with the given observation counts, channels drawn with repeats (duplicate rows)"""
    rng = np.random.default_rng(seed)
    T, P = [], []
    for n in counts:
        w = (rng.uniform(0, 60000), rng.uniform(0, 60000), -50.0 if fix_z else rng.uniform(-1200, 0))
        ch = rng.integers(0, len(cable), n)
        P.append(cable[ch])
        T.append(O.arrivals(cable[ch], w, rng.uniform(0, 100), C0, 2e-3, rng))
    return np.concatenate(T), np.concatenate(P), np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)


# ------------------------------------------------------------------------------ oracle against the reference
def test_oracle_matches_golden_reference(golden):
    g = golden("loc")
    cable = g["cable"]
    for k, (x, y, z, fz) in enumerate(g["cases"]):
        fz = bool(fz)
        T = g[f"T{k}"]
        n, traj = O.gauss_newton(T, cable, C0, np.r_[O.REF_GUESS, T.min()], 10, fz)
        assert np.array_equal(n, g[f"n{k}"])
        lines = g[f"stdout{k}"].item().splitlines()
        assert len(lines) == 10 and lines[-1].startswith("Iteration 10: x = ")
        var = O.variance(T, cable, n, C0, fz)
        assert rel(var, g[f"var{k}"]) <= 1e-15
        C, singular = O.covariance_unscaled(cable, n, C0, fz)
        assert not singular and rel(var * C, g[f"cov{k}"]) <= 1e-15
        assert rel(np.sqrt(var * np.diag(C)), g[f"unc{k}"]) <= 1e-15
    # the fixed first guess diverges for the second and third whales and converges for the first
    assert np.hypot(*(g["n0"][:2] - g["cases"][0][:2])) < 50
    for k in (1, 2):
        assert np.hypot(*(g[f"n{k}"][:2] - g["cases"][k][:2])) > 10000
    C, singular = O.covariance_unscaled(g["flat_cable"], g["flat_whale"], C0, False)
    assert singular and rel(g["flat_var"] * C, g["flat_cov"]) <= 1e-15
    assert g["flat_covout"].item() == "Matrix is singular\nMatrix is singular\n"


@pytest.mark.skipif(not ref_loader.available(), reason="reference not available")
@pytest.mark.parametrize("fix_z", [False, True])
@pytest.mark.parametrize("whale", [(38000., 21000., -80.), (12000., 30000., -50.), (55000., 10000., -300.)])
def test_oracle_matches_live_reference(fix_z, whale):
    L = loc_golden.load_loc()
    cable = O.bent_cable(1000)
    T = O.arrivals(cable, whale, 2.0, C0, 2e-3, np.random.default_rng(7))
    with contextlib.redirect_stdout(io.StringIO()):
        n = L.solve_lq(T, cable, C0, Nbiter=7, fix_z=fix_z)
        var = L.cal_variance_residuals(T, L.calc_arrival_times(n[-1], cable, n[:3], C0), fix_z)
        unc = L.calc_uncertainty_position(cable, n, C0, var, fix_z)
    no, vo, uo, _ = O.solve(T, cable, C0, None, 7, fix_z)
    assert np.array_equal(no, n) and rel(vo, var) <= 1e-15 and rel(uo, unc) <= 1e-13
    # the host helpers of loc.py are the reference's
    w = np.r_[whale, 0.0]
    assert np.array_equal(loc.calc_arrival_times(1.5, cable, whale, C0), L.calc_arrival_times(1.5, cable, whale, C0))
    for f in ("calc_distance_matrix", "calc_radii_matrix", "calc_theta_vector", "calc_phi_vector"):
        assert np.array_equal(getattr(loc, f)(cable, w[:3] if f == "calc_distance_matrix" else w),
                              getattr(L, f)(cable, w[:3] if f == "calc_distance_matrix" else w)), f
    assert loc.cal_variance_residuals(T, T[::-1], fix_z) == L.cal_variance_residuals(T, T[::-1], fix_z)


# ------------------------------------------------------------------------------ host emulation of the kernel bodies
@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    out = os.path.join(str(tmp_path_factory.mktemp("loc")), "loc_emul")
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "--expt-relaxed-constexpr", "-arch=sm_90a", "-o", out,
                        os.path.join(EMUL, "loc_emul.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    return out


def _emulate(exe, tmp, mode, T, pos, off, nbiter=10, fix_z=False, n0=None, axes=None):
    B, p = len(off) - 1, 3 if fix_z else 4
    nx, ny, nz = (len(a) for a in axes) if axes else (1, 1, 1)
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    with open(fin, "wb") as f:
        f.write(np.array([mode, B, len(T), nbiter, int(fix_z), n0 is not None, nx, ny, nz], np.int64).tobytes())
        f.write(np.float64(C0).tobytes())
        for a in [np.asarray(off, np.int64), T, pos] + ([] if n0 is None else [n0]) + (list(axes) if axes else []):
            f.write(np.ascontiguousarray(a).tobytes())
    subprocess.run([exe, fin, fout], check=True)
    raw = open(fout, "rb").read()
    if mode == 0:
        index = np.frombuffer(raw, np.int64, B)
        rest = np.frombuffer(raw, np.float64, offset=8 * B)
        return index, rest[:B], rest[B:].reshape(B, 4)
    a = np.frombuffer(raw, np.float64)
    sizes = dict(n=4 * B, var=B, unc=p * B, cinv=p * p * B, cond=B, traj=4 * nbiter * B)
    out, k = {}, 0
    for name, s in sizes.items():
        out[name] = a[k:k + s]
        k += s
    return out


@pytest.mark.parametrize("fix_z", [False, True])
def test_gn_emulation_vs_oracle(exe, tmp_path, fix_z):
    cable = O.bent_cable(3000)
    counts = [0, 1, 3, 4, 5, 40, 700, 3000, 2, 1500]
    T, P, off = ragged_batch(11 + fix_z, counts, cable, fix_z)
    p = 3 if fix_z else 4
    for n0 in (None, np.random.default_rng(3).uniform([0, 0, -800, 0], [60000, 60000, -10, 50], (len(counts), 4))):
        e = _emulate(exe, str(tmp_path), 1, T, P, off, 10, fix_z, n0)
        n, var, unc = O.solve_batch(T, P, off, C0, n0, 10, fix_z)
        assert rel(e["n"], n.ravel()) <= TOL_N
        assert rel(e["var"], var) <= TOL_VAR
        assert rel(e["unc"], unc.ravel()) <= TOL_UNC
        assert np.all(np.isnan(e["var"][np.array(counts) <= p]))
        assert np.all(np.isnan(e["n"][:4]))                     # the empty call
        b = counts.index(700)
        guess = np.r_[O.REF_GUESS, T[off[b]:off[b + 1]].min()] if n0 is None else n0[b]
        _, traj = O.gauss_newton(T[off[b]:off[b + 1]], P[off[b]:off[b + 1]], C0, guess, 10, fix_z)
        assert rel(e["traj"].reshape(-1, 10, 4)[b], traj) <= TOL_N


def test_singular_covariance_branch_emulation(exe, tmp_path, golden):
    g = golden("loc")
    flat, whale = g["flat_cable"], g["flat_whale"]
    off = np.array([0, len(flat)])
    e = _emulate(exe, str(tmp_path), 1, np.zeros(len(flat)), flat, off, 0, False, np.r_[whale[:3], 0.0][None])
    assert e["cond"][0] > 1 / np.finfo(float).eps
    assert rel(g["flat_var"] * e["cinv"].reshape(4, 4), g["flat_cov"]) <= TOL_UNC
    for k, (_, _, _, fz) in enumerate(g["cases"]):
        p = 3 if fz else 4
        e = _emulate(exe, str(tmp_path), 1, g[f"T{k}"], g["cable"], np.array([0, len(g["cable"])]), 0, bool(fz),
                     np.r_[g[f"n{k}"]][None])
        assert e["cond"][0] < 1 / np.finfo(float).eps
        assert rel(g[f"var{k}"] * e["cinv"].reshape(p, p), g[f"cov{k}"]) <= TOL_UNC


@pytest.mark.parametrize("fix_z,shape", [(True, (31, 23, 1)), (False, (13, 11, 5))])
def test_grid_emulation_vs_oracle(exe, tmp_path, fix_z, shape):
    cable = O.bent_cable(3000)
    counts = [0, 2, 4, 60, 900, 3000]
    T, P, off = ragged_batch(5, counts, cable, fix_z)
    grid = ((-10000, 70000, shape[0]), (-10000, 70000, shape[1]), (-50, -50, 1) if fix_z else (-1200, 0, shape[2]))
    axes = [np.linspace(*a) for a in grid]
    index, score, n0 = _emulate(exe, str(tmp_path), 0, T, P, off, fix_z=fix_z, axes=axes)
    nodes = O.grid_nodes(grid)
    p = 3 if fix_z else 4
    assert index[0] == -1 and np.isnan(score[0]) and np.all(np.isnan(n0[0]))
    for b in range(1, len(counts)):
        s = slice(off[b], off[b + 1])
        sc, t0 = O.grid_scores(T[s], P[s], C0, nodes, fix_z)
        i = index[b]
        assert np.array_equal(n0[b, :3], nodes[i])
        if counts[b] <= p:
            assert np.isnan(score[b])
            continue
        assert abs(score[b] - sc[i]) <= 1e-9 * sc[i]
        assert sc[i] <= (1 + 1e-9) * sc.min()
        assert abs(n0[b, 3] - t0[i]) <= 1e-12 * abs(t0[i])


# ------------------------------------------------------------------------------ host bookkeeping and argument checks
def test_picks_to_batch_is_select_picked_times():
    rng = np.random.default_rng(9)
    nch, fs = 400, 200.0
    idx_tp = detect.convert_pick_times([np.sort(rng.choice(20000, rng.integers(0, 12), replace=False)) for _ in range(nch)])
    cable = O.bent_cable(nch)
    windows = [(0.0, 10.0), (10.0, 10.0), (12.5, 40.005), (99.0, 98.0), (50.0, 100.0), (0.0, 1000.0), (30.0, 30.0 + 1 / fs)]
    T, P, off = loc.picks_to_batch(idx_tp, fs, windows, cable)
    for w, (a, b) in enumerate(windows):
        ch, tt = detect.select_picked_times(idx_tp, a, b, fs)
        assert np.array_equal(T[off[w]:off[w + 1]], tt / fs) and np.array_equal(P[off[w]:off[w + 1]], cable[ch])


def test_value_errors_before_any_device_work():
    T, P, off = ragged_batch(1, [10, 5], O.bent_cable(100))
    grid = ((0, 1, 2), (0, 1, 2), (0, 1, 2))
    bad = [dict(offsets=[0, 12, 11]), dict(offsets=[0, 5, 16]), dict(offsets=[-1, 15]), dict(offsets=[0.0, 15.0]),
           dict(offsets=[3]), dict(fix_z=True, grid=grid), dict(n0=np.zeros(4), grid=grid), dict(n0=np.zeros((3, 4))),
           dict(T=T[:-1]), dict(pos=P[:, :2]), dict(T=T[:, None]), dict(c0=0.0), dict(Nbiter=-1),
           dict(grid=((0, 1, 2), (0, 1, 0), (0, 1, 1))), dict(grid=((0, 1, 2), (0, 1, 2)))]
    for kw in bad:
        args = dict(T=T, pos=P, offsets=off, c0=C0)
        args.update(kw)
        with pytest.raises(ValueError):
            loc.solve_lq_batch(args.pop("T"), args.pop("pos"), args.pop("offsets"), args.pop("c0"), **args)
    with pytest.raises(ValueError):
        loc.grid_search(T, P, off, C0, ((0, 1, 2), (0, 1, 2), (0, 1, 3)), fix_z=True)
    with pytest.raises(ValueError):
        loc.solve_lq(T, P[:-1], C0)
    with pytest.raises(ValueError):
        loc.localize_picks(np.zeros((2, 3), np.int64), 200.0, [(0.0, 1.0)], np.zeros((5, 2)), C0)
    with pytest.raises(ValueError):
        loc.picks_to_batch(np.array([[0, 9], [1, 2]]), 200.0, [(0.0, 1.0)], np.zeros((5, 3)))


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    T, P, off = ragged_batch(1, [10, 5], O.bent_cable(100))
    with pytest.raises(RuntimeError):
        loc.solve_lq_batch(T, P, off, C0)
    with pytest.raises(RuntimeError):
        loc.solve_lq_batch(T, P, off, C0, fix_z=True, grid=((0, 1, 2), (0, 1, 2), (0, 0, 1)))
    with pytest.raises(RuntimeError):
        loc.solve_lq(T[:10], P[:10], C0)
    with pytest.raises(RuntimeError):
        loc.calc_uncertainty_position(P, np.r_[1000., 2000., -50., 0.], C0, 1e-6)
