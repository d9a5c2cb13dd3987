"""CPU: pick association.  The float64 oracle (oracle/assoc_oracle.py) against the invariants of back-projection; the kernel
bodies of csrc/assoc_kernels.cuh run block by block on the host (tests/host_emul/assoc_emul.cu) against the oracle, which
must agree exactly (labels, nodes, t0 and counts), since every bin is computed with the same float64 roundings; and every
ValueError of loc.associate_picks / localize_calls before device work."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from das4whales_b200 import loc
from oracle import assoc_oracle as A

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
EMUL = os.path.join(ROOT, "tests", "host_emul")
C0, FS, TOL = 1500.0, 200.0, 0.05
DXC = 10.0                                                   # channel spacing of the test cable (m)
GRID = ((0.0, 6000.0, 31), (0.0, 3000.0, 16), (0.0, 0.0, 1))
# on grid nodes; t0 far enough apart that no pick of one call falls in another's window (|t0_a - t0_b| > |a - b| / c0 +
# tol), while their move-outs overlap in time
SOURCES = [((1000.0, 1000.0, 0.0), 10.0), ((3000.0, 2000.0, 0.0), 11.7), ((5000.0, 600.0, 0.0), 13.5)]


def node_index(grid, w):
    nodes = A.grid_nodes(grid)
    return int(np.flatnonzero(np.all(nodes == np.asarray(w), axis=1))[0])


def scene(seed=0, nch=600, every=1, false_frac=0.0, sources=SOURCES):
    cable = A.straight_cable(nch, DXC)
    ch, s, truth = A.synth_picks(cable, sources, FS, C0, np.random.default_rng(seed), every, false_frac, t_max=20.0)
    return cable, ch, s, truth


# ------------------------------------------------------------------------------ oracle invariants
def test_oracle_finds_three_overlapping_calls():
    cable, ch, s, truth = scene()
    T = s / FS
    for a in range(2):                                        # consecutive calls' move-outs overlap in time
        ta, tb = T[truth == a], T[truth == a + 1]
        assert max(ta.min(), tb.min()) < min(ta.max(), tb.max())
    labels, node, t0, count = A.associate(ch, s, FS, cable, C0, GRID, TOL, min_picks=20)
    assert len(node) == 3
    # calls come out by decreasing score; every source covers the whole cable, so map them by node
    want = [node_index(GRID, w) for w, _ in SOURCES]
    perm = [want.index(g) for g in node]
    assert sorted(perm) == [0, 1, 2]
    for k, src in enumerate(perm):
        assert np.array_equal(labels == k, truth == src)
        assert count[k] == np.sum(truth == src)
        assert abs(t0[k] - SOURCES[src][1]) <= TOL
    assert np.all(np.diff(count) <= 0)


def test_oracle_shuffle_permutes_labels():
    cable, ch, s, _ = scene(false_frac=0.2, seed=3)
    ref = A.associate(ch, s, FS, cable, C0, GRID, TOL, min_picks=20)
    o = np.random.default_rng(5).permutation(len(ch))
    got = A.associate(ch[o], s[o], FS, cable, C0, GRID, TOL, min_picks=20)
    assert np.array_equal(got[0], ref[0][o])
    for a, b in zip(got[1:], ref[1:]):
        assert np.array_equal(a, b)


def test_oracle_noise_below_min_picks_and_max_calls():
    cable = A.straight_cable(600, DXC)
    rng = np.random.default_rng(1)
    ch, s = rng.integers(0, 600, 300), rng.integers(0, int(20 * FS), 300)
    labels, node, _, _ = A.associate(ch, s, FS, cable, C0, GRID, TOL, min_picks=40)
    assert len(node) == 0 and np.all(labels == -1)
    _, ch, s, _ = scene()
    labels, node, t0, count = A.associate(ch, s, FS, cable, C0, GRID, TOL, min_picks=20, max_calls=2)
    assert len(node) == 2 and len(t0) == 2 and set(np.unique(labels)) == {-1, 0, 1}
    assert np.sum(labels >= 0) == count.sum()


# ------------------------------------------------------------------------------ host emulation of the kernel bodies
@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    out = os.path.join(str(tmp_path_factory.mktemp("assoc")), "assoc_emul")
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "--expt-relaxed-constexpr", "-arch=sm_90a", "-Xcompiler",
                        "-ffp-contract=off", "-o", out, os.path.join(EMUL, "assoc_emul.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    return out


def emulate(exe, tmp, ch, s, cable, grid, tol, min_picks, max_calls=64):
    """(status, labels, node, t0, count) of the host loop of d4w_loc_associate; picks in CSR (channel-major) order"""
    assert np.all(np.diff(ch) >= 0)
    nch = len(cable)
    off = np.zeros(nch + 1, np.int32)
    off[1:] = np.cumsum(np.bincount(ch, minlength=nch))
    axes = [np.linspace(a, b, int(n)) for a, b, n in grid]
    h = tol / 2.0
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    with open(fin, "wb") as f:
        f.write(np.array([nch, len(s)] + [len(a) for a in axes] + [min_picks, max_calls], np.int64).tobytes())
        f.write(np.array([FS, C0, h, 1.0 / h], np.float64).tobytes())
        for a in [off, np.asarray(s, np.int32), np.ascontiguousarray(cable, np.float64)] + axes:
            f.write(np.ascontiguousarray(a).tobytes())
    subprocess.run([exe, fin, fout], check=True)
    raw = open(fout, "rb").read()
    status, K, _ = np.frombuffer(raw, np.int64, 3)
    n = len(s)
    o = 24
    labels = np.frombuffer(raw, np.int64, n, o); o += 8 * n
    node = np.frombuffer(raw, np.int64, K, o); o += 8 * K
    t0 = np.frombuffer(raw, np.float64, K, o); o += 8 * K
    count = np.frombuffer(raw, np.int64, K, o)
    return int(status), labels, node, t0, count


CASES = {
    # a straight cable with a grid on both sides: every node ties with its mirror image, the lower index wins
    "mirror": dict(grid=((0.0, 6000.0, 31), (-3000.0, 3000.0, 31), (0.0, 0.0, 1))),
    "empty_channels": dict(every=3),
    "nz": dict(grid=((0.0, 6000.0, 16), (0.0, 3000.0, 16), (-200.0, 0.0, 3)),
               sources=[((1200.0, 1000.0, 0.0), 10.0), ((3200.0, 2000.0, -100.0), 11.7), ((4800.0, 600.0, -200.0), 13.5)]),
    "single_node": dict(grid=((3000.0, 3000.0, 1), (2000.0, 2000.0, 1), (0.0, 0.0, 1))),
    "false_picks": dict(false_frac=0.2),
}


@pytest.mark.parametrize("case", list(CASES))
def test_emulation_equals_oracle(exe, tmp_path, case):
    kw = dict(CASES[case])
    grid = kw.pop("grid", GRID)
    cable, ch, s, _ = scene(seed=11, **kw)
    min_picks = 5 if case == "single_node" else 20
    status, *got = emulate(exe, str(tmp_path), ch, s, cable, grid, TOL, min_picks)
    ref = A.associate(ch, s, FS, cable, C0, grid, TOL, min_picks)
    assert status == 0
    assert len(ref[1]) >= 1
    for a, b in zip(got, ref):
        assert a.dtype == b.dtype and np.array_equal(a, b), case
    if case == "mirror":                                     # found at the mirror images, y <= 0
        assert np.all(A.grid_nodes(grid)[ref[1], 1] <= 0)


def test_emulation_refuses_an_oversized_histogram(exe, tmp_path):
    cable, ch, s, _ = scene()
    status, labels, node, _, _ = emulate(exe, str(tmp_path), ch, s, cable, GRID, 1e-5, 20)
    assert status == 2 and len(node) == 0


# ------------------------------------------------------------------------------ argument checks
def test_value_errors_before_any_device_work():
    cable, ch, s, _ = scene()
    picks = np.array([ch, s])
    good = dict(picks=picks, fs=FS, cable_pos=cable, c0=C0, grid=GRID, tol=TOL, min_picks=20)
    bad = [dict(grid=((0, 1, 2), (0, 1, 0), (0, 0, 1))), dict(grid=((0, 1, 2), (0, 1, 2))), dict(grid="x"),
           dict(grid=((0, np.inf, 2), (0, 1, 2), (0, 0, 1))),
           dict(tol=0.0), dict(tol=-1.0), dict(tol=np.nan), dict(tol=np.inf), dict(fs=0.0), dict(fs=np.inf),
           dict(c0=0.0), dict(c0=-1500.0), dict(c0=np.nan), dict(min_picks=0), dict(min_picks=2.5), dict(max_calls=0),
           dict(picks=np.array([ch, s])[:, :-1].T), dict(picks=np.array([np.r_[ch, 600], np.r_[s, 10]])),
           dict(picks=np.array([np.r_[ch, -1], np.r_[s, 10]])), dict(picks=np.array([ch, np.r_[s[:-1], -3]])),
           dict(cable_pos=cable[:, :2]), dict(cable_pos=np.where(cable == cable[5, 0], np.nan, cable)),
           dict(tol=1e-5)]                                  # 2e8 bins of tol / 2: the histogram does not fit
    for kw in bad:
        args = dict(good)
        args.update(kw)
        with pytest.raises(ValueError):
            loc.associate_picks(**args)
        with pytest.raises(ValueError):
            loc.localize_calls(**args)
    with pytest.raises(ValueError, match="raise tol or shorten the record"):
        loc.associate_picks(**dict(good, tol=1e-5))
    with pytest.raises(ValueError, match="nz = 1"):
        loc.localize_calls(**dict(good, grid=((0, 1, 2), (0, 1, 2), (0, 1, 2))), fix_z=True)


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    cable, ch, s, _ = scene()
    with pytest.raises(RuntimeError):
        loc.associate_picks(np.array([ch, s]), FS, cable, C0, GRID, TOL, 20)
    with pytest.raises(RuntimeError):
        loc.localize_calls(np.array([ch, s]), FS, cable, C0, GRID, TOL, 20, fix_z=True)
