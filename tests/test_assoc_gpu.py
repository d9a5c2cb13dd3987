"""GPU: pick association (d4w_loc_associate through loc.associate_picks / localize_calls).  The device result must equal the
float64 oracle (oracle/assoc_oracle.py) exactly, as the host emulation does (tests/test_assoc_host.py): every bin is
computed with the same roundings, counts are integers and every reduction has a fixed order."""
import numpy as np
import pytest

from das4whales_b200 import loc
from oracle import assoc_oracle as A

pytestmark = pytest.mark.gpu
C0, FS = 1500.0, 200.0
NCH, DXC = 2000, 10.0                                        # a 20 km straight cable along x
TOL_E2E = 20.0                                               # m, test_end_to_end_mfdetect_pipeline


def nodes_on(grid, xy):
    """grid nodes nearest to the given (x, y, z) points"""
    nodes = A.grid_nodes(grid)
    return [tuple(nodes[np.argmin(np.sum((nodes - np.asarray(p)) ** 2, 1))]) for p in xy]


def scene(grid, seed=0, every=1, false_frac=0.0, fs=FS):
    cable = A.straight_cable(NCH, DXC)
    pts = nodes_on(grid, [(4000.0, 1500.0, 0.0), (9000.0, 3000.0, -100.0), (15000.0, 800.0, -300.0)])
    sources = list(zip(pts, (10.0, 13.0, 17.0)))
    ch, s, truth = A.synth_picks(cable, sources, fs, C0, np.random.default_rng(seed), every, false_frac, t_max=40.0)
    return cable, ch, s, truth


def device_csr(ch, s, nch):
    import torch
    off = np.zeros(nch + 1, np.int32)
    off[1:] = np.cumsum(np.bincount(ch, minlength=nch))
    return torch.from_numpy(off).cuda(), torch.from_numpy(s.astype(np.int32)).cuda()


G61 = ((0.0, 20000.0, 61), (0.0, 6000.0, 61), (0.0, 0.0, 1))
G31 = ((0.0, 20000.0, 31), (0.0, 6000.0, 31), (-300.0, 0.0, 4))
CASES = {
    "mirror": (((0.0, 20000.0, 61), (-6000.0, 6000.0, 61), (0.0, 0.0, 1)), {}),
    "empty_channels": (G61, dict(every=3)),
    "nz": (G31, {}),
    "single_node": (((9000.0, 9000.0, 1), (3000.0, 3000.0, 1), (0.0, 0.0, 1)), {}),
    "false_picks_61": (G61, dict(false_frac=0.2)),
    "false_picks_31": (G31, dict(false_frac=0.2)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_device_equals_oracle(case):
    import torch
    grid, kw = CASES[case]
    cable, ch, s, _ = scene(grid, seed=4, **kw)
    tol, mp = 0.05, (5 if case == "single_node" else 50)
    o = np.random.default_rng(2).permutation(len(ch))          # host picks in any order
    ref = A.associate(ch[o], s[o], FS, cable, C0, grid, tol, mp)
    assert len(ref[1]) >= 3
    got = loc.associate_picks(np.array([ch[o], s[o]]), FS, cable, C0, grid, tol, mp)
    assert all(isinstance(a, np.ndarray) for a in got)
    for a, b in zip(got, ref):
        assert a.dtype == b.dtype and np.array_equal(a, b), case
    # device CSR in: CUDA tensors out, labels in CSR order, the same calls; and a second run is bit-identical
    picks = device_csr(ch, s, NCH)
    d1 = loc.associate_picks(picks, FS, cable, C0, grid, tol, mp)
    d2 = loc.associate_picks(picks, FS, cable, C0, grid, tol, mp)
    assert all(isinstance(a, torch.Tensor) and a.is_cuda for a in d1)
    for a, b in zip(d1, d2):
        assert torch.equal(a, b)
    ref_csr = A.associate(ch, s, FS, cable, C0, grid, tol, mp)
    for a, b in zip(d1, ref_csr):
        assert np.array_equal(a.cpu().numpy(), b), case
    for a, b in zip(d1[1:], got[1:]):
        assert np.array_equal(a.cpu().numpy(), b)
    if case == "mirror":
        assert np.all(A.grid_nodes(grid)[ref[1], 1] <= 0)


def test_no_picks_and_max_calls():
    cable, ch, s, _ = scene(G61)
    res = loc.associate_picks(np.zeros((2, 0), np.int64), FS, cable, C0, G61, 0.05, 1)
    assert res.labels.shape == (0,) and res.node.shape == (0,)
    res = loc.associate_picks(np.array([ch, s]), FS, cable, C0, G61, 0.05, 50, max_calls=2)
    ref = A.associate(ch, s, FS, cable, C0, G61, 0.05, 50, max_calls=2)
    assert len(res.node) == 2
    for a, b in zip(res, ref):
        assert np.array_equal(a, b)


def test_oversized_histogram_from_device_picks_is_a_value_error():
    cable, ch, s, _ = scene(G61)
    with pytest.raises(ValueError, match="raise tol or shorten the record"):
        loc.associate_picks(device_csr(ch, s, NCH), FS, cable, C0, G61, 1e-5, 50)


def test_localize_calls_is_solve_lq_batch_of_the_calls():
    """Off-grid sources at fs = 10 kHz (sample rounding 0.05 ms, 7.5 cm of range): every call is found whole and localised
    within 1 m.  tol = 0.5 s: at the nearest node of this 61 x 61 grid the picks' origin times spread by at most
    2 * 174 m / c0 = 0.23 s, less than one bin of tol / 2, and the calls are 25 s apart.  The grid starts 100 m off the
    cable: on the cable line (y = 0) a straight cable gives the solver no y gradient, and when several nodes hold a whole
    call the lowest index, the lowest y, wins."""
    import torch
    fs = 10000.0
    grid = ((0.0, 20000.0, 61), (100.0, 6100.0, 61), (0.0, 0.0, 1))
    cable = A.straight_cable(NCH, DXC)
    whales = [(4123.0, 1456.0, 0.0), (9871.0, 2954.0, 0.0), (15432.0, 777.0, 0.0)]
    ch, s, truth = A.synth_picks(cable, list(zip(whales, (10.0, 35.0, 60.0))), fs, C0, None)
    picks = device_csr(ch, s, NCH)
    assoc, res = loc.localize_calls(picks, fs, cable, C0, grid, 0.5, 100, fix_z=True)
    K = assoc.node.numel()
    assert K == 3
    lab = assoc.labels.cpu().numpy()
    order = []
    for k in range(K):
        src = np.unique(truth[lab == k])
        assert len(src) == 1 and np.array_equal(lab == k, truth == src[0])
        order.append(int(src[0]))
    # the composition: solve_lq_batch of the calls' picks in CSR order from (node, t0)
    rows = np.concatenate([np.flatnonzero(lab == k) for k in range(K)])
    off = np.r_[0, np.cumsum([np.sum(lab == k) for k in range(K)])]
    nodes = A.grid_nodes(grid)[assoc.node.cpu().numpy()]
    n0 = np.column_stack([nodes, assoc.t0.cpu().numpy()])
    T = torch.from_numpy(s[rows] / fs).cuda()
    P = torch.from_numpy(cable[ch[rows]]).cuda()
    want = loc.solve_lq_batch(T, P, off, C0, fix_z=True, n0=n0)
    for a, b in zip(res, want):
        assert torch.equal(a, b)
    n = res.n.cpu().numpy()
    err = [np.hypot(*(n[k, :2] - np.asarray(whales[order[k]][:2]))) for k in range(K)]
    assert max(err) <= 1.0, err
    # host picks in: the same calls, ndarrays out
    ah, rh = loc.localize_calls(np.array([ch, s]), fs, cable, C0, grid, 0.5, 100, fix_z=True)
    assert np.array_equal(ah.labels, lab) and np.array_equal(rh.n, n)
    # no call: empty results
    a0, r0 = loc.localize_calls(picks, fs, cable, C0, grid, 0.5, 10 ** 6, fix_z=True)
    assert a0.node.numel() == 0 and r0.n.shape == (0, 4)


def test_end_to_end_mfdetect_pipeline():
    """synth.synth_strain -> MfDetectPipeline.process_device -> localize_calls on the device HF picks.  The generator puts a
    call at (c dx, 500, 0) with its chirp starting at sample floor((t0 + d / 1500) fs) on every channel; seed 225 gives
    8 calls at least 3.6 s apart, all inside the 60 s record.  The picks are envelope peaks quantised to 5 ms (7.5 m of range)
    and shifted by the template's constant lag, which moves t0 but not the position.  Grid: 102 m along the cable, 50 m
    across from y = 50 (not on the cable line, where a straight cable gives no y gradient); at the nearest node a call's
    origin times spread by at most 2 * 57 m / c0 = 0.08 s plus the pick jitter, inside one bin of tol / 2 = 0.125 s.
    On an H100 the eight calls came out 0.4-4.7 m from the truth (picks quantised to 7.5 m of range, some 1 750 per call);
    TOL_E2E = 20 m holds that with a margin of four times the worst case and is five times finer than the grid the solver
    starts from."""
    from das4whales_b200 import pipeline, synth
    nx, ns, seed, dx, fs = 2000, 12000, 225, synth.DX, synth.FS
    x = synth.synth_strain(nx, ns, seed=seed)
    rng = np.random.default_rng(seed)
    truth = []
    for _ in range(int(round(8 * ns / fs / 60.0))):
        c = float(rng.integers(0, nx))
        t0 = float(rng.uniform(0, max(ns / fs - 10.0, 1.0)))
        truth.append((c * dx, 500.0, t0))
    assert len(truth) == 8
    pipe = pipeline.MfDetectPipeline(nx, ns, [0, nx, 1], dx, fs, 1.0)
    out = pipe.process_device(x)
    picks = out["picks_hf"]
    cable = A.straight_cable(nx, dx)
    grid = ((0.0, nx * dx, 41), (50.0, 2000.0, 40), (0.0, 0.0, 1))
    assoc, res = loc.localize_calls(picks, fs, cable, 1500.0, grid, 0.25, nx // 4, fix_z=True)
    n = res.n.cpu().numpy()
    assert len(n) == len(truth)
    for xt, yt, t0 in truth:
        # two of these whales are 77 m apart: a call is matched by position and origin time together
        hit = (np.hypot(n[:, 0] - xt, n[:, 1] - yt) <= TOL_E2E) & (np.abs(n[:, 3] - t0) <= 0.5)
        assert np.sum(hit) == 1, (xt, t0, n)
