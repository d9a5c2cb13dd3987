"""Localisation of whale calls from arrival times picked along the cable (reference: das4whales/loc.py).

The geometry helpers and `cal_variance_residuals` are host NumPy, as in the reference.  `solve_lq`,
`calc_covariance_matrix` and `calc_uncertainty_position` keep the reference's signatures and run on the GPU
(d4w_loc_solve); `solve_lq_batch` solves many calls in one launch, optionally from the best node of a grid search
(d4w_loc_grid), and `localize_picks` solves the calls of a pick list cut by time windows.  `associate_picks` groups a
file's picks into calls by back-projection over a source grid (d4w_loc_associate), and `localize_calls` solves every call
it finds, so no time window is needed.  Everything is float64.
"""
import sys
from collections import namedtuple

import numpy as np

from . import _lib

Localisation = namedtuple("Localisation", "n var unc nobs n0")
Localisation.__doc__ = """Result of solve_lq_batch for B calls: n [B, 4] = (x, y, z, t0); var [B] = cal_variance_residuals at n;
unc [B, p] = sqrt(var diag C) in the order of the unknowns, (x, y, z, t0) or (x, y, t0) with fix_z; nobs [B]; n0 [B, 4] the
first guess.  var and unc are NaN for a call with nobs <= p; a call with no observation is NaN throughout."""

# ------------------------------------------------------------------------------ host geometry (loc.py:13-54, :131-153)
def calc_arrival_times(t0, cable_pos, pos, c0):
    """t0 + |cable_pos - pos| / c0 for every cable position"""
    x, y, z = pos
    return t0 + np.sqrt((cable_pos[:, 0] - x) ** 2 + (cable_pos[:, 1] - y) ** 2 + (cable_pos[:, 2] - z) ** 2) / c0


def calc_distance_matrix(cable_pos, whale_pos):
    return np.sqrt(np.sum((cable_pos - whale_pos) ** 2, axis=1))


def calc_radii_matrix(cable_pos, whale_pos):
    """horizontal distances"""
    return np.sqrt(np.sum((cable_pos[:, :2] - whale_pos[:2]) ** 2, axis=1))


def calc_theta_vector(cable_pos, whale_pos):
    """elevation angle atan2(|z_whale - z_cable|, r)"""
    return np.arctan2(abs(whale_pos[2] - cable_pos[:, 2]), calc_radii_matrix(cable_pos, whale_pos))


def calc_phi_vector(cable_pos, whale_pos):
    """azimuth atan2(y_whale - y_cable, x_whale - x_cable)"""
    return np.arctan2(whale_pos[1] - cable_pos[:, 1], whale_pos[0] - cable_pos[:, 0])


def cal_variance_residuals(arrtimes, predic_arrtimes, fix_z=False):
    """sum of squared residuals / (n - 3) with fix_z, / (n - 4) otherwise"""
    residuals = arrtimes - predic_arrtimes
    return 1 / (len(residuals) - (3 if fix_z else 4)) * np.sum(residuals ** 2)


# ------------------------------------------------------------------------------ argument checks (host, before device work)
def _torch():
    import torch
    if not torch.cuda.is_available():
        raise _lib.D4WError("das4whales_b200 needs a CUDA device (no CPU fallback)")
    return torch


def _is_tensor(x):
    return type(x).__module__.startswith("torch") and hasattr(x, "is_cuda")


def _offsets(offsets, nobs):
    off = np.asarray(offsets.cpu() if _is_tensor(offsets) else offsets)
    if off.ndim != 1 or off.size < 2 or not np.issubdtype(off.dtype, np.integer):
        raise ValueError("offsets must be a 1-D integer array of B + 1 >= 2 entries")
    off = off.astype(np.int64)
    if off[0] < 0 or off[-1] > nobs or np.any(np.diff(off) < 0):
        raise ValueError(f"offsets must be non-decreasing within [0, {nobs}]")
    return off


def _grid_axes(grid, fix_z):
    try:
        axes = [(float(a), float(b), int(n)) for a, b, n in grid]
    except (TypeError, ValueError):
        raise ValueError("grid must be ((x0, x1, nx), (y0, y1, ny), (z0, z1, nz))") from None
    if len(axes) != 3 or any(n < 1 for _, _, n in axes):
        raise ValueError("grid must be ((x0, x1, nx), (y0, y1, ny), (z0, z1, nz)) with every n >= 1")
    if fix_z and axes[2][2] != 1:
        raise ValueError("fix_z holds z at the first guess: the grid needs nz = 1")
    return [np.linspace(a, b, n) for a, b, n in axes]


def _check(T, pos, offsets, c0, Nbiter, fix_z, n0, grid):
    """validated host-side description of a batch; raises ValueError before any device work"""
    tensor = _is_tensor(T)
    if tensor != _is_tensor(pos):
        raise ValueError("T and pos must both be ndarrays or both be CUDA tensors")
    if tensor:
        import torch
        if not (T.is_cuda and pos.is_cuda and T.dtype == torch.float64 and pos.dtype == torch.float64):
            raise ValueError("tensor inputs must be float64 CUDA tensors")
    else:
        T, pos = np.asarray(T, dtype=np.float64), np.asarray(pos, dtype=np.float64)
    if T.ndim != 1 or pos.ndim != 2 or pos.shape[1] != 3 or pos.shape[0] != T.shape[0]:
        raise ValueError(f"T must be [n_obs] and pos [n_obs, 3], got {tuple(T.shape)} and {tuple(pos.shape)}")
    off = _offsets(offsets, T.shape[0])
    B = off.size - 1
    if not (np.isfinite(c0) and c0 > 0):
        raise ValueError("c0 must be a positive speed")
    if int(Nbiter) != Nbiter or Nbiter < 0:
        raise ValueError("Nbiter must be an integer >= 0")
    if n0 is not None and grid is not None:
        raise ValueError("n0 and grid are mutually exclusive")
    if n0 is not None:
        n0 = np.asarray(n0.cpu() if _is_tensor(n0) else n0, dtype=np.float64)
        if n0.shape == (4,):
            n0 = np.broadcast_to(n0, (B, 4))
        if n0.shape != (B, 4):
            raise ValueError(f"n0 must be [4] or [{B}, 4], got {n0.shape}")
    axes = _grid_axes(grid, fix_z) if grid is not None else None
    return tensor, T, pos, off, n0, axes


def _dev(a, device):
    torch = _torch()
    if _is_tensor(a):
        return a.contiguous()
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def _pd(t):
    return _lib.ptr(t, "double*")


# ------------------------------------------------------------------------------ device calls
def _grid(Td, Pd, offd, B, c0, fix_z, axes):
    torch = _torch()
    L = _lib.lib()
    gx, gy, gz = (_dev(a, Td.device) for a in axes)
    ws = torch.empty(max(1, int(L.d4w_loc_grid_workspace_bytes(B, gx.numel(), gy.numel(), gz.numel()))),
                     dtype=torch.uint8, device=Td.device)
    index = torch.empty(B, dtype=torch.int64, device=Td.device)
    score = torch.empty(B, dtype=torch.float64, device=Td.device)
    n0 = torch.empty((B, 4), dtype=torch.float64, device=Td.device)
    _lib.check(L.d4w_loc_grid(_pd(Td), _pd(Pd), _lib.ptr(offd, "long long*"), B, float(c0), int(bool(fix_z)),
                              _pd(gx), gx.numel(), _pd(gy), gy.numel(), _pd(gz), gz.numel(), _lib.ptr(ws),
                              _lib.ptr(index, "long long*"), _pd(score), _pd(n0), _lib.stream_ptr()), "loc_grid")
    return index, score, n0


def _solve(Td, Pd, offd, B, c0, Nbiter, fix_z, n0d, cinv=False, traj=False):
    torch = _torch()
    p = 3 if fix_z else 4
    dev = Td.device
    o = dict(n=torch.empty((B, 4), dtype=torch.float64, device=dev), var=torch.empty(B, dtype=torch.float64, device=dev),
             unc=torch.empty((B, p), dtype=torch.float64, device=dev), cond=torch.empty(B, dtype=torch.float64, device=dev),
             n0=torch.empty((B, 4), dtype=torch.float64, device=dev))
    if cinv:
        o["cinv"] = torch.empty((B, p, p), dtype=torch.float64, device=dev)
    if traj:
        o["traj"] = torch.empty((B, max(1, Nbiter), 4), dtype=torch.float64, device=dev)
    null = _lib.ffi.NULL
    _lib.check(_lib.lib().d4w_loc_solve(
        _pd(Td), _pd(Pd), _lib.ptr(offd, "long long*"), B, float(c0), int(Nbiter), int(bool(fix_z)),
        null if n0d is None else _pd(n0d), _pd(o["n"]), _pd(o["var"]), _pd(o["unc"]),
        _pd(o["cinv"]) if cinv else null, _pd(o["cond"]), _pd(o["traj"]) if traj else null, _pd(o["n0"]),
        _lib.stream_ptr()), "loc_solve")
    return o


def _device_of(tensor, T):
    torch = _torch()
    return T.device if tensor else torch.device("cuda", torch.cuda.current_device())


def grid_search(T, pos, offsets, c0, grid, fix_z=False):
    """Best node of `grid` for every call: (index [B] int64, score [B], n0 [B, 4]).

    grid = ((x0, x1, nx), (y0, y1, ny), (z0, z1, nz)): nodes numpy.linspace(x0, x1, nx) x ..., node index
    (iz * ny + iy) * nx + ix.  score = sum (T - t0* - d / c0)^2 / (nobs - p) with t0* = mean(T - d / c0), the residual
    variance at the best emission time; the minimising node (ties to the lowest index) and its t0* are n0.  An empty
    call gets index -1 and NaN; a call with nobs <= p gets the node of least squared residual and a NaN score."""
    tensor, T, pos, off, _, axes = _check(T, pos, offsets, c0, 0, fix_z, None, grid)
    dev = _device_of(tensor, T)
    with _torch().cuda.device(dev):
        index, score, n0 = _grid(_dev(T, dev), _dev(pos, dev), _dev(off, dev), off.size - 1, c0, fix_z, axes)
    if tensor:
        return index, score, n0
    return index.cpu().numpy(), score.cpu().numpy(), n0.cpu().numpy()


def solve_lq_batch(T, pos, offsets, c0, Nbiter=10, fix_z=False, n0=None, grid=None):
    """loc.solve_lq for B calls in one launch.  Call b is T[offsets[b]:offsets[b + 1]] (s) at pos[...] ([n_obs, 3], m);
    two picks of one channel are two rows.  First guess: n0=None is the reference's [40000, 23000, -60, min(T)] per call;
    n0 [4] or [B, 4] is used as given; grid (see grid_search) starts each call at its best node.  With fix_z, z stays at
    the first guess.  Returns a Localisation; ndarrays in give ndarrays out, float64 CUDA tensors in give tensors out
    (computed on the current stream)."""
    tensor, T, pos, off, n0, axes = _check(T, pos, offsets, c0, Nbiter, fix_z, n0, grid)
    torch = _torch()
    B = off.size - 1
    dev = _device_of(tensor, T)
    with torch.cuda.device(dev):
        Td, Pd, offd = _dev(T, dev), _dev(pos, dev), _dev(off, dev)
        if axes is not None:
            n0d = _grid(Td, Pd, offd, B, c0, fix_z, axes)[2]
        elif n0 is not None:
            n0d = _dev(np.ascontiguousarray(n0), dev)
        else:
            n0d = None
        o = _solve(Td, Pd, offd, B, c0, int(Nbiter), fix_z, n0d)
        res = Localisation(o["n"], o["var"], o["unc"], offd[1:] - offd[:-1], o["n0"])
    if tensor:
        return res
    return Localisation(*(t.cpu().numpy() for t in res))


def picks_to_batch(idx_tp, fs, windows, cable_pos):
    """(T, pos, offsets) of the calls of a pick list: call w is detect.select_picked_times(idx_tp, *windows[w], fs), in
    the pick list's order, with arrival times sample / fs at cable_pos[channel].  Host bookkeeping on the picks."""
    ch = np.asarray(idx_tp[0])
    sm = np.asarray(idx_tp[1])
    cable_pos = np.asarray(cable_pos, dtype=np.float64)
    win = np.asarray(windows, dtype=np.float64)
    if win.ndim != 2 or win.shape[1] != 2 or win.shape[0] == 0:
        raise ValueError("windows must be a non-empty list of (tstart, tend) pairs")
    if cable_pos.ndim != 2 or cable_pos.shape[1] != 3:
        raise ValueError(f"cable_pos must be [channels, 3], got {cable_pos.shape}")
    if ch.shape != sm.shape or ch.ndim != 1:
        raise ValueError("idx_tp must be [[channel ...], [sample ...]]")
    if ch.size and (ch.min() < 0 or ch.max() >= cable_pos.shape[0]):
        raise ValueError("a picked channel is outside cable_pos")
    # picks ordered by sample: a window is a contiguous run of that order, taken back to the pick list's own order
    order = np.argsort(sm, kind="stable")
    ss = sm[order]
    sel = []
    for tstart, tend in win:
        lo = np.searchsorted(ss, tstart * fs, side="left")      # first sample >= tstart * fs
        hi = np.searchsorted(ss, tend * fs, side="right")       # first sample > tend * fs
        sel.append(np.sort(order[lo:max(lo, hi)]))
    offsets = np.concatenate([[0], np.cumsum([len(x) for x in sel])]).astype(np.int64)
    rows = np.concatenate(sel).astype(np.int64)
    return sm[rows] / fs, cable_pos[ch[rows]], offsets


def localize_picks(idx_tp, fs, windows, cable_pos, c0, Nbiter=10, fix_z=False, grid=None):
    """Localise the calls of a pick list: idx_tp = [[channel ...], [sample ...]] as detect.convert_pick_times and the
    pipelines' picks_to_host return it, windows = [(tstart, tend), ...] in seconds, cable_pos [channels, 3] in metres.
    Call w is detect.select_picked_times(idx_tp, *windows[w], fs) (picks_to_batch); all calls are solved by one
    solve_lq_batch, whose Localisation (ndarrays) is returned."""
    T, pos, offsets = picks_to_batch(idx_tp, fs, windows, cable_pos)
    return solve_lq_batch(T, pos, offsets, c0, Nbiter=Nbiter, fix_z=fix_z, grid=grid)


# ------------------------------------------------------------------------------ association of picks into calls
Association = namedtuple("Association", "labels node t0 count")
Association.__doc__ = """Result of associate_picks for K calls: labels [n_picks] int64, the call of each pick or -1; node [K] int64,
the grid node index of each call; t0 [K] float64, its origin time (s); count [K] int64, its number of picks.  Calls are
numbered in extraction order (highest score first)."""


def _assoc_picks(picks, ncable):
    """('device', offsets int32, samples int32) or ('host', ch int64, s int64), validated"""
    if isinstance(picks, (tuple, list)) and len(picks) == 2 and all(_is_tensor(a) for a in picks):
        import torch
        offsets, idx = picks
        if not (offsets.is_cuda and idx.is_cuda and offsets.dtype == torch.int32 and idx.dtype == torch.int32
                and offsets.ndim == 1 and idx.ndim == 1 and offsets.numel() >= 2):
            raise ValueError("device picks must be (offsets int32 [n_channels + 1], idx int32 [n_picks]) CUDA tensors")
        if offsets.numel() - 1 > ncable:
            raise ValueError(f"a picked channel is outside cable_pos: the picks have {offsets.numel() - 1} channels, "
                             f"cable_pos {ncable} rows")
        return "device", offsets.contiguous(), idx.contiguous()
    try:
        a = np.asarray(picks)
    except (TypeError, ValueError):
        raise ValueError("picks must be [[channel ...], [sample ...]] or the device (offsets, idx)") from None
    if a.ndim != 2 or a.shape[0] != 2 or not (a.size == 0 or np.issubdtype(a.dtype, np.integer)):
        raise ValueError("picks must be [[channel ...], [sample ...]] of integers or the device (offsets, idx)")
    ch, s = a[0].astype(np.int64), a[1].astype(np.int64)
    if ch.size and (ch.min() < 0 or ch.max() >= ncable):
        raise ValueError("a picked channel is outside cable_pos")
    if s.size and s.min() < 0:
        raise ValueError("a pick has a negative sample")
    if s.size and s.max() > np.iinfo(np.int32).max:
        raise ValueError("pick samples must be below 2**31")
    return "host", ch, s


def _assoc_check(picks, fs, cable_pos, c0, grid, tol, min_picks, max_calls):
    for name, v in (("fs", fs), ("c0", c0), ("tol", tol)):
        if not (isinstance(v, (int, float, np.integer, np.floating)) and np.isfinite(v) and v > 0):
            raise ValueError(f"{name} must be positive and finite")
    for name, v in (("min_picks", min_picks), ("max_calls", max_calls)):
        if int(v) != v or v < 1:
            raise ValueError(f"{name} must be an integer >= 1")
    axes = _grid_axes(grid, False)
    if not all(np.all(np.isfinite(a)) for a in axes):
        raise ValueError("grid bounds must be finite")
    cable_pos = np.asarray(cable_pos.cpu() if _is_tensor(cable_pos) else cable_pos, dtype=np.float64)
    if cable_pos.ndim != 2 or cable_pos.shape[1] != 3 or cable_pos.shape[0] == 0 or not np.all(np.isfinite(cable_pos)):
        raise ValueError(f"cable_pos must be finite [channels, 3], got {cable_pos.shape}")
    kind, a, b = _assoc_picks(picks, cable_pos.shape[0])
    h = float(tol) / 2.0
    r = 1.0 / h
    if kind == "host" and a.size:
        # the histogram bound the device applies to the picks' range, checked here before any device work
        used = cable_pos[np.unique(a)]
        box = np.r_[used.min(0), used.max(0), [x.min() for x in axes], [x.max() for x in axes]]
        _assoc_bins(b.min() / float(fs), b.max() / float(fs), box, float(c0), r)
    return kind, a, b, cable_pos, axes, h, r


def _assoc_bins(tmin, tmax, box, c0, r):
    L = _lib.lib()
    box = np.ascontiguousarray(box, dtype=np.float64)
    jlo, nb = _lib.ffi.new("long long*"), _lib.ffi.new("int*")
    rc = L.d4w_loc_assoc_bins(float(tmin), float(tmax), _lib.ffi.cast("double*", box.ctypes.data), c0, r, jlo, nb)
    _assoc_rc(rc)


def _assoc_rc(rc):
    if rc == 2:           # D4W_ERR_UNSUPPORTED: the vote's histogram does not fit shared memory
        msg = _lib.ffi.string(_lib.lib().d4w_last_error()).decode(errors="replace")
        raise ValueError(f"associate_picks: {msg}: raise tol or shorten the record")
    _lib.check(rc, "loc_associate")


def _associate_device(offsets, samples, fs, cable_pos, c0, axes, h, r, min_picks, max_calls):
    """device CSR in, (labels, node, t0, count) CUDA tensors out (labels in CSR order)"""
    torch = _torch()
    L = _lib.lib()
    dev = offsets.device
    nch, npk = offsets.numel() - 1, samples.numel()
    P = _dev(cable_pos, dev)
    gx, gy, gz = (_dev(a, dev) for a in axes)
    ws = torch.empty(max(1, int(L.d4w_loc_assoc_workspace_bytes(npk, gx.numel(), gy.numel(), gz.numel()))),
                     dtype=torch.uint8, device=dev)
    labels = torch.empty(npk, dtype=torch.int64, device=dev)
    node = torch.empty(max_calls, dtype=torch.int64, device=dev)
    t0 = torch.empty(max_calls, dtype=torch.float64, device=dev)
    count = torch.empty(max_calls, dtype=torch.int64, device=dev)
    K = _lib.ffi.new("int*")
    _assoc_rc(L.d4w_loc_associate(_lib.ptr(offsets, "int*"), _lib.ptr(samples, "int*"), nch, npk, float(fs), _pd(P),
                                  float(c0), _pd(gx), gx.numel(), _pd(gy), gy.numel(), _pd(gz), gz.numel(), h, r,
                                  int(min_picks), int(max_calls), _lib.ptr(ws), _lib.ptr(labels, "long long*"),
                                  _lib.ptr(node, "long long*"), _pd(t0), _lib.ptr(count, "long long*"), K,
                                  _lib.stream_ptr()))
    k = int(K[0])
    return Association(labels, node[:k], t0[:k], count[:k])


def _host_csr(ch, s, ncable, dev):
    """host picks -> (order, device offsets int32, device samples int32) in channel-major, stable order"""
    torch = _torch()
    order = np.argsort(ch, kind="stable")
    off = np.zeros(ncable + 1, dtype=np.int32)
    off[1:] = np.cumsum(np.bincount(ch, minlength=ncable))
    return order, _dev(off, dev), _dev(s[order].astype(np.int32), dev)


def associate_picks(picks, fs, cable_pos, c0, grid, tol, min_picks, max_calls=64):
    """Group picks into calls by back-projection over a source grid, on the GPU.

    picks: the host [[channel ...], [sample ...]] of detect.convert_pick_times / picks_to_host, or the device
    (offsets, idx) of a pipeline's process_device.  cable_pos [n_channels, 3] (m), row c = channel c; c0 the sound speed;
    grid = ((x0, x1, nx), (y0, y1, ny), (z0, z1, nz)) as grid_search.  For every node g each pick implies an origin time
    T - |pos - g| / c0, binned on a grid of step tol / 2; a call is the node and window of width tol (two adjacent bins)
    holding the most unassigned picks, taken while it holds at least min_picks, at most max_calls times.  The exact rule
    is d4w_loc_associate's (include/d4w.h).  Two picks of one channel count separately.  A straight cable cannot tell a
    source from its mirror image: the lower node index wins, so restrict the grid to one side of the cable.

    Returns an Association.  Host picks give ndarrays with labels in the given order; device picks give CUDA tensors
    with labels in CSR order (picks_to_host's order).  ValueError for bad arguments, and when the origin times span more
    bins than fit shared memory (raise tol or shorten the record)."""
    kind, a, b, cable_pos, axes, h, r = _assoc_check(picks, fs, cable_pos, c0, grid, tol, min_picks, max_calls)
    torch = _torch()
    if kind == "device":
        with torch.cuda.device(a.device):
            return _associate_device(a, b, fs, cable_pos, c0, axes, h, r, min_picks, max_calls)
    dev = _device_of(False, None)
    with torch.cuda.device(dev):
        order, offd, sd = _host_csr(a, b, cable_pos.shape[0], dev)
        res = _associate_device(offd, sd, fs, cable_pos, c0, axes, h, r, min_picks, max_calls)
        lab_csr = res.labels.cpu().numpy()
    labels = np.empty_like(lab_csr)
    labels[order] = lab_csr
    return Association(labels, res.node.cpu().numpy(), res.t0.cpu().numpy(), res.count.cpu().numpy())


def localize_calls(picks, fs, cable_pos, c0, grid, tol, min_picks, max_calls=64, Nbiter=10, fix_z=False):
    """associate_picks, then one solve_lq_batch over the calls: call k's observations are its picks in CSR order
    (channel, then pick order within the channel), T = sample / fs at cable_pos[channel], from the first guess
    n0 = (node x, y, z, t0).  fix_z needs nz = 1.  Returns (Association, Localisation), both ndarrays for host picks and
    CUDA tensors for device picks; with no call the Localisation has 0 rows."""
    if fix_z:
        _grid_axes(grid, True)
    kind, a, b, cable_pos, axes, h, r = _assoc_check(picks, fs, cable_pos, c0, grid, tol, min_picks, max_calls)
    torch = _torch()
    dev = a.device if kind == "device" else _device_of(False, None)
    with torch.cuda.device(dev):
        if kind == "device":
            offd, sd = a, b
        else:
            order, offd, sd = _host_csr(a, b, cable_pos.shape[0], dev)
        res = _associate_device(offd, sd, fs, cable_pos, c0, axes, h, r, min_picks, max_calls)
        T, pos, off, n0 = _calls_batch(res, offd, sd, fs, cable_pos, axes, dev)
        K = res.node.numel()
        if K:
            loc_ = solve_lq_batch(T, pos, off, c0, Nbiter=Nbiter, fix_z=fix_z, n0=n0)
        else:
            p = 3 if fix_z else 4
            z = lambda *s: torch.empty(s, dtype=torch.float64, device=dev)     # noqa: E731
            loc_ = Localisation(z(0, 4), z(0), z(0, p), torch.empty(0, dtype=torch.int64, device=dev), z(0, 4))
    if kind == "device":
        return res, loc_
    labels = np.empty(res.labels.numel(), dtype=np.int64)
    labels[order] = res.labels.cpu().numpy()
    assoc = Association(labels, res.node.cpu().numpy(), res.t0.cpu().numpy(), res.count.cpu().numpy())
    return assoc, Localisation(*(t.cpu().numpy() for t in loc_))


def _calls_batch(res, offd, sd, fs, cable_pos, axes, dev):
    """(T, pos, offsets, n0) of solve_lq_batch for the calls of an association, gathered on the device: call k's picks in
    CSR order, its first guess (node, t0)"""
    torch = _torch()
    K = res.node.numel()
    nch = offd.numel() - 1
    ch = torch.repeat_interleave(torch.arange(nch, device=dev), (offd[1:] - offd[:-1]).long())
    lab = res.labels
    keep = torch.nonzero(lab >= 0).flatten()
    rows = keep[torch.argsort(lab[keep], stable=True)]
    # divided by a device tensor: torch multiplies by the reciprocal of a Python scalar, which is not s / fs to the bit
    T = sd[rows].double() / torch.tensor(float(fs), dtype=torch.float64, device=dev)
    pos = _dev(cable_pos, dev)[ch[rows]]
    off = torch.zeros(K + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(res.count, 0)
    nx, ny = len(axes[0]), len(axes[1])
    gx, gy, gz = (_dev(a, dev) for a in axes)
    g = res.node
    n0 = torch.stack([gx[g % nx], gy[(g // nx) % ny], gz[g // (nx * ny)], res.t0], 1)
    return T.contiguous(), pos.contiguous(), off, n0


# ------------------------------------------------------------------------------ reference signatures on the GPU
def _one_call(Ti, cable_pos):
    Ti = np.asarray(Ti, dtype=np.float64)
    cable_pos = np.asarray(cable_pos, dtype=np.float64)
    if Ti.ndim != 1 or cable_pos.shape != (Ti.size, 3):
        raise ValueError(f"Ti must be 1-D and cable_pos [{Ti.size}, 3], got {Ti.shape} and {cable_pos.shape}")
    return Ti, cable_pos, np.array([0, Ti.size], dtype=np.int64)


def solve_lq(Ti, cable_pos, c0, Nbiter=10, fix_z=False):
    """loc.solve_lq on the GPU: Gauss-Newton from [40000, 23000, -60, min(Ti)]; prints the reference's line per
    iteration and returns n = [x, y, z, t0]."""
    Ti, cable_pos, off = _one_call(Ti, cable_pos)
    if Ti.size == 0:
        raise ValueError("Ti is empty")
    _check(Ti, cable_pos, off, c0, Nbiter, fix_z, None, None)
    torch = _torch()
    dev = _device_of(False, Ti)
    with torch.cuda.device(dev):
        o = _solve(_dev(Ti, dev), _dev(cable_pos, dev), _dev(off, dev), 1, c0, int(Nbiter), fix_z, None, traj=True)
        traj = o["traj"][0].cpu().numpy()
        n = o["n"][0].cpu().numpy()
    for j in range(int(Nbiter)):
        v = traj[j]
        print(f'Iteration {j+1}: x = {v[0]:.4f} m, y = {v[1]:.4f}, z = {v[2]:.4f}, ti = {v[3]:.4f}')
    return n


def _cov_unscaled(cable_pos, whale_pos, c0, fix_z):
    cable_pos = np.asarray(cable_pos, dtype=np.float64)
    if cable_pos.ndim != 2 or cable_pos.shape[1] != 3 or cable_pos.shape[0] == 0:
        raise ValueError(f"cable_pos must be [channels, 3], got {cable_pos.shape}")
    w = np.asarray(whale_pos, dtype=np.float64).ravel()
    if w.size not in (3, 4):
        raise ValueError("whale_pos must be [x, y, z] or [x, y, z, t0]")
    n0 = np.r_[w[:3], 0.0][None]
    off = np.array([0, cable_pos.shape[0]], dtype=np.int64)
    _check(np.zeros(cable_pos.shape[0]), cable_pos, off, c0, 0, fix_z, None, None)
    torch = _torch()
    dev = _device_of(False, None)
    with torch.cuda.device(dev):
        # no iteration: the epilogue at n0 gives G^T G, its condition number and the inverse
        o = _solve(_dev(np.zeros(cable_pos.shape[0]), dev), _dev(cable_pos, dev), _dev(off, dev), 1, c0, 0, fix_z,
                   _dev(n0, dev), cinv=True)
        C, cond = o["cinv"][0].cpu().numpy(), float(o["cond"][0])
    if cond > 1 / sys.float_info.epsilon:
        print('Matrix is singular')
    return C


def calc_covariance_matrix(cable_pos, whale_pos, c0, var, fix_z=False):
    """loc.calc_covariance_matrix on the GPU: var * inv(G^T G) at whale_pos, or var * inv(G^T G + 1e-5 I) (printing
    'Matrix is singular') when cond(G^T G) > 1 / eps"""
    return var * _cov_unscaled(cable_pos, whale_pos, c0, fix_z)


def calc_uncertainty_position(cable_pos, whale_pos, c0, var, fix_z=False):
    """loc.calc_uncertainty_position: sqrt(diag(calc_covariance_matrix(...)))"""
    return np.sqrt(np.diag(calc_covariance_matrix(cable_pos, whale_pos, c0, var, fix_z)))
