"""TEST INFRASTRUCTURE -- float64 NumPy restatement of the reference's localisation (das4whales/loc.py:57-216) for
ragged batches of calls and any first guess, plus the grid score of loc.solve_lq_batch's first guess.

Call b is T[off[b]:off[b + 1]], pos[off[b]:off[b + 1]].  p = 4 unknowns (x, y, z, t0), or 3 with z held (fix_z)."""
import numpy as np

LAMBDA = 1e-5
REF_GUESS = (40000.0, 23000.0, -60.0)


def g_matrix(P, v, c0, fix_z):
    """G of loc.py:92-110 at the estimate v = (x, y, z, ...)"""
    r = np.sqrt((P[:, 0] - v[0]) ** 2 + (P[:, 1] - v[1]) ** 2)
    th = np.arctan2(np.abs(v[2] - P[:, 2]), r)
    ph = np.arctan2(v[1] - P[:, 1], v[0] - P[:, 0])
    cols = [np.cos(th) * np.cos(ph) / c0, np.cos(th) * np.sin(ph) / c0]
    if not fix_z:
        cols.append(np.sin(th) / c0)
    cols.append(np.ones_like(th))
    return np.array(cols).T


def residuals(T, P, v, c0):
    return T - (v[3] + np.sqrt(np.sum((P - v[:3]) ** 2, axis=1)) / c0)


def gauss_newton(T, P, c0, n0, nbiter=10, fix_z=False):
    """loc.solve_lq from the first guess n0; returns (n, trajectory [nbiter, 4])"""
    n = np.array(n0, dtype=np.float64)
    idx = [0, 1, 3] if fix_z else [0, 1, 2, 3]
    traj = []
    for j in range(nbiter):
        G = g_matrix(P, n, c0, fix_z)
        dt = residuals(T, P, n, c0)
        dn = np.linalg.inv(G.T @ G + LAMBDA * np.eye(G.shape[1])) @ G.T @ dt
        n[idx] += (0.7 if j < 4 else 1.0) * dn
        traj.append(n.copy())
    return n, np.array(traj).reshape(nbiter, 4)


def variance(T, P, n, c0, fix_z=False):
    """loc.cal_variance_residuals at n; NaN when there are no more observations than unknowns"""
    p = 3 if fix_z else 4
    return float(np.sum(residuals(T, P, n, c0) ** 2) / (len(T) - p)) if len(T) > p else np.nan


def covariance_unscaled(P, n, c0, fix_z=False):
    """(C, singular): C = inv(G^T G), or inv(G^T G + 1e-5 I) when cond(G^T G) > 1 / eps (loc.py:175-189)"""
    G = g_matrix(P, n, c0, fix_z)
    A = G.T @ G
    singular = bool(np.linalg.cond(A) > 1 / np.finfo(float).eps)
    return np.linalg.inv(A + LAMBDA * np.eye(A.shape[0]) if singular else A), singular


def solve(T, P, c0, n0=None, nbiter=10, fix_z=False):
    """One call: (n, var, unc, n0 used); n0=None is the reference's guess"""
    p = 3 if fix_z else 4
    if len(T) == 0:
        return np.full(4, np.nan), np.nan, np.full(p, np.nan), np.full(4, np.nan)
    n0 = np.r_[REF_GUESS, np.min(T)] if n0 is None else np.asarray(n0, dtype=np.float64)
    n, _ = gauss_newton(T, P, c0, n0, nbiter, fix_z)
    var = variance(T, P, n, c0, fix_z)
    C, _ = covariance_unscaled(P, n, c0, fix_z)
    return n, var, np.sqrt(var * np.diag(C)), n0


def solve_batch(T, pos, off, c0, n0=None, nbiter=10, fix_z=False):
    B = len(off) - 1
    p = 3 if fix_z else 4
    out_n, out_var, out_unc = np.empty((B, 4)), np.empty(B), np.empty((B, p))
    for b in range(B):
        s = slice(off[b], off[b + 1])
        guess = None if n0 is None else (n0 if np.ndim(n0) == 1 else n0[b])
        out_n[b], out_var[b], out_unc[b], _ = solve(T[s], pos[s], c0, guess, nbiter, fix_z)
    return out_n, out_var, out_unc


def grid_nodes(grid):
    (x0, x1, nx), (y0, y1, ny), (z0, z1, nz) = grid
    gx, gy, gz = np.linspace(x0, x1, nx), np.linspace(y0, y1, ny), np.linspace(z0, z1, nz)
    Z, Y, X = np.meshgrid(gz, gy, gx, indexing="ij")          # node index (iz * ny + iy) * nx + ix
    return np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1)


def grid_scores(T, P, c0, nodes, fix_z=False, block=512):
    """(score, t0*) at every node: score = sum (T - t0* - d / c0)^2 / (n - p), t0* = mean(T - d / c0)"""
    p = 3 if fix_z else 4
    score, t0 = np.empty(len(nodes)), np.empty(len(nodes))
    for k in range(0, len(nodes), block):
        R = T[None] - np.sqrt(np.sum((P[None] - nodes[k:k + block, None]) ** 2, axis=-1)) / c0
        m = R.mean(1)
        t0[k:k + block] = m
        score[k:k + block] = np.sum((R - m[:, None]) ** 2, axis=1) / (len(T) - p) if len(T) > p else np.nan
    return score, t0


def bent_cable(nch=3000, length=60000.0):
    """Test geometry: a cable of `length` m whose heading turns from 20 to 90 degrees (a straight cable leaves a mirror
    ambiguity no solver can resolve), descending from 200 to 1200 m."""
    s = np.linspace(0, 1, nch)
    ang = np.deg2rad(20 + 70 * s ** 2)
    xy = np.cumsum(np.stack([np.cos(ang), np.sin(ang)], 1) * (length / nch), 0)
    return np.column_stack([xy, -200 - 1000 * s])


def arrivals(cable, whale, t0, c0, noise, rng):
    return t0 + np.sqrt(np.sum((cable - np.asarray(whale, dtype=np.float64)) ** 2, axis=1)) / c0 + rng.normal(0, noise, len(cable))
