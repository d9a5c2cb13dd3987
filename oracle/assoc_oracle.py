"""TEST INFRASTRUCTURE -- float64 NumPy restatement of the pick association of loc.associate_picks (d4w_loc_associate).

Picks are (channel c_p, sample s_p).  T_p = s_p / fs; tau(g, c) = sqrt(dx*dx + dy*dy + dz*dz) / c0 with
dx = cable_pos[c, 0] - g_x, evaluated left to right with every operation rounded on its own (NumPy does not fuse);
o(g, p) = T_p - tau(g, c_p); h = tol / 2, r = 1 / h; bin j(g, p) = floor(o(g, p) * r).  n(g, j) counts the unassigned picks
with j(g, p) = j and (g, j) scores n(g, j) + n(g, j + 1).  Repeatedly: the (g, j) of highest score (ties to the lowest node
index, then the lowest j); stop when the score is below min_picks or after max_calls calls; else call k gets node g,
t0 = (j + 1) * h and the unassigned picks with j(g, p) in {j, j + 1}."""
import numpy as np


def grid_nodes(grid):
    (x0, x1, nx), (y0, y1, ny), (z0, z1, nz) = grid
    gx, gy, gz = np.linspace(x0, x1, int(nx)), np.linspace(y0, y1, int(ny)), np.linspace(z0, z1, int(nz))
    Z, Y, X = np.meshgrid(gz, gy, gx, indexing="ij")          # node index (iz * ny + iy) * nx + ix
    return np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1)


def bins(ch, s, fs, cable_pos, c0, nodes, tol):
    """j(g, p) for every node and pick: int64 [n_nodes, n_picks]"""
    h = tol / 2.0
    r = 1.0 / h
    T = np.asarray(s, dtype=np.int64).astype(np.float64) / fs
    q = np.asarray(cable_pos, dtype=np.float64)[np.asarray(ch, dtype=np.int64)]
    dx = q[None, :, 0] - nodes[:, None, 0]
    dy = q[None, :, 1] - nodes[:, None, 1]
    dz = q[None, :, 2] - nodes[:, None, 2]
    tau = np.sqrt(dx * dx + dy * dy + dz * dz) / c0
    return np.floor((T[None, :] - tau) * r).astype(np.int64)


def associate(ch, s, fs, cable_pos, c0, grid, tol, min_picks, max_calls=64):
    """(labels [n_picks], node [K], t0 [K], count [K]) in the given pick order"""
    nodes = grid_nodes(grid)
    J = bins(ch, s, fs, cable_pos, c0, nodes, tol)
    h = tol / 2.0
    n = J.shape[1]
    labels = np.full(n, -1, dtype=np.int64)
    node, t0, count = [], [], []
    if n == 0:
        return labels, np.zeros(0, np.int64), np.zeros(0), np.zeros(0, np.int64)
    jlo = int(J.min()) - 1                                       # the window (jmin - 1, jmin) holds bin jmin alone
    nb = int(J.max()) - jlo + 2                                  # one more: the partner of the last bin is 0
    while len(node) < max_calls:
        free = labels < 0
        best = (-1, 0, 0)
        for g in range(len(nodes)):                              # ascending node, then ascending j: ties keep the first
            cnt = np.bincount(J[g, free] - jlo, minlength=nb)
            score = cnt[:-1] + cnt[1:]
            j = int(np.argmax(score))
            if score[j] > best[0]:
                best = (int(score[j]), g, j + jlo)
        sc, g, j = best
        if sc < min_picks:
            break
        sel = free & ((J[g] == j) | (J[g] == j + 1))
        k = len(node)
        labels[sel] = k
        node.append(g)
        t0.append((j + 1) * h)
        count.append(int(sel.sum()))
    return labels, np.array(node, np.int64), np.array(t0, np.float64), np.array(count, np.int64)


def straight_cable(nch, dx):
    """channel c at (c dx, 0, 0)"""
    return np.column_stack([np.arange(nch) * dx, np.zeros(nch), np.zeros(nch)])


def synth_picks(cable_pos, sources, fs, c0, rng, every=1, false_frac=0.0, t_max=None):
    """Noise-free picks of calls from `sources` = [((x, y, z), t0), ...]: sample round((t0 + d / c0) fs) on every `every`-th
    channel, plus false picks (a fraction of the true count) at uniform channels and samples.  Returns (ch, s, truth) with
    truth[p] = the call of pick p or -1, in channel-major order."""
    ch, s, truth = [], [], []
    for k, (w, t0) in enumerate(sources):
        c = np.arange(0, len(cable_pos), every)
        d = np.sqrt(np.sum((cable_pos[c] - np.asarray(w, np.float64)) ** 2, axis=1))
        ch.append(c)
        s.append(np.round((t0 + d / c0) * fs).astype(np.int64))
        truth.append(np.full(len(c), k))
    n = sum(len(c) for c in ch)
    nf = int(round(false_frac * n))
    if nf:
        hi = max(int(np.concatenate(s).max()), 1) if t_max is None else int(t_max * fs)
        ch.append(rng.integers(0, len(cable_pos), nf))
        s.append(rng.integers(0, hi + 1, nf))
        truth.append(np.full(nf, -1))
    ch, s, truth = np.concatenate(ch), np.concatenate(s), np.concatenate(truth)
    o = np.lexsort((s, ch))
    return ch[o], s[o], truth[o]
