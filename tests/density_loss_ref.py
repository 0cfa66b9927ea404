"""fp64 NumPy reference of the correspondence-free density loss (DESIGN.md §4, DensityMatchingLoss): the deposit m_i = sum_p m_p w_ip with
p2g's stencil (base = int(x / dx - 0.5) by truncation, quadratic B-spline, particles whose 3x3x3 stencil leaves the grid deposit nothing),
L = w_d sum_i (m_i - m*_i)^2 + w_s sum_i m_i phi*_i, and its adjoints with the stencil base held fixed:
x_p = m_p sum_i gbar_i grad w_ip and dL/dm_p = sum_i gbar_i w_ip, gbar_i = 2 w_d (m_i - m*_i) + w_s phi*_i."""
import numpy as np

OFFS = np.array([(i, j, k) for i in range(3) for j in range(3) for k in range(3)])   # node t = 9 i + 3 j + k, as the kernels number them


def stencil(x, n_grid):
    """ok (P,), node ids (P, 27), weights (P, 27) and their x-gradients (P, 27, 3) (zero rows where not ok)"""
    x = np.asarray(x, dtype=np.float64).reshape(-1, 3)
    g = x * n_grid
    t = g - 0.5
    ok = ((t > -1.0) & (t < n_grid - 2)).all(axis=1)
    base = np.where(ok[:, None], np.trunc(np.where(np.isfinite(t), t, 0.0)), 0.0).astype(np.int64)
    fx = g - base
    w1 = np.stack([0.5 * (1.5 - fx) ** 2, 0.75 - (fx - 1.0) ** 2, 0.5 * (fx - 0.5) ** 2], axis=1)     # (P, offset, axis)
    d1 = np.stack([-(1.5 - fx), -2.0 * (fx - 1.0), fx - 0.5], axis=1) * n_grid                        # d w1 / d x
    wa, wb, wc = w1[:, OFFS[:, 0], 0], w1[:, OFFS[:, 1], 1], w1[:, OFFS[:, 2], 2]
    da, db, dc = d1[:, OFFS[:, 0], 0], d1[:, OFFS[:, 1], 1], d1[:, OFFS[:, 2], 2]
    w = wa * wb * wc
    dw = np.stack([da * wb * wc, wa * db * wc, wa * wb * dc], axis=-1)
    nodes = ((base[:, None, 0] + OFFS[None, :, 0]) * n_grid + base[:, None, 1] + OFFS[None, :, 1]) * n_grid + base[:, None, 2] + OFFS[None, :, 2]
    w[~ok] = 0.0; dw[~ok] = 0.0; nodes[~ok] = 0
    return ok, nodes, w, dw


def selection(x, used, mat, matching_mat, n_grid):
    """the particles that deposit: used, of the matched material, stencil inside the grid"""
    ok, _, _, _ = stencil(x, n_grid)
    return ok & (np.asarray(used) != 0) & np.isin(np.asarray(mat), np.atleast_1d(matching_mat))


def deposit(x, mass, sel, n_grid):
    _, nodes, w, _ = stencil(x, n_grid)
    m = np.zeros(n_grid ** 3)
    mp = np.broadcast_to(np.asarray(mass, dtype=np.float64), (len(nodes),))
    np.add.at(m, nodes[sel].reshape(-1), (mp[sel, None] * w[sel]).reshape(-1))
    return m


def _vol(v, G):
    return np.zeros(G) if v is None else np.asarray(v, dtype=np.float64).reshape(G)


def loss(m, target, sdf, wd, ws):
    t, phi = _vol(target, len(m)), _vol(sdf, len(m))
    return float(wd * ((m - t) ** 2).sum() + ws * (m * phi).sum())


def adjoint(x, mass, sel, n_grid, target, sdf, wd, ws):
    """(L, x adjoint (P, 3), dL/dm_p (P,)) of one frame"""
    m = deposit(x, mass, sel, n_grid)
    t, phi = _vol(target, len(m)), _vol(sdf, len(m))
    gbar = 2.0 * wd * (m - t) + ws * phi
    _, nodes, w, dw = stencil(x, n_grid)
    mp = np.broadcast_to(np.asarray(mass, dtype=np.float64), (len(nodes),))
    gb = gbar[nodes]
    gx = np.where(sel[:, None], mp[:, None] * (gb[:, :, None] * dw).sum(1), 0.0)
    dm = np.where(sel, (gb * w).sum(1), 0.0)
    return loss(m, target, sdf, wd, ws), gx, dm
