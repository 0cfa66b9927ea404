"""fp64 NumPy reference of the correspondence-free momentum loss (DESIGN.md §4, MomentumMatchingLoss): with density_loss_ref's stencil,
d_ip = (o_i - fx_p) dx, u_ip = v_p + C_p d_ip, the deposit m_i = sum_p m_p w_ip and P_i = sum_p m_p w_ip u_ip (p2g's (momentum, mass) with
zero stress), L = w_d sum_i (m_i - m*_i)^2 + w_s sum_i m_i phi*_i + w_m sum_i |P_i - P*_i|^2, and its adjoints with the stencil base held
fixed: a_i = 2 w_d (m_i - m*_i) + w_s phi*_i, b_i = 2 w_m (P_i - P*_i),
v_p = m_p sum_i w_ip b_i, C_p = m_p sum_i w_ip b_i d_ip^T, x_p = m_p sum_i [grad w_ip (a_i + b_i . u_ip) - w_ip C_p^T b_i],
dL/dm_p = sum_i w_ip (a_i + b_i . u_ip)."""
import numpy as np

import density_loss_ref as dref


def offsets(x, n_grid):
    """d_ip = (o_i - fx_p) dx, (P, 27, 3), in the kernels' node order (zero where the stencil leaves the grid)"""
    x = np.asarray(x, dtype=np.float64).reshape(-1, 3)
    ok, _, _, _ = dref.stencil(x, n_grid)
    g = x * n_grid
    base = np.where(ok[:, None], np.trunc(np.where(np.isfinite(g), g - 0.5, 0.0)), 0.0)
    d = (dref.OFFS[None, :, :] - (g - base)[:, None, :]) / n_grid
    d[~ok] = 0.0
    return d


def _u(x, v, C, n_grid):
    d = offsets(x, n_grid)
    return d, np.asarray(v, np.float64)[:, None, :] + np.einsum('pab,ptb->pta', np.asarray(C, np.float64), d)


def deposit(x, v, C, mass, sel, n_grid):
    """(P (G, 3), m (G,)) that the selected particles deposit"""
    _, nodes, w, _ = dref.stencil(x, n_grid)
    _, u = _u(x, v, C, n_grid)
    mp = np.broadcast_to(np.asarray(mass, dtype=np.float64), (len(nodes),))
    mw = mp[:, None] * w
    m = np.zeros(n_grid ** 3)
    pm = np.zeros((n_grid ** 3, 3))
    np.add.at(m, nodes[sel].reshape(-1), mw[sel].reshape(-1))
    np.add.at(pm, nodes[sel].reshape(-1), (mw[:, :, None] * u)[sel].reshape(-1, 3))
    return pm, m


def _vol(a, shape):
    return np.zeros(shape) if a is None else np.asarray(a, dtype=np.float64).reshape(shape)


def loss(pm, m, target_m, target_p, sdf, wd, ws, wm):
    t, tp, phi = _vol(target_m, m.shape), _vol(target_p, pm.shape), _vol(sdf, m.shape)
    return float(wd * ((m - t) ** 2).sum() + ws * (m * phi).sum() + wm * ((pm - tp) ** 2).sum())


def adjoint(x, v, C, mass, sel, n_grid, target_m, target_p, sdf, wd, ws, wm):
    """(L, x adjoint (P, 3), v adjoint (P, 3), C adjoint (P, 3, 3), dL/dm_p (P,)) of one frame"""
    pm, m = deposit(x, v, C, mass, sel, n_grid)
    t, tp, phi = _vol(target_m, m.shape), _vol(target_p, pm.shape), _vol(sdf, m.shape)
    a = 2.0 * wd * (m - t) + ws * phi
    b = 2.0 * wm * (pm - tp)
    _, nodes, w, dw = dref.stencil(x, n_grid)
    d, u = _u(x, v, C, n_grid)
    mp = np.broadcast_to(np.asarray(mass, dtype=np.float64), (len(nodes),))
    an, bn = a[nodes], b[nodes]                                   # (P, 27), (P, 27, 3)
    s = an + (bn * u).sum(-1)
    bw = w[:, :, None] * bn                                       # w_ip b_i
    gv = mp[:, None] * bw.sum(1)
    gC = mp[:, None, None] * np.einsum('pta,ptb->pab', bw, d)
    gx = mp[:, None] * ((s[:, :, None] * dw).sum(1) - np.einsum('pab,pa->pb', np.asarray(C, np.float64), bw.sum(1)))
    dm = (w * s).sum(1)
    z = ~np.asarray(sel, bool)
    gx[z] = 0.0; gv[z] = 0.0; gC[z] = 0.0; dm = np.where(z, 0.0, dm)
    return loss(pm, m, target_m, target_p, sdf, wd, ws, wm), gx, gv, gC, dm
