"""fp64 reference of the loss gradients with respect to the material parameters and gravity, on top of the oracle.

`ParamGradOracle` is `oracle.OracleSim` whose backward substep also accumulates, per particle, dL/dmu, dL/dlam and dL/dmass and, for the scene,
dL/dgravity.  They are computed in NumPy float64 from what the oracle exposes after its own `substep_grad(f)`: the state of frame f, its forward
grid and the adjoint of that grid (the oracle clears both at the start of every backward substep).  With P = 2 mu (F~ - R) F~^T + lam J (J - 1) I,
A = k_stress P + m C, the scatter v_in_i += w_i (m v + A d_i), mass_i += w_i m and grid_op v = v_in / m + dt g:
    gA = sum_i w_i a_i (x) d_i,  a_i = adjoint of v_in_i,  am_i = adjoint of mass_i
    dmu += 2 k_stress gA : ((F~ - R) F~^T)     dlam += k_stress J (J - 1) tr(gA)     dmass += v . sum_i w_i a_i + gA : C + sum_i w_i am_i
    dg += dt * sum over nodes with mass of m_i a_i   (a_i = (adjoint of v_in / m + dt g) / m_i there)
The tests check these against central differences through the oracle's forward and against torch.autograd (tests/test_param_grad.py)."""
import numpy as np

from oracle import oracle as orc


class ParamGradOracle(orc.OracleSim):
    def __init__(self, n_grid, particles, gravity=(0.0, -10.0, 0.0), boundary=None, max_substeps_local=50, precision=64, dt=2e-4, n_substeps=10):
        super().__init__(n_grid, particles, gravity=gravity, boundary=boundary, max_substeps_local=max_substeps_local, precision=precision, dt=dt,
                         n_substeps=n_substeps)
        self.dt = float(dt)
        self.dx = 1.0 / n_grid
        self.inv_dx = float(n_grid)
        self.p_vol = (self.dx * 0.5) ** 2
        self.k_stress = -self.dt * self.p_vol * 4 * self.inv_dx * self.inv_dx   # MPM:343
        self.reset_param_grad()

    def reset_param_grad(self):
        self.pg = dict(mu=np.zeros(self.N), lam=np.zeros(self.N), mass=np.zeros(self.N), gravity=np.zeros(3))

    def reset_grad(self):
        super().reset_grad()
        self.reset_param_grad()

    def get_param_grad(self):
        return {k: v.copy() for k, v in self.pg.items()}

    def substep_grad(self, f, none_action=True):
        super().substep_grad(f, none_action)
        _, m_grid, _ = self.get_grid()
        ga_vin, ga_m, _ = self.get_grid_grad()
        t = param_grad_terms(self.get_frame(f), m_grid, ga_vin, ga_m, self.n_grid, self.dt)
        self.pg['gravity'] += t['gravity']
        p = t['p']
        if len(p) == 0:
            return
        for k in ('mu', 'lam', 'mass'):
            np.add.at(self.pg[k], p, t[k])


def param_grad_terms(fr, m_grid, ga_vin, ga_m, n, dt):
    """the terms of the formula above from a frame `fr` (get_frame's dict), the forward grid's mass and the grid adjoint (of v_in and of the
    mass): `p` the used particles, per used particle `mu`, `lam`, `mass`, and the scene's `gravity` (3,)"""
    dx, inv_dx = 1.0 / n, float(n)
    k_stress = -dt * (dx * 0.5) ** 2 * 4 * inv_dx * inv_dx   # MPM:343
    has = m_grid > 1e-12
    out = dict(gravity=dt * (ga_vin[has] * m_grid[has, None]).sum(0))
    p = out['p'] = np.where(fr['used'] != 0)[0]
    if len(p) == 0:
        return out
    x, v, Cm, F = fr['x'][p], fr['v'][p], fr['C'][p], fr['F'][p]
    base = (x * inv_dx - 0.5).astype(np.int64)   # cast(int) truncates toward zero (MPM:335)
    fx = x * inv_dx - base
    w = np.stack([0.5 * (1.5 - fx) ** 2, 0.75 - (fx - 1.0) ** 2, 0.5 * (fx - 0.5) ** 2], 1)   # [P, 3 (offset), 3 (axis)]
    gA = np.zeros((len(p), 3, 3)); gvp = np.zeros((len(p), 3)); sam = np.zeros(len(p))
    for i in range(3):
        for j in range(3):
            for k in range(3):
                o = np.array([i, j, k])
                wt = w[:, i, 0] * w[:, j, 1] * w[:, k, 2]
                g = ((base[:, 0] + i) * n + base[:, 1] + j) * n + base[:, 2] + k
                a = ga_vin[g]
                d = (o[None] - fx) * dx
                gA += wt[:, None, None] * a[:, :, None] * d[:, None, :]
                gvp += wt[:, None] * a
                sam += wt * ga_m[g]
    Ft = (np.eye(3)[None] + dt * Cm) @ F
    U, s, Vt = np.linalg.svd(Ft)
    R = U @ Vt                                            # the rotation of the polar decomposition (det F~ > 0)
    J = np.linalg.det(Ft)
    gP = k_stress * gA
    MFt = (Ft - R) @ np.transpose(Ft, (0, 2, 1))
    out['mu'] = 2.0 * (gP * MFt).sum((1, 2))
    out['lam'] = J * (J - 1.0) * np.trace(gP, axis1=1, axis2=2)
    out['mass'] = (v * gvp).sum(1) + sam + (gA * Cm).sum((1, 2))
    return out
