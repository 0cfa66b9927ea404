"""Shared body of tests/test_smoke_layouts.py: the smoke solver's kernels (fluidlab_b200/csrc/fsmk_smoke.cu) ONE launch at a time against the
fp64 oracle (oracle/smoke_oracle.hpp), on grid / band / obstacle layouts that force each boundary branch.  Each launch is compared with the
oracle phase started from the kernel's OWN inputs (set_free / set_state / set_grad), so errors do not compound along the chain:

    fsmk_free_space        is_free[s]                                   equal to fp64 except cells with |sdf| < AMB_SDF (fp32 oracle there)
    fsmk_advect            v_tmp[s], every plane of q[s+1]              per cell and component, C['advect'] 2^-23 S_i
                           v[s+1], v_tmp[s] of non-free cells           exactly 0;  q[s+1] = q[s] there, bit for bit
    fsmk_divergence        div[s] on free cells                         C['div'] 2^-23 S_i
    fsmk_pressure          p[s+1] on free cells                         bit-identical to the fp32 oracle's sweeps; C['jacobi'] 2^-23 S_i
    fsmk_project           v[s+1] on free cells                         C['project'] 2^-23 S_i
    fsmk_project_grad      gv_tmp[s] (free cells), gp[s+1]              C['project_grad'] 2^-23 S_i
    fsmk_pressure_grad     gp[s], gdiv[s]                               C['jacobi_grad'] 2^-23 S_i
    fsmk_divergence_grad   gv_tmp[s]                                    C['div_grad'] 2^-23 S_i
    fsmk_advect_grad       gv[s], every plane of gq[s]                  C['advect_grad'] 2^-23 S_i; cells no lookup reaches keep their adjoint
                           the 9 air-conditioner adjoints of substep f  C['air'] 2^-23 sum |per-cell term|

S_i is a first-order error scale in fp64: for the linear phases the same expression on absolute values (for the Jacobi chains, the abs-value
recursion summed over the sweeps); for advection the trilerp's sum w|f| / W plus |d out / d p| times a bound on the fp32 error of the backtrace
points (`backtrace`), and for its adjoint the abs-value replay of the gather-scatter chain with the same point terms.

One documented difference: the oracle's subtract_gradient_grad adds gv[s+1] into gv_tmp[s] of non-free cells too, k_project_grad does not (v_tmp
of a non-free cell is the constant 0, so that adjoint is a dead end).  gv_tmp[s] is compared on free cells, and the kernel must leave the non-free
ones as they were.

Before each launch every output range the launch must not touch holds a sentinel (other ring frames, non-free cells of p[s+1] / div[s], the
adjoints of other substeps); after it, every buffer outside the launch's write set must come back bit-identical.  Inputs a kernel may read through
loc() hold real data.

Ambiguous cells: a cell whose fp64 sdf is within AMB_SDF of 0 (the mask may flip), and a free cell whose fp64 backtrace point p1, p2 or pe lies
within twice its fp32 error bound of a cell plane (floorf and sign(t) may flip) are compared with the fp32 oracle instead, and so are the adjoint cells
their lookups reach.  They must stay rarer than AMB_FRAC of the free cells."""
import ctypes as C
import itertools
import time

import numpy as np

U = 2.0 ** -23
DT = 0.5
SEED = 3
T_SUB = 10
F_CORNER, F_BAND = 3, 7          # substeps whose air conditioner sits near a grid corner / inside the band
AMB_SDF = 1e-5
AMB_FRAC = 0.005
JT_OUT, JT_HALO, JT_HMAX = 16, 8, 8
SENT = np.float32(1234.5)
SENT_U8 = 0xA5
# Bars in units of 2^-23 S_i, each 4-6x the largest ratio measured over every layout on an H100 (80 GB HBM3, 700 W power limit) and on the CPU
# shim with and without FMA contraction (measured: advect 0.72, div 1.39, jacobi 0.23, project 0.96, project_grad 1.15, jacobi_grad 0.44, div_grad
# 0.98, advect_grad 0.93, air 0.081).  The Jacobi scales sum the abs recursion over every sweep, so their ratios fall with the sweep count.
C_BAR = dict(advect=4.0, div=6.0, jacobi=1.0, project=4.0, project_grad=5.0, jacobi_grad=2.0, div_grad=4.0, advect_grad=4.0, air=0.4)

# res, (lower_y, higher_y), q_dim, solver_iters, statics: (centre, radius) spheres in world units, SDF volume resolution
LAYOUTS = {
    'interior': dict(res=20, band=(6, 12), qd=3, iters=13, vres=24,
                     statics=[((0.0, 0.45, 0.5), 0.15), ((0.5, 0.5, 1.0), 0.15), ((0.6, 0.45, 0.3), 0.12), ((0.25, 0.55, 0.75), 0.1)]),
    'floor': dict(res=24, band=(-1, 6), qd=2, iters=9, vres=24, statics=[((0.0, 0.1, 0.3), 0.15), ((0.7, 0.0, 1.0), 0.2), ((0.5, 0.15, 0.5), 0.08)]),
    'ceiling': dict(res=24, band=(17, 24), qd=4, iters=8, vres=24,
                    statics=[((0.0, 0.9, 0.6), 0.15), ((0.4, 1.0, 1.0), 0.2), ((0.6, 0.85, 0.4), 0.1), ((0.2, 0.95, 0.2), 0.08)]),
    'thin': dict(res=33, band=(10, 12), qd=3, iters=17, vres=24, statics=[((0.0, 0.35, 0.4), 0.15), ((0.5, 0.35, 1.0), 0.15)]),
    'tall8': dict(res=16, band=(3, 12), qd=3, iters=16, vres=24, statics=[((0.0, 0.5, 0.5), 0.2), ((0.6, 0.4, 1.0), 0.2), ((0.5, 0.6, 0.4), 0.12)]),
    'tall9': dict(res=16, band=(3, 13), qd=1, iters=5, vres=24, statics=[((0.0, 0.5, 0.5), 0.2), ((0.6, 0.4, 1.0), 0.2), ((0.5, 0.6, 0.4), 0.12)]),
    'whole': dict(res=12, band=(-3, 15), qd=2, iters=3, vres=24,
                  statics=[((0.0, 0.5, 0.5), 0.25), ((0.5, 0.5, 1.0), 0.25), ((0.5, 0.0, 0.3), 0.2), ((0.6, 1.0, 0.6), 0.2)]),
    'empty': dict(res=16, band=(9, 10), qd=3, iters=4, vres=24, statics=[((0.5, 0.5, 0.5), 0.2)]),
    'reference': dict(res=128, band=(60, 68), qd=3, iters=500, vres=48,
                      statics=[((0.0, 0.5, 0.5), 0.1), ((0.5, 0.5, 1.0), 0.1), ((0.5, 0.5, 0.5), 0.05), ((0.3, 0.5, 0.7), 0.03)]),
}
SHIM_LAYOUTS = [k for k in LAYOUTS if k != 'reference']
# what each layout exists for: census counts it must reach (about half the seed's counts)
MIN = {
    'interior': dict(free=600, blocked_band=100, nb_blocked_ym=200, nb_blocked_yp=200, nb_blocked_xm=10, nb_blocked_zp=10, nb_out_xm=20, tri_out_blocked=20,
                     tri_out_free=20, tri_blocked=200, out_of_grid=10, zero_v=5, tiles_last_width=4, launches=2),
    'floor': dict(free=1500, nb_out_ym=200, nb_blocked_yp=200, nb_blocked_zp=5, tri_out_blocked=50, tri_out_free=50, out_of_grid=30, zero_v=5),
    'ceiling': dict(free=1500, nb_out_yp=200, nb_blocked_ym=200, nb_blocked_xm=5, tri_out_blocked=50, tri_out_free=50, out_of_grid=30, zero_v=5),
    'thin': dict(free=500, nb_blocked_ym=500, nb_blocked_yp=500, nb_out_xm=10, tri_out_blocked=20, out_of_grid=10, zero_v=2),
    'tall8': dict(free=800, nb_blocked_xm=10, nb_blocked_zp=10, tri_out_blocked=20, tri_out_free=20, out_of_grid=10, zero_v=5, launches=2),
    'tall9': dict(free=900, nb_blocked_xm=10, nb_blocked_zp=10, tri_out_blocked=20, tri_out_free=20, out_of_grid=10, zero_v=5, launches=5),
    'whole': dict(free=500, nb_out_ym=30, nb_out_yp=30, nb_blocked_xm=5, tri_out_blocked=20, tri_out_free=20, out_of_grid=20, zero_v=5, launches=3),
    'empty': dict(),
    'reference': dict(free=80000, nb_blocked_ym=5000, nb_blocked_yp=5000, nb_blocked_xm=5, nb_blocked_zp=5, tri_out_blocked=50, tri_out_free=50,
                      out_of_grid=50, zero_v=20, launches=63, last_sweeps=4),
}
# the shape of each layout: band height, q planes, the Jacobi plan (asserted exactly)
SHAPE = {
    'interior': dict(H=5, qd=3, tiled=True, launches=2, last_sweeps=5, tiles=2, tiles_last_width=4, j0=7, j1=11),
    'floor': dict(H=6, qd=2, tiled=True, launches=2, last_sweeps=1, tiles=2, tiles_last_width=8, j0=0, j1=5),
    'ceiling': dict(H=6, qd=4, tiled=True, launches=1, last_sweeps=8, tiles=2, tiles_last_width=8, j0=18, j1=23),
    'thin': dict(H=1, qd=3, tiled=True, launches=3, last_sweeps=1, tiles=3, tiles_last_width=1, j0=11, j1=11),
    'tall8': dict(H=8, qd=3, tiled=True, launches=2, last_sweeps=8, tiles=1, tiles_last_width=16, j0=4, j1=11),
    'tall9': dict(H=9, qd=1, tiled=False, launches=5, last_sweeps=1, j0=4, j1=12),
    'whole': dict(H=12, qd=2, tiled=False, launches=3, last_sweeps=1, j0=0, j1=11),
    'empty': dict(H=0, qd=3),
    'reference': dict(H=7, qd=3, tiled=True, launches=63, last_sweeps=4, tiles=8, tiles_last_width=16, j0=61, j1=67),
}
DIRS = [(d, sg) for d in range(3) for sg in (-1, 1)]
SIDE = {(0, -1): 'xm', (0, 1): 'xp', (1, -1): 'ym', (1, 1): 'yp', (2, -1): 'zm', (2, 1): 'zp'}
CORNERS = np.array([[m >> 2, (m >> 1) & 1, m & 1] for m in range(8)])


# ------------------------------------------------------------------------------------------------------------------ layouts and state
def band_rows(cfg):
    n, (lo, hi) = cfg['res'], cfg['band']
    j0, j1 = max(lo + 1, 0), min(hi - 1, n - 1)
    return j0, j1, max(j1 - j0 + 1, 0)


def jacobi_plan(cfg):
    _, _, H = band_rows(cfg)
    tiled = H <= JT_HMAX
    per = JT_HALO if tiled else 1
    it = cfg['iters']
    launches = 1 if it == 0 else (it + per - 1) // per
    n = cfg['res']
    tiles = (n + JT_OUT - 1) // JT_OUT
    return dict(tiled=tiled, launches=launches, last_sweeps=it - per * (launches - 1), tiles=tiles, tiles_last_width=n - JT_OUT * (tiles - 1))


def sphere_static(centre, radius, vres):
    """an SDF volume of a sphere on vres^3 voxels spanning world [-0.1, 1.1]^3, and its T_mesh_to_voxels (world -> voxel coordinates)"""
    sc = (vres - 1) / 1.2
    ax = np.arange(vres) / sc - 0.1
    X, Y, Z = np.meshgrid(ax, ax, ax, indexing='ij')
    vox = (np.sqrt((X - centre[0]) ** 2 + (Y - centre[1]) ** 2 + (Z - centre[2]) ** 2) - radius).astype(np.float32)
    T = np.array([[sc, 0, 0, 0.1 * sc], [0, sc, 0, 0.1 * sc], [0, 0, sc, 0.1 * sc], [0, 0, 0, 1]], np.float32).astype(np.float64)
    return vox, T


def sdf64(vox, T, pw):
    """sdf_lookup in fp64 at world points pw (N, 3): trilinear, 1 outside the volume"""
    R = vox.shape[0]
    pv = pw @ np.asarray(T, np.float64)[:3, :3].T + np.asarray(T, np.float64)[:3, 3]
    b = np.floor(pv).astype(np.int64)
    ok = ((b >= 0) & (b < R - 1)).all(1)
    bb = np.clip(b, 0, R - 2)
    sd = np.zeros(len(pw))
    for o in CORNERS:
        t = pv - (bb + o)
        w = np.prod(1.0 - np.abs(t), 1)
        sd += w * vox[bb[:, 0] + o[0], bb[:, 1] + o[1], bb[:, 2] + o[2]].astype(np.float64)
    return np.where(ok, sd, 1.0)


def q_rot(q, v):
    q, v = np.asarray(q, np.float64), np.asarray(v, np.float64)
    uv = np.array([q[2] * v[2] - q[3] * v[1], q[3] * v[0] - q[1] * v[2], q[1] * v[1] - q[2] * v[0]])
    uu = np.array([q[2] * uv[2] - q[3] * uv[1], q[3] * uv[0] - q[1] * uv[2], q[1] * uv[1] - q[2] * uv[0]])
    return v + 2 * (q[0] * uv + uu)


def make_layout(name, seed=SEED):
    """the configuration and the fp32 state of one layout"""
    cfg = dict(LAYOUTS[name], name=name)
    rng = np.random.RandomState(seed + 17 * list(LAYOUTS).index(name))
    n, qd = cfg['res'], cfg['qd']
    G = n ** 3
    j0, j1, H = band_rows(cfg)
    cfg.update(S=2, s=1, n=n, G=G, j0=j0, j1=j1, H=H, inject_v=(-0.3, 0.2, 1.0))
    cfg['static_vols'] = [sphere_static(c, r, cfg['vres']) for c, r in cfg['statics']]
    # velocity: |v| dt up to ~3 cells, exactly zero in a box inside the band
    v = (rng.uniform(-1, 1, (G, 3)) * (6.0 / np.sqrt(3)) * rng.uniform(0, 1, (G, 1))).astype(np.float32)
    I = np.stack(np.unravel_index(np.arange(G), (n,) * 3), 1)
    zb = (np.abs(I[:, 0] - n // 2) <= max(n // 10, 1)) & (I[:, 2] >= 1) & (I[:, 2] <= max(n // 6, 2))
    v[zb] = 0
    cfg['zero_box'] = zb
    q = rng.uniform(0, 1, (qd, G)).astype(np.float32)
    p = rng.uniform(-1, 1, G).astype(np.float32)
    air = np.zeros((T_SUB + 1, 9))
    air[:, 3] = 1
    ymid = (j0 + j1 + 1) / 2 / n if H else 0.5
    for f, pos, s_, r in ((F_CORNER, (0.01, 0.01, 0.99), 2.5, n / 3), (F_BAND, (0.4, ymid, 0.6), 3.0, 2.0)):
        qt = rng.randn(4); qt /= np.linalg.norm(qt)
        air[f] = [*pos, *qt, s_, r]
    cfg['air'] = air
    return cfg, dict(v=v, q=q, p=p)


def mask64(cfg):
    """the free-space mask in fp64 (Static.is_collide on every statics), and the cells whose |sdf| is within AMB_SDF of 0"""
    n, G = cfg['n'], cfg['G']
    I = np.stack(np.unravel_index(np.arange(G), (n,) * 3), 1)
    band = (I[:, 1] > cfg['band'][0]) & (I[:, 1] < cfg['band'][1])
    pw = (I + 0.5) * (1.0 / n)
    free, amb = band.copy(), np.zeros(G, bool)
    for vox, T in cfg['static_vols']:
        sd = sdf64(vox, T, pw)
        free &= ~(sd <= 0)
        amb |= band & (np.abs(sd) < AMB_SDF)
    return free, amb, band


# ------------------------------------------------------------------------------------------------------------------ fp64 host replay
def neighbours(free, n):
    """per direction (axis, sign): in-grid flag, free_at flag, and loc() index of every cell (the neighbour when free, else the centre)"""
    G = n ** 3
    I = np.stack(np.unravel_index(np.arange(G), (n,) * 3), 1)
    out = {}
    for d, sg in DIRS:
        J = I.copy(); J[:, d] += sg
        ing = (J[:, d] >= 0) & (J[:, d] < n)
        nb = np.ravel_multi_index(tuple(np.clip(J, 0, n - 1).T), (n,) * 3)
        fa = ing & free[nb]
        out[(d, sg)] = dict(ingrid=ing, free=fa, loc=np.where(fa, nb, np.arange(G)), nb=nb)
    return out


class Tri:
    """the trilinear lookup of SF:325-347 at N points (cell units): clamped corner indices, weights, and d w / d p"""

    def __init__(self, pts, free, n):
        pI = pts - 0.5
        base = np.floor(pI).astype(np.int64)
        g = base[:, None, :] + CORNERS[None]
        t = pI[:, None, :] - g
        wx = 1.0 - np.abs(t)
        sg = np.sign(t)
        self.w = np.prod(wx, 2)
        self.dwdp = np.stack([-sg[..., 0] * wx[..., 1] * wx[..., 2], -wx[..., 0] * sg[..., 1] * wx[..., 2], -wx[..., 0] * wx[..., 1] * sg[..., 2]], 2)
        gc = np.clip(g, 0, n - 1)
        self.idx = (gc[..., 0] * n + gc[..., 1]) * n + gc[..., 2]
        self.out = (g != gc).any(2)
        self.blocked = ~free[self.idx]
        self.W = self.w.sum(1)
        self.base = base
        self.pI = pI

    def look(self, F):
        """F (G, C): value, sum w|f| / W, and sum_d |d value / d p_d| (N, C)"""
        fm = F[self.idx]
        val = (self.w[..., None] * fm).sum(1) / self.W[:, None]
        absv = (self.w[..., None] * np.abs(fm)).sum(1) / self.W[:, None]
        lip = np.einsum('nmc,nmd->nc', np.abs(fm - val[:, None, :]), np.abs(self.dwdp)) / self.W[:, None]
        return val, absv, lip

    def adj(self, F, val, go, go_abs, ep):
        """adjoint of one lookup with output adjoint go (N, C): the point adjoint, its abs scale, and the abs scale of each corner's scatter
        (N, 8, C); ep = the point's fp32 error bound in units of 2^-23"""
        fm = F[self.idx]
        diff = fm - val[:, None, :]
        W = self.W[:, None]
        gw = np.einsum('nc,nmc->nm', go, diff) / W
        gp = np.einsum('nm,nmd->nd', gw, self.dwdp)
        _, _, lip = self.look(F)
        Dw = np.abs(self.dwdp).sum((1, 2))
        gw_abs = (np.einsum('nc,nmc->nm', go_abs, np.abs(fm) + np.abs(val)[:, None, :]) / W
                  + ep[:, None] * np.einsum('nc,nmc->nm', np.abs(go), lip[:, None, :] + np.abs(diff) * (Dw / self.W)[:, None, None]) / W)
        gp_abs = np.einsum('nm,nmd->nd', gw_abs, np.abs(self.dwdp))
        contrib = (go_abs[:, None, :] * self.w[..., None] + ep[:, None, None] * np.abs(go)[:, None, :] * np.abs(self.dwdp).sum(2)[..., None]) / W[..., None]
        return gp, gp_abs, contrib

    def near_plane(self, tol):
        """a coordinate within tol (N,) of a cell plane, but not on it"""
        d = np.abs(self.pI - np.round(self.pI))
        return ((d > 0) & (d <= tol[:, None])).any(1)


def impulse(cfg, f, cells):
    a = cfg['air'][f]
    n = cfg['n']
    I = np.stack(np.unravel_index(cells, (n,) * 3), 1).astype(np.float64)
    dirv = q_rot(a[3:7], cfg['inject_v'])
    d = I - np.asarray(a[0:3]) / (1.0 / n)
    dist = np.sqrt((d * d).sum(1) + 1e-12)
    factor = np.exp(-dist / a[8])
    return dirv, d, dist, factor, a[7], a[8]


def backtrace(cfg, free, v, cells):
    """RK3 backtrace (SF:349-360) of the free cells in fp64 with the fp32 error bound of each point (units of 2^-23, first order: rounding of
    the point update plus |d v / d p| times the error of the previous point)"""
    n, dt = cfg['n'], DT
    I = np.stack(np.unravel_index(cells, (n,) * 3), 1).astype(np.float64)
    p0 = I + 0.5
    t0 = Tri(p0, free, n); v1, a1, _ = t0.look(v)
    p1 = p0 - 0.5 * dt * v1
    e1 = np.abs(p1).max(1) + 0.5 * dt * 10 * a1.max(1) + 2
    t1 = Tri(p1, free, n); v2, a2, l2 = t1.look(v)
    ev2 = 10 * a2.max(1) + l2.max(1) * e1
    p2 = p0 - 0.75 * dt * v2
    e2 = np.abs(p2).max(1) + 0.75 * dt * ev2 + 2
    t2 = Tri(p2, free, n); v3, a3, l3 = t2.look(v)
    ev3 = 10 * a3.max(1) + l3.max(1) * e2
    pe = p0 - dt * (2.0 / 9.0 * v1 + 1.0 / 3.0 * v2 + 4.0 / 9.0 * v3)
    ee = np.abs(pe).max(1) + dt * (2.0 / 9.0 * 10 * a1.max(1) + 1.0 / 3.0 * ev2 + 4.0 / 9.0 * ev3) + 4
    te = Tri(pe, free, n)
    amb = t1.near_plane(2 * e1 * U) | t2.near_plane(2 * e2 * U) | te.near_plane(2 * ee * U)
    return dict(tris=(t0, t1, t2, te), pts=(p0, p1, p2, pe), vs=(v1, v2, v3), eps=(np.zeros(len(cells)), e1, e2, ee), amb=amb)


def census(cfg, free, v):
    """the branch counts of one layout from the fp64 replay on the mask `free`"""
    n = cfg['n']
    _, _, band = mask64(cfg)
    c = dict(free=int(free.sum()), blocked_band=int((band & ~free).sum()))
    c.update(jacobi_plan(cfg), H=cfg['H'], qd=cfg['qd'], j0=cfg['j0'], j1=cfg['j1'])
    nbs = neighbours(free, n)
    for (d, sg), nb in nbs.items():
        c['nb_out_' + SIDE[(d, sg)]] = int((free & ~nb['ingrid']).sum())
        c['nb_blocked_' + SIDE[(d, sg)]] = int((free & nb['ingrid'] & ~nb['free']).sum())
    cells = np.nonzero(free)[0]
    c.update(tri_out_blocked=0, tri_out_free=0, tri_blocked=0, out_of_grid=0, zero_v=0, amb_points=0)
    bt = None
    if len(cells):
        bt = backtrace(cfg, free, v, cells)
        for t in bt['tris'][1:]:
            live = t.w > 0
            c['tri_out_blocked'] += int((live & t.out & t.blocked).sum())
            c['tri_out_free'] += int((live & t.out & ~t.blocked).sum())
            c['tri_blocked'] += int((live & ~t.out & t.blocked).sum())
        c['out_of_grid'] = int(((bt['pts'][3] < 0) | (bt['pts'][3] > n)).any(1).sum())
        c['zero_v'] = int((np.abs(bt['vs'][0]).max(1) == 0).sum())
        c['amb_points'] = int(bt['amb'].sum())
    return c, bt


def check_census(name, c):
    for k, v in SHAPE[name].items():
        assert c[k] == v, f'layout {name}: {k} = {c[k]}, the layout exists for {v}'
    for k, v in MIN[name].items():
        assert c[k] >= v, f'layout {name} drifted off its branch: {k} = {c[k]} < {v} ({c})'
    assert c['amb_points'] <= AMB_FRAC * max(c['free'], 1), f'layout {name}: {c["amb_points"]} ambiguous backtraces of {c["free"]} free cells'


# ------------------------------------------------------------------------------------------------------------------ the device side
class Dev:
    """the C ABI of include/fluidsmoke.h on torch tensors of `device` (CPU tensors on the shim)"""

    def __init__(self, L, cfg, device):
        import torch
        from fluidlab_b200 import _lib
        self.L, self.cfg, self.torch = L, cfg, torch
        self.dev = torch.device(device)
        S, G, qd = cfg['S'], cfg['G'], cfg['qd']
        z = lambda *sh, dt=torch.float32: torch.zeros(sh, dtype=dt, device=self.dev)
        self.b = dict(v=z(S + 1, G, 4), v_tmp=z(S + 1, G, 4), div=z(S + 1, G), p=z(S + 1, G), q=z(S + 1, qd, G), is_free=z(S + 1, G, dt=torch.uint8),
                      gv=z(S + 1, G, 4), gv_tmp=z(S + 1, G, 4), gdiv=z(S + 1, G), gp=z(S + 1, G), gq=z(S + 1, qd, G), tmp_a=z(G), tmp_b=z(G), acc=z(G))
        self.air = dict(pos=z(T_SUB + 1, 3), quat=z(T_SUB + 1, 4), s=z(T_SUB + 1), r=z(T_SUB + 1), gpos=z(T_SUB + 1, 3), gquat=z(T_SUB + 1, 4),
                        gs=z(T_SUB + 1), gr=z(T_SUB + 1))
        a = cfg['air']
        for k, sl in (('pos', slice(0, 3)), ('quat', slice(3, 7))):
            self.air[k].copy_(torch.from_numpy(a[:, sl].astype(np.float32)))
        self.air['s'].copy_(torch.from_numpy(a[:, 7].astype(np.float32))); self.air['r'].copy_(torch.from_numpy(a[:, 8].astype(np.float32)))
        c = _lib.FsmkConfig()
        c.res, c.max_steps_local, c.q_dim, c.solver_iters, c.dt = cfg['n'], S, qd, cfg['iters'], DT
        c.lower_y, c.higher_y, c.low_T, c.device = cfg['band'][0], cfg['band'][1], 0.0, (self.dev.index or 0) if self.dev.type == 'cuda' else 0
        c.inject_v = (C.c_float * 3)(*cfg['inject_v'])
        self.h = C.c_void_p()
        assert L.fsmk_create(C.byref(c), C.byref(self.h)) == 0
        bb = _lib.FsmkBuffers()
        for k, t in self.b.items():
            setattr(bb, k, t.data_ptr())
        self.ck(L.fsmk_bind(self.h, C.byref(bb)))
        ab = _lib.FsmkAircon()
        for k, t in self.air.items():
            setattr(ab, k, t.data_ptr())
        self.ck(L.fsmk_set_aircon(self.h, C.byref(ab)))
        self.vox = [torch.from_numpy(vx.reshape(-1)).to(self.dev) for vx, _ in cfg['static_vols']]
        arr = (_lib.FmpmSdfMesh * 4)()
        for i, ((vx, T), t) in enumerate(zip(cfg['static_vols'], self.vox)):
            arr[i].voxels, arr[i].res = t.data_ptr(), vx.shape[0]
            arr[i].T_mesh_to_voxels = (C.c_float * 16)(*[float(x) for x in T.reshape(-1)])
        self.ck(L.fsmk_set_statics(self.h, len(self.vox), arr))

    def __del__(self):
        try:
            self.L.fsmk_destroy(self.h)
        except Exception:
            pass

    def ck(self, rc):
        assert rc == 0, self.L.fsmk_last_error(self.h).decode()

    def launch(self, name, *args):
        self.ck(getattr(self.L, 'fsmk_' + name)(self.h, *args, None))
        if self.dev.type == 'cuda':
            self.torch.cuda.synchronize()

    def snap(self):
        return {k: t.cpu().numpy().copy() for k, t in itertools.chain(self.b.items(), (('air_' + k, t) for k, t in self.air.items()))}


def _bits(a):
    return a.view(np.uint8) if a.dtype == np.uint8 else a.view(np.uint32)


def assert_untouched(tag, before, after, allowed):
    """every buffer outside the launch's write set comes back bit for bit; allowed: key -> bool mask of before[key]'s shape (or True)"""
    for k in before:
        m = allowed.get(k, False)
        if m is True:
            continue
        bad = _bits(before[k]) != _bits(after[k])
        if m is not False:
            bad &= ~np.broadcast_to(m, bad.shape)
        assert not bad.any(), f'{tag} wrote outside its outputs: {k} at {np.argwhere(bad)[:4].tolist()} ({int(bad.sum())} elements)'


def ratio(got, ref, S):
    with np.errstate(divide='ignore', invalid='ignore'):
        r = np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64)) / (U * np.maximum(np.asarray(S, np.float64), 1e-30))
    return r


def check_bar(tag, key, got, ref, S, sel, err, amb_tag=''):
    if not np.any(sel):
        return
    r = ratio(got, ref, S)
    r = np.where(np.broadcast_to(sel, r.shape), r, 0.0)
    rm = float(r.max())
    where = np.unravel_index(int(np.argmax(r)), r.shape)
    assert rm <= C_BAR[key], (f'{tag}: {key}{amb_tag} off by {rm:.3g} x 2^-23 S_i (bar {C_BAR[key]}) at {where}: got {np.asarray(got)[where]!r}, '
                              f'ref {np.asarray(ref)[where]!r}, S {np.asarray(S)[where]!r}')
    err[key] = max(err.get(key, 0.0), rm)


# ------------------------------------------------------------------------------------------------------------------ oracle feeding
def _oracle(cfg, prec):
    from oracle.smoke import SmokeOracle
    o = SmokeOracle(res=cfg['n'], dt=DT, solver_iters=cfg['iters'], q_dim=cfg['qd'], max_steps_local=cfg['S'], max_substeps_local=T_SUB,
                    lower_y=cfg['band'][0], higher_y=cfg['band'][1], inject_v=tuple(float(np.float32(x)) for x in cfg['inject_v']), precision=prec)
    for vox, T in cfg['static_vols']:
        o.add_static(vox, T)
    for f in range(T_SUB + 1):
        o.set_aircon(f, np.asarray(cfg['air'][f], np.float32))
    return o


def _frame(b, s, grad=False):
    g = 'g' if grad else ''
    return dict(v=b[g + 'v'][s, :, :3], v_tmp=b[g + 'v_tmp'][s, :, :3], div=b[g + 'div'][s], p=b[g + 'p'][s], q=b[g + 'q'][s].T)


def feed(os_, b, s, grad=False):
    """both frames s, s+1 (state, and adjoints when grad) of the device buffers into the oracles; the mask of frame s"""
    for o in os_:
        o.set_free(s, b['is_free'][s])
        for fr in (s, s + 1):
            o.set_state(fr, _frame(b, fr))
            if grad:
                o.set_grad(fr, _frame(b, fr, True))


def ostate(o, s, grad=False):
    """frame s of an oracle (its adjoint when grad) in the flat layouts: (G, C) fields, (G,) scalars"""
    st = o.get_grad(s) if grad else o.get_state(s)
    return {k: v.reshape(-1, v.shape[-1]) if v.ndim == 4 else v.reshape(-1) for k, v in st.items()}


# ------------------------------------------------------------------------------------------------------------------ abs-value scales of the linear phases
def div_scale(vt, free, nbs):
    S = np.zeros(len(free))
    for (d, sg), nb in nbs.items():
        S += 0.5 * np.where(nb['free'], np.abs(vt[nb['nb'], d]), np.abs(vt[:, d]))
    return S


def jacobi_scales(free, nbs, x0, rhs, iters):
    """the abs-value recursion of `iters` Jacobi sweeps from |x0| with |rhs|: A_t (abs iterate), E_t (accumulated first-order rounding scale);
    returns A, E at the end and the sums over the sweeps' inputs (for the adjoint's running sum)"""
    A = np.where(free, np.abs(x0), 0.0)
    E = np.zeros_like(A)
    sumAE = np.zeros_like(A)
    locs = [nb['loc'] for nb in nbs.values()]
    r = np.where(free, np.abs(rhs), 0.0)
    for _ in range(iters):
        sumAE += A + E
        NA = sum(A[l] for l in locs)
        NE = sum(E[l] for l in locs)
        A, E = np.where(free, (NA + r) / 6.0, 0.0), np.where(free, (NE + NA + r) / 6.0, 0.0)
    return A, E, sumAE


# ------------------------------------------------------------------------------------------------------------------ the run
def run(name, device, L, seed=SEED, log=None):
    """every launch of one step and of its adjoint on one layout; returns the census counts, the largest ratios and timings"""
    import torch
    cfg, st = make_layout(name, seed)
    n, G, S, s, qd = cfg['n'], cfg['G'], cfg['S'], cfg['s'], cfg['qd']
    tag = f'{name} ({device})'
    err, tm = {}, {}
    dev = Dev(L, cfg, device)
    b0 = dev.b
    rng = np.random.RandomState(seed + 1000)
    # state of frame s, sentinels everywhere else
    for k in ('v', 'v_tmp', 'gv', 'gv_tmp'):
        b0[k].fill_(float(SENT))
    for k in ('div', 'p', 'q', 'gdiv', 'gp', 'gq'):
        b0[k].fill_(float(SENT))
    b0['is_free'].fill_(SENT_U8)
    for k in ('gpos', 'gquat', 'gs', 'gr'):
        dev.air[k].fill_(float(SENT))
    v4 = np.zeros((G, 4), np.float32); v4[:, :3] = st['v']
    dev.b['v'][s].copy_(torch.from_numpy(v4))
    dev.b['q'][s].copy_(torch.from_numpy(st['q']))
    dev.b['p'][s].copy_(torch.from_numpy(st['p']))
    o64, o32 = _oracle(cfg, 64), _oracle(cfg, 32)
    band = mask64(cfg)[2]

    # 1. free space
    before = dev.snap()
    dev.launch('free_space', s)
    after = dev.snap()
    fr_k = after['is_free'][s]
    inb = np.zeros_like(before['is_free'], bool); inb[s] = band
    assert_untouched(f'{tag} fsmk_free_space', before, after, dict(is_free=inb))
    assert set(np.unique(fr_k[band])) <= {0, 1} and (fr_k[~band] == SENT_U8).all(), f'{tag} fsmk_free_space: bytes outside the band must keep the sentinel'
    o64.free_space(s); o32.free_space(s)
    f64, f32 = o64.is_free(s).reshape(-1) != 0, o32.is_free(s).reshape(-1) != 0
    _, amb_sdf, _ = mask64(cfg)
    free = fr_k == 1
    assert np.array_equal(free[~amb_sdf], f64[~amb_sdf]), f'{tag} fsmk_free_space: mask differs from fp64 at {np.nonzero((free != f64) & ~amb_sdf)[0][:8]}'
    assert np.array_equal(free[amb_sdf], f32[amb_sdf]), f'{tag} fsmk_free_space: mask differs from the fp32 oracle on the ambiguous cells'
    assert amb_sdf.sum() <= AMB_FRAC * max(free.sum(), 1), f'{tag}: {amb_sdf.sum()} cells with |sdf| < {AMB_SDF}'
    # the host zeroes is_free outside the band (the later kernels read it there through loc())
    dev.b['is_free'][s][torch.from_numpy(~band).to(dev.dev)] = 0
    cen, bt = census(cfg, free, st['v'].astype(np.float64))
    cen['amb_sdf'] = int(amb_sdf.sum())
    check_census(name, cen)
    nbs = neighbours(free, n)
    cells = np.nonzero(free)[0]
    if log:
        log(f'{tag} census {cen}')

    # 2. advection, twice: the corner and the band air conditioner
    v64, q64 = st['v'].astype(np.float64), st['q'].T.astype(np.float64)
    for f in (F_CORNER, F_BAND):
        dev.b['v_tmp'].fill_(float(SENT)); dev.b['v'][s + 1].fill_(float(SENT)); dev.b['q'][s + 1].fill_(float(SENT))
        before = dev.snap()
        t = time.perf_counter()
        dev.launch('advect', s, f)
        tm['advect'] = time.perf_counter() - t
        after = dev.snap()
        al = dict(v_tmp=np.zeros(before['v_tmp'].shape, bool), v=np.zeros(before['v'].shape, bool), q=np.zeros(before['q'].shape, bool))
        al['v_tmp'][s] = True; al['v'][s + 1][~free] = True; al['q'][s + 1] = True
        assert_untouched(f'{tag} fsmk_advect(f={f})', before, after, al)
        nf = ~free
        assert (after['v_tmp'][s][nf] == 0).all() and (after['v'][s + 1][nf] == 0).all(), f'{tag} fsmk_advect: v_tmp / v[s+1] of non-free cells must be 0'
        assert np.array_equal(_bits(after['q'][s + 1][:, nf]), _bits(after['q'][s][:, nf])), f'{tag} fsmk_advect: q[s+1] = q[s] on non-free cells, every plane'
        assert (after['v_tmp'][s][:, 3] == 0).all()
        feed((o64, o32), after, s)
        o64.advect(s, f); o32.advect(s, f)
        r64, r32 = ostate(o64, s), ostate(o32, s)
        q1_64, q1_32 = ostate(o64, s + 1)['q'], ostate(o32, s + 1)['q']
        if len(cells):
            te = bt['tris'][3]
            ee = bt['eps'][3]
            vf, av, lv = te.look(v64)
            qf, aq, lq = te.look(q64)
            dirv, _, dist, fac, sa, ra = impulse(cfg, f, cells)
            imp = np.abs(dirv)[None] * sa * fac[:, None] * DT
            Sv = np.zeros((G, 3)); Sq = np.zeros((G, qd))
            Sv[cells] = av + lv * ee[:, None] + imp * (4 + dist / ra)[:, None]
            Sq[cells] = (1 - fac[:, None]) * (aq + lq * ee[:, None]) + np.abs(qf) * fac[:, None] * (4 + dist / ra)[:, None]
            amb = np.zeros(G, bool); amb[cells[bt['amb']]] = True
            ok = free & ~amb
            check_bar(tag + f' fsmk_advect(f={f})', 'advect', after['v_tmp'][s][:, :3], r64['v_tmp'], Sv, ok[:, None], err)
            check_bar(tag + f' fsmk_advect(f={f})', 'advect', after['q'][s + 1].T, q1_64, Sq, ok[:, None], err)
            check_bar(tag + f' fsmk_advect(f={f})', 'advect', after['v_tmp'][s][:, :3], r32['v_tmp'], 2 * Sv, amb[:, None], err, ' (ambiguous, fp32 oracle)')
            check_bar(tag + f' fsmk_advect(f={f})', 'advect', after['q'][s + 1].T, q1_32, 2 * Sq, amb[:, None], err, ' (ambiguous, fp32 oracle)')

    # 3. divergence
    dev.b['div'].fill_(float(SENT))
    before = dev.snap()
    dev.launch('divergence', s)
    after = dev.snap()
    al = np.zeros(before['div'].shape, bool); al[s] = free
    assert_untouched(f'{tag} fsmk_divergence', before, after, dict(div=al))
    feed((o64,), after, s)
    o64.divergence(s)
    vt = after['v_tmp'][s][:, :3].astype(np.float64)
    check_bar(tag + ' fsmk_divergence', 'div', after['div'][s], ostate(o64, s)['div'], div_scale(vt, free, nbs), free, err)

    # 4. pressure: p[s] random on free cells, sentinel elsewhere (the chain must never read a non-free cell)
    p_in = np.where(free, st['p'], SENT).astype(np.float32)
    dev.b['p'][s].copy_(torch.from_numpy(p_in)); dev.b['p'][s + 1].fill_(float(SENT))
    before = dev.snap()
    t = time.perf_counter()
    dev.launch('pressure', s)
    tm['pressure'] = time.perf_counter() - t
    after = dev.snap()
    al = np.zeros(before['p'].shape, bool); al[s + 1] = free
    assert_untouched(f'{tag} fsmk_pressure', before, after, dict(p=al, tmp_a=True, tmp_b=True))
    if cfg['H']:
        feed((o64, o32), after, s)
        t = time.perf_counter()
        o64.pressure(s)
        tm['oracle64_pressure'] = time.perf_counter() - t
        o32.pressure(s)
        p32 = ostate(o32, s + 1)['p'].astype(np.float32)
        diff = free & (_bits(after['p'][s + 1]) != _bits(p32))
        assert not diff.any(), f'{tag} fsmk_pressure: not bit-identical to the fp32 oracle\'s sweeps at {np.nonzero(diff)[0][:8]} ({int(diff.sum())} cells)'
        A, E, _ = jacobi_scales(free, nbs, p_in.astype(np.float64), after['div'][s].astype(np.float64), cfg['iters'])
        check_bar(tag + ' fsmk_pressure', 'jacobi', after['p'][s + 1], ostate(o64, s + 1)['p'], A + E, free, err)

    # 5. projection
    dev.b['v'][s + 1][torch.from_numpy(free).to(dev.dev)] = float(SENT)
    before = dev.snap()
    dev.launch('project', s)
    after = dev.snap()
    al = np.zeros(before['v'].shape, bool); al[s + 1][free] = True
    assert_untouched(f'{tag} fsmk_project', before, after, dict(v=al))
    feed((o64,), after, s)
    o64.project(s)
    p1 = after['p'][s + 1].astype(np.float64)
    Sp = np.abs(vt).copy()
    for d in range(3):
        Sp[:, d] += 0.5 * (np.abs(p1[nbs[(d, 1)]['loc']]) + np.abs(p1[nbs[(d, -1)]['loc']]))
    check_bar(tag + ' fsmk_project', 'project', after['v'][s + 1][:, :3], ostate(o64, s + 1)['v'], Sp, free[:, None], err)
    assert (after['v'][s + 1][:, 3][free] == 0).all()

    # ---------------------------------------------------------------- adjoint: random O(1) adjoints, sentinels on every cell that must not move
    for k in ('gv', 'gv_tmp', 'gdiv', 'gp', 'gq'):
        dev.b[k].fill_(float(SENT))
    rnd = lambda *sh: torch.from_numpy(rng.randn(*sh).astype(np.float32))
    g4 = rnd(G, 4); g4[:, 3] = 0
    dev.b['gv'][s + 1].copy_(torch.where(torch.from_numpy(free)[:, None], g4, torch.tensor(SENT)).to(dev.dev))
    gvt0 = rnd(G, 4); gvt0[:, 3] = 0
    dev.b['gv_tmp'][s].copy_(torch.where(torch.from_numpy(free)[:, None], gvt0, torch.tensor(SENT)).to(dev.dev))
    dev.b['gp'][s + 1].copy_(torch.where(torch.from_numpy(free), rnd(G), torch.tensor(SENT)).to(dev.dev))
    fT = torch.from_numpy(free).to(dev.dev)

    # 6. project_grad
    before = dev.snap()
    dev.launch('project_grad', s)
    after = dev.snap()
    al_gvt = np.zeros(before['gv_tmp'].shape, bool); al_gvt[s][free] = True
    al_gp = np.zeros(before['gp'].shape, bool); al_gp[s + 1] = free
    assert_untouched(f'{tag} fsmk_project_grad', before, after, dict(gv_tmp=al_gvt, gp=al_gp))
    o64.reset_grad(); feed((o64,), before, s, grad=True)
    o64.project_grad(s)
    gv1 = np.where(free[:, None], before['gv'][s + 1][:, :3], 0).astype(np.float64)
    gvt_in = before['gv_tmp'][s][:, :3].astype(np.float64)
    check_bar(tag + ' fsmk_project_grad', 'project_grad', after['gv_tmp'][s][:, :3], ostate(o64, s, True)['v_tmp'], np.abs(gvt_in) + np.abs(gv1),
              free[:, None], err)
    Sgp = np.abs(before['gp'][s + 1].astype(np.float64))
    for d in range(3):
        fm, fp = nbs[(d, -1)]['free'], nbs[(d, 1)]['free']
        gc = np.abs(gv1[:, d])
        Sgp += 0.5 * (np.where(fm, np.abs(gv1[nbs[(d, -1)]['nb'], d]), 0) + np.where(fp, 0, gc) + np.where(fp, np.abs(gv1[nbs[(d, 1)]['nb'], d]), 0) + np.where(fm, 0, gc))
    check_bar(tag + ' fsmk_project_grad', 'project_grad', after['gp'][s + 1], ostate(o64, s + 1, True)['p'], Sgp, free, err)

    # 7. pressure_grad: gp[s], gdiv[s] random on free cells
    dev.b['gp'][s].copy_(torch.where(fT, rnd(G).to(dev.dev), torch.tensor(SENT, device=dev.dev)))
    dev.b['gdiv'][s].copy_(torch.where(fT, rnd(G).to(dev.dev), torch.tensor(SENT, device=dev.dev)))
    before = dev.snap()
    dev.launch('pressure_grad', s)
    after = dev.snap()
    al_gp = np.zeros(before['gp'].shape, bool); al_gp[s] = free
    al_gd = np.zeros(before['gdiv'].shape, bool); al_gd[s] = free
    assert_untouched(f'{tag} fsmk_pressure_grad', before, after, dict(gp=al_gp, gdiv=al_gd, tmp_a=True, tmp_b=True, acc=True))
    if cfg['H']:
        o64.reset_grad(); feed((o64,), before, s, grad=True)
        t = time.perf_counter()
        o64.pressure_grad(s)
        tm['oracle64_pressure_grad'] = time.perf_counter() - t
        A, E, sumAE = jacobi_scales(free, nbs, before['gp'][s + 1].astype(np.float64), np.zeros(G), cfg['iters'])
        r = ostate(o64, s, True)
        check_bar(tag + ' fsmk_pressure_grad', 'jacobi_grad', after['gp'][s], r['p'], np.abs(before['gp'][s].astype(np.float64)) + A + E, free, err)
        check_bar(tag + ' fsmk_pressure_grad', 'jacobi_grad', after['gdiv'][s], r['div'], np.abs(before['gdiv'][s].astype(np.float64)) + sumAE / 6, free, err)

    # 8. divergence_grad
    before = dev.snap()
    dev.launch('divergence_grad', s)
    after = dev.snap()
    al = np.zeros(before['gv_tmp'].shape, bool); al[s][free] = True
    assert_untouched(f'{tag} fsmk_divergence_grad', before, after, dict(gv_tmp=al))
    o64.reset_grad(); feed((o64,), before, s, grad=True)
    o64.divergence_grad(s)
    gd = np.where(free, before['gdiv'][s], 0).astype(np.float64)
    Sdg = np.abs(before['gv_tmp'][s][:, :3].astype(np.float64))
    for d in range(3):
        fm, fp = nbs[(d, -1)]['free'], nbs[(d, 1)]['free']
        Sdg[:, d] += 0.5 * (np.where(fm, np.abs(gd[nbs[(d, -1)]['nb']]), 0) + np.where(fp, np.abs(gd[nbs[(d, 1)]['nb']]), 0) + np.abs(gd) * (~fm + ~fp))
    check_bar(tag + ' fsmk_divergence_grad', 'div_grad', after['gv_tmp'][s][:, :3], ostate(o64, s, True)['v_tmp'], Sdg, free[:, None], err)

    # 9. advect_grad, on the advection's own v[s], q[s]; gv[s], gq[s] random (they accumulate), gq[s+1] random everywhere
    for f in (F_CORNER, F_BAND):
        gv0 = rnd(G, 4); gv0[:, 3] = 0
        dev.b['gv'][s].copy_(gv0); dev.b['gq'][s].copy_(rnd(qd, G)); dev.b['gq'][s + 1].copy_(rnd(qd, G))
        for k in ('gpos', 'gquat', 'gs', 'gr'):
            dev.air[k][f] = 0
        before = dev.snap()
        t = time.perf_counter()
        dev.launch('advect_grad', s, f)
        tm['advect_grad'] = time.perf_counter() - t
        after = dev.snap()
        al_gv = np.zeros(before['gv'].shape, bool); al_gv[s] = True
        al_gq = np.zeros(before['gq'].shape, bool); al_gq[s] = True
        al_air = {('air_' + k): (np.arange(T_SUB + 1) == f).reshape((-1,) + (1,) * (before['air_' + k].ndim - 1)) for k in ('gpos', 'gquat', 'gs', 'gr')}
        assert_untouched(f'{tag} fsmk_advect_grad(f={f})', before, after, dict(gv=al_gv, gq=al_gq, **al_air))
        o64.reset_grad(); o32.reset_grad()
        feed((o64, o32), before, s, grad=True)
        o64.advect_grad(s, f); o32.advect_grad(s, f)
        r64, r32 = ostate(o64, s, True), ostate(o32, s, True)
        gv_in, gq_in, gq1 = before['gv'][s][:, :3].astype(np.float64), before['gq'][s].T.astype(np.float64), before['gq'][s + 1].T.astype(np.float64)
        Sgv, Sgq = np.abs(gv_in).copy(), np.abs(gq_in).copy()
        Sgq[~free] += np.abs(gq1[~free])
        reach, amb_t = np.zeros(G, bool), np.zeros(G, bool)
        air_abs = np.zeros(9)
        tag_f = tag + f' fsmk_advect_grad(f={f})'
        if len(cells):
            t0, t1, t2, te = bt['tris']
            e0, e1, e2, ee = bt['eps']
            gvt = before['gv_tmp'][s][cells, :3].astype(np.float64)
            go_q = gq1[cells]
            dirv, dd, dist, fac, sa, ra = impulse(cfg, f, cells)
            qf, _, lq = te.look(q64)
            vf, _, _ = te.look(v64)
            relf = fac * (4 + dist / ra)             # abs error scale of factor
            gqf = (1 - fac)[:, None] * go_q
            gqf_abs = np.abs(go_q) * ((1 - fac) + relf)[:, None]
            g_pe, g_pe_abs = np.zeros((len(cells), 3)), np.zeros((len(cells), 3))
            for a in range(qd):
                gp_, gpa, con = te.adj(q64[:, a:a + 1], qf[:, a:a + 1], gqf[:, a:a + 1], gqf_abs[:, a:a + 1], ee)
                g_pe += gp_; g_pe_abs += gpa
                np.add.at(Sgq[:, a], te.idx.reshape(-1), con[..., 0].reshape(-1))
            gp_, gpa, con = te.adj(v64, vf, gvt, np.abs(gvt), ee)
            g_pe += gp_; g_pe_abs += gpa
            np.add.at(Sgv, te.idx.reshape(-1), con.reshape(-1, 3))
            g_v3, g_v3a = -DT * 4 / 9 * g_pe, DT * 4 / 9 * g_pe_abs
            g_p2, g_p2a, con = t2.adj(v64, bt['vs'][2], g_v3, g_v3a, e2)
            np.add.at(Sgv, t2.idx.reshape(-1), con.reshape(-1, 3))
            g_v2, g_v2a = -DT / 3 * g_pe - 0.75 * DT * g_p2, DT / 3 * g_pe_abs + 0.75 * DT * g_p2a
            g_p1, g_p1a, con = t1.adj(v64, bt['vs'][1], g_v2, g_v2a, e1)
            np.add.at(Sgv, t1.idx.reshape(-1), con.reshape(-1, 3))
            g_v1, g_v1a = -DT * 2 / 9 * g_pe - 0.5 * DT * g_p1, DT * 2 / 9 * g_pe_abs + 0.5 * DT * g_p1a
            _, _, con = t0.adj(v64, bt['vs'][0], g_v1, g_v1a, e0)
            np.add.at(Sgv, t0.idx.reshape(-1), con.reshape(-1, 3))
            for tt in bt['tris']:
                reach[tt.idx.reshape(-1)] = True
            ac = cells[bt['amb']]
            for tt in bt['tris'][1:]:       # the corners an ambiguous cell's fp32 lookups may take instead
                base = tt.base[bt['amb']]
                for o in itertools.product(range(-1, 3), repeat=3):
                    gc = np.clip(base + np.array(o), 0, n - 1)
                    amb_t[(gc[:, 0] * n + gc[:, 1]) * n + gc[:, 2]] = True
            reach |= amb_t
            # the air conditioner's per-cell terms on absolute values
            dot_abs = (np.abs(gvt) * np.abs(dirv)[None]).sum(1) * (1 + relf)
            gfac_abs = (np.abs(go_q) * (np.abs(qf) + lq * ee[:, None])).sum(1) + dot_abs * abs(sa) * DT
            gdir_abs = np.abs(gvt).sum(1) * abs(sa) * fac * DT * (1 + relf)
            qa = np.abs(cfg['air'][f][3:7]).sum()
            air_abs[0:3] = ((gfac_abs * fac / ra * (1 + relf) * n)[:, None] * np.abs(dd) / dist[:, None]).sum(0)
            air_abs[3:7] = (gdir_abs * np.abs(cfg['inject_v']).sum() * 4 * (1 + qa) ** 2).sum()
            air_abs[7] = (dot_abs * fac * DT).sum()
            air_abs[8] = (gfac_abs * fac * dist / ra ** 2 * (1 + relf)).sum()
            assert len(ac) <= AMB_FRAC * len(cells)
        ok = ~amb_t
        check_bar(tag_f, 'advect_grad', after['gv'][s][:, :3], r64['v'], Sgv, ok[:, None], err)
        check_bar(tag_f, 'advect_grad', after['gq'][s].T, r64['q'], Sgq, ok[:, None], err)
        check_bar(tag_f, 'advect_grad', after['gv'][s][:, :3], r32['v'], 2 * Sgv, amb_t[:, None], err, ' (ambiguous, fp32 oracle)')
        check_bar(tag_f, 'advect_grad', after['gq'][s].T, r32['q'], 2 * Sgq, amb_t[:, None], err, ' (ambiguous, fp32 oracle)')
        # exact: a cell no lookup reaches keeps its adjoint; non-free unreached cells of gq[s] get exactly gq[s] + gq[s+1]
        un = ~reach
        assert np.array_equal(_bits(after['gv'][s][un]), _bits(before['gv'][s][un])), f'{tag_f}: gv[s] of a cell no lookup reaches changed'
        fu = un & free
        assert np.array_equal(_bits(after['gq'][s][:, fu]), _bits(before['gq'][s][:, fu])), f'{tag_f}: gq[s] of a free cell no lookup reaches changed'
        nu = un & ~free
        want = (before['gq'][s][:, nu] + before['gq'][s + 1][:, nu]).astype(np.float32)
        assert np.array_equal(_bits(after['gq'][s][:, nu]), _bits(want)), f'{tag_f}: gq[s] += gq[s+1] of the non-free cells'
        cen.setdefault('unreached', 0)
        cen['unreached'] = max(cen['unreached'], int(un.sum()))
        ga = np.concatenate([after['air_gpos'][f], after['air_gquat'][f], [after['air_gs'][f]], [after['air_gr'][f]]]).astype(np.float64)
        gb = o64.aircon_grad(f)
        if len(cells):
            check_bar(tag_f, 'air', ga, gb, air_abs, np.ones(9, bool), err)
        else:
            assert (ga == 0).all(), f'{tag_f}: no free cell, the air conditioner adjoints must stay 0'
    del dev
    return dict(counts=cen, err=err, time=tm)
