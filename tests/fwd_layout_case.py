"""Shared body of tests/test_fwd_layouts.py: ONE launch of k_fwd (csrc/fmpm_forward.cu: g2p of frame f + p2g of frame f+1) on particle layouts
built to force each of its footprint branches, against the fp64 oracle; and one stored-grid backward substep on the same layouts.

k_fwd serves the 3x3x3 stencils of a warp's 32 particles in one of four ways, chosen from the warp-wide box of stencil bases (nx, ny, nz = the
box's extent + 2 nodes per axis):
    tma8       nx, ny <= 4, nz <= 8          footprint tile of 4 x 4 node columns of 8 nodes, by TMA (fwd mask bit 3, tensor map tm_gv8)
    tma16      nx, ny <= 4, 9 <= nz <= 16    the same with 16-node columns (tm_gv16)
    (staged)   the same two boxes with TMA off: plain loads into the same tile (masks 1 / 3; the only form the CPU shim compiles)
    unstaged   any other box: every lane gathers its 27 nodes from L2
`census` replays that decision on the host, so that every layout asserts that it reaches the branch it exists for and cannot pass by missing
it.  A staged warp is an "edge" warp when its TMA box reaches past the grid (bx0 + 4 > n, by0 + 4 > n or bz0 + rows > n): the tensor map then
fills the nodes outside with zeros.  The backward kernels (k_g2p, k_particle_grad) stage a footprint of their own (footprint_of,
csrc/fmpm_scatter.cuh: one node column, at most G2P_ZMAX = 32 nodes, else L2); its decision is replayed too.

What one launch is compared with:
  - the gather half (x, v, C of frame f+1): the oracle's p2g / grid_op / g2p of frame f, started from the same fp32 frame.  The error of each
    particle is scaled by the field's RMS over the used particles: a max-norm bar over the whole state lets a few wrong particles hide behind
    the largest value;
  - the scatter half (the accumulator of frame f+1 and F[f+2]): the oracle's p2g of frame f+1 started from the kernel's OWN frame f+1, so
    that both sides scatter identical inputs.  Per node and component |got - ref| <= GRID_C 2^-23 S_i, with S_i = sum_p |w_ip| |term_p|
    evaluated in fp64: a bar relative to the node's own value means nothing where momenta cancel or the mass is small;
  - TMA against plain staging (same kernel instantiation): the tile holds the same floats and the gather code is the same, so frame f+1 and
    F[f+2] must agree bit for bit; the accumulators differ only in the order of the float reductions (the per-node bar above);
  - unused and frozen slots: carried over bit for bit."""
import itertools

import numpy as np

from conftest import make_particles

U = 2.0 ** -23
# Bars, with the largest errors measured over every layout (H100 at n = 32 and 64, and the CPU shim with and without FMA contraction):
# per-node accumulator ratio 2.5; per particle x 7.5e-8, v 3.6e-5, C 1.2e-4, F 1.5e-6; adjoints (max-norm) 3.3e-6.
GRID_C = 16   # per-node bar of the accumulators, in units of 2^-23 S_i
# per-particle bars (error / RMS of the field over the used particles); x, v, C: gather half against the oracle chain from frame f;
# F: F[f+2], written by the scatter half, against the oracle's p2g from the kernel's own frame f+1
BARS = {'x': 5e-7, 'v': 1e-4, 'C': 5e-4, 'F': 1e-5}
GRAD_BAR = 1e-4
GRAVITY = (0.3, -10.0, 0.0)
BOUNDARY = dict(type='cube', lower=(0.05, 0.05, 0.05), upper=(0.95, 0.95, 0.95))
LAYOUTS = ('dense', 'zruns', 'long', 'high_edge', 'low_edge', 'ragged')
CLASSES = ('tma8', 'tma16', 'unstaged', 'empty')
# the branches each layout exists for: minimum number of warps per census class, at n = 32 and n = 64 alike
MIN_COUNTS = {
    'dense': dict(tma8=60),
    'zruns': dict(tma16=50, edge=5, bwd_staged=50),
    'long': dict(unstaged=20, bwd_staged=5, bwd_l2=10),
    'high_edge': dict(tma8=30, edge=30, bwd_staged=30),
    'low_edge': dict(tma8=30),
    'ragged': dict(tma8=10, partial_warps=18),
}


# ------------------------------------------------------------------------------------------------------------------ host replay of the kernels' choices
def replay_base(x, n):
    """base_fx (csrc/fmpm_common.cuh) in float32: ok (the whole stencil inside the grid) and the stencil base, per particle"""
    t = np.asarray(x, np.float32) * np.float32(n) - np.float32(0.5)
    with np.errstate(invalid='ignore'):
        ok = np.all((t > np.float32(-1.0)) & (t < np.float32(n - 2)), axis=1)
    b = np.zeros(t.shape, np.int64)
    b[ok] = np.trunc(t[ok]).astype(np.int64)   # cast(int): truncation toward zero
    return ok, b


def census(x_slots, used_slots, n):
    """per warp of 32 slots (particles in SLOT order): k_fwd's footprint branch, whether its TMA box reaches past the grid, and footprint_of's
    choice (staged / l2) in the backward kernels"""
    ok, b = replay_base(x_slots, n)
    live = ok & (np.asarray(used_slots) != 0)
    N = len(live)
    W = (N + 31) // 32
    cls, bwd, edge = [], [], np.zeros(W, bool)
    partial = 0
    for w in range(W):
        sl = slice(32 * w, min(32 * w + 32, N))
        partial += int(not live[sl].all())
        bb = b[sl][live[sl]]
        if len(bb) == 0:
            cls.append('empty'); bwd.append('empty')
            continue
        lo, hi = bb.min(0), bb.max(0)
        nx, ny, nz = (hi - lo + 3).tolist()
        if nx <= 4 and ny <= 4 and nz <= 16:
            rows = 8 if nz <= 8 else 16
            cls.append('tma8' if rows == 8 else 'tma16')
            edge[w] = lo[0] + 4 > n or lo[1] + 4 > n or lo[2] + rows > n
        else:
            cls.append('unstaged')
        same = bool((bb[:, 0] == bb[0, 0]).all() and (bb[:, 1] == bb[0, 1]).all())   # footprint_of: the column of the first valid lane
        bwd.append('staged' if same and nz <= 32 else 'l2')
    cls, bwd = np.array(cls), np.array(bwd)
    counts = {k: int((cls == k).sum()) for k in CLASSES}
    counts.update(edge=int(edge.sum()), bwd_staged=int((bwd == 'staged').sum()), bwd_l2=int((bwd == 'l2').sum()), partial_warps=partial)
    return dict(ok=ok, live=live, cls=cls, bwd=bwd, edge=edge, counts=counts)


def check_counts(name, counts):
    for k, v in MIN_COUNTS[name].items():
        assert counts[k] >= v, f'layout {name} drifted off its branch: {k} = {counts[k]} < {v} ({counts})'


# ------------------------------------------------------------------------------------------------------------------ layouts
def _in_cells(rng, cells):
    """one particle per row of `cells` (stencil bases), in grid units: t = g - 0.5 lies in [b + 0.05, b + 0.95], at least 0.05 cells from the
    freeze thresholds (a substep moves a particle by < 0.01 cells here)"""
    cells = np.asarray(cells, np.int64)
    return cells + 0.55 + 0.9 * rng.rand(*cells.shape)


def _column(cx, cy, z0, counts):
    """stencil bases of a run of cells along z, counts[i] particles in cell z0 + i"""
    return np.repeat(np.array([[cx, cy, z0 + i] for i in range(len(counts))], np.int64), counts, axis=0)


def weights(g):
    """stencil bases and quadratic B-spline weights [p, offset, axis] of positions in grid units (MPM:335-337)"""
    b = np.trunc(g - 0.5).astype(np.int64)
    fx = g - b
    return b, fx, np.stack([0.5 * (1.5 - fx) ** 2, 0.75 - (fx - 1.0) ** 2, 0.5 * (fx - 0.5) ** 2], 1)


def _cancelling(g, n):
    """particles with a negative weight on a node whose summed weight is below half its summed |weight| (the node's velocity p / m would
    amplify the rounding of both sums)"""
    b, _, w = weights(g)
    m, S = np.zeros(n ** 3), np.zeros(n ** 3)
    nodes, wts = [], []
    for o in itertools.product(range(3), repeat=3):
        wt = w[:, o[0], 0] * w[:, o[1], 1] * w[:, o[2], 2]
        node = ((b[:, 0] + o[0]) * n + b[:, 1] + o[1]) * n + b[:, 2] + o[2]
        np.add.at(m, node, wt); np.add.at(S, node, np.abs(wt))
        nodes.append(node); wts.append(wt)
    bad = (S > 0) & (m < 0.5 * S)
    return np.where(np.any([(wt < 0) & bad[node] for node, wt in zip(nodes, wts)], axis=0))[0]


def _block(lo, hi):
    return np.stack(np.meshgrid(*[np.arange(a, b) for a, b in zip(lo, hi)], indexing='ij'), -1).reshape(-1, 3)


def layout(name, n, rng):
    """positions (float32, original particle order), used, frozen (used slots outside the grid) and whether frame f is cell-sorted before the
    launch; unsorted layouts are built warp by warp in slot order.  Sorted layouts keep every node column at a multiple of 32 particles, so
    that warps do not straddle columns."""
    c = n // 2 - 3
    frozen = None
    if name == 'dense':        # 12 - 16 particles per cell in a 6^3 block, shuffled, then cell-sorted: a warp spans 2 - 4 cells in z (tma8)
        cells = _block((c, c, c), (c + 6, c + 6, c + 6))
        g = _in_cells(rng, np.repeat(cells, rng.randint(12, 17, len(cells)), axis=0))
        sort = True
    elif name == 'zruns':      # 28 node columns of 2 warps, 2 - 3 particles per cell: a sorted warp spans 11 - 14 cells in z (tma16); every other column ends at the top
        cols = []
        for k, (cx, cy) in enumerate(itertools.product(range(c, c + 7), range(c + 1, c + 5))):
            cnt = []
            for _ in range(2):   # 3 k3 + 2 k2 = 32 particles on k3 + k2 cells
                k3, k2 = [(10, 1), (8, 4), (6, 7), (4, 10)][rng.randint(4)]
                cnt += list(rng.permutation([3] * k3 + [2] * k2))
            z0 = n - 2 - len(cnt) if k % 2 else rng.randint(0, n - 1 - len(cnt))
            cols.append(_column(cx, cy, z0, cnt))
        g = _in_cells(rng, np.concatenate(cols))
        sort = True
    elif name == 'long':       # no sort: 12 warps on one column each over 17 - 32 cells (nz > 16), then 10 warps of a cloud across the grid (nx > 4)
        parts = []
        for k in range(12):
            L = rng.randint(17, min(32, n - 2) + 1)
            cnt = np.ones(L, np.int64)
            cnt[rng.choice(L, 32 - L, replace=False)] += 1
            parts.append(_column(c + k % 4, c + k // 4, rng.randint(0, n - 1 - L), cnt)[rng.permutation(32)])
        parts.append(rng.randint(2, n - 4, size=(320, 3)))
        g = _in_cells(rng, np.concatenate(parts))
        sort = False
    elif name in ('high_edge', 'low_edge'):   # stencil bases at the last (n - 3) / first (0) cell in x, in y, in z and in all three, 8 per cell
        e = n - 3 if name == 'high_edge' else 0
        ze = (n - 6, n - 2) if name == 'high_edge' else (0, 4)
        cells = np.concatenate([
            np.repeat(_block((e, c, c), (e + 1, c + 4, c + 8)), 8, axis=0),       # x at the edge: 4 columns of 64
            np.repeat(_block((c, e, c), (c + 4, e + 1, c + 8)), 8, axis=0),       # y
            np.repeat(_block((c, c, ze[0]), (c + 4, c + 4, ze[1])), 8, axis=0),   # z: 16 columns of 32
            np.repeat(_block((e, e, c), (e + 1, e + 1, c + 4)), 8, axis=0),       # x and y
            np.repeat([[e, e, e]], 32, axis=0)])                                  # the corner cell
        g = _in_cells(rng, cells)
        if name == 'low_edge':   # along one of its edge axes, a quarter of the particles at x * inv_dx in (-0.5, 0.5) (base 0 by truncation toward
            # zero, fx < 0.5, w1 < 0.5 and negative below fx = 0.134) and a quarter just above 0.5; the rest keeps the nodes' masses well away from
            # zero (negative weights along two axes of one particle, or too many of them, could cancel a node's mass)
            for p in np.where((cells == 0).any(1))[0]:
                d = rng.choice(np.where(cells[p] == 0)[0])
                r = rng.rand()
                if r < 0.5:
                    g[p, d] = rng.uniform(-0.45, 0.45) if r < 0.25 else rng.uniform(0.55, 0.7)
            for _ in range(200):   # a node whose mass the negative weights cut below half the sum of the |weights|: some of its particles with negative weights go back to the cell's bulk
                movers = _cancelling(g, n)
                if len(movers) == 0:
                    break
                movers = rng.choice(movers, (len(movers) + 3) // 4, replace=False)
                neg = g[movers] < 0.134
                g[movers] = np.where(neg, rng.uniform(0.55, 1.45, neg.shape), g[movers])
            assert len(_cancelling(g, n)) == 0
        sort = True
    elif name == 'ragged':     # no sort: columns of 6 cells x 6 particles back to back, N = 32 k + 17, 81 unused slots interleaved, 8 used slots outside the grid
        N, n_unused = 32 * 20 + 17, 81
        body = _in_cells(rng, np.concatenate([_column(c + i, c + j, c, [6] * 6) for i in range(4) for j in range(4)]))
        assert len(body) == N - n_unused
        unused = np.zeros(N, bool)
        unused[rng.choice(N, n_unused, replace=False)] = True
        g = rng.uniform(0, n, size=(N, 3))
        g[~unused] = body
        frozen = np.zeros(N, bool)
        fz = rng.choice(np.where(~unused)[0], 8, replace=False)
        frozen[fz] = True
        for i, p in enumerate(fz):   # one coordinate beyond a freeze threshold (t >= n - 1.95 or t <= -1.05)
            g[p, i % 3] = rng.uniform(n - 1.45, n - 0.6) if i % 2 else rng.uniform(-1.4, -0.55)
        used = (~unused).astype(np.int32)
        return dict(x=(g / n).astype(np.float32), used=used, frozen=frozen, sort=False)
    else:
        raise KeyError(name)
    N = len(g)
    perm = rng.permutation(N) if sort else np.arange(N)
    return dict(x=(g[perm] / n).astype(np.float32), used=np.ones(N, np.int32), frozen=np.zeros(N, bool), sort=sort)


def _state(rng, N, liquid):
    """materials and v, C, F of frame f: |v| < 0.5, C ~ 2, F near I (all-liquid: s I, and a general F for every 7th particle)"""
    from fluidlab_b200 import macros as M
    mats = [M.WATER, M.MILK, M.COFFEE] if liquid else [M.WATER, M.ELASTIC, M.ICECREAM]
    mat = np.array(mats, np.int32)[rng.randint(3, size=N)]
    v = rng.uniform(-0.28, 0.28, size=(N, 3)).astype(np.float32)
    C = (rng.randn(N, 3, 3) * 2.0).astype(np.float32)
    if liquid:
        F = np.eye(3)[None] * (1.0 + rng.randn(N) * 0.02)[:, None, None]
        F[::7] += rng.randn(len(F[::7]), 3, 3) * 0.02
    else:
        F = np.eye(3)[None] + rng.randn(N, 3, 3) * 0.05
    return mat, v, C, F.astype(np.float32)


def _sim(n, P, device, grad=False):
    from fluidlab_b200 import MPMSimulator
    s = MPMSimulator(dim=3, quality=n / 64, gravity=GRAVITY, horizon=10, max_substeps_local=10, max_substeps_global=1000, ckpt_dest='cpu', device=device,
                     sort_every=0)
    s.use_graphs = False
    if grad:
        s.store_grids = True
    s.setup_boundary(**BOUNDARY)
    s.build(None, None, [], P)
    return s


def _setup(name, n, liquid, device, seed, grad=False):
    rng = np.random.RandomState(seed)
    lay = layout(name, n, rng)
    x, used, frozen = lay['x'], lay['used'], lay['frozen']
    N = len(x)
    mat, v0, C0, F0 = _state(rng, N, liquid)
    P = make_particles(x, mat, n, used=used)
    s = _sim(n, P, device, grad)
    if grad:
        s.enable_grad()
    s.setframe(0, x, v0, C0, F0, used)
    if lay['sort']:
        s.sort_frame(0)
    ids = s._frame_ord[0].ids
    ids = np.arange(N) if ids is None else ids.cpu().numpy().astype(np.int64)
    cen = census(x[ids], used[ids], n)
    check_counts(name, cen['counts'])
    ok = np.empty(N, bool); ok[ids] = cen['ok']
    live = (used != 0) & ~frozen   # the oracle does not freeze particles: the frozen ones are unused there
    assert np.array_equal(ok & (used != 0), live), 'every used particle must be inside the grid at frame f, except the frozen ones'
    warp_of = np.empty(N, np.int64); warp_of[ids] = np.arange(N) // 32
    Po = make_particles(x, mat, n, used=live.astype(np.int32))
    return dict(rng=rng, x=x, used=used, live=live, v=v0, C=C0, F=F0, P=P, Po=Po, s=s, cen=cen, warp_of=warp_of, n=n, name=name)


# ------------------------------------------------------------------------------------------------------------------ bars
def particle_errors(got, ref, live):
    """per used particle: max |got - ref| over the components, over the RMS of the field over the used particles"""
    k = int(live.sum())
    a = np.asarray(got, np.float64)[live].reshape(k, -1)
    b = np.asarray(ref, np.float64)[live].reshape(k, -1)
    return np.abs(a - b).max(1) / max(np.sqrt(np.mean(b * b)), 1e-30)


def _check_particles(ctx, what, got, ref, key, bar):
    e = particle_errors(got, ref, ctx['live'])
    i = int(np.argmax(e))
    pid = int(np.where(ctx['live'])[0][i])
    w = int(ctx['warp_of'][pid])
    assert e[i] < bar, f'{ctx["name"]} n={ctx["n"]} {what}: {key} error {e[i]:.3g} (bar {bar:g}) at particle {pid}, warp {w} ({ctx["cen"]["cls"][w]}, backward {ctx["cen"]["bwd"][w]})'
    return float(e[i])


def scatter_scale(n, x, v, C, F, P, live, dt=2e-4):
    """S_i of the per-node bar, in fp64: sum_p |w_ip| (|m v_k| + sum_j |B_kj| (|fx_j| + o_j)) per momentum component (k_fwd's q = m v - B fx plus
    B o, B = dx (k_stress stress + m C)) and sum_p |w_ip| m for the mass; p over the used particles of frame f+1.  |B| is taken before the
    cancellations inside the stress, as fp32 evaluates it: 2 mu (|F~| + |R|) |F~|^T + lam |J| (D + 1) I, D = the sum of the absolute products
    of det F~ (J - 1 loses the digits J and 1 share)."""
    G = n ** 3
    x, v, C, F = [np.asarray(a, np.float64)[live] for a in (x, v, C, F)]
    m, mu, lam = P['mass'][live], P['mu'][live], P['lam'][live]
    dx = 1.0 / n
    k_stress = -dt * (dx * 0.5) ** 2 * 4 * n * n
    b, fx, w = weights(x * n)
    Ft = (np.eye(3)[None] + dt * C) @ F
    J = np.linalg.det(Ft)
    Us, _, Vt = np.linalg.svd(Ft)
    R = Us @ Vt
    A = np.abs(Ft)
    D = sum(A[:, 0, i] * A[:, 1, j] * A[:, 2, k] for i, j, k in itertools.permutations(range(3)))
    stress = 2 * mu[:, None, None] * (A + np.abs(R)) @ np.transpose(A, (0, 2, 1)) + (lam * np.abs(J) * (D + 1))[:, None, None] * np.eye(3)[None]
    Babs = (abs(k_stress) * stress + np.abs(m[:, None, None] * C)) * dx
    mv = np.abs(m[:, None] * v)
    Sv, Sm = np.zeros((G, 3)), np.zeros(G)
    for o in itertools.product(range(3), repeat=3):
        wt = np.abs(w[:, o[0], 0] * w[:, o[1], 1] * w[:, o[2], 2])
        node = ((b[:, 0] + o[0]) * n + b[:, 1] + o[1]) * n + b[:, 2] + o[2]
        T = mv + np.einsum('pkj,pj->pk', Babs, np.abs(fx) + np.array(o, np.float64))
        np.add.at(Sv, node, wt[:, None] * T)
        np.add.at(Sm, node, wt * m)
    return Sv, Sm


def grid_ratio(got, ref, S):
    """max over nodes of |got - ref| / (2^-23 S); a node without contributions must be exactly zero"""
    d = np.abs(np.asarray(got, np.float64) - ref)
    with np.errstate(divide='ignore', invalid='ignore'):
        r = np.where(S > 0, d / (U * S), np.where(d > 0, np.inf, 0.0))
    return float(r.max())


def _check_grid(what, got, ref, S):
    for k, (a, b, s) in {'momentum': (got[0], ref[0], S[0]), 'mass': (got[1], ref[1], S[1])}.items():
        r = grid_ratio(a, b, s)
        assert r <= GRID_C, f'{what}: {k} of the f+1 accumulator off by {r:.3g} x 2^-23 S_i (bar {GRID_C})'
    assert np.array_equal(got[1] != 0, ref[1] != 0), f'{what}: the nodes with mass differ'


# ------------------------------------------------------------------------------------------------------------------ one k_fwd launch
def run(name, n, liquid, masks, device=None, seed=0):
    """p2g(f) -> grid_op(f) -> fwd_step(f, full) under each fwd mask in turn (the grid of frame f is built once; fmpm_clear_grid between the launches
    zeroes only the accumulator, and k_fwd reads frame f and writes only frame f+1, F[f+2] and the accumulator), compared as described above.
    Returns the census counts and the largest errors."""
    from oracle import oracle as orc
    ctx = _setup(name, n, liquid, device, seed)
    s, live, used = ctx['s'], ctx['live'], ctx['used']
    f = 0
    s.phase('clear_grid', f); s.phase('p2g', f, 1); s.phase('grid_op', f, 1)
    s._frame_ord[f + 1] = s._frame_ord[f + 2] = s._frame_ord[f]
    on_gpu = s.device.type == 'cuda'
    out = {}
    for mask in masks:
        s._ck(s._lib.fmpm_clear_grid(s._h, s._stream()), 'fmpm_clear_grid')
        s._ck(s._lib.fmpm_set_fwd_mask(s._h, int(mask)), 'fmpm_set_fwd_mask')
        path = int(s._lib.fmpm_fwd_path(s._h))
        want = mask & (11 if liquid else 9)
        if not on_gpu:   # the shim compiles the TMA branch out
            assert not mask & 8
        assert path == want, f'mask {mask}: fmpm_fwd_path = {path}, expected {want} (bit 3: TMA tiles, required on the H100)'
        s._ck(s._lib.fmpm_fwd_step(s._h, f, 1, s._stream()), 'fmpm_fwd_step')
        fr = s.readframe(f + 1)
        fr['F2'] = s.readframe(f + 2, ('F',))['F']
        fr['vin'], fr['m'], _ = s.read_grid()
        out[mask] = fr
    # the oracle's gather half from the same fp32 frame f
    o = orc.OracleSim(n, ctx['Po'], gravity=GRAVITY, boundary=BOUNDARY, precision=64, max_substeps_local=10)
    o.set_frame(f, ctx['x'], ctx['v'], ctx['C'], ctx['F'], live)
    L = o.L
    L.orc_phase_reset_grid(o.h); L.orc_phase_p2g(o.h, f, 1); L.orc_phase_grid_op(o.h, f); L.orc_phase_g2p(o.h, f)
    ref = o.get_frame(f + 1)
    err = {}
    ok0 = ctx['cen']['ok']
    for mask, fr in out.items():
        what = f'{name} n={n} {"liquid" if liquid else "general"} mask {mask}'
        assert np.array_equal(fr['used'], used)
        ok1, _ = replay_base(fr['x'], n)
        assert np.array_equal(ok1[used != 0], live[used != 0]), f'{what}: a particle crossed a freeze threshold in the launch'
        for k in ('x', 'v', 'C'):
            err[(mask, k)] = _check_particles(ctx, what, fr[k], ref[k], k, BARS[k])
        idle = ~live   # unused and frozen slots: frame f+1 = frame f, F[f+2] = F[f+1] = F[f]
        for k, a in (('x', ctx['x']), ('v', ctx['v']), ('C', ctx['C']), ('F2', ctx['F'])):
            assert np.array_equal(fr[k][idle], a[idle]), f'{what}: unused / frozen slots must be carried over untouched ({k})'
        # the scatter half against the oracle's p2g of frame f+1 from the kernel's own frame f+1
        o.set_frame(f + 1, fr['x'], fr['v'], fr['C'], fr['F'], live)
        L.orc_phase_reset_grid(o.h); L.orc_phase_p2g(o.h, f + 1, 1)
        rvin, rm, _ = o.get_grid()
        err[(mask, 'F')] = _check_particles(ctx, what, fr['F2'], o.get_frame(f + 2)['F'], 'F[f+2]', BARS['F'])
        Sv, Sm = scatter_scale(n, fr['x'], fr['v'], fr['C'], fr['F'], ctx['P'], live)
        _check_grid(what, (fr['vin'], fr['m']), (rvin, rm), (Sv, Sm))
        err[(mask, 'grid')] = max(grid_ratio(fr['vin'], rvin, Sv), grid_ratio(fr['m'], rm, Sm))
        out[mask]['S'] = (Sv, Sm)
    # TMA tiles against plain staging, same instantiation
    for a, b in ((9, 1), (11, 3)):
        if a in out and b in out:
            for k in ('x', 'v', 'C', 'F2'):
                assert np.array_equal(out[a][k], out[b][k]), f'{name} n={n}: the gather from TMA tiles (mask {a}) differs from plain staging (mask {b}) in {k}'
            _check_grid(f'{name} n={n} mask {a} vs {b}', (out[a]['vin'], out[a]['m']), (out[b]['vin'], out[b]['m']), out[b]['S'])
    return dict(counts=ctx['cen']['counts'], err=err)


# ------------------------------------------------------------------------------------------------------------------ one backward substep
def run_backward(name, n, liquid, device=None, seed=0):
    """frame f forward through fmpm_substep_store (its k_g2p stages footprints like k_particle_grad), then fmpm_substep_grad_stored from random
    O(1) adjoints of frame f+1, against the fp64 oracle's substep_grad; unused and frozen slots pass their adjoint through unchanged"""
    from oracle import oracle as orc
    ctx = _setup(name, n, liquid, device, seed + 1, grad=True)
    s, live, rng = ctx['s'], ctx['live'], ctx['rng']
    N = len(live)
    s.substep(0, True)
    assert s._pm_ring is not None and s._ring_valid[0], 'the stored-grid substep must have run'
    s.cur_substep_global = 1
    g = {k: rng.randn(*sh).astype(np.float32) for k, sh in (('x', (N, 3)), ('v', (N, 3)), ('C', (N, 3, 3)), ('F', (N, 3, 3)))}
    s.reset_grad(); s.set_grad(g['x'], g['v'], g['C'], g['F'])
    s.cur_substep_global = 0
    s.substep_grad(0, True)
    gg = s.get_grad()
    o = orc.OracleSim(n, ctx['Po'], gravity=GRAVITY, boundary=BOUNDARY, precision=64, max_substeps_local=10)
    o.set_frame(0, ctx['x'], ctx['v'], ctx['C'], ctx['F'], live)
    o.substep(0)
    o.reset_grad(); o.set_grad_frame(1, g['x'], g['v'], g['C'], g['F'])
    o.substep_grad(0)
    og = o.get_grad_frame(0)
    err = {}
    for k in ('x', 'v', 'C', 'F'):
        a, b = gg[k].astype(np.float64), og[k]
        err[k] = float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))
        assert err[k] < GRAD_BAR, f'{name} n={n}: adjoint of {k} off by {err[k]:.3g} (bar {GRAD_BAR:g})'
        assert np.array_equal(gg[k][~live], g[k][~live]), f'{name} n={n}: unused / frozen slots must pass the adjoint of {k} through'
    return dict(counts=ctx['cen']['counts'], err=err)
