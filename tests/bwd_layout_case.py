"""Shared body of tests/test_bwd_layouts.py: the kernels of the backward substep ONE launch at a time, on the particle layouts of
tests/fwd_layout_case.py, against the fp64 oracle.  Each launch is compared with an oracle phase started from the kernel's OWN inputs (the
forward grid, the grid adjoints the previous launch left on the device), passed in through set_frame / set_grid / set_grid_grad, so that errors
do not compound along the chain:
    1  k_p2g (write_F = 0: the recompute of fmpm_substep_grad; write_F = 1: the forward, also F[f+1])   per node, GRID_C 2^-23 S_i
    2  k_grid_op + k_g2p (the stored-grid forward: x, v, C of frame f+1)                                 per particle, over the field's RMS
    3  k_g2p_grad_scatter (the v_out adjoint)                                                           per node and component, SC_C 2^-23 S_i
    4  k_grid_op_grad (the (v_in, mass) adjoint, the wall-reflection adjoint)                           per node, ulp-scale
    5  k_particle_grad (the adjoint of frame f)                                                         per particle, over the field's RMS
    6  4 and 5 again in their parameter-gradient instantiations, and the per-row dL/d(mu, lam, mass), dL/dg and dL/d(restitution) against
       fp64 sums of their terms                                                                         per row, BETA sum |term|

What each layout has to reach is asserted from a host replay of the kernels' choices (`bwd_census`), on the slot order the device produced:
  - k_g2p_grad_scatter's register window: it runs SC_ROUNDS = 4 rounds of 32 slots per warp of 128 and keeps its window across rounds.  Every
    cell run is a carry (a round's smallest cell is the one the window is on: no run start), a z+1 shift or a full move; a round past N is
    skipped (`rem <= 0`), a round with fewer than 32 slots is partial;
  - footprint_of in k_particle_grad (staged tile / L2), as in fwd_layout_case.census;
  - the plastic pairs (i, j) of constitutive_grad, from the fp64 singular values of F~ = (I + dt C) F: both pass the clamp, mixed (one
    clamped, or both at different bounds: the line with 1 / (s_j^2 - s_i^2)), both clamped at the same bound;
  - param_grad_reduce: warps whose 32 lanes share one material row (butterfly), warps whose live lanes hold several rows, partial warps;
  - with a per-particle material field (`field`): particles with mu_p = 0 (k_particle_grad<2, true> takes one more svd3 for their dL/dmu) and
    particles of a liquid-class row with mu_p > 0 (the constitutive model's SVD path on a liquid row).

With `field`, every launch runs its material-field instantiation (k_p2g_field, k_particle_grad<2, *>): mu and lam per particle from
material_field_case.random_field (within 2x of the row's, 15 % of the particles at mu_p = 0, WATER particles mostly at mu_p > 0).  Step 6 then
checks k_particle_grad<2, true>'s per-slot accumulator `gfield` particle by particle (a read-modify-write add into a random prefill; unused and
frozen slots keep the prefill bit for bit), that the rows' dL/dmu and dL/dlam stay exactly 0 while dL/dmass is still reduced per row, and that
get_param_grad() maps the slot-order accumulator into original particle order (MPMSimulator._flush_field_grad) and sums it per row.

F is well conditioned by construction: F~ = Q1 diag(s) Q2^T is drawn and F = (I + dt C)^-1 F~ rounded to fp32; a particle whose fp64 F~ has two
singular values closer than 1e-2 (1e-3 for a pair inside the plastic window, whose adjoint takes no 1 / (s_j^2 - s_i^2)), or, in a plastic
row, a singular value within 2e-4 of a clamp bound, is drawn again.  Repeated singular values are out of scope: U and V are not unique there,
fp32 and fp64 may take different branches, and the reference's clamp turns the adjoint into O(1e8) x 0."""
import itertools

import numpy as np

from conftest import make_particles
from material_field_case import random_field
from fwd_layout_case import (BOUNDARY, GRAVITY, GRID_C, LAYOUTS, U, _sim, census, check_counts, grid_ratio, layout, particle_errors, replay_base,
                             scatter_scale, weights)
from param_grad_ref import param_grad_terms

DT = 2e-4
SEED = 11   # dense gets N = 32 k here: only ragged ends in a partial scatter round
SC_ROUNDS = 4
PL_LO, PL_HI = 0.998, 1.003   # the plastic clamp of constitutive_grad (fp32 constants; kept 2e-4 away from them)
# Bars, each with the largest error measured over every layout, liquid and general, on the H100 (80 GB HBM3, 700 W) at n = 32 and 64 and on
# the CPU shim at n = 32 with and without FMA contraction; k_p2g's accumulators keep fwd_layout_case's GRID_C = 16 (measured 2.6).
SC_C = 8           # k_g2p_grad_scatter, per node and component, in units of 2^-23 S_i (measured 2.1)
GOP_C = 8          # k_grid_op_grad: v_in adjoint in units of 2^-23 |gv_out| / m, mass adjoint in units of 2^-23 sum_k |p_k gv_k| / m^2 (2.2)
# per particle, error over the field's RMS: k_g2p (x, v, C of frame f+1; measured 7.4e-8, 1.9e-6, 4.2e-6) and k_p2g (F[f+1]; 1.2e-6)
BARS = {'x': 5e-7, 'v': 1e-5, 'C': 2e-5, 'F': 5e-6}
GRAD_BARS = {'x': 1e-4, 'v': 1e-5, 'C': 2e-5, 'F': 5e-5}   # k_particle_grad, adjoint of frame f (measured 2.8e-5, 1.7e-6, 5.8e-6, 1.1e-5)
# parameter gradients, |got - ref| <= BETA sum |term| per row and component (measured mu 1.5e-6, lam 5.0e-6, mass 4.1e-8; gravity 1.1e-8,
# restitution 2.5e-8; lam loses the digits J and 1 share in J - 1)
BETA = dict(mu=5e-6, lam=2e-5, mass=2e-7, gravity=5e-8, restitution=1e-7)
# k_particle_grad<2, true>: dL/dmu_p and dL/dlam_p per slot, in units of 2^-23 S_p (field_grad_scale), on top of one ulp of the prefill
# (measured over the same runs: mu 0.21, lam 0.79).  With a field the bars above hold with these largest errors: k_p2g 3.0, F[f+1] 1.2e-6;
# k_g2p 7.5e-8, 1.9e-6, 5.9e-6; adjoints 4.0e-5, 2.6e-6, 6.7e-6, 1.2e-5; rows mu 1.0e-6, lam 9.5e-6, mass 5.6e-8
FIELD_C = 4
AMBIG_FRAC = 0.05  # the wall nodes whose branch is within rounding of v = 0 (excluded) must stay this rare
# the branches each layout exists for, at n = 32 and n = 64 alike, about half the counts of the seed (`plastic_*` count pairs, general
# materials only; the rest count warps, rounds or runs).  zruns and the edge layouts fill whole cells per round of 32, so their rounds shift.
MIN_BWD = {
    'dense': dict(carry=30, shift=90, move=15, bwd_staged=30, bwd_l2=15, row_uniform=30, row_mixed=15),
    'zruns': dict(shift=300, bwd_staged=28, row_uniform=28),
    'long': dict(move=150, shift=130, bwd_l2=5, row_mixed=11),
    'high_edge': dict(shift=50, move=8, bwd_staged=17, row_uniform=17),
    'low_edge': dict(shift=50, move=8, bwd_staged=17, row_uniform=17),
    'ragged': dict(carry=6, move=7, partial_rounds=1, skipped_rounds=3, bwd_l2=7, row_mixed=10, row_partial=10),
}
MIN_PLASTIC = dict(plastic_pass=30, plastic_mixed=150, plastic_same=100)
# with a material field: the live particles at mu_p = 0 and the live liquid-class particles at mu_p > 0, at n = 32 and n = 64 alike (about
# half the counts of the seed)
FIELD_ZERO_FRAC = 0.15
MIN_FIELD = {
    'dense': dict(field_mu0=210, field_liquid_mu=490),
    'zruns': dict(field_mu0=134, field_liquid_mu=300),
    'long': dict(field_mu0=51, field_liquid_mu=114),
    'high_edge': dict(field_mu0=82, field_liquid_mu=136),
    'low_edge': dict(field_mu0=70, field_liquid_mu=194),
    'ragged': dict(field_mu0=47, field_liquid_mu=89),
}


# ------------------------------------------------------------------------------------------------------------------ host replay of the choices
def scatter_census(x_slots, used_slots, n):
    """k_g2p_grad_scatter's window, replayed per warp of 32 SC_ROUNDS slots: scatter_rank stages a round in ascending cell order (cells
    packed as bx << 20 | by << 10 | bz, keyless slots last); each distinct cell of the round is a carry (the round's smallest cell equals the
    window's: no run start), a z+1 shift (cell = window + 1) or a full move (any other cell, the window open).  Returns the counts."""
    ok, b = replay_base(x_slots, n)
    live = ok & (np.asarray(used_slots) != 0)
    key = np.where(live, (b[:, 0] << 20) | (b[:, 1] << 10) | b[:, 2], -1)
    N = len(key)
    c = dict(carry=0, shift=0, move=0, place=0, partial_rounds=0, skipped_rounds=0)
    for s0 in range(0, N, 32 * SC_ROUNDS):
        cur = -1
        for r in range(SC_ROUNDS):
            rem = N - (s0 + 32 * r)
            if rem <= 0:   # the kernel breaks: this round and the ones after it
                c['skipped_rounds'] += SC_ROUNDS - r
                break
            c['partial_rounds'] += rem < 32
            ks = np.unique(key[s0 + 32 * r: s0 + 32 * r + min(rem, 32)])
            for i, k in enumerate(ks[ks >= 0]):
                if i == 0 and k == cur:
                    c['carry'] += 1
                    continue
                c['shift' if cur >= 0 and k == cur + 1 else 'move' if cur >= 0 else 'place'] += 1
                cur = k
    return c


def f_tilde(F, C, dt=DT):
    """F~ = (I + dt C) F in fp64 from the fp32 F and C"""
    return (np.eye(3)[None] + dt * np.asarray(C, np.float64)) @ np.asarray(F, np.float64)


def plastic_pairs(sig):
    """per particle, the number of pairs (i, j) of constitutive_grad in each branch: [both pass, mixed, both clamped at the same bound]"""
    lo, hi = np.float32(PL_LO), np.float32(PL_HI)
    side = np.where(sig <= lo, -1, np.where(sig >= hi, 1, 0))   # 0: passes the clamp
    out = np.zeros((len(sig), 3), np.int64)
    for i, j in ((0, 1), (0, 2), (1, 2)):
        a, b = side[:, i], side[:, j]
        out[:, 0] += (a == 0) & (b == 0)
        out[:, 2] += (a != 0) & (a == b)
        out[:, 1] += ~(((a == 0) & (b == 0)) | ((a != 0) & (a == b)))
    return out


def row_census(rows_slots, live_slots):
    """param_grad_reduce per warp of 32 slots: every lane live and of one row (butterfly), live lanes of several rows (group path), a warp
    with idle lanes (group path through the live ballot)"""
    N = len(rows_slots)
    c = dict(row_uniform=0, row_mixed=0, row_partial=0)
    for s0 in range(0, N, 32):
        r, l = rows_slots[s0:s0 + 32], live_slots[s0:s0 + 32]
        if not l.any():
            continue
        if len(l) < 32 or not l.all():
            c['row_partial'] += 1
        if len(np.unique(r[l])) > 1:
            c['row_mixed'] += 1
        elif len(l) == 32 and l.all():
            c['row_uniform'] += 1
    return c


def bwd_census(x_slots, used_slots, rows_slots, n):
    cen = census(x_slots, used_slots, n)
    cen['counts'].update(scatter_census(x_slots, used_slots, n))
    cen['counts'].update(row_census(np.asarray(rows_slots), cen['live']))
    return cen


def field_counts(P, mu, live):
    """the live particles of a material field at mu_p = 0 and the live liquid-class particles at mu_p > 0"""
    from fluidlab_b200 import macros as M
    return dict(field_mu0=int(((mu == 0) & live).sum()), field_liquid_mu=int(((P['cls'] == M.MAT_LIQUID) & (mu > 0) & live).sum()))


def check_bwd_counts(name, counts, plastic, field=False):
    want = dict(MIN_BWD[name], **(MIN_PLASTIC if plastic else {}), **(MIN_FIELD[name] if field else {}))
    for k, v in want.items():
        assert counts[k] >= v, f'layout {name} drifted off its branch: {k} = {counts[k]} < {v} ({counts})'


# ------------------------------------------------------------------------------------------------------------------ particle state
def materials(liquid):
    from fluidlab_b200 import macros as M
    return [M.WATER, M.MILK, M.COFFEE] if liquid else [M.WATER, M.MILK_VIS, M.ELASTIC, M.ICECREAM, M.PLASTIC_DEMO]


def _rot(rng):
    q, _ = np.linalg.qr(rng.randn(3, 3))
    return q if np.linalg.det(q) > 0 else -q


def _sigmas(rng, plastic):
    """target singular values of F~: near 1 with gaps >= 1e-2; a plastic particle takes one of three shapes: two inside the clamp window and
    one outside (both pass), one inside between one below and one above (mixed), all three beyond the same bound (both clamped)"""
    if not plastic:
        return 1.0 + np.array([-0.08, 0.0, 0.08]) + rng.uniform(-0.02, 0.02, 3)
    u = rng.rand()
    if u < 0.3:
        a = rng.uniform(0.9984, 0.9998)
        return np.array([a, rng.uniform(a + 0.0012, 1.0026), rng.choice([0.95, 1.05]) + rng.uniform(-0.02, 0.02)])
    if u < 0.65:
        return np.array([rng.uniform(0.9984, 1.0026), rng.uniform(0.90, 0.98), rng.uniform(1.02, 1.10)])
    base = rng.uniform(1.008, 1.02) if rng.rand() < 0.5 else rng.uniform(0.90, 0.94)
    return base + np.array([0.0, 0.02, 0.04]) + rng.uniform(-0.004, 0.004, 3)


def _well_conditioned(sig, plastic):
    s = np.sort(sig)
    gaps = np.diff(s)
    inside = (s > PL_LO + 2e-4) & (s < PL_HI - 2e-4)
    need = np.where(inside[:-1] & inside[1:], 1e-3, 1e-2) if plastic else 1e-2
    if (gaps < need).any():
        return False
    return not (plastic and (np.abs(s[:, None] - np.array([PL_LO, PL_HI])[None]) < 2e-4).any())


def bwd_state(rng, x, n, sort, liquid):
    """materials and v, C, F of frame f (see the module docstring).  Sorted layouts take the material of the particle's stencil column, so that
    the cell-sorted warps hold one row; unsorted layouts draw it per particle, so that warps mix rows."""
    from fluidlab_b200 import macros as M
    mats = np.array(materials(liquid), np.int32)
    N = len(x)
    b = np.trunc(np.asarray(x, np.float64) * n - 0.5).astype(np.int64)
    mat = mats[(b[:, 0] * 3 + b[:, 1]) % len(mats)] if sort else mats[rng.randint(len(mats), size=N)]
    v = rng.uniform(-0.28, 0.28, size=(N, 3)).astype(np.float32)
    C = (rng.randn(N, 3, 3) * 2.0).astype(np.float32)
    plastic = np.isin(mat, [M.ICECREAM, M.PLASTIC_DEMO])
    F = np.empty((N, 3, 3), np.float32)
    for p in range(N):
        for _ in range(100):
            Ft = _rot(rng) @ np.diag(_sigmas(rng, plastic[p])) @ _rot(rng).T
            F[p] = (np.linalg.solve(np.eye(3) + DT * C[p].astype(np.float64), Ft)).astype(np.float32)
            if _well_conditioned(np.linalg.svd(f_tilde(F[p:p + 1], C[p:p + 1])[0], compute_uv=False), plastic[p]):
                break
        else:
            raise AssertionError('no well-conditioned F drawn')
    return mat, v, C, F, plastic


# ------------------------------------------------------------------------------------------------------------------ setup
def setup(name, n, liquid, device, seed=SEED, field=False):
    """the simulator with frame 0 of the layout (cell-sorted where the layout says so) and the census; field: general materials only, a
    random per-particle (mu, lam) bound with set_material_field, and ctx['P'] / ctx['Po'] carry it for the oracle and the bars"""
    assert not (field and liquid), 'a material field runs the general kernels'
    rng = np.random.RandomState(seed)
    lay = layout(name, n, rng)
    x, used, frozen = lay['x'], lay['used'], lay['frozen']
    N = len(x)
    mat, v0, C0, F0, plastic = bwd_state(rng, x, n, lay['sort'], liquid)
    P = make_particles(x, mat, n, used=used)
    s = _sim(n, P, device)
    if field:
        mu_p, lam_p = random_field(P, rng, zero_frac=FIELD_ZERO_FRAC)
        P = dict(P, mu=mu_p, lam=lam_p)
        s.set_material_field(mu_p, lam_p)
    s.enable_grad()
    s.setframe(0, x, v0, C0, F0, used)
    if lay['sort']:
        s.sort_frame(0)
    ids = s._frame_ord[0].ids
    ids = np.arange(N) if ids is None else ids.cpu().numpy().astype(np.int64)
    table = s.get_material_table()
    row = np.searchsorted(table['mat'], mat)
    assert np.array_equal(table['mat'][row], mat), 'one material-table row per material'
    cen = bwd_census(x[ids], used[ids], row[ids], n)
    check_counts(name, cen['counts'])
    live = (used != 0) & ~frozen   # the oracle does not freeze particles: the frozen ones are unused there
    sig = np.linalg.svd(f_tilde(F0, C0), compute_uv=False)
    pairs = plastic_pairs(sig) * (plastic & live)[:, None]
    cen['counts'].update(plastic_pass=int(pairs[:, 0].sum()), plastic_mixed=int(pairs[:, 1].sum()), plastic_same=int(pairs[:, 2].sum()))
    if field:
        cen['counts'].update(field_counts(P, P['mu'], live))
    check_bwd_counts(name, cen['counts'], not liquid, field)
    ok = np.empty(N, bool); ok[ids] = cen['ok']
    assert np.array_equal(ok & (used != 0), live), 'every used particle must be inside the grid at frame f, except the frozen ones'
    warp_of = np.empty(N, np.int64); warp_of[ids] = np.arange(N) // 32
    Po = dict(make_particles(x, mat, n, used=live.astype(np.int32)), mu=P['mu'], lam=P['lam'])
    return dict(rng=rng, x=x, used=used, live=live, v=v0, C=C0, F=F0, P=P, Po=Po, s=s, cen=cen, warp_of=warp_of, n=n, name=name, row=row,
                pairs=pairs, plastic=plastic, liquid=liquid, field=field, ids=ids)


# ------------------------------------------------------------------------------------------------------------------ bars
def _where(ctx, pid):
    w = int(ctx['warp_of'][pid])
    pp = ctx['pairs'][pid]
    br = f'plastic pairs pass/mixed/same {pp[0]}/{pp[1]}/{pp[2]}' if ctx['plastic'][pid] else 'not plastic'
    mu = f', mu_p {ctx["P"]["mu"][pid]:.6g}' if ctx['field'] else ''
    return f'particle {pid} (row {ctx["row"][pid]}{mu}, {br}), warp {w} (backward footprint {ctx["cen"]["bwd"][w]})'


def _check_particles(ctx, what, got, ref, key, bar):
    e = particle_errors(got, ref, ctx['live'])
    i = int(np.argmax(e))
    pid = int(np.where(ctx['live'])[0][i])
    assert e[i] < bar, f'{what}: {key} error {e[i]:.3g} (bar {bar:g}) at {_where(ctx, pid)}'
    return float(e[i])


def g2p_grad_scale(n, x, gx, gv, gC, live, dt=DT):
    """S_i of the v_out adjoint bar, in fp64: sum_p |w_ip| (|gv_p + dt gx_p|_k + sum_j |4 inv_dx gC_p,kj| (|fx_j| + o_j)), per component k; p over
    the used particles of frame f (k_g2p_grad_scatter's q = gv + dt gx - B fx plus B o, B = 4 inv_dx gC)"""
    G = n ** 3
    x, gx, gv, gC = [np.asarray(a, np.float64)[live] for a in (x, gx, gv, gC)]
    b, fx, w = weights(x * n)
    Babs = np.abs(4.0 * n * gC)
    q = np.abs(gv + dt * gx)
    S = np.zeros((G, 3))
    for o in itertools.product(range(3), repeat=3):
        wt = np.abs(w[:, o[0], 0] * w[:, o[1], 1] * w[:, o[2], 2])
        node = ((b[:, 0] + o[0]) * n + b[:, 1] + o[1]) * n + b[:, 2] + o[2]
        np.add.at(S, node, wt[:, None] * (q + np.einsum('pkj,pj->pk', Babs, np.abs(fx) + np.array(o, np.float64))))
    return S


def walls(vin, m, n):
    """the cube's wall test of grid_op at every node in fp64 from the fp32 grid: v = p / m + dt g, per axis whether the node is past a wall
    (`past`), whether it reflects (`hit`) and whether fp32 may decide otherwise (`ambiguous`: |v| <= 8 U (|p / m| + dt |g|))"""
    G = n ** 3
    idx = np.stack(np.unravel_index(np.arange(G), (n, n, n)), 1).astype(np.float64)
    pos = idx * np.float64(np.float32(1.0 / n))
    lo, hi = np.float32(BOUNDARY['lower']).astype(np.float64), np.float32(BOUNDARY['upper']).astype(np.float64)
    m = np.asarray(m, np.float64)
    has = m > np.float64(np.float32(1e-12))
    with np.errstate(divide='ignore', invalid='ignore'):
        pm = np.where(has[:, None], np.asarray(vin, np.float64) / m[:, None], 0.0)
    g = DT * np.asarray(GRAVITY, np.float64)
    v = pm + g
    up, down = pos >= hi, pos <= lo
    hit = has[:, None] & ((up & (v >= 0)) | (down & (v <= 0)))
    ambiguous = has[:, None] & (up | down) & (np.abs(v) <= 8 * U * (np.abs(pm) + np.abs(g)))
    return dict(has=has, past=has[:, None] & (up | down), hit=hit, ambiguous=ambiguous, v=v)


def field_grad_scale(n, x, C, F, ga_vin, dt=DT):
    """S_p of the per-slot bar of dL/dmu_p and dL/dlam_p, in fp64, per particle of x (already restricted to the live ones): the terms
    2 k_stress gA : ((F~ - R) F~^T) and k_stress J (J - 1) tr gA with every factor taken in absolute value before its cancellations, as fp32
    evaluates them.  |gA| = dx sum_i |w_i| |a_i| (o_i + |fx|)^T (k_particle_grad forms gA = dx (sum_i w_i a_i o_i^T - (sum_i w_i a_i) fx^T)); the
    mu term takes (|F~| + |R|) |F~|^T, the lam term |J| (D + 1) with D the sum of the absolute products of det F~ (J - 1 loses the digits J and
    1 share)."""
    x, C, F = [np.asarray(a, np.float64) for a in (x, C, F)]
    ga_vin = np.asarray(ga_vin, np.float64)
    dx = 1.0 / n
    k_stress = abs(-dt * (dx * 0.5) ** 2 * 4 * n * n)
    b, fx, w = weights(x * n)
    gA = np.zeros((len(x), 3, 3))
    for o in itertools.product(range(3), repeat=3):
        wt = np.abs(w[:, o[0], 0] * w[:, o[1], 1] * w[:, o[2], 2])
        node = ((b[:, 0] + o[0]) * n + b[:, 1] + o[1]) * n + b[:, 2] + o[2]
        gA += wt[:, None, None] * np.abs(ga_vin[node])[:, :, None] * ((np.array(o, np.float64) + np.abs(fx)) * dx)[:, None, :]
    Ft = f_tilde(F, C)
    J = np.linalg.det(Ft)
    Us, _, Vt = np.linalg.svd(Ft)
    A = np.abs(Ft)
    D = sum(A[:, 0, i] * A[:, 1, j] * A[:, 2, k] for i, j, k in itertools.permutations(range(3)))
    s_mu = 2 * k_stress * (gA * ((A + np.abs(Us @ Vt)) @ np.transpose(A, (0, 2, 1)))).sum((1, 2))
    s_lam = k_stress * np.abs(J) * (D + 1) * np.trace(gA, axis1=1, axis2=2)
    return s_mu, s_lam


# ------------------------------------------------------------------------------------------------------------------ the launches
def _sentinel(t):
    t.fill_(1234.5)


def run(name, n, liquid, device=None, seed=SEED, field=False):
    """steps 1 - 6 of the module docstring on one layout, with the material table or (field) a per-particle material field; returns the
    census counts and the largest errors"""
    import torch
    from oracle import oracle as orc
    ctx = setup(name, n, liquid, device, seed, field)
    s, live, used, rng = ctx['s'], ctx['live'], ctx['used'], ctx['rng']
    N, G, f = len(live), n ** 3, 0
    idle = ~live
    tag = f'{name} n={n} {"field" if field else "liquid" if liquid else "general"}'
    err = {}
    s._frame_ord[f + 1] = s._frame_ord[f]
    o = orc.OracleSim(n, ctx['Po'], gravity=GRAVITY, boundary=BOUNDARY, precision=64, max_substeps_local=10)
    L = o.L
    o.set_frame(f, ctx['x'], ctx['v'], ctx['C'], ctx['F'], live)
    # 1. k_p2g: the recompute (write_F = 0), then the forward (write_F = 1, also F[f+1])
    L.orc_phase_reset_grid(o.h); L.orc_phase_p2g(o.h, f, 1)
    rvin, rm, _ = o.get_grid()
    Sv, Sm = scatter_scale(n, ctx['x'], ctx['v'], ctx['C'], ctx['F'], ctx['P'], live)
    for wf in (0, 1):
        s.phase('clear_grid', f); s.phase('p2g', f, wf)
        vin, m, _ = s.read_grid()
        r = max(grid_ratio(vin, rvin, Sv), grid_ratio(m, rm, Sm))
        assert r <= GRID_C, f'{tag} k_p2g(write_F={wf}): accumulator off by {r:.3g} x 2^-23 S_i (bar {GRID_C})'
        assert np.array_equal(m != 0, rm != 0), f'{tag} k_p2g(write_F={wf}): the nodes with mass differ'
        err['p2g'] = max(err.get('p2g', 0.0), r)
    F1 = s.readframe(f + 1, ('F',))['F']
    err['F'] = _check_particles(ctx, f'{tag} k_p2g(write_F=1)', F1, o.get_frame(f + 1)['F'], 'F[f+1]', BARS['F'])
    # 2. k_grid_op + k_g2p, against the oracle's grid_op and g2p on the kernel's accumulator
    s.phase('grid_op', f, 0)
    vin, m, vout = s.read_grid()
    s.phase('g2p', f)
    fr = s.readframe(f + 1)
    o.set_grid(vin, m); L.orc_phase_grid_op(o.h, f); L.orc_phase_g2p(o.h, f)
    ref = o.get_frame(f + 1)
    for k in ('x', 'v', 'C'):
        err[k] = _check_particles(ctx, f'{tag} k_g2p', fr[k], ref[k], k, BARS[k])
    for k, a in (('x', ctx['x']), ('v', ctx['v']), ('C', ctx['C']), ('F', ctx['F'])):
        assert np.array_equal(fr[k][idle], a[idle]), f'{tag} k_g2p: unused / frozen slots must be carried over untouched ({k})'
    # the adjoint of frame f+1, random O(1)
    g = {k: rng.randn(*sh).astype(np.float32) for k, sh in (('x', (N, 3)), ('v', (N, 3)), ('C', (N, 3, 3)), ('F', (N, 3, 3)))}
    for pg in (False, True):
        what = f'{tag}{" param_grad" if pg else ""}'
        s.param_grad = pg
        s.cur_substep_global = f + 1
        s.reset_grad(); s.set_grad(g['x'], g['v'], g['C'], g['F'])
        s.cur_substep_global = f
        s._ensure_grad_order(s._frame_ord[f])
        # 3. k_g2p_grad_scatter
        s.phase('g2p_grad_scatter', f)
        _, _, ggv = s.read_grid_grad()
        o.reset_grad(); o.set_grad_frame(f + 1, g['x'], g['v'], g['C'], g['F'])
        o.set_grid_grad(np.zeros((G, 3)), np.zeros(G), np.zeros((G, 3)))
        L.orc_phase_g2p_grad(o.h, f)
        _, _, rggv = o.get_grid_grad()
        S = g2p_grad_scale(n, ctx['x'], g['x'], g['v'], g['C'], live)
        r = grid_ratio(ggv, rggv, S)
        assert r <= SC_C, f'{what} k_g2p_grad_scatter: v_out adjoint off by {r:.3g} x 2^-23 S_i (bar {SC_C}) at node {tuple(int(i) for i in np.unravel_index(int(np.argmax(np.abs(ggv - rggv).max(1))), (n, n, n)))}'
        err['scatter'] = max(err.get('scatter', 0.0), r)
        # 4. k_grid_op_grad on the kernel's grid and v_out adjoint; nodes outside the active blocks keep what they held
        _sentinel(s._ggrid_pm)
        blk = s._blk_flags.cpu().numpy().copy()
        s.phase('grid_op_grad', f)
        gvin, gm, _ = s.read_grid_grad()
        o.set_grid_grad(np.zeros((G, 3)), np.zeros(G), ggv)
        L.orc_phase_grid_op_grad(o.h, f)
        rgvin, rgm, _ = o.get_grid_grad()
        nb = n // 8
        I = np.stack(np.unravel_index(np.arange(G), (n, n, n)), 1) // 8
        active = blk[(I[:, 0] * nb + I[:, 1]) * nb + I[:, 2]] != 0
        W = walls(vin, m, n)
        has = W['has']
        assert (gvin[~active] == 1234.5).all() and (gm[~active] == 1234.5).all(), f'{what} k_grid_op_grad wrote outside the active blocks'
        assert has[~active].sum() == 0, 'a node with mass outside the active blocks'
        dead = active & ~has
        assert (gvin[dead] == 0).all() and (gm[dead] == 0).all(), f'{what} k_grid_op_grad: nodes without mass must be exactly 0'
        amb = W['ambiguous']
        mm = np.where(has, np.asarray(m, np.float64), 1.0)
        gvabs = np.abs(ggv.astype(np.float64))
        with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
            rv = np.where(has[:, None] & ~amb, np.abs(gvin - rgvin) / (U * np.maximum(gvabs, 1e-30) / mm[:, None]), 0.0)
            mscale = (np.abs(np.asarray(vin, np.float64)) * gvabs).sum(1) / mm ** 2
            rmass = np.where(has & ~amb.any(1), np.abs(gm - rgm) / (U * np.maximum(mscale, 1e-300)), 0.0)
        n_past, n_amb = int(W['past'].sum()), int(amb.sum())
        assert n_amb <= AMBIG_FRAC * max(n_past, 1), f'{what}: {n_amb} of {n_past} wall node axes are within rounding of v = 0'
        if name in ('high_edge', 'low_edge'):
            assert n_past - n_amb >= 100, f'{what}: only {n_past - n_amb} wall node axes checked'
        bad = int(np.argmax(rv.max(1)))
        assert rv.max() <= GOP_C, f'{what} k_grid_op_grad: v_in adjoint off by {rv.max():.3g} ulp-scale (bar {GOP_C}) at node {tuple(int(i) for i in np.unravel_index(bad, (n, n, n)))}, wall axes {W["past"][bad]}'
        assert rmass.max() <= GOP_C, f'{what} k_grid_op_grad: mass adjoint off by {rmass.max():.3g} ulp-scale (bar {GOP_C})'
        err['grid_op_grad'] = max(err.get('grid_op_grad', 0.0), float(rv.max()), float(rmass.max()))
        err['walls'] = (n_past, n_amb)
        fr0 = dict(x=ctx['x'].astype(np.float64), v=ctx['v'].astype(np.float64), C=ctx['C'].astype(np.float64), F=ctx['F'].astype(np.float64),
                   used=live.astype(np.int32))
        if pg:   # the parameter-gradient terms per particle, from the kernel's own grid adjoint
            t_k = param_grad_terms(fr0, np.asarray(m, np.float64), np.asarray(gvin, np.float64), np.asarray(gm, np.float64), n, DT)
        if pg and field:   # gfield is a read-modify-write add per live slot: prefill it with values the size of the terms
            pre = np.stack([rng.randn(N) * np.sqrt(np.mean(t_k[k] ** 2)) for k in ('mu', 'lam')], 1).astype(np.float32)
            s._gfield.copy_(torch.from_numpy(pre).to(s._gfield.device))
        # 5. k_particle_grad on the kernel's grid adjoint
        s.phase('particle_grad', f)
        gg = s.get_grad()
        L.orc_phase_reset_grid(o.h); o.set_grid(vin, m); L.orc_phase_grid_op(o.h, f)
        o.reset_grad(); o.set_grad_frame(f + 1, g['x'], g['v'], g['C'], g['F'])
        L.orc_phase_g2p_grad(o.h, f)
        _, _, og_vout = o.get_grid_grad()
        o.set_grid_grad(gvin, gm, og_vout)   # after g2p_grad, which writes the grid adjoint too
        L.orc_phase_p2g_grad(o.h, f); L.orc_phase_unused_grad(o.h, f)
        og = o.get_grad_frame(f)
        for k in ('x', 'v', 'C', 'F'):
            err[f'g{k}'] = max(err.get(f'g{k}', 0.0), _check_particles(ctx, f'{what} k_particle_grad', gg[k], og[k], f'adjoint of {k}', GRAD_BARS[k]))
            assert np.array_equal(gg[k][idle], g[k][idle]), f'{what} k_particle_grad: unused / frozen slots must pass the adjoint of {k} through'
        if not pg:
            continue
        # 6. the parameter gradients, against fp64 sums of their terms built from the kernel's own inputs
        p = t_k['p']
        if field:
            err.update(_check_field_grad(ctx, what, pre, t_k, gvin))
        got = s.get_param_grad()
        if field:   # the slot-order accumulator (prefill removed above) in original particle order, and its sums per row
            ids = ctx['ids']
            d = ctx.pop('gfield_left').astype(np.float64)
            for j, k in enumerate(('mu_field', 'lam_field')):
                want = np.zeros(N); want[ids] = d[:, j]
                assert np.array_equal(got[k], want), f'{what}: get_param_grad()[{k!r}] is not the slot-order accumulator mapped through ids'
                rows = np.bincount(ctx['row'], weights=want, minlength=len(got['mu']))
                key = k[:-6]
                assert np.allclose(got[key], rows, rtol=1e-12, atol=1e-300), f'{what}: get_param_grad()[{key!r}] is not the row sum of {k!r}'
        # the reflected axes as the kernel decided them (at an ambiguous node, the zero it wrote)
        hit = np.where(amb, (gvin == 0) & (ggv != 0), W['hit'])
        vb = np.where(hit, 0.0, ggv.astype(np.float64))   # restitution 0: a reflected axis passes no adjoint
        ga_ref = np.where(has[:, None], vb / mm[:, None], 0.0)
        t = param_grad_terms(fr0, np.asarray(m, np.float64), ga_ref, np.asarray(gm, np.float64), n, DT)
        pv = float(np.float32(s.p_vol))
        for k, key, fac in (('mu', 'mu', 1.0), ('lam', 'lam', 1.0), ('mass', 'rho', pv)):
            for r in range(len(got[key])):
                sel = ctx['row'][p] == r
                want, scale = t_k[k][sel].sum() * fac, np.abs(t_k[k][sel]).sum() * fac
                e = abs(got[key][r] - want) / max(scale, 1e-300)
                assert e <= BETA[k], f'{what}: dL/d{k} of row {r} off by {e:.3g} x sum |term| (bar {BETA[k]:g}): {got[key][r]!r} vs {want!r}'
                err[f'd{k}'] = max(err.get(f'd{k}', 0.0), e)
        gscale = DT * np.abs(vb[has]).sum(0)
        eg = np.abs(got['gravity'] - t['gravity']) / np.maximum(gscale, 1e-300)
        assert eg.max() <= BETA['gravity'], f'{what}: dL/dg off by {eg} x sum |term| (bar {BETA["gravity"]:g})'
        wv = W['v']
        rest = -(np.where(hit, wv * ggv, 0.0)).sum()
        rscale = np.abs(np.where(W['past'], wv * ggv, 0.0)).sum()
        er = abs(got['restitution'] - rest) / max(rscale, 1e-300)
        assert er <= BETA['restitution'], f'{what}: dL/d(restitution) off by {er:.3g} x sum |term| (bar {BETA["restitution"]:g}): {got["restitution"]!r} vs {rest!r}'
        err['dg'], err['drest'] = float(eg.max()), er
    s.param_grad = False
    return dict(counts=ctx['cen']['counts'], err=err)


def _check_field_grad(ctx, what, pre, t_k, gvin):
    """k_particle_grad<2, true> against the terms t_k, on the raw slot-order accumulators: per live slot got - prefill against the particle's
    dL/dmu_p, dL/dlam_p (FIELD_C 2^-23 S_p plus one ulp of the prefill), the prefill untouched in unused and frozen slots, the rows' dL/dmu and
    dL/dlam exactly 0.  Leaves got - prefill (fp32) in the accumulator and in ctx['gfield_left'], for the check through get_param_grad()."""
    import torch
    s, ids, live = ctx['s'], ctx['ids'], ctx['live']
    N = len(live)
    raw = s._gfield.cpu().numpy().copy()
    gmat = s._gmat.cpu().numpy()
    assert (gmat[:, 0:2] == 0).all(), f'{what}: with a material field the rows\' dL/dmu and dL/dlam must not be written ({gmat[:, 0:2]})'
    live_s = live[ids]
    idle_s = np.where(~live_s)[0]
    assert np.array_equal(raw[idle_s].view(np.int32), pre[idle_s].view(np.int32)), \
        f'{what}: unused / frozen slots {idle_s[(raw[idle_s] != pre[idle_s]).any(1)][:8].tolist()} must keep their gfield prefill'
    inv = np.empty(N, np.int64); inv[ids] = np.arange(N)
    p = t_k['p']
    sl = inv[p]   # the slot of each live particle
    s_mu, s_lam = field_grad_scale(ctx['n'], ctx['x'][p], ctx['C'][p], ctx['F'][p], gvin)
    err = {}
    for j, (k, S) in enumerate((('mu', s_mu), ('lam', s_lam))):
        got = raw[sl, j].astype(np.float64) - pre[sl, j].astype(np.float64)
        ulp = np.spacing(np.abs(pre[sl, j])).astype(np.float64)
        r = np.maximum(np.abs(got - t_k[k]) - ulp, 0.0) / (U * S)
        i = int(np.argmax(r))
        assert r[i] <= FIELD_C, (f'{what} k_particle_grad<2, true>: dL/d{k}_p off by {r[i]:.3g} x 2^-23 S_p (bar {FIELD_C}) at {_where(ctx, int(p[i]))}: '
                                 f'{got[i]:.9g} vs {t_k[k][i]:.9g} (slot {sl[i]})')
        err[f'field_{k}'] = float(r[i])
    left = raw - pre
    s._gfield.copy_(torch.from_numpy(left).to(s._gfield.device))
    ctx['gfield_left'] = left
    return err
