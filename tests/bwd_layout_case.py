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

With `field='mass'` a random density field (density_field_case.random_rho) is bound too: k_p2g_field_mass and k_particle_grad<3, *>, whose
dL/dm_p goes to the per-slot `gmass` (checked like gfield, MASS_C) and the rows' dL/dmass stays 0 as well.  With `field='plastic'` per-particle
plastic limits are bound on top (random_limits: log-uniform, theta_c = 0, theta_s = 0, both 0, wide windows): k_p2g_field_plastic and
k_particle_grad<4, *>, and each plastic particle's F~ is drawn against its own window (_sigmas_in; with lo == hi one axis below 1 and one above,
clamped at different bounds to the same value).  The oracle clamps to the constants, so its F[f+1] is clamped again to the particles' own
windows and its adjoint of frame f gets plastic_grad_ref.limit_grad's correction; the plastic record's accumulator `gpfield` holds
(dmu, dlam, dlo, dhi) per slot: dlo / dhi against limit_grad's fp64 sums where the particle has an axis at that bound (LIM_C), the prefill bit
for bit where it has none, and the field's own `gfield`, whose pointer slots the record takes, untouched.

F is well conditioned by construction: F~ = Q1 diag(s) Q2^T is drawn and F = (I + dt C)^-1 F~ rounded to fp32; a particle whose fp64 F~ has two
singular values closer than 1e-2 (1e-3 for a pair inside the plastic window, whose adjoint takes no 1 / (s_j^2 - s_i^2)), or, in a plastic
row, a singular value within 2e-4 of a clamp bound, is drawn again.  Repeated singular values are out of scope: U and V are not unique there,
fp32 and fp64 may take different branches, and the reference's clamp turns the adjoint into O(1e8) x 0."""
import itertools

import numpy as np

from conftest import make_particles
from density_field_case import particle_mass, random_rho
from material_field_case import random_field
from plastic_grad_ref import limit_grad, limits, reclamp
from plastic_limits_case import random_theta
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
# With a mass field and with plastic limits (k_particle_grad<3 | 4, *>), the largest errors over every layout on the H100 (80 GB HBM3, 700 W)
# at n = 32 and 64 / on the CPU shim at n = 32 with and without FMA contraction: k_p2g 3.0 / 2.7, F[f+1] 1.3e-6 / 1.1e-6; k_g2p 7.5e-8,
# 2.9e-6, 6.7e-6 / 7.4e-8, 2.6e-6, 5.6e-6; scatter 2.1 / 2.0; grid_op_grad 2.0 / 2.1; adjoints 7.3e-5, 8.8e-6, 1.3e-5, 2.5e-5 / 3.6e-5,
# 4.8e-6, 1.5e-5, 1.5e-5; per slot mu 0.34 / 0.16, lam 1.05 / 0.86, mass 2.4 / 1.35 (MASS_C), lo 16.1 / 15, hi 17.2 / 12 (LIM_C); rows mu
# 1.2e-6 / 1.4e-6, lam 6.7e-6 / 2.8e-6, mass 5.6e-8 / 8.1e-8; gravity 9.4e-9 / 1.1e-8, restitution 2.6e-8 / 2.0e-8.  dL/dlo_p and dL/dhi_p
# take U and V of the fp32 SVD, whose axes turn by about 2^-23 / (gap of the singular values, >= 1e-2 for a clamped axis) against fp64's
MASS_C = 12   # k_particle_grad<3 | 4, true>: dL/dm_p per slot (gmass), in units of 2^-23 S_p (mass_grad_scale), on top of one ulp of the prefill
LIM_C = 85    # k_particle_grad<4, true>: dL/dlo_p, dL/dhi_p per slot (gpfield.zw), in units of 2^-23 sum_d (|U|^T |gF'| |V|)_dd
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
# with per-particle plastic limits (setup(field='plastic'), about half the counts of the seed at n = 32 and n = 64): the pairs as above, counted
# against each particle's own window; `cross` the pairs clamped at different bounds to the same value (lo == hi); the live plastic particles
# with an axis clamped at lo = 1 (`lo1`) or hi = 1 (`hi1`) exactly, with a wide window (nothing clamps) and with an axis at lo / hi (their
# dL/dlo / dL/dhi gets a term)
MIN_PLASTIC_FIELD = {
    'dense': dict(plastic_pass=381, plastic_mixed=657, plastic_same=660, plastic_cross=71, plastic_lo1=87, plastic_hi1=83, plastic_wide=93, plastic_dlo=343, plastic_dhi=341),
    'zruns': dict(plastic_pass=224, plastic_mixed=386, plastic_same=442, plastic_cross=51, plastic_lo1=49, plastic_hi1=53, plastic_wide=53, plastic_dlo=202, plastic_dhi=208),
    'long': dict(plastic_pass=88, plastic_mixed=136, plastic_same=166, plastic_cross=16, plastic_lo1=20, plastic_hi1=20, plastic_wide=20, plastic_dlo=74, plastic_dhi=74),
    'high_edge': dict(plastic_pass=125, plastic_mixed=249, plastic_same=249, plastic_cross=29, plastic_lo1=32, plastic_hi1=33, plastic_wide=28, plastic_dlo=118, plastic_dhi=132),
    'low_edge': dict(plastic_pass=79, plastic_mixed=200, plastic_same=201, plastic_cross=22, plastic_lo1=25, plastic_hi1=23, plastic_wide=16, plastic_dlo=101, plastic_dhi=100),
    'ragged': dict(plastic_pass=75, plastic_mixed=151, plastic_same=114, plastic_cross=15, plastic_lo1=17, plastic_hi1=19, plastic_wide=17, plastic_dlo=70, plastic_dhi=68),
}
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


def clamp_sides(sig, lo=PL_LO, hi=PL_HI):
    """per axis, where constitutive_grad's clamp puts it (the tie rule of plastic_grad_ref.clamp): -1 at lo, +1 at hi, 0 passes; and the clamped
    value sp.  lo, hi: scalars or one per particle (rounded to fp32 either way)"""
    lo, hi = [np.broadcast_to(np.asarray(a, np.float32).astype(np.float64), (len(sig),))[:, None] for a in (lo, hi)]
    side = np.where(sig <= lo, -1, np.where(sig >= hi, 1, 0))
    return side, np.where(side < 0, lo, np.where(side > 0, hi, sig))


def plastic_pairs(sig, lo=PL_LO, hi=PL_HI):
    """per particle, the number of pairs (i, j) of constitutive_grad in each branch, counted by value as the kernel branches: [both pass, mixed,
    both clamped to the same value (sp_i == sp_j), of those the pairs clamped at different bounds (lo == hi: one axis below, one above)]"""
    side, sp = clamp_sides(sig, lo, hi)
    out = np.zeros((len(sig), 4), np.int64)
    for i, j in ((0, 1), (0, 2), (1, 2)):
        a, b = side[:, i], side[:, j]
        both = (a == 0) & (b == 0)
        same = (a != 0) & (b != 0) & (sp[:, i] == sp[:, j])
        out[:, 0] += both
        out[:, 2] += same
        out[:, 3] += same & (a != b)
        out[:, 1] += ~(both | same)
    return out


def plastic_counts(sig, sel, lo=PL_LO, hi=PL_HI, wide=None):
    """the census of the plastic pairs over the particles `sel` (live, plasto-elastic) and, with per-particle windows, the particles with an
    axis clamped at lo = 1 / at hi = 1 exactly, the wide-window particles (`wide`) and the particles whose dL/dlo / dL/dhi gets a term"""
    pairs = plastic_pairs(sig, lo, hi) * sel[:, None]
    c = dict(plastic_pass=int(pairs[:, 0].sum()), plastic_mixed=int(pairs[:, 1].sum()), plastic_same=int(pairs[:, 2].sum()))
    if wide is not None:
        side, _ = clamp_sides(sig, lo, hi)
        at_lo, at_hi = sel & (side < 0).any(1), sel & (side > 0).any(1)
        lo32, hi32 = [np.asarray(a, np.float32) for a in (lo, hi)]
        c.update(plastic_cross=int(pairs[:, 3].sum()), plastic_lo1=int((at_lo & (lo32 == 1)).sum()), plastic_hi1=int((at_hi & (hi32 == 1)).sum()),
                 plastic_wide=int((sel & wide).sum()), plastic_dlo=int(at_lo.sum()), plastic_dhi=int(at_hi.sum()))
    return pairs, c


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
    want = dict(MIN_BWD[name], **(MIN_PLASTIC_FIELD[name] if field == 'plastic' else MIN_PLASTIC if plastic else {}),
                **(MIN_FIELD[name] if field else {}))
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


def _sigmas_in(rng, lo, hi):
    """_sigmas relative to a particle's own window [lo, hi]: a wide window (hi - lo >= 0.1) holds all three axes (nothing clamps); lo == hi
    mostly takes one axis below 1 and one above (clamped at different bounds to the same value), else all three beyond one bound; other
    windows draw the three shapes of _sigmas that fit in them (both pass needs a width of 2e-3, mixed 1e-3), 4e-4 inside the bounds"""
    w = hi - lo
    if w >= 0.1:
        return 1.0 + np.array([-0.04, 0.0, 0.04]) + rng.uniform(-0.005, 0.005, 3)
    if w == 0 and rng.rand() < 0.7:
        far = lo - rng.uniform(0.07, 0.12) if rng.rand() < 0.5 else hi + rng.uniform(0.07, 0.12)
        return np.array([lo - rng.uniform(0.005, 0.05), hi + rng.uniform(0.005, 0.05), far])
    shapes = [('same', 0.35)] + ([('mixed', 0.35)] if w >= 1e-3 else []) + ([('pass', 0.3)] if w >= 2e-3 else [])
    p = np.array([q for _, q in shapes])
    shape = shapes[rng.choice(len(shapes), p=p / p.sum())][0]
    if shape == 'pass':
        a = rng.uniform(lo + 4e-4, hi - 1.6e-3)
        return np.array([a, rng.uniform(a + 1.2e-3, hi - 4e-4), lo - rng.uniform(0.03, 0.07) if rng.rand() < 0.5 else hi + rng.uniform(0.03, 0.07)])
    if shape == 'mixed':
        return np.array([rng.uniform(lo + 4e-4, hi - 4e-4), lo - rng.uniform(0.02, 0.10), hi + rng.uniform(0.02, 0.10)])
    base = hi + rng.uniform(0.005, 0.017) if rng.rand() < 0.5 else lo - rng.uniform(0.06, 0.10)
    return base + np.array([0.0, 0.02, 0.04]) + rng.uniform(-0.004, 0.004, 3)


def _well_conditioned(sig, plastic, lo=PL_LO, hi=PL_HI):
    s = np.sort(sig)
    gaps = np.diff(s)
    inside = (s > lo + 2e-4) & (s < hi - 2e-4)
    need = np.where(inside[:-1] & inside[1:], 1e-3, 1e-2) if plastic else 1e-2
    if (gaps < need).any():
        return False
    return not (plastic and (np.abs(s[:, None] - np.array([lo, hi])[None]) < 2e-4).any())


PL_WIDE = (0.05, 0.3)   # theta_c, theta_s of a wide window: 1 +- 0.045 stays inside it


def random_limits(rng, N):
    """theta_c, theta_s per particle (fp32-representable) and the wide-window mask: 55 % log-uniform over 1/4 .. 4x the defaults
    (plastic_limits_case.random_theta), 10 % theta_c = 0 (lo = 1), 10 % theta_s = 0 (hi = 1), 10 % both 0 (lo == hi), 15 % a wide window"""
    tc, ts = random_theta(N, rng)
    k = np.digitize(rng.rand(N), [0.55, 0.65, 0.75, 0.85])   # 0 random, 1 theta_c = 0, 2 theta_s = 0, 3 both, 4 wide
    tc[(k == 1) | (k == 3)] = 0.0
    ts[(k == 2) | (k == 3)] = 0.0
    wide = k == 4
    for t in (tc, ts):
        t[wide] = rng.uniform(*PL_WIDE, int(wide.sum())).astype(np.float32)
    return tc, ts, wide


def bwd_state(rng, x, n, sort, liquid, lim=None):
    """materials and v, C, F of frame f (see the module docstring).  Sorted layouts take the material of the particle's stencil column, so that
    the cell-sorted warps hold one row; unsorted layouts draw it per particle, so that warps mix rows.  lim: (lo, hi) per particle, the plastic
    particles' own windows (_sigmas_in); None keeps the constants."""
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
        own = lim is not None and plastic[p]
        win = (lim[0][p], lim[1][p]) if own else (PL_LO, PL_HI)
        for _ in range(100):
            Ft = _rot(rng) @ np.diag(_sigmas_in(rng, *win) if own else _sigmas(rng, plastic[p])) @ _rot(rng).T
            F[p] = (np.linalg.solve(np.eye(3) + DT * C[p].astype(np.float64), Ft)).astype(np.float32)
            if _well_conditioned(np.linalg.svd(f_tilde(F[p:p + 1], C[p:p + 1])[0], compute_uv=False), plastic[p], *win):
                break
        else:
            raise AssertionError('no well-conditioned F drawn')
    return mat, v, C, F, plastic


# ------------------------------------------------------------------------------------------------------------------ setup
FIELDS = {False: 'table', True: 'field', 'mass': 'mass', 'plastic': 'plastic'}   # the field states of setup, by the kind names of the tests


def draw(name, n, liquid, seed=SEED, field=False):
    """the host half of setup: the layout, frame 0 and the per-particle fields, in the order setup draws them"""
    assert field in FIELDS and not (field and liquid), 'a material field runs the general kernels'
    rng = np.random.RandomState(seed)
    lay = layout(name, n, rng)
    N = len(lay['x'])
    theta = random_limits(rng, N) if field == 'plastic' else None
    lim = limits(*theta[:2]) if theta else None
    mat, v0, C0, F0, plastic = bwd_state(rng, lay['x'], n, lay['sort'], liquid, lim)
    P = Pt = make_particles(lay['x'], mat, n, used=lay['used'])
    if field:
        mu_p, lam_p = random_field(P, rng, zero_frac=FIELD_ZERO_FRAC)
        P = dict(P, mu=mu_p, lam=lam_p)
    if field in ('mass', 'plastic'):   # random_rho's own spread (x 1/4 .. 4 of the row's, bounded below by (n / 64)^2)
        rho = random_rho(P, rng, n=n)
        P = dict(P, rho=rho, mass=particle_mass(rho, (0.5 / n) ** 2))
    return dict(rng=rng, lay=lay, mat=mat, v=v0, C=C0, F=F0, plastic=plastic, P=P, Pt=Pt, theta=theta, lim=lim)


def setup(name, n, liquid, device, seed=SEED, field=False):
    """the simulator with frame 0 of the layout (cell-sorted where the layout says so) and the census; field (general materials only): True, a
    random per-particle (mu, lam) bound with set_material_field; 'mass', that and a random density field (set_density_field); 'plastic', those
    and per-particle plastic limits (set_plastic_field, random_limits) with each plastic particle's F drawn against its own window.
    ctx['P'] / ctx['Po'] carry the fields (mu, lam, mass) for the oracle and the bars, ctx['lim'] the windows (lo, hi)."""
    d = draw(name, n, liquid, seed, field)
    rng, lay, mat, v0, C0, F0, plastic, P, lim = [d[k] for k in ('rng', 'lay', 'mat', 'v', 'C', 'F', 'plastic', 'P', 'lim')]
    x, used, frozen = lay['x'], lay['used'], lay['frozen']
    N = len(x)
    s = _sim(n, d['Pt'], device)   # (built on the material table's rows)
    if field:
        s.set_material_field(P['mu'], P['lam'])
    if field in ('mass', 'plastic'):
        assert s.p_vol == (0.5 / n) ** 2
        s.set_density_field(P['rho'])
    if field == 'plastic':
        s.set_plastic_field(*d['theta'][:2])
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
    pairs, pc = plastic_counts(sig, plastic & live, *(lim or (PL_LO, PL_HI)), None if lim is None else d['theta'][2])
    cen['counts'].update(pc)
    if field:
        cen['counts'].update(field_counts(P, P['mu'], live))
    check_bwd_counts(name, cen['counts'], not liquid, field)
    ok = np.empty(N, bool); ok[ids] = cen['ok']
    assert np.array_equal(ok & (used != 0), live), 'every used particle must be inside the grid at frame f, except the frozen ones'
    warp_of = np.empty(N, np.int64); warp_of[ids] = np.arange(N) // 32
    Po = dict(make_particles(x, mat, n, used=live.astype(np.int32)), mu=P['mu'], lam=P['lam'], mass=P['mass'])
    return dict(rng=rng, x=x, used=used, live=live, v=v0, C=C0, F=F0, P=P, Po=Po, s=s, cen=cen, warp_of=warp_of, n=n, name=name, row=row,
                pairs=pairs, plastic=plastic, liquid=liquid, field=field, ids=ids, lim=lim, own=None if lim is None else plastic & live)


def own_clamp(ctx, Fn, C, F):
    """the oracle's F[f+1] (Fn, in place) from frame f (C, F) with the live plastic particles clamped to their own windows (the oracle clamps
    to the constants)"""
    if ctx['lim'] is not None:
        reclamp(Fn, C, F, np.where(ctx['own'])[0], *ctx['lim'], DT)


# ------------------------------------------------------------------------------------------------------------------ bars
def _where(ctx, pid):
    w = int(ctx['warp_of'][pid])
    pp = ctx['pairs'][pid]
    br = f'plastic pairs pass/mixed/same/cross {pp[0]}/{pp[1]}/{pp[2]}/{pp[3]}' if ctx['plastic'][pid] else 'not plastic'
    if ctx['plastic'][pid] and ctx['lim'] is not None:
        br += f' in [{ctx["lim"][0][pid]:.9g}, {ctx["lim"][1][pid]:.9g}]'
    mu = f', mu_p {ctx["P"]["mu"][pid]:.6g}, m_p {ctx["P"]["mass"][pid]:.6g}' if ctx['field'] else ''
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
    tag = f'{name} n={n} {FIELDS[field] if field else "liquid" if liquid else "general"}'
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
    rF1 = o.get_frame(f + 1)['F']
    own_clamp(ctx, rF1, ctx['C'], ctx['F'])
    err['F'] = _check_particles(ctx, f'{tag} k_p2g(write_F=1)', F1, rF1, 'F[f+1]', BARS['F'])
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
        if pg and field:   # the per-slot accumulators are read-modify-write adds per live slot: prefill them with values the size of the terms
            pre = {'gfield': np.stack([rng.randn(N) * np.sqrt(np.mean(t_k[k] ** 2)) for k in ('mu', 'lam')], 1).astype(np.float32)}
            if field == 'plastic':   # (dmu, dlam, dlo, dhi) go to the plastic record; the field's own accumulator keeps a sentinel
                pre['gpfield'] = np.concatenate([pre['gfield'], rng.randn(N, 2).astype(np.float32)], 1)
                pre['gfield'] = np.full((N, 2), 1234.5, np.float32)
            if field in ('mass', 'plastic'):
                pre['gmass'] = (rng.randn(N) * np.sqrt(np.mean(t_k['mass'] ** 2))).astype(np.float32)
            for k, a in pre.items():
                getattr(s, '_' + k).copy_(torch.from_numpy(a).to(s.device))
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
        if ctx['lim'] is not None:   # the oracle's p2g adjoint takes the constants' clamp: the particles' own windows, and dL/dlo, dL/dhi
            q = np.where(ctx['own'])[0]
            dlim = np.zeros((N, 2))
            dlim[q, 0], dlim[q, 1] = limit_grad(og, g['F'].astype(np.float64), ctx['C'], ctx['F'], q, *ctx['lim'], ctx['own'], DT)
        for k in ('x', 'v', 'C', 'F'):
            err[f'g{k}'] = max(err.get(f'g{k}', 0.0), _check_particles(ctx, f'{what} k_particle_grad', gg[k], og[k], f'adjoint of {k}', GRAD_BARS[k]))
            assert np.array_equal(gg[k][idle], g[k][idle]), f'{what} k_particle_grad: unused / frozen slots must pass the adjoint of {k} through'
        if not pg:
            continue
        # 6. the parameter gradients, against fp64 sums of their terms built from the kernel's own inputs
        p = t_k['p']
        if field:
            err.update(_check_field_grad(ctx, what, pre, t_k, gvin, gm, g['F'], dlim if ctx['lim'] is not None else None))
        got = s.get_param_grad()
        if field:   # the slot-order accumulators (prefill removed above) in original particle order, and their sums per row
            ids = ctx['ids']
            left = {k: a.astype(np.float64) for k, a in ctx.pop('grad_left').items()}
            d = left['gpfield'] if field == 'plastic' else left['gfield']
            cols = [('mu_field', d[:, 0], 'mu'), ('lam_field', d[:, 1], 'lam')]
            if field in ('mass', 'plastic'):   # dL/drho = p_vol dL/dm
                cols.append(('rho_field', left['gmass'] * float(np.float32(s.p_vol)), 'rho'))
            if field == 'plastic':   # dL/dtheta_c = -dL/dlo, dL/dtheta_s = dL/dhi
                cols += [('theta_c_field', -d[:, 2], 'theta_c'), ('theta_s_field', d[:, 3], 'theta_s')]
            for k, a, key in cols:
                want = np.zeros(N); want[ids] = a
                assert np.array_equal(got[k], want), f'{what}: get_param_grad()[{k!r}] is not the slot-order accumulator mapped through ids'
                rows = np.bincount(ctx['row'], weights=want, minlength=len(got['mu']))
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


def _check_field_grad(ctx, what, pre, t_k, gvin, gm, gF1, dlim):
    """k_particle_grad<2 | 3 | 4, true> against the terms t_k, on the raw slot-order accumulators `pre` names (prefilled with those values):
      - per live slot got - prefill against the particle's dL/dmu_p, dL/dlam_p (gfield, or gpfield.xy with a plastic field; FIELD_C 2^-23 S_p
        plus one ulp of the prefill) and, with a mass field, dL/dm_p (gmass; MASS_C 2^-23 S_p, mass_grad_scale);
      - with a plastic field, dL/dlo_p and dL/dhi_p (gpfield.zw) against `dlim` (plastic_grad_ref.limit_grad, from the fp64 F~ and the adjoint
        gF1 of F[f+1]) where the particle has an axis at that bound (LIM_C 2^-23 sum_d (|U|^T |gF1| |V|)_dd), the prefill bit for bit elsewhere;
        gfield, whose pointer slots the plastic record takes, keeps its sentinel in every slot;
      - unused and frozen slots keep every prefill bit for bit; the rows' dL/dmu, dL/dlam (and with a mass field dL/dmass) stay exactly 0.
    Leaves got - prefill (fp32) in the accumulators and in ctx['grad_left'], for the check through get_param_grad()."""
    import torch
    s, ids, live, field = ctx['s'], ctx['ids'], ctx['live'], ctx['field']
    N = len(live)
    kern = f'k_particle_grad<{ {True: 2, "mass": 3, "plastic": 4}[field] }, true>'
    raw = {k: getattr(s, '_' + k).cpu().numpy().copy() for k in pre}
    gmat = s._gmat.cpu().numpy()
    nrow = 2 if field is True else 3
    assert (gmat[:, 0:nrow] == 0).all(), f'{what}: with a {FIELDS[field]} field the rows\' first {nrow} parameter gradients must not be written ({gmat[:, 0:nrow]})'
    live_s = live[ids]
    idle_s = np.where(~live_s)[0]
    for k in pre:
        keep = np.arange(N) if field == 'plastic' and k == 'gfield' else idle_s
        a, b = raw[k].reshape(N, -1)[keep], pre[k].reshape(N, -1)[keep]
        bad = keep[(a.view(np.int32) != b.view(np.int32)).any(1)]
        assert len(bad) == 0, f'{what}: slots {bad[:8].tolist()} must keep their {k} prefill ({"every slot" if len(keep) == N else "unused / frozen"})'
    inv = np.empty(N, np.int64); inv[ids] = np.arange(N)
    p = t_k['p']
    sl = inv[p]   # the slot of each live particle
    err = {}

    def check(key, col, ref, S, bar, label, k=slice(None)):   # over the live particles p[k]
        a, b = raw[key].reshape(N, -1)[sl[k], col], pre[key].reshape(N, -1)[sl[k], col]
        got = a.astype(np.float64) - b.astype(np.float64)
        r = np.maximum(np.abs(got - ref[k]) - np.spacing(np.abs(b)).astype(np.float64), 0.0) / (U * S[k])
        if len(r) == 0:
            return 0.0
        i = int(np.argmax(r))
        assert r[i] <= bar, (f'{what} {kern}: {label} off by {r[i]:.3g} x 2^-23 S_p (bar {bar}) at {_where(ctx, int(p[k][i]))}: '
                             f'{got[i]:.9g} vs {ref[k][i]:.9g} (slot {sl[k][i]})')
        return float(r[i])
    x, v, C, F = ctx['x'][p], ctx['v'][p], ctx['C'][p], ctx['F'][p]
    s_mu, s_lam = field_grad_scale(ctx['n'], x, C, F, gvin)
    mk = 'gpfield' if field == 'plastic' else 'gfield'
    err['field_mu'] = check(mk, 0, t_k['mu'], s_mu, FIELD_C, 'dL/dmu_p')
    err['field_lam'] = check(mk, 1, t_k['lam'], s_lam, FIELD_C, 'dL/dlam_p')
    if 'gmass' in pre:
        err['field_mass'] = check('gmass', 0, t_k['mass'], mass_grad_scale(ctx['n'], x, v, C, gvin, gm), MASS_C, 'dL/dm_p')
    if field == 'plastic':
        side, _ = clamp_sides(np.linalg.svd(f_tilde(F, C), compute_uv=False), ctx['lim'][0][p], ctx['lim'][1][p])
        S = lim_grad_scale(F, C, gF1[p])
        for col, (lab, at) in enumerate((('dL/dlo_p', (side < 0).any(1) & ctx['own'][p]), ('dL/dhi_p', (side > 0).any(1) & ctx['own'][p]))):
            a, b = raw['gpfield'][sl[~at], 2 + col], pre['gpfield'][sl[~at], 2 + col]
            bad = p[~at][a.view(np.int32) != b.view(np.int32)]
            assert len(bad) == 0, f'{what} {kern}: {lab} written for particles without an axis at that bound, e.g. {_where(ctx, int(bad[0]))}'
            err[('field_dlo', 'field_dhi')[col]] = check('gpfield', 2 + col, dlim[p, col], S, LIM_C, lab, np.where(at)[0])
    left = {k: raw[k] - pre[k] for k in pre if not (field == 'plastic' and k == 'gfield')}
    for k, a in left.items():
        getattr(s, '_' + k).copy_(torch.from_numpy(a).to(s.device))
    if field == 'plastic':
        s._gfield.zero_()   # (the flush adds it into the field's gradient)
    ctx['grad_left'] = left
    return err


def mass_grad_scale(n, x, v, C, ga_vin, ga_m):
    """S_p of the per-slot bar of dL/dm_p, in fp64, per particle of x (the live ones): sum_i |w_i| |am_i| + |v| . sum_i |w_i| |a_i| + |gA| : |C|,
    with |gA| as in field_grad_scale"""
    x, v, C = [np.asarray(a, np.float64) for a in (x, v, C)]
    ga_vin, ga_m = np.abs(np.asarray(ga_vin, np.float64)), np.abs(np.asarray(ga_m, np.float64))
    dx = 1.0 / n
    b, fx, w = weights(x * n)
    gA, ga, sam = np.zeros((len(x), 3, 3)), np.zeros((len(x), 3)), np.zeros(len(x))
    for o in itertools.product(range(3), repeat=3):
        wt = np.abs(w[:, o[0], 0] * w[:, o[1], 1] * w[:, o[2], 2])
        node = ((b[:, 0] + o[0]) * n + b[:, 1] + o[1]) * n + b[:, 2] + o[2]
        gA += wt[:, None, None] * ga_vin[node][:, :, None] * ((np.array(o, np.float64) + np.abs(fx)) * dx)[:, None, :]
        ga += wt[:, None] * ga_vin[node]
        sam += wt * ga_m[node]
    return sam + (np.abs(v) * ga).sum(1) + (gA * np.abs(C)).sum((1, 2))


def lim_grad_scale(F, C, gF1):
    """S_p of the per-slot bar of dL/dlo_p and dL/dhi_p: sum_d (|U|^T |gF1| |V|)_dd with U, V of the fp64 F~"""
    Us, _, Vt = np.linalg.svd(f_tilde(F, C))
    A = np.transpose(np.abs(Us), (0, 2, 1)) @ np.abs(np.asarray(gF1, np.float64)) @ np.transpose(np.abs(Vt), (0, 2, 1))
    return np.trace(A, axis1=1, axis2=2)
