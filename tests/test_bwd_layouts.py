"""The backward substep's kernels one launch at a time against the fp64 oracle (tests/bwd_layout_case.py), on the layouts of
tests/fwd_layout_case.py: k_p2g (recompute and forward), k_grid_op + k_g2p, k_g2p_grad_scatter, k_grid_op_grad and k_particle_grad, the last
two also in their parameter-gradient instantiations, each fed the kernel's own upstream output.  The general materials run k_particle_grad<0>
(SVD adjoint, plastic clamps), the mu = 0 liquids k_particle_grad<1>, a per-particle material field k_p2g_field and k_particle_grad<2>, a
density field too k_p2g_field_mass and k_particle_grad<3>, per-particle plastic limits on top k_p2g_field_plastic and k_particle_grad<4>.

The CPU shim (tests/cuda_emu) runs n = 32 under `-m "not gpu"`; an H100 runs n = 32 and n = 64."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'cuda_emu'))
import harness  # noqa: E402

import bwd_layout_case as case  # noqa: E402

FIELD = {'field': True, 'mass': 'mass', 'plastic': 'plastic'}   # the field states of case.setup by kind


@pytest.fixture
def emu():
    L = harness.enable()
    yield L
    harness.disable()


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')


def _stable_sort_order(x, used, n):
    """the slot order fmpm_sort gives a frame in identity order: a stable sort on the stencil base cell, unused and frozen slots last"""
    ok, b = case.replay_base(x, n)
    key = np.where(ok & (used != 0), (b[:, 0] * n + b[:, 1]) * n + b[:, 2], n ** 3)
    return np.argsort(key, kind='stable')


@pytest.mark.parametrize('liquid', [True, False], ids=['liquid', 'general'])
@pytest.mark.parametrize('n', [32, 64])
@pytest.mark.parametrize('layout', case.LAYOUTS)
def test_every_layout_reaches_the_backward_branches_it_exists_for(layout, n, liquid):
    """the host census without a device, on the replayed sort order: scatter-window carries, shifts, full moves, partial and skipped rounds;
    the backward footprint; the material rows per warp; the plastic branches of the general set (the runs assert the same on the device's
    slot order)"""
    rng = np.random.RandomState(case.SEED)
    lay = case.layout(layout, n, rng)
    x, used, frozen = lay['x'], lay['used'], lay['frozen']
    mat, _, C, F, plastic = case.bwd_state(rng, x, n, lay['sort'], liquid)
    row = np.searchsorted(np.unique(mat), mat)
    ids = _stable_sort_order(x, used, n) if lay['sort'] else np.arange(len(x))
    cen = case.bwd_census(x[ids], used[ids], row[ids], n)
    live = (used != 0) & ~frozen
    pairs = case.plastic_pairs(np.linalg.svd(case.f_tilde(F, C), compute_uv=False)) * (plastic & live)[:, None]
    cen['counts'].update(plastic_pass=int(pairs[:, 0].sum()), plastic_mixed=int(pairs[:, 1].sum()), plastic_same=int(pairs[:, 2].sum()))
    case.check_bwd_counts(layout, cen['counts'], not liquid)
    if layout == 'ragged':   # N = 32 * 20 + 17: the last warp of 128 slots starts at slot 640, runs one round of 17 and skips three
        assert len(x) == 657 and cen['counts']['partial_rounds'] == 1 and cen['counts']['skipped_rounds'] == 3
    else:
        assert len(x) % 32 == 0 and cen['counts']['partial_rounds'] == 0
    sig = np.linalg.svd(case.f_tilde(F, C), compute_uv=False)
    gaps = np.abs(np.diff(np.sort(sig, 1), axis=1)).min(1)
    assert gaps.min() >= 1e-3 and (gaps[~plastic] >= 1e-2).all(), 'singular values of F~ must stay apart'


@pytest.mark.parametrize('n', [32, 64])
@pytest.mark.parametrize('layout', case.LAYOUTS)
def test_every_layout_reaches_the_material_field_branches_it_exists_for(layout, n):
    """the census of the field runs without a device: particles at mu_p = 0 and liquid-class particles at mu_p > 0, on top of the plastic pairs
    and the material rows per warp of the general set"""
    rng = np.random.RandomState(case.SEED)
    lay = case.layout(layout, n, rng)
    x, used, frozen = lay['x'], lay['used'], lay['frozen']
    mat, _, C, F, plastic = case.bwd_state(rng, x, n, lay['sort'], False)
    P = case.make_particles(x, mat, n, used=used)
    mu, lam = case.random_field(P, rng, zero_frac=case.FIELD_ZERO_FRAC)
    row = np.searchsorted(np.unique(mat), mat)
    ids = _stable_sort_order(x, used, n) if lay['sort'] else np.arange(len(x))
    cen = case.bwd_census(x[ids], used[ids], row[ids], n)
    live = (used != 0) & ~frozen
    pairs = case.plastic_pairs(np.linalg.svd(case.f_tilde(F, C), compute_uv=False)) * (plastic & live)[:, None]
    cen['counts'].update(plastic_pass=int(pairs[:, 0].sum()), plastic_mixed=int(pairs[:, 1].sum()), plastic_same=int(pairs[:, 2].sum()))
    cen['counts'].update(case.field_counts(P, mu, live))
    case.check_bwd_counts(layout, cen['counts'], True, field=True)
    # the field stays within 2x of each row's value where the row's is non-zero, and is fp32-representable
    nz = (P['mu'] != 0) & (mu != 0)
    assert (mu[nz] / P['mu'][nz] <= 2.0 + 1e-6).all() and (mu[nz] / P['mu'][nz] >= 0.5 - 1e-6).all()
    assert np.array_equal(mu.astype(np.float32).astype(np.float64), mu) and np.array_equal(lam.astype(np.float32).astype(np.float64), lam)


@pytest.mark.parametrize('n', [32, 64])
@pytest.mark.parametrize('layout', case.LAYOUTS)
def test_every_layout_reaches_the_plastic_field_branches_it_exists_for(layout, n):
    """the census of the plastic-field runs without a device, on the replayed sort order: the plastic pairs against each particle's own window
    (cross-bound pairs of lo == hi among them), the particles clamped at lo = 1 and at hi = 1, the wide windows, the particles whose dL/dlo and
    dL/dhi get a term; rho and theta fp32-representable, and every singular value of F~ 2e-4 or more from its particle's own bounds"""
    d = case.draw(layout, n, False, case.SEED, 'plastic')
    lay, P, plastic, (tc, ts, wide), (lo, hi) = d['lay'], d['P'], d['plastic'], d['theta'], d['lim']
    x, used, frozen = lay['x'], lay['used'], lay['frozen']
    row = np.searchsorted(np.unique(d['mat']), d['mat'])
    ids = _stable_sort_order(x, used, n) if lay['sort'] else np.arange(len(x))
    cen = case.bwd_census(x[ids], used[ids], row[ids], n)
    live = (used != 0) & ~frozen
    sig = np.linalg.svd(case.f_tilde(d['F'], d['C']), compute_uv=False)
    _, pc = case.plastic_counts(sig, plastic & live, lo, hi, wide)
    cen['counts'].update(pc)
    cen['counts'].update(case.field_counts(P, P['mu'], live))
    case.check_bwd_counts(layout, cen['counts'], True, field='plastic')
    for a in (P['rho'], tc, ts):
        assert np.array_equal(a.astype(np.float32).astype(np.float64), a)
    assert np.array_equal(P['mass'], (np.float32((0.5 / n) ** 2) * P['rho'].astype(np.float32)).astype(np.float64))
    assert ((lo == 1) & (hi == 1)).any() and (wide == ((1 - lo >= 0.05) & (hi - 1 >= 0.05))).all()
    margin = np.minimum(np.abs(sig - lo[:, None]), np.abs(sig - hi[:, None])).min(1)
    assert margin[plastic].min() >= 2e-4, 'a singular value of a plastic particle within 2e-4 of its own bounds'
    side, _ = case.clamp_sides(sig, lo, hi)
    assert not (side[plastic & wide] != 0).any(), 'a wide window clamps'


@pytest.mark.parametrize('kind', ['liquid', 'general', 'field', 'mass', 'plastic'])
@pytest.mark.parametrize('layout', case.LAYOUTS)
def test_backward_kernels_one_launch_at_a_time_match_the_fp64_oracle_on_the_shim(emu, layout, kind):
    """field: k_p2g_field<false | true>, k_particle_grad<2, false> and, with parameter gradients, k_particle_grad<2, true> and its per-slot
    gfield; mass: k_p2g_field_mass and k_particle_grad<3, *> with gfield and gmass; plastic: k_p2g_field_plastic and k_particle_grad<4, *> with
    the plastic record's gpfield (dmu, dlam, dlo, dhi) and gmass"""
    case.run(layout, 32, kind == 'liquid', device='cpu', field=FIELD.get(kind, False))


@pytest.mark.gpu
@pytest.mark.parametrize('n', [32, 64])
@pytest.mark.parametrize('kind', ['liquid', 'general', 'field', 'mass', 'plastic'])
@pytest.mark.parametrize('layout', case.LAYOUTS)
def test_backward_kernels_one_launch_at_a_time_match_the_fp64_oracle(layout, kind, n):
    _need_gpu()
    case.run(layout, n, kind == 'liquid', field=FIELD.get(kind, False))
