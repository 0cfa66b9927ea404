"""k_fwd's footprint branches one launch at a time against the fp64 oracle, at particle layouts that force each branch (tests/fwd_layout_case.py):
dense cell-sorted clouds (8-node tiles), sparse runs along z (16-node tiles), long runs and unsorted clouds (L2 gathers), stencils against the
high and the low edge of the grid (TMA boxes past the grid, truncation to base 0 with negative weights), and ragged warps with unused and
frozen slots.  The same layouts go through one stored-grid backward substep, whose kernels stage footprints of their own.  With a per-particle
material field, k_p2g_field and k_fwd<2, false, false> run the same launch; with fwd mask 0, fmpm_g2p2g runs the agent-free k_g2p2g and
k_g2p2g_field (write_vc 0 and 1) on the same layouts, its write set included.

The CPU shim (tests/cuda_emu) runs the plain staged tile (masks 1 / 3) at n = 32 under `-m "not gpu"`; an H100 runs TMA tiles too (masks 9 / 11),
at n = 32 and n = 64."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'cuda_emu'))
import harness  # noqa: E402

import fwd_layout_case as case  # noqa: E402

FIELD = {'field': True, 'mass': 'mass', 'plastic': 'plastic'}   # the field states of bwd_layout_case.setup by kind
G2P2G = {'g2p2g-table': False, 'g2p2g-field': True, 'g2p2g-mass': 'mass', 'g2p2g-plastic': 'plastic'}


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


@pytest.mark.parametrize('n', [32, 64])
@pytest.mark.parametrize('layout', case.LAYOUTS)
def test_every_layout_reaches_the_branches_it_exists_for(layout, n):
    """the host census of each layout, without a device: the warps of every layout take the branch it exists for, in enough numbers (the runs
    below assert the same counts on the slot order the device produced)"""
    lay = case.layout(layout, n, np.random.RandomState(0))
    x, used = lay['x'], lay['used']
    ids = _stable_sort_order(x, used, n) if lay['sort'] else np.arange(len(x))
    c = case.census(x[ids], used[ids], n)
    case.check_counts(layout, c['counts'])
    if layout == 'ragged':
        assert len(x) % 32 != 0 and (used == 0).sum() > 0.1 * len(x) and lay['frozen'].sum() > 0
    if layout == 'low_edge':   # base 0 with fx < 0.5, and a negative middle weight, in enough particles
        b, fx, w = case.weights(x.astype(np.float64) * n)
        assert ((b == 0) & (fx < 0.5)).any(1).sum() >= 100 and (w[:, 1] < 0).any(1).sum() >= 40, (((b == 0) & (fx < 0.5)).any(1).sum(), (w[:, 1] < 0).any(1).sum())


@pytest.mark.parametrize('kind', ['liquid', 'general', 'field', 'mass', 'plastic'])
@pytest.mark.parametrize('layout', case.LAYOUTS)
def test_one_k_fwd_launch_matches_the_fp64_oracle_on_the_shim(emu, layout, kind):
    """k_fwd<1> (all-liquid, masks 3), k_fwd<0> (masks 1) and, with a material field, k_p2g_field<true> then k_fwd<2, false, false> (mask 1),
    with the plain staged tile; with a density field too (mass) k_p2g_field_mass<true> then k_fwd<3, false, false>, with plastic limits per
    particle too (plastic) k_p2g_field_plastic<true> then k_fwd<4, false, false>"""
    case.run(layout, 32, kind == 'liquid', [1, 3] if kind == 'liquid' else [1], device='cpu', field=FIELD.get(kind, False))


@pytest.mark.parametrize('write_vc', [0, 1])
@pytest.mark.parametrize('kind', list(G2P2G))
@pytest.mark.parametrize('layout', case.LAYOUTS)
def test_one_k_g2p2g_launch_matches_the_fp64_oracle_on_the_shim(emu, layout, kind, write_vc):
    """the agent-free k_g2p2g<write_vc, false> / k_g2p2g_field / k_g2p2g_field_mass / k_g2p2g_field_plastic<write_vc, false> (fwd mask 0), with
    its write set"""
    case.run_g2p2g(layout, 32, G2P2G[kind], write_vc, device='cpu')


@pytest.mark.parametrize('layout', case.LAYOUTS)
def test_one_stored_grid_backward_substep_matches_the_fp64_oracle_on_the_shim(emu, layout):
    case.run_backward(layout, 32, False, device='cpu')


@pytest.mark.gpu
@pytest.mark.parametrize('n', [32, 64])
@pytest.mark.parametrize('kind', ['liquid', 'general', 'field', 'mass', 'plastic'])
@pytest.mark.parametrize('layout', case.LAYOUTS)
def test_one_k_fwd_launch_matches_the_fp64_oracle(layout, kind, n):
    """plain staged tiles (masks 1 / 3) and TMA tiles (masks 9 / 11; the H100 must report TMA), and TMA against plain bit for bit; the
    material, mass and plastic fields run k_fwd<2 | 3 | 4, false, false> under masks 1 and 9"""
    _need_gpu()
    case.run(layout, n, kind == 'liquid', [1, 3, 9, 11] if kind == 'liquid' else [1, 9], field=FIELD.get(kind, False))


@pytest.mark.gpu
@pytest.mark.parametrize('n', [32, 64])
@pytest.mark.parametrize('write_vc', [0, 1])
@pytest.mark.parametrize('kind', list(G2P2G))
@pytest.mark.parametrize('layout', case.LAYOUTS)
def test_one_k_g2p2g_launch_matches_the_fp64_oracle(layout, kind, write_vc, n):
    _need_gpu()
    case.run_g2p2g(layout, n, G2P2G[kind], write_vc)


@pytest.mark.gpu
@pytest.mark.parametrize('n', [32, 64])
@pytest.mark.parametrize('liquid', [True, False], ids=['liquid', 'general'])
@pytest.mark.parametrize('layout', case.LAYOUTS)
def test_one_stored_grid_backward_substep_matches_the_fp64_oracle(layout, liquid, n):
    _need_gpu()
    case.run_backward(layout, n, liquid)
