"""The backward substep's kernels one launch at a time against the fp64 oracle (tests/bwd_layout_case.py), on the layouts of
tests/fwd_layout_case.py: k_p2g (recompute and forward), k_grid_op + k_g2p, k_g2p_grad_scatter, k_grid_op_grad and k_particle_grad, the last
two also in their parameter-gradient instantiations, each fed the kernel's own upstream output.  The general materials run k_particle_grad<0>
(SVD adjoint, plastic clamps), the mu = 0 liquids k_particle_grad<1>.

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


@pytest.mark.parametrize('liquid', [True, False], ids=['liquid', 'general'])
@pytest.mark.parametrize('layout', case.LAYOUTS)
def test_backward_kernels_one_launch_at_a_time_match_the_fp64_oracle_on_the_shim(emu, layout, liquid):
    case.run(layout, 32, liquid, device='cpu')


@pytest.mark.gpu
@pytest.mark.parametrize('n', [32, 64])
@pytest.mark.parametrize('liquid', [True, False], ids=['liquid', 'general'])
@pytest.mark.parametrize('layout', case.LAYOUTS)
def test_backward_kernels_one_launch_at_a_time_match_the_fp64_oracle(layout, liquid, n):
    _need_gpu()
    case.run(layout, n, liquid)
