"""The smoke solver's kernels one launch at a time against the fp64 oracle (tests/smoke_layout_case.py), on band, grid and obstacle layouts that
force each boundary branch: q_dim 1-4, bands on the grid's bottom and top faces, band heights 0, 1, 8, 9 and 12, one partial tile and a last
tile one column wide, statics that block cells on the grid faces inside the band, backtraces that leave the grid, a zero-velocity region, and the
reference's configuration (128^3, 500 sweeps: 63 chained tile launches, the last one 4 sweeps).

The CPU shim (tests/cuda_emu) runs every layout except `reference` under `-m "not gpu"`; an H100 runs all of them."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'cuda_emu'))
import harness  # noqa: E402

import smoke_layout_case as case  # noqa: E402


@pytest.fixture
def emu():
    L = harness.enable()
    yield L
    harness.disable()


@pytest.mark.parametrize('layout', list(case.LAYOUTS))
def test_every_layout_reaches_the_branches_it_exists_for(layout):
    """the host census in fp64, without a device: band rows, Jacobi plan, blocked and out-of-grid neighbours per side, the loc() fallbacks of
    the trilinear corners, backtraces outside the grid, zero-velocity cells (the runs assert the same on the kernel's own mask)"""
    cfg, st = case.make_layout(layout)
    free, amb, _ = case.mask64(cfg)
    cen, _ = case.census(cfg, free, st['v'].astype(np.float64))
    print(layout, cen)
    case.check_census(layout, cen)
    assert amb.sum() == 0, 'no cell centre within AMB_SDF of a static surface at the seed'


def test_the_layouts_cover_the_issue_s_shapes():
    """band heights 0, 1, 8, 9; both grid faces in y; q_dim 2, 3, 4; the 63-launch chain with its 4-sweep tail; four statics at least once"""
    sh = case.SHAPE
    assert {0, 1, 8, 9} <= {v['H'] for v in sh.values()}
    assert any(v.get('j0') == 0 for v in sh.values()) and any(v.get('j1') == case.LAYOUTS[k]['res'] - 1 for k, v in sh.items())
    assert {2, 3, 4} <= {v['qd'] for v in sh.values()}
    assert sh['reference']['launches'] == 63 and sh['reference']['last_sweeps'] == 4
    assert max(len(v['statics']) for v in case.LAYOUTS.values()) == 4


@pytest.mark.parametrize('layout', case.SHIM_LAYOUTS)
def test_smoke_kernels_one_launch_at_a_time_match_the_fp64_oracle_on_the_shim(emu, layout):
    out = case.run(layout, 'cpu', emu)
    print(layout, out['err'])


def test_smoke_kernels_are_order_independent_under_a_shuffled_schedule():
    """the tile kernel's shared-memory sweeps and the air conditioner's block reduction under CUEMU_SCHED=shuffle (another thread order inside
    every block): a missing barrier would change the result"""
    env = dict(os.environ, CUEMU_SCHED='shuffle')
    r = subprocess.run([sys.executable, '-m', 'pytest', os.path.abspath(__file__), '-q', '-p', 'no:cacheprovider',
                        '-k', 'match_the_fp64_oracle_on_the_shim and interior'],
                       capture_output=True, text=True, timeout=1500, env=env, cwd=os.path.dirname(HERE))
    tail = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else ''
    assert r.returncode == 0 and '1 passed' in tail, r.stdout[-3000:] + r.stderr[-1000:]


@pytest.mark.gpu
@pytest.mark.parametrize('layout', list(case.LAYOUTS))
def test_smoke_kernels_one_launch_at_a_time_match_the_fp64_oracle(layout):
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from fluidlab_b200 import _lib
    out = case.run(layout, 'cuda', _lib.load())
    print(layout, out['err'], out['time'])
