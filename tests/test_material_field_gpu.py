"""Per-particle mu and lam (MPMSimulator.set_material_field) on the H100: the cases of tests/material_field_case.py against the fp64 oracle, a
full-size directional derivative against central differences of the device forward and the stiff-core identification at 256k particles."""
import numpy as np
import pytest
import torch

from conftest import make_particles
from fluidlab_b200 import macros as M
import material_field_case as mfc

pytestmark = pytest.mark.gpu


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip('needs an H100')


@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('case', ['elastic', 'mixed'])
def test_field_equal_to_the_table_reproduces_the_table_run_gpu(case, sort):
    _need_gpu()
    mfc.field_equals_table_case(None, case, sort)


@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('case', ['elastic', 'icecream', 'milk_vis', 'mixed', 'mixed-mu0'])
def test_heterogeneous_field_matches_the_oracle_gpu(case, sort):
    _need_gpu()
    mfc.heterogeneous_case(None, case.replace('-mu0', ''), sort, zero_frac=0.2 if case.endswith('mu0') else 0.0)


@pytest.mark.parametrize('sort_every', [0, 1])
def test_field_gradients_across_sort_epochs_and_the_checkpoint_ring_gpu(sort_every):
    _need_gpu()
    mfc.ring_case(None, sort_every)


def test_field_full_size_directional_derivative():
    """1M ELASTIC particles in C2's box at 128^3 with a smooth random field (x 0.5 .. 2 of the table), pre-strained; L = sum w . x_T after one
    step (forward on the fused k_fwd<2> path, backward on the stored grids): the derivative along a smooth random field perturbation against
    central differences of the device forward, 0.5 % bar"""
    _need_gpu()
    from fluidlab_b200 import MPMSimulator
    N = 1_000_000
    rs = np.random.RandomState(4)
    x = rs.uniform((0.25, 0.30, 0.25), (0.75, 0.54, 0.75), size=(N, 3))
    P = make_particles(x, M.ELASTIC, 128)
    s = MPMSimulator(dim=3, quality=2, gravity=(0.0, -10.0, 0.0), horizon=100, max_substeps_local=50, max_substeps_global=100000, ckpt_dest='gpu')
    s.build(None, None, [], P)
    tp = 2 * np.pi
    smooth = lambda a, b, c: np.sin(tp * (a * x[:, 0] + 0.3)) * np.cos(tp * (b * x[:, 1] + 0.1)) * np.sin(tp * (c * x[:, 2] + 0.7))
    mu = P['mu'] * np.exp(0.7 * smooth(2, 3, 2)); lam = P['lam'] * np.exp(0.7 * smooth(3, 2, 3))
    dmu = 0.02 * mu * smooth(1, 2, 3); dlam = 0.02 * lam * smooth(2, 1, 2)
    v0 = (0.2 * np.stack([np.sin(tp * x[:, 1] * 2), np.cos(tp * x[:, 2] * 3), np.sin(tp * x[:, 0] * 2 + 1.0)], 1)).astype(np.float32)
    w = np.stack([np.cos(tp * (x[:, 0] * 2 + 0.3)), np.sin(tp * (x[:, 1] * 3 + x[:, 0])), np.cos(tp * x[:, 2] * 3)], 1).astype(np.float32)
    base = s.get_state(); base['v'] = v0; base['F'] = np.tile(np.diag([0.97, 1.0, 1.03]).astype(np.float32), (N, 1, 1))

    def run(m, l):
        s.set_material_field(m, l)
        s.cur_substep_global = 0
        s.set_state(0, base)
        s.step(None)
        return float((s.get_state()['x'].astype(np.float64) * w).sum())
    s.param_grad = True
    s.enable_grad()
    run(mu, lam)
    s.reset_grad()
    z3, z9 = np.zeros((N, 3), np.float32), np.zeros((N, 3, 3), np.float32)
    s.set_grad(w, z3, z9, z9)
    s.step_grad(None)
    g = s.get_param_grad()
    an = float((g['mu_field'] * dmu).sum() + (g['lam_field'] * dlam).sum())
    s.disable_grad()
    fd = (run(mu + dmu, lam + dlam) - run(mu - dmu, lam - dlam)) / 2
    assert an != 0.0 and abs(fd - an) < 5e-3 * abs(an), (fd, an)



def test_fused_forward_with_a_field_matches_the_oracle_gpu():
    _need_gpu()
    mfc.fused_forward_case(None)


@pytest.mark.parametrize('fuse', [True, False], ids=['fused', 'per-substep'])
def test_injector_with_a_field_matches_the_oracle_gpu(fuse):
    _need_gpu()
    mfc.injector_case(None, fuse)


def test_field_identification_256k():
    """the stiff-core identification of tests/material_field_case.py with 256k particles on 64^3: the field error drops at least 1.5x, the core's
    mean stiffness scale rises above 3 (truth 4) and the shell's falls below 1.5 (truth 1)"""
    _need_gpu()
    hist = mfc.identification_case(None, n_grid=64, N=262_144)
    (e0, _, _), (e1, core, shell) = hist[0], hist[-1]
    assert e1 <= e0 / 1.5 and core >= 3.0 and shell <= 1.5, hist
