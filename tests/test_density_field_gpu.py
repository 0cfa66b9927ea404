"""Per-particle density (MPMSimulator.set_density_field) on the H100: the cases of tests/density_field_case.py against the fp64 oracle and the
loss references on 32^3 and 64^3 grids (particle counts grown with the grid), a full-size directional derivative against central differences of the device forward and the dense-core identification at
256k particles."""
import numpy as np
import pytest
import torch

from conftest import make_particles
from fluidlab_b200 import macros as M
import density_field_case as dfc

pytestmark = pytest.mark.gpu


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip('needs an H100')


@pytest.mark.parametrize('with_field', [False, True], ids=['rho', 'rho+mu-lam'])
@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('case', ['elastic', 'mixed'])
@pytest.mark.parametrize('n', [32, 64])
def test_density_field_equal_to_the_rows_reproduces_the_table_run_gpu(case, sort, with_field, n):
    _need_gpu()
    dfc.equals_table_case(None, case, sort, with_field, n=n)


@pytest.mark.parametrize('with_field', [False, True], ids=['rho', 'rho+mu-lam'])
@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('case', ['elastic', 'icecream', 'milk_vis', 'water', 'mixed'])
@pytest.mark.parametrize('n', [32, 64])
def test_heterogeneous_density_matches_the_oracle_gpu(case, sort, with_field, n):
    _need_gpu()
    dfc.heterogeneous_case(None, case, sort, with_field, n=n)


@pytest.mark.parametrize('sort_every', [0, 1])
@pytest.mark.parametrize('n', [32, 64])
def test_density_gradients_across_sort_epochs_and_the_checkpoint_ring_gpu(sort_every, n):
    _need_gpu()
    dfc.ring_case(None, sort_every, n=n)


@pytest.mark.parametrize('n', [32, 64])
def test_density_gradients_match_central_differences_of_the_oracle_gpu(n):
    _need_gpu()
    dfc.central_difference_case(None, n=n)


@pytest.mark.parametrize('n', [32, 64])
def test_fused_forward_with_a_density_field_matches_the_oracle_gpu(n):
    _need_gpu()
    dfc.fused_forward_case(None, n=n)


@pytest.mark.parametrize('n', [32, 64])
def test_fused_stored_grad_path_with_a_density_field_matches_the_oracle_gpu(n):
    _need_gpu()
    dfc.heterogeneous_case(None, 'mixed', True, with_field=True, fuse=True, n=n)


@pytest.mark.parametrize('fuse', [True, False], ids=['fused', 'per-substep'])
@pytest.mark.parametrize('n', [32, 64])
def test_injector_with_a_density_field_matches_the_oracle_gpu(fuse, n):
    _need_gpu()
    dfc.injector_case(None, fuse, n_grid=n)


@pytest.mark.parametrize('n', [32, 64])
def test_rigid_bodies_with_a_density_field_match_the_oracle_gpu(n):
    _need_gpu()
    dfc.rigid_case(None, n_grid=n)


@pytest.mark.parametrize('n', [32, 64])
def test_loss_kernels_with_a_density_field_match_the_references_gpu(n):
    _need_gpu()
    dfc.loss_kernel_case(None, n=n, N=400 * n // 16)


@pytest.mark.parametrize('n', [32, 64])
def test_density_loss_env_gradient_matches_central_differences_gpu(n):
    _need_gpu()
    dfc.env_case(None, n=n, N=600 * n // 16)


def test_density_field_full_size_directional_derivative():
    """1M ELASTIC particles in C2's box at 128^3 with a smooth random rho (x 0.5 .. 2 of the row), pre-strained; L = sum w . x_T after one step
    (forward on the fused k_fwd<3> path, backward on the stored grids): the derivative along a smooth random rho perturbation against central
    differences of the device forward, 0.5 % bar"""
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
    rho = np.asarray(P['rho'], np.float64) * np.exp(0.7 * smooth(2, 3, 2))
    drho = 0.02 * rho * smooth(1, 2, 3)
    v0 = (0.2 * np.stack([np.sin(tp * x[:, 1] * 2), np.cos(tp * x[:, 2] * 3), np.sin(tp * x[:, 0] * 2 + 1.0)], 1)).astype(np.float32)
    w = np.stack([np.cos(tp * (x[:, 0] * 2 + 0.3)), np.sin(tp * (x[:, 1] * 3 + x[:, 0])), np.cos(tp * x[:, 2] * 3)], 1).astype(np.float32)
    base = s.get_state(); base['v'] = v0; base['F'] = np.tile(np.diag([0.97, 1.0, 1.03]).astype(np.float32), (N, 1, 1))

    def run(r):
        s.set_density_field(r)
        s.cur_substep_global = 0
        s.set_state(0, base)
        s.step(None)
        return float((s.get_state()['x'].astype(np.float64) * w).sum())
    s.param_grad = True
    s.enable_grad()
    run(rho)
    s.reset_grad()
    z3, z9 = np.zeros((N, 3), np.float32), np.zeros((N, 3, 3), np.float32)
    s.set_grad(w, z3, z9, z9)
    s.step_grad(None)
    an = float((s.get_param_grad()['rho_field'] * drho).sum())
    s.disable_grad()
    fd = (run(rho + drho) - run(rho - drho)) / 2
    assert an != 0.0 and abs(fd - an) < 5e-3 * abs(an), (fd, an)


def test_density_identification_256k():
    """the dense-core identification of tests/density_field_case.py with 256k particles on 64^3: the field error drops at least 1.5x (measured
    2.14x on an H100) and the core's mean ends at least 1.5x the shell's (measured 2.5x)"""
    _need_gpu()
    hist = dfc.identification_case(None, n_grid=64, N=262_144)
    (e0, _, _), (e1, core, shell) = hist[0], hist[-1]
    assert e1 <= e0 / 1.5 and core > 1.5 * shell, hist
