"""Plastic yield limits (MPMSimulator.set_plastic_limits / set_plastic_field) on the H100: the cases of tests/plastic_limits_case.py against
the fp64 oracle on 32^3 and 64^3 grids (particle counts grown with the grid), a full-size directional derivative in (theta_c, theta_s) against
central differences of the device forward, and the identification of an ICECREAM block's limits at 256k particles."""
import numpy as np
import pytest
import torch

from conftest import make_particles
from fluidlab_b200 import macros as M
import plastic_limits_case as plc

pytestmark = pytest.mark.gpu


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip('needs an H100')


@pytest.mark.parametrize('with_field', [False, True], ids=['limits', 'limits+mu-lam'])
@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('case', ['icecream', 'mixed'])
def test_default_limits_reproduce_the_runs_without_them_gpu(case, sort, with_field):
    _need_gpu()
    plc.defaults_case(None, case, sort, with_field)


@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('case', ['icecream', 'plastic_demo', 'mixed'])
@pytest.mark.parametrize('n', [32, 64])
def test_random_limits_match_the_oracle_gpu(case, sort, n):
    _need_gpu()
    plc.heterogeneous_case(None, case, sort, n=n)


@pytest.mark.parametrize('n', [32, 64])
def test_random_row_limits_and_the_fused_stored_grad_path_gpu(n):
    _need_gpu()
    plc.heterogeneous_case(None, 'mixed', True, n=n, per_row=True)
    plc.heterogeneous_case(None, 'mixed', True, fuse=True, n=n)


@pytest.mark.parametrize('sort_every', [0, 1])
@pytest.mark.parametrize('n', [32, 64])
def test_limit_gradients_across_sort_epochs_and_the_checkpoint_ring_gpu(sort_every, n):
    _need_gpu()
    plc.ring_case(None, sort_every, n=n)


@pytest.mark.parametrize('n', [32, 64])
def test_fused_forward_and_rigid_bodies_with_limits_gpu(n):
    _need_gpu()
    plc.fused_forward_case(None, n=n)
    plc.rigid_case(None, n_grid=n)


@pytest.mark.parametrize('fuse', [True, False], ids=['fused', 'per-substep'])
def test_injected_icecream_with_limits_gpu(fuse):
    """the shim's 16^3 scene: on 32^3 and 64^3 this pour clamps no singular value within its three steps (the oracle's dL/dtheta is 0)"""
    _need_gpu()
    plc.injector_case(None, fuse)


def test_fields_set_and_cleared_in_any_order_keep_the_gradients_gpu():
    _need_gpu()
    plc.composition_case(None, 'lrm', 'mlr')


def test_full_size_directional_derivative_matches_central_differences_of_the_device_forward():
    """1M ICECREAM particles on 64^3 with random F and C: dL/dtheta of the row (one step, seed . frame) along a direction in (theta_c,
    theta_s) against central differences of the device's own forward.  (ICECREAM on 128^3 is beyond the fixed time step: dt c / dx > 1, and
    the state turns NaN within a step.)"""
    _need_gpu()
    rng = np.random.RandomState(7)
    N, n = 1 << 20, 64
    x = rng.uniform(0.25, 0.75, size=(N, 3))
    P = make_particles(x, M.ICECREAM, n)
    s = plc._sim(None, P, n, True)
    st = s.get_state()
    st['v'][:] = (rng.randn(N, 3) * 0.5).astype(np.float32)
    st['F'][:] = (np.eye(3)[None] + rng.randn(N, 3, 3) * 0.05).astype(np.float32)
    st['C'][:] = (rng.randn(N, 3, 3) * 0.5).astype(np.float32)
    seed = {k: torch.from_numpy(rng.randn(*sh).astype(np.float32)).cuda() for k, sh in (('x', (N, 3)), ('F', (N, 3, 3)))}
    th = np.array([plc.THETA_C, plc.THETA_S])
    d = th * np.array([1.0, -0.5])

    def loss(t, grad=False):
        s.set_plastic_limits([t[0]], [t[1]])
        s.cur_substep_global = 0
        s.set_state(0, st)
        s.enable_grad()
        s.step(None)
        fr = s.readframe(10)
        L = sum(float((seed[k].double().cpu().numpy() * np.asarray(fr[k], np.float64)).sum()) for k in ('x', 'F'))
        if grad:
            s.reset_grad()
            z3, z9 = np.zeros((N, 3), np.float32), np.zeros((N, 3, 3), np.float32)
            s.set_grad(seed['x'].cpu().numpy(), z3, z9, seed['F'].cpu().numpy())
            s.step_grad(None)
            g = s.get_param_grad()
            return L, float(g['theta_c'][0] * d[0] + g['theta_s'][0] * d[1])
        return L
    _, an = loss(th, grad=True)
    h = 1e-2
    fd = (loss(th + h * d) - loss(th - h * d)) / (2 * h)
    print('directional', fd, an)
    # measured on an H100: -1.7607 against -1.8501 (5.1 %).  The loss is piecewise smooth in the limits: every axis that sits at a limit
    # after a substep's clamp moves off it by about dt |C| in the next, and the step h theta moves the limit by a fifth of that, so the
    # secant crosses the kinks of many of the 3M axes (the fp64 oracle shows the same secant bias, 0.2 .. 0.7 % on 200 particles at this h,
    # and agrees to 2e-8 at h = 1e-5, which fp32 cannot resolve); a sign or factor error in the adjoint is off by order 1
    assert abs(fd - an) <= 0.1 * abs(fd), (fd, an)


def test_identification_recovers_the_limits_at_256k_particles():
    _need_gpu()
    hist = plc.identification_case(None, n_grid=64, N=1 << 18)
    print('identification', hist)
    # measured on an H100 (64^3, 256k particles, 25 Adam steps from the defaults): the loss falls 185x by step 7, at (5.73e-3, 1.061e-3)
    # against the truth (6e-3, 1e-3), 4.5 % and 6.1 %; Adam then overshoots in theta_c and ends at (4.32e-3, 0.77e-3).  The fit is the
    # iterate of least loss
    tc, ts, loss = min(hist, key=lambda h: h[2])
    assert loss < 1e-2 * hist[0][2], hist
    assert abs(tc / 6e-3 - 1) < 0.1 and abs(ts / 1e-3 - 1) < 0.1, hist
