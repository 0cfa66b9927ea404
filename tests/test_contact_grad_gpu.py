"""Loss gradients with respect to the contact parameters on an H100: the CUDA kernels against the fp64 oracle on every scene of
tests/contact_grad_case.py, a 256k-particle ICECREAM block pushed by a soft box collider against central differences of the fp32 forward
loss, and the static-friction identification at full speed."""
import numpy as np
import pytest
import torch

import contact_grad_case as cgc

pytestmark = pytest.mark.gpu


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')


@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('scene', list(cgc.SCENES))
def test_contact_grad_kernels_match_the_oracle(scene, sort):
    _need_gpu()
    got, _, want = cgc.sim_run(scene, None, sort)
    cgc.assert_contact_close(got, want, scene)


@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
def test_contact_accumulator_leaves_the_other_gradients_alone(sort):
    _need_gpu()
    cgc.assert_bound_unbound_agree('rigid_both_s50', None, sort)


def _icecream_push(n_grid=64, N=262144):
    """an ICECREAM block on the floor of a cube with restitution 0.3, pushed sideways and down by a soft box collider (friction 8, softness
    100: the cone of agent_icecreamdynamic.yaml) at collide_type 'both'; loss = sum w . x after 4 steps"""
    from conftest import make_particles, box_sdf
    from fluidlab_b200 import TaichiEnv, macros as M
    rng = np.random.RandomState(17)
    x = rng.uniform((0.3, 0.205, 0.3), (0.7, 0.45, 0.7), size=(N, 3))
    P = make_particles(x, M.ICECREAM, n_grid)
    env = TaichiEnv(quality=n_grid / 64, max_substeps_local=50, gravity=(0.0, -10.0, 0.0), horizon=5)
    s = env.simulator
    s.use_graphs, s.param_grad = False, True
    vox, T = box_sdf((0.06, 0.06, 0.15), 0.2)
    env.setup_agent(dict(type='AgentRigid', params=dict(collide_type='both'), effectors=[dict(
        type='Rigid', params=dict(init_pos=(0.28, 0.4, 0.5), init_euler=(0.0, 0.0, 0.0), action_dim=3),
        mesh=dict(file='box.obj', material=M.STIRRER, softness=100.0, sdf=dict(voxels=vox, T_mesh_to_voxels=T)),
        boundary=dict(type='cube', lower=(0.05,) * 3, upper=(0.95,) * 3))]))
    env.setup_boundary(type='cube', lower=(0.2, 0.2, 0.2), upper=(0.8, 0.8, 0.8), restitution=0.3)
    env.particle_bodies.get = lambda: P
    env.build()
    s.set_contact_params(rigid_friction=8.0)
    st0 = s.get_state()
    st0['v'][:] = np.array([0.0, -1.0, 0.0], dtype=np.float32)
    w = np.tile(np.array([1.0, 1.0, 0.5]), (N, 1))   # one direction for every particle: the contact's push and drag add up instead of cancelling
    actions = np.array([[0.006, -0.003, 0.0]] * 4, dtype=np.float32)

    def loss(**params):
        s.set_contact_params(**params)
        env.set_state(st0, grad_enabled=True)
        env.apply_agent_action_p(np.array([0.28, 0.4, 0.5], dtype=np.float32))
        for a in actions:
            env.step(a)
        return float((w * s.get_state()['x'].astype(np.float64)).sum())
    return s, env, w, actions, loss


def test_icecream_push_contact_gradients_match_central_differences():
    """dL/d(rigid friction, rigid softness, restitution) of a 256k-particle scene against central differences of the fp32 forward.  Step:
    2 % of the value (friction 0.16, softness 2, restitution 0.006).  A smaller step drowns in the fp32 noise of the loss (run-to-run
    reordering of the scatter's float atomics moves it by about 1e-5 relative), a larger one averages over the kinks of the contact map
    (the max(0, .) of the friction cone, the min(., 1) of the influence).  The hit test has no derivative but moves a few particles across
    its threshold inside the step: for friction and restitution the bar is 5 % of the larger of the two values.  For softness that threshold
    is sd = ln(10) / softness itself, so the difference quotient also counts the particles it sweeps over, a term the adjoint leaves out by
    the rule that branch conditions carry no gradient (measured: about half the quotient on a small version of this scene); only the sign is
    checked there."""
    _need_gpu()
    s, env, w, actions, loss = _icecream_push()
    base = dict(rigid_friction=8.0, rigid_softness=100.0, restitution=0.3)
    L0 = loss(**base)
    env.reset_grad()
    s.set_grad((w).astype(np.float32), np.zeros_like(w, np.float32), np.zeros((len(w), 3, 3), np.float32), np.zeros((len(w), 3, 3), np.float32))
    for a in actions[::-1]:
        env.step_grad(a)
    g = s.get_param_grad()
    assert np.isfinite(L0)
    res = {}
    for k, v in base.items():
        h = 0.02 * v
        fd = (loss(**dict(base, **{k: v + h})) - loss(**dict(base, **{k: v - h}))) / (2 * h)
        res[k] = (fd, g[k])
    print('contact gradients (fd, analytic):', res)
    for k, (fd, an) in res.items():
        assert abs(an) > 0, (k, res)
        if k == 'rigid_softness':
            assert np.sign(fd) == np.sign(an), (k, res)
        else:
            assert abs(fd - an) <= 0.05 * max(abs(fd), abs(an)), (k, res)


def test_static_friction_identification_at_full_speed():
    _need_gpu()
    hist = cgc.friction_sysid_case(None)
    assert abs(hist[-1] - 0.3) < 0.03, hist
