"""Scenes for the contact-parameter gradients (MPMSimulator.param_grad: dL/d static friction, rigid friction, rigid softness and restitution):
the fp64 oracle against central differences through its own forward (tests/test_contact_grad.py), and the CUDA kernels on an H100
(tests/test_contact_grad_gpu.py) and on the CPU execution-model shim (tests/test_contact_grad.py) against the oracle (the fp64 reference
of tests/contact_grad_ref.py)."""
import numpy as np

from conftest import make_particles, box_sdf
from fluidlab_b200 import macros as M
from contact_grad_ref import ContactGradOracle

N_GRID = 16
CUBE = dict(type='cube', lower=(0.32, 0.32, 0.32), upper=(0.68, 0.68, 0.68))
CYL = dict(type='cylinder', xz_radius=0.2, xz_center=(0.5, 0.5), y_range=(0.32, 0.7))
RIGID_POS = (0.5, 0.515, 0.5)   # the Rigid box: 0.2 x 0.04 x 0.2, its lower face inside the top of the cloud, its medial plane above it


def _walls(bnd, restitution):
    return dict(bnd, restitution=restitution)


# name -> scene: boundary, cloud velocity, optional static box (friction), optional Rigid box (collide_type, friction, softness)
SCENES = {
    'cube_r0': dict(bnd=_walls(CUBE, 0.0), vel=(0.3, -3.0, 0.2)),
    'cube_r04': dict(bnd=_walls(CUBE, 0.4), vel=(0.3, -3.0, 0.2)),
    'cylinder': dict(bnd=_walls(CYL, 0.4), vel=(0.2, -3.0, 0.1)),
    'static': dict(bnd=_walls(CUBE, 0.0), vel=(1.5, -2.0, 1.0), static=0.3),
    **{f'rigid_{ct}_s{int(s)}': dict(bnd=_walls(CUBE, 0.0), vel=(0.0, 0.0, 0.0), rigid=(ct, 0.5, s))
       for ct in ('particle', 'grid', 'both') for s in (0.0, 50.0)},
    'rigid_sticky': dict(bnd=_walls(CUBE, 0.0), vel=(0.0, 0.0, 0.0), rigid=('both', 12.0, 50.0)),
}


def static_box():
    """an off-centre box SDF: 0.24 x 0.04 x 0.24 centred at (0.46, 0.36, 0.53), under the cloud (mesh T includes the placement)"""
    vox, T = box_sdf((0.12, 0.02, 0.12), 0.3)
    T = T.copy(); T[:3, 3] -= T[0, 0] * np.array([0.46, 0.36, 0.53])
    return vox, T


def rigid_box():
    """the Rigid mesh (centred at the mesh origin; the effector pose places it)"""
    return box_sdf((0.1, 0.02, 0.1), 0.2)


def cloud(scene, N=300, seed=7):
    rng = np.random.RandomState(seed)
    x = rng.uniform((0.38, 0.325, 0.38), (0.62, 0.5, 0.62), size=(N, 3))
    P = make_particles(x, M.ELASTIC, N_GRID)
    v = np.asarray(SCENES[scene]['vel'])[None] + rng.randn(N, 3) * 0.3
    C = rng.randn(N, 3, 3) * 2.0
    F = np.eye(3)[None] + rng.randn(N, 3, 3) * 0.02
    wts = {k: rng.randn(*a.shape) for k, a in (('x', x), ('v', v), ('C', C), ('F', F))}
    return P, dict(x=x, v=v, C=C, F=F, used=P['used']), wts


def rigid_pose(f):
    """pose of the Rigid box at frame f: moving down and sideways (collider velocity (1, -2, 0.5))"""
    dt = 2e-4
    return np.array([RIGID_POS[0] + 1.0 * dt * f, RIGID_POS[1] - 2.0 * dt * f, RIGID_POS[2] + 0.5 * dt * f, 1.0, 0.0, 0.0, 0.0, 0.0])


def oracle_params(scene):
    sc = SCENES[scene]
    p = dict(restitution=float(sc['bnd']['restitution']))
    if 'static' in sc:
        p['static_friction'] = float(sc['static'])
    if 'rigid' in sc:
        p['rigid_friction'], p['rigid_softness'] = float(sc['rigid'][1]), float(sc['rigid'][2])
    return p


def oracle_run(scene, params=None, n_sub=3, grads=False):
    """the scene on the fp64 oracle for n_sub substeps; loss = sum w * (x, v, C, F) of the last frame.  params overrides the contact
    parameters (keys of oracle_params).  Returns the loss, and with grads the contact gradients of that loss"""
    sc = SCENES[scene]
    p = dict(oracle_params(scene), **(params or {}))
    P, st, wts = cloud(scene)
    o = ContactGradOracle(N_GRID, P, gravity=(0.0, -10.0, 0.0), boundary=dict(sc['bnd'], restitution=p['restitution']), precision=64,
                      max_substeps_local=10)
    if 'static' in sc:
        o.add_static(*static_box(), friction=p['static_friction'])
    if 'rigid' in sc:
        o.add_effector(type=0, action_dim=3, boundary=dict(type='cube', lower=(0.05,) * 3, upper=(0.95,) * 3), max_action_steps=4, init_pos=RIGID_POS)
        o.set_rigid_mesh(*rigid_box(), friction=p['rigid_friction'], softness=p['rigid_softness'], collide_type=sc['rigid'][0])
        for f in range(n_sub + 1):
            o.set_effector_state(0, f, rigid_pose(f))
    o.set_frame(0, st['x'], st['v'], st['C'], st['F'], st['used'])
    for f in range(n_sub):
        o.substep(f)
    fr = o.get_frame(n_sub)
    loss = sum(float((wts[k] * fr[k]).sum()) for k in 'xvCF')
    if not grads:
        return loss
    o.reset_grad()
    o.set_grad_frame(n_sub, wts['x'], wts['v'], wts['C'], wts['F'])
    for f in reversed(range(n_sub)):
        o.substep_grad(f)
    g = o.get_contact_grad()
    return loss, dict(static_friction=float(g['static_friction'][0]), rigid_friction=g['rigid_friction'], rigid_softness=g['rigid_softness'],
                      restitution=g['restitution'])


def checked_params(scene):
    """the parameters a scene exercises, with the derivative expected to be non-zero (False: exactly zero)"""
    sc = SCENES[scene]
    out = {}
    if 'rigid' not in sc:
        out['restitution'] = True
    if 'static' in sc:
        out['static_friction'] = True
    if 'rigid' in sc:
        sticky = sc['rigid'][1] > 10.0
        out['rigid_friction'] = not sticky
        out['rigid_softness'] = sc['rigid'][2] > 0.0 and not sticky
    return out


# ---------------------------------------------------------------------------------------------------------- the CUDA simulator
def sim_run(scene, device, sort, contact_bound=True, n_steps=1):
    """the scene through TaichiEnv / MPMSimulator with param_grad: one step of 10 substeps (the Rigid box moved by the action), then a random
    adjoint seed on the last frame and one backward step.  sort=True: cell-sorted slots and the stored-grid backward; False: no sort and the
    recompute backward.  contact_bound=False unbinds the contact accumulator (the material one stays bound).  Returns the simulator's
    get_param_grad(), the state adjoint and the oracle's contact gradients for the same run."""
    from fluidlab_b200 import TaichiEnv
    sc = SCENES[scene]
    P, st, wts = cloud(scene)
    N = len(P['x'])
    kw = dict(ckpt_dest='cpu', device='cpu') if device == 'cpu' else dict(ckpt_dest='gpu')
    env = TaichiEnv(quality=N_GRID / 64, max_substeps_local=20, gravity=(0.0, -10.0, 0.0), horizon=n_steps + 1, **kw)
    s = env.simulator
    s.use_graphs, s.fuse_g2p2g, s.sort_every, s.store_grids, s.param_grad = False, False, 1 if sort else 0, sort, True
    ebnd = dict(type='cube', lower=(0.05,) * 3, upper=(0.95,) * 3)
    if 'rigid' in sc:
        vox, T = rigid_box()
        env.setup_agent(dict(type='AgentRigid', params=dict(collide_type=sc['rigid'][0]), effectors=[dict(
            type='Rigid', params=dict(init_pos=RIGID_POS, init_euler=(0.0, 0.0, 0.0), action_dim=3),
            mesh=dict(file='box.obj', material=M.STIRRER, softness=sc['rigid'][2], sdf=dict(voxels=vox, T_mesh_to_voxels=T)), boundary=ebnd)]))
    env.setup_boundary(**sc['bnd'])
    if 'static' in sc:
        vox, T = box_sdf((0.12, 0.02, 0.12), 0.3)
        env.add_static(file='box.obj', material=M.CUP, has_dynamics=True, pos=(0.46, 0.36, 0.53), sdf=dict(voxels=vox, T_mesh_to_voxels=T))
    env.particle_bodies.get = lambda: P
    env.build()
    cp = {}
    if 'static' in sc:
        cp['static_friction'] = [sc['static']]
    if 'rigid' in sc:
        cp['rigid_friction'] = sc['rigid'][1]
    s.set_contact_params(**cp)
    state = s.get_state()
    state['v'][:] = st['v']; state['C'][:] = st['C']; state['F'][:] = st['F']
    env.set_state(state, grad_enabled=True)
    action = np.array([0.002, -0.004, 0.001], dtype=np.float32) if 'rigid' in sc else None   # the box moves at (1, -2, 0.5)
    if action is not None:
        env.apply_agent_action_p(np.array(RIGID_POS, dtype=np.float32))
    env.step(action)
    env.reset_grad()
    if not contact_bound:
        s._ensure_grad_buffers()
        assert s._lib.fmpm_set_contact_grad(s._h, None) == 0
    f32 = {k: wts[k].astype(np.float32) for k in 'xvCF'}
    s.set_grad(f32['x'], f32['v'], f32['C'], f32['F'])
    env.step_grad(action)
    got = s.get_param_grad()
    state_grad = s.get_grad()
    # the oracle: the same step (the Rigid pose chain driven by the same action) and the same seed
    o = ContactGradOracle(N_GRID, P, gravity=(0.0, -10.0, 0.0), boundary=sc['bnd'], precision=64, max_substeps_local=20)
    if 'static' in sc:
        for st_ in env.statics:
            o.add_static(st_.sdf_voxels_np, st_.T_mesh_to_voxels_np, friction=st_.friction)
    if 'rigid' in sc:
        o.add_effector(type=0, action_dim=3, boundary=ebnd, max_action_steps=n_steps + 1, init_pos=RIGID_POS)
        mesh = env.agent.rigid.mesh
        o.set_rigid_mesh(mesh.sdf_voxels_np, mesh.T_mesh_to_voxels_np, friction=mesh.friction, softness=mesh.softness, collide_type=sc['rigid'][0])
    o.enable_grad()
    o.set_frame(0, P['x'], st['v'].astype(np.float32), st['C'].astype(np.float32), st['F'].astype(np.float32), P['used'])
    if action is not None:
        o.set_effector_state(0, 0, np.array([*RIGID_POS, 1, 0, 0, 0, 0.0])); o.apply_action_p(np.array(RIGID_POS, dtype=np.float32))
    o.step(None if action is None else action.astype(np.float64))
    o.reset_grad()
    o.set_grad_frame(o.cur_substep_local, f32['x'], f32['v'], f32['C'], f32['F'])
    o.step_grad(None if action is None else action.astype(np.float64))
    want = o.get_contact_grad()
    return got, state_grad, want


def assert_bound_unbound_agree(scene, device, sort):
    """binding the contact accumulator leaves the state adjoint and the material / gravity gradients as they were (up to the order of the
    unordered float reductions of the scatters, which differs from run to run whether or not it is bound)"""
    a, ga, _ = sim_run(scene, device, sort, contact_bound=True)
    b, gb, _ = sim_run(scene, device, sort, contact_bound=False)
    for k in 'xvCF':
        err = float(np.abs(ga[k] - gb[k]).max() / max(np.abs(gb[k]).max(), 1e-30))
        assert err < 1e-3, ('state adjoint changed by the contact accumulator', k, err)
    for k in ('mu', 'lam', 'rho', 'gravity'):
        err = float(np.abs(np.asarray(a[k]) - np.asarray(b[k])).max() / max(np.abs(np.asarray(b[k])).max(), 1e-30))
        assert err < 1e-3, ('material / gravity gradient changed by the contact accumulator', k, err)
    assert np.abs(b['restitution']) == 0.0 and np.abs(np.asarray(b['static_friction'])).sum() == 0.0, 'unbound: nothing accumulated'


def assert_contact_close(got, want, scene, bar=1e-3):
    """per exercised parameter: |got - want| <= bar * max(1, |want|); non-zero where the scene exercises the parameter, 0 where it must be.
    The comparison covers a whole step (10 substeps) of the fp32 forward and backward against fp64, whose contact maps are only piecewise smooth
    (hit and influence thresholds): measured differences are up to 3e-4 on the emulated device."""
    errs = {}
    for k, nonzero in checked_params(scene).items():
        w = float(want['static_friction'][0]) if k == 'static_friction' else float(want[k])
        g = float(np.asarray(got[k]).reshape(-1)[0]) if k == 'static_friction' else float(got[k])
        if nonzero:
            assert abs(w) > 1e-6, (scene, k, 'the oracle gradient is zero: the scene does not exercise this parameter', w)
        else:
            assert w == 0.0 and g == 0.0, (scene, k, 'the sticky branch has zero derivative', w, g)
        errs[k] = abs(g - w) / max(1.0, abs(w))
    assert max(errs.values()) < bar, (scene, errs, got, want)
    return errs


def friction_sysid_case(device, iters=12, lr=0.5, n_steps=2, N=600):
    """system identification of a static friction: a cloud sliding over the static box with friction 0.3 gives the target trajectory; gradient
    steps on the friction of the static, started at 0.1, with the loss sum |x_T - x_T(target)|^2 and a step normalised by the first gradient.
    Returns the friction before every iteration and after the last."""
    from fluidlab_b200 import TaichiEnv
    rng = np.random.RandomState(3)
    x = rng.uniform((0.38, 0.385, 0.38), (0.54, 0.45, 0.54), size=(N, 3))
    P = make_particles(x, M.ELASTIC, N_GRID)
    kw = dict(ckpt_dest='cpu', device='cpu') if device == 'cpu' else dict(ckpt_dest='gpu')
    env = TaichiEnv(quality=N_GRID / 64, max_substeps_local=10 * n_steps + 10, gravity=(0.0, -10.0, 0.0), horizon=n_steps + 1, **kw)
    s = env.simulator
    s.use_graphs, s.param_grad = device != 'cpu', True
    env.setup_boundary(**CUBE)
    vox, T = box_sdf((0.12, 0.02, 0.12), 0.3)
    env.add_static(file='box.obj', material=M.CUP, has_dynamics=True, pos=(0.46, 0.36, 0.53), sdf=dict(voxels=vox, T_mesh_to_voxels=T))
    env.particle_bodies.get = lambda: P
    env.build()
    st0 = s.get_state()
    st0['v'][:] = np.array([3.0, -2.0, 2.0], dtype=np.float32)

    def rollout():
        s.cur_substep_global = 0
        s.set_state(0, st0)
        for _ in range(n_steps):
            s.step(None)
        return s.get_state()['x'].astype(np.float64)
    s.enable_grad()
    s.set_contact_params(static_friction=[0.3])
    tgt = rollout()
    mu, hist, scale = 0.1, [], None
    z3, z9 = np.zeros((N, 3), np.float32), np.zeros((N, 3, 3), np.float32)
    for _ in range(iters):
        hist.append(mu)
        s.set_contact_params(static_friction=[mu])
        xT = rollout()
        s.reset_grad()
        s.set_grad((2.0 * (xT - tgt)).astype(np.float32), z3, z9, z9)
        for _ in range(n_steps):
            s.step_grad(None)
        g = float(s.get_param_grad()['static_friction'][0])
        scale = scale or abs(g) / 0.1   # the first step moves the friction by lr * 0.1
        mu = max(0.0, mu - lr * g / scale)
    hist.append(mu)
    return hist
