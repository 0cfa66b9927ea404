"""Scenes for the parameter-gradient tests (MPMSimulator.param_grad: dL/d(mu, lam, rho) per material row and dL/dgravity): the same bodies run
on an H100 (tests/test_param_grad_gpu.py) and on the CPU execution-model shim (tests/test_param_grad.py), each against the fp64 oracle."""
import numpy as np

from conftest import make_particles
from fluidlab_b200 import macros as M
from param_grad_ref import ParamGradOracle


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def oracle_rows(og, P, table, p_vol):
    """per-particle oracle gradients summed into the simulator's material rows (matched on (material, rho)), in get_param_grad()'s units; `scale`
    holds the sums of the magnitudes of the per-particle terms (what an fp32 sum of them is accurate relative to)"""
    out = {k: np.zeros(len(table['mat'])) for k in ('mu', 'lam', 'rho')}
    out['scale'] = {k: np.zeros(len(table['mat'])) for k in ('mu', 'lam', 'rho')}
    pv = float(np.float32(p_vol))
    for r, (m, rh) in enumerate(zip(table['mat'], table['rho'])):
        sel = (np.asarray(P['mat']) == m) & (np.asarray(P['rho']).astype(np.float32).astype(np.float64) == rh)   # the table keeps rho in f32
        for k, a, f in (('mu', og['mu'], 1.0), ('lam', og['lam'], 1.0), ('rho', og['mass'], pv)):
            out[k][r] = a[sel].sum() * f
            out['scale'][k][r] = np.abs(a[sel]).sum() * f
    out['gravity'] = og['gravity']
    out['scale']['gravity'] = np.full(3, np.abs(og['gravity']).max())
    return out


def assert_param_grads_close(got, want, bar, what):
    """per component: |got - want| <= bar * max(|want|, the sum of the magnitudes of its terms)"""
    errs = {k: float((np.abs(np.asarray(got[k]) - want[k]) / np.maximum(np.abs(want[k]), np.maximum(want['scale'][k], 1e-30))).max())
            for k in ('mu', 'lam', 'rho', 'gravity')}
    assert max(errs.values()) < bar, (what, errs, got, want)
    return errs


CASE_MATS = {'water': [M.WATER], 'elastic': [M.ELASTIC], 'icecream': [M.ICECREAM], 'milk_vis': [M.MILK_VIS],
             'mixed': [M.WATER, M.ELASTIC, M.ICECREAM, M.MILK_VIS]}


def substep_case(device, case, sort):
    """one backward substep (the last of a 10-substep step) with a random adjoint seed: 300 particles, 15 % unused, random v / C / F.
    sort=True: cell-sorted slots and the stored-grid backward (fmpm_substep_grad_stored); False: no sort (mixed rows inside warps in the 'mixed'
    case) and the recompute backward (fmpm_substep_grad).  The parameter gradients must match the oracle's, and turning param_grad on must
    leave the state adjoint as it was."""
    from fluidlab_b200 import MPMSimulator
    rng = np.random.RandomState(11)
    n, N = 16, 300
    mats = CASE_MATS[case]
    x = rng.uniform(0.35, 0.65, size=(N, 3))
    mat = np.array([mats[i % len(mats)] for i in range(N)], dtype=np.int32)
    used = (rng.rand(N) > 0.15).astype(np.int32)
    v0 = (rng.randn(N, 3) * 0.5).astype(np.float32)
    F0 = (np.eye(3)[None] + rng.randn(N, 3, 3) * 0.05).astype(np.float32)
    C0 = (rng.randn(N, 3, 3) * 0.5).astype(np.float32)
    P = make_particles(x, mat, n, used=used)
    bnd = dict(type='cube', lower=(0.3, 0.3, 0.3), upper=(0.7, 0.7, 0.7))
    grav = (0.5, -10.0, 0.2)
    seed = {k: rng.randn(*s).astype(np.float32) for k, s in (('x', (N, 3)), ('v', (N, 3)), ('C', (N, 3, 3)), ('F', (N, 3, 3)))}
    res = {}
    for pg in (False, True):
        s = MPMSimulator(dim=3, quality=n / 64, gravity=grav, horizon=50, max_substeps_local=20, max_substeps_global=1000, ckpt_dest='gpu' if device is None else 'cpu',
                         device=device, sort_every=1 if sort else 0)
        s.use_graphs, s.store_grids, s.fuse_g2p2g, s.param_grad = False, sort, False, pg
        s.setup_boundary(**bnd)
        s.build(None, None, [], P)
        st = s.get_state(); st['v'][:] = v0; st['F'][:] = F0; st['C'][:] = C0; s.set_state(0, st)
        s.enable_grad()
        s.step(None)
        s.reset_grad(); s.set_grad(seed['x'], seed['v'], seed['C'], seed['F'])
        s.cur_substep_global -= 1
        s.substep_grad(9, True)
        res[pg] = (s.get_grad(), s.get_param_grad() if pg else None, s.get_material_table(), s.p_vol)
    for k in 'xvCF':   # equal up to the order of the unordered float reductions of the scatters, which differs from run to run with or without param_grad
        assert rel(res[True][0][k], res[False][0][k]) < 1e-3, ('state adjoint changed by param_grad', k, rel(res[True][0][k], res[False][0][k]))
    o = ParamGradOracle(n, P, gravity=grav, boundary=bnd, precision=64, max_substeps_local=20)
    o.set_frame(0, x, v0, C0, F0, used)
    for f in range(10):
        o.substep(f)
    o.reset_grad(); o.set_grad_frame(10, seed['x'], seed['v'], seed['C'], seed['F'])
    o.substep_grad(9)
    _, got, table, p_vol = res[True]
    want = oracle_rows(o.get_param_grad(), P, table, p_vol)
    return assert_param_grads_close(got, want, 1e-4, (case, sort))


def latteart_case(device, sort_every, n_steps=3, T=20):
    """LatteArt-like TaichiEnv (AgentInjector pouring MILK into COFFEE, LatteArtLoss, the call sequence of optimizer/solver.py:23-59) with
    param_grad: a ring of T substeps for a 3-step horizon, so the backward pass re-simulates a chunk.  dL/d(mu, lam, rho, g) against the oracle;
    loss and dLoss/dAction as in the run without param_grad."""
    from fluidlab_b200 import TaichiEnv, LatteArtLoss
    n_grid, n_coffee, n_milk, flux = 16, 400, 120, 2
    rng = np.random.RandomState(21)
    x = np.concatenate([np.tile(M.NOWHERE, (n_milk, 1)), rng.uniform((0.38, 0.36, 0.38), (0.62, 0.45, 0.62), size=(n_coffee, 3))])
    mat = np.concatenate([np.full(n_milk, M.MILK), np.full(n_coffee, M.COFFEE)])
    used = np.concatenate([np.zeros(n_milk), np.ones(n_coffee)]).astype(np.int32)
    P = make_particles(x, mat, n_grid, used=used)
    bnd = dict(type='cylinder', xz_radius=0.2, xz_center=(0.5, 0.5), y_range=(0.34, 0.9))
    ebnd = dict(type='cylinder', xz_radius=0.12, xz_center=(0.5, 0.5), y_range=(0.55, 0.55))
    cfg = dict(type='AgentInjector', effectors=[dict(type='Injector', params=dict(radius=0.0075, flux=flux, init_pos=(0.5, 0.5, 0.5), action_dim=3, inject_v=(0.0, -3.0, 0.0),
                                                                                 action_scale_p=(1.0, 1.0, 1.0), action_scale_v=(1.0, 1.0, 1.0), locally_random=True), boundary=ebnd)])
    tgt = [rng.uniform(0.4, 0.6, size=x.shape).astype(np.float32) for _ in range(n_steps)]
    actions = rng.uniform(-0.004, 0.004, size=(n_steps, 3)).astype(np.float32)
    action_p = np.array([0.47, 0.55, 0.52], dtype=np.float32)
    res = {}
    for pg in (False, True):
        kw = dict(ckpt_dest='cpu', device='cpu') if device == 'cpu' else dict(ckpt_dest='gpu')
        env = TaichiEnv(quality=n_grid / 64, max_substeps_local=T, gravity=(0.0, -20.0, 0.0), horizon=n_steps, **kw)
        env.simulator.use_graphs, env.simulator.fuse_g2p2g, env.simulator.sort_every = False, False, sort_every
        env.simulator.param_grad = pg
        np.random.seed(5)
        env.setup_agent(cfg)
        env.particle_bodies.get = lambda: P
        env.setup_boundary(**bnd)
        env.setup_loss(loss_cls=LatteArtLoss, type='diff', target=tgt, weights={'chamfer': 1.0})
        env.build()
        rv = env.agent.effectors[0].random_vector_np
        env.set_state(env.get_state()['state'], grad_enabled=True)
        env.apply_agent_action_p(action_p)
        for i in range(n_steps):
            env.step(actions[i])
        info = env.get_final_loss()
        env.reset_grad(); env.get_final_loss_grad()
        for i in range(n_steps - 1, -1, -1):
            env.step_grad(actions[i])
        env.apply_agent_action_p_grad(action_p)
        sim = env.simulator
        res[pg] = (info['loss'], env.agent.get_grad(n_steps), sim.get_param_grad() if pg else None, sim.get_material_table(), sim.p_vol)
    assert abs(res[False][0] - res[True][0]) <= 1e-5 * abs(res[False][0]) and rel(res[True][1], res[False][1]) < 1e-4, 'loss / dLoss/dAction changed by param_grad'
    o = ParamGradOracle(n_grid, P, gravity=(0, -20, 0), boundary=bnd, precision=64, max_substeps_local=T)
    o.add_effector(type=1, action_dim=3, boundary=ebnd, radius=0.0075, flux=flux, inject_v=(0, -3, 0), inject_p=(0, 0, 0), locally_random=True, random_vector=rv,
                   act_range=np.where(used == 0)[0], max_action_steps=n_steps + 1)
    N = len(x)
    o.enable_grad()
    o.set_frame(0, P['x'], np.zeros((N, 3)), np.zeros((N, 3, 3)), np.tile(np.eye(3), (N, 1, 1)), P['used'])
    o.set_effector_state(0, 0, np.array([0.5, 0.5, 0.5, 1, 0, 0, 0, 0.0]))
    o.apply_action_p(action_p)
    for i in range(n_steps):
        o.step(actions[i])
    o.reset_grad()
    for i in range(n_steps - 1, -1, -1):
        o.loss_seed(o.cur_substep_local, M.MILK, 1.0, tgt[i]); o.step_grad(actions[i])
    _, _, got, table, p_vol = res[True]
    want = oracle_rows(o.get_param_grad(), P, table, p_vol)
    assert np.abs(want['lam']).max() > 0 and np.abs(want['gravity']).max() > 0
    return assert_param_grads_close(got, want, 1e-4, ('latteart', sort_every))


def sysid_case(device, n_grid=16, N=1200, iters=20, lr=0.06, gamma=0.85, n_steps=2, seed=0):
    """system identification: an ELASTIC block thrown against the floor, mu and lam started 30 % off (mu high, lam low); torch.optim.Adam on
    (log mu, log lam) with gradients from get_param_grad and an exponentially decaying step (gamma), loss = sum |x_T - x_T(true)|^2 after n_steps
    steps.  Returns the relative parameter
    error max(|mu/mu* - 1|, |lam/lam* - 1|) before every iteration and after the last."""
    import torch
    from fluidlab_b200 import MPMSimulator
    rng = np.random.RandomState(seed)
    x = rng.uniform((0.35, 0.32, 0.35), (0.65, 0.5, 0.65), size=(N, 3))
    P = make_particles(x, M.ELASTIC, n_grid)
    s = MPMSimulator(dim=3, quality=n_grid / 64, gravity=(0.0, -10.0, 0.0), horizon=50, max_substeps_local=10 * n_steps + 10, max_substeps_global=100000,
                     ckpt_dest='gpu' if device is None else 'cpu', device=device)
    s.use_graphs = device is None
    s.setup_boundary(type='cube', lower=(0.3, 0.3, 0.3), upper=(0.7, 0.7, 0.7))
    s.param_grad = True
    s.build(None, None, [], P)
    st0 = s.get_state()
    c = x.mean(0)
    st0['v'] = (np.array([0.0, -1.5, 0.0]) + 6.0 * np.cross(np.array([0.3, 1.0, 0.2]), x - c)).astype(np.float32)   # falling and spinning: shear and compression
    true = s.get_material_table()
    mu_t, lam_t = float(true['mu'][0]), float(true['lam'][0])

    def rollout(grad_seed=None):
        s.cur_substep_global = 0
        s.set_state(0, st0)
        for _ in range(n_steps):
            s.step(None)
        return s.get_state()['x'].astype(np.float64)
    s.enable_grad()
    tgt = rollout()
    logp = torch.tensor([np.log(mu_t * 1.3), np.log(lam_t * 0.7)], dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([logp], lr=lr)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma)
    errs = []
    for _ in range(iters):
        mu, lam = (float(v) for v in torch.exp(logp.detach()))
        errs.append(max(abs(mu / mu_t - 1), abs(lam / lam_t - 1)))
        s.set_material_table(mu=[mu], lam=[lam])
        xT = rollout()
        s.reset_grad()
        z3, z9 = np.zeros((N, 3), np.float32), np.zeros((N, 3, 3), np.float32)
        s.set_grad((2.0 * (xT - tgt)).astype(np.float32), z3, z9, z9)
        for _ in range(n_steps):
            s.step_grad(None)
        g = s.get_param_grad()
        opt.zero_grad()
        logp.grad = torch.tensor([g['mu'][0] * mu, g['lam'][0] * lam], dtype=torch.float64)
        opt.step()
        sched.step()
    mu, lam = (float(v) for v in torch.exp(logp.detach()))
    errs.append(max(abs(mu / mu_t - 1), abs(lam / lam_t - 1)))
    return errs
