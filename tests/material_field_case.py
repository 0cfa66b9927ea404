"""Scenes for the per-particle material-field tests (MPMSimulator.set_material_field): the same bodies run on an H100
(tests/test_material_field_gpu.py) and on the CPU execution-model shim (tests/test_material_field.py), each against the fp64 oracle, which takes
mu and lam per particle.  The oracle's per-particle parameter adjoints (tests/param_grad_ref.py, ParamGradOracle.pg) are the reference for
get_param_grad()['mu_field'] / ['lam_field']; their row sums (param_grad_case.oracle_rows) for the row keys."""
import numpy as np

from conftest import make_particles
from fluidlab_b200 import macros as M
from param_grad_ref import ParamGradOracle
import param_grad_case as pgc

rel = pgc.rel
CUBE = dict(type='cube', lower=(0.3, 0.3, 0.3), upper=(0.7, 0.7, 0.7))
GRAV = (0.5, -10.0, 0.2)
CASE_MATS = {'elastic': [M.ELASTIC], 'icecream': [M.ICECREAM], 'milk_vis': [M.MILK_VIS], 'mixed': [M.WATER, M.ELASTIC, M.ICECREAM, M.MILK_VIS]}


def random_field(P, rng, zero_frac=0.0, spread=2.0):
    """per-particle (mu, lam) around each particle's row value (x 1/spread .. spread), fp32-representable; a fraction of the particles gets mu = 0"""
    mu = (P['mu'] * np.exp(rng.uniform(-np.log(spread), np.log(spread), len(P['mu'])))).astype(np.float32)
    lam = (P['lam'] * np.exp(rng.uniform(-np.log(spread), np.log(spread), len(P['lam'])))).astype(np.float32)
    water = P['mu'] == 0
    mu[water] = rng.uniform(0.0, 300.0, water.sum()).astype(np.float32)   # liquids with mu_p > 0 (and some left at 0 below)
    if zero_frac > 0:
        mu[rng.rand(len(mu)) < zero_frac] = 0.0
    return mu.astype(np.float64), lam.astype(np.float64)


def _scene(case, N=300, n=16, seed=11):
    rng = np.random.RandomState(seed)
    mats = CASE_MATS[case]
    x = rng.uniform(0.35, 0.65, size=(N, 3))
    mat = np.array([mats[i % len(mats)] for i in range(N)], dtype=np.int32)
    used = (rng.rand(N) > 0.15).astype(np.int32)
    st = dict(x=x, v=(rng.randn(N, 3) * 0.5).astype(np.float32), F=(np.eye(3)[None] + rng.randn(N, 3, 3) * 0.05).astype(np.float32),
              C=(rng.randn(N, 3, 3) * 0.5).astype(np.float32), used=used)
    P = make_particles(x, mat, n, used=used)
    seed_g = {k: rng.randn(*s).astype(np.float32) for k, s in (('x', (N, 3)), ('v', (N, 3)), ('C', (N, 3, 3)), ('F', (N, 3, 3)))}
    return rng, P, st, seed_g


def _sim(device, P, n, sort, T=20, pg=True, fuse=False):
    from fluidlab_b200 import MPMSimulator
    s = MPMSimulator(dim=3, quality=n / 64, gravity=GRAV, horizon=50, max_substeps_local=T, max_substeps_global=1000, ckpt_dest='gpu' if device is None else 'cpu',
                     device=device, sort_every=1 if sort else 0)
    s.use_graphs, s.store_grids, s.fuse_g2p2g, s.param_grad = device is None, sort, fuse, pg
    s.setup_boundary(**CUBE)
    s.build(None, None, [], P)
    return s


def _run_one_substep_grad(s, st, seed_g, field=None):
    """one step forward, then the backward substep of its last substep with the adjoint seed; returns (frame after the step, state adjoint,
    get_param_grad())"""
    if field is not None:
        s.set_material_field(*field)
    g = s.get_state(); g['v'][:] = st['v']; g['F'][:] = st['F']; g['C'][:] = st['C']; s.set_state(0, g)
    s.enable_grad()
    s.step(None)
    fr = s.readframe(10)
    s.reset_grad(); s.set_grad(seed_g['x'], seed_g['v'], seed_g['C'], seed_g['F'])
    s.cur_substep_global -= 1
    s.substep_grad(9, True)
    return fr, s.get_grad(), s.get_param_grad()


def field_equals_table_case(device, case, sort):
    """a field equal to every particle's row values reproduces the table run: states, state adjoint and the row keys of get_param_grad()"""
    _, P, st, seed_g = _scene(case)
    res = {}
    for use_field in (False, True):
        s = _sim(device, P, 16, sort)
        res[use_field] = _run_one_substep_grad(s, st, seed_g, (P['mu'], P['lam']) if use_field else None)
    (fa, ga, pa), (fb, gb, pb) = res[False], res[True]
    for k in ('x', 'v', 'C', 'F'):
        assert rel(fb[k], fa[k]) < 1e-5, ('state', k, rel(fb[k], fa[k]))
        assert rel(gb[k], ga[k]) < 1e-3, ('state adjoint', k, rel(gb[k], ga[k]))   # unordered scatter reductions differ from run to run
    for k in ('mu', 'lam', 'rho', 'gravity'):
        assert rel(pb[k], pa[k]) < 1e-3, ('row key', k, pb[k], pa[k])
    np.testing.assert_allclose(pb['mu_field'].sum(), pb['mu'].sum(), rtol=1e-9)
    assert 'mu_field' not in pa


def heterogeneous_case(device, case, sort, zero_frac=0.0, fuse=False):
    """random per-particle (mu, lam) against the fp64 oracle: the frame after one step, and one backward substep's state adjoint and per-particle
    dL/d(mu, lam) (the oracle's unreduced ParamGradOracle.pg) at the 1e-4 bar, the row sums against oracle_rows.  fuse (with sort: the stored-grid
    path): the forward step runs the fused g2p2g kernels (fmpm_substeps_fused_store: k_g2p2g_field<true, false>).  Returns the errors."""
    rng, P, st, seed_g = _scene(case)
    mu, lam = random_field(P, rng, zero_frac)
    s = _sim(device, P, 16, sort, fuse=fuse)
    fr, g, pg = _run_one_substep_grad(s, st, seed_g, (mu, lam))
    Pf = dict(P, mu=mu, lam=lam)
    o = ParamGradOracle(16, Pf, gravity=GRAV, boundary=CUBE, precision=64, max_substeps_local=20)
    o.set_frame(0, st['x'], st['v'], st['C'], st['F'], st['used'])
    for f in range(10):
        o.substep(f)
    want_fr = o.get_frame(10)
    o.reset_grad(); o.set_grad_frame(10, seed_g['x'], seed_g['v'], seed_g['C'], seed_g['F'])
    o.substep_grad(9)
    og, opg = o.get_grad_frame(9), o.get_param_grad()
    errs = {('frame', k): rel(fr[k], want_fr[k]) for k in ('x', 'v', 'C', 'F')}
    errs.update({('adjoint', k): rel(g[k], og[k]) for k in ('x', 'v', 'C', 'F')})
    errs[('field', 'mu')] = rel(pg['mu_field'], opg['mu'])
    errs[('field', 'lam')] = rel(pg['lam_field'], opg['lam'])
    # fp32 after 10 substeps; the rest 1e-4.  The all-plastic scene is worse conditioned per particle (the clamp of the singular values): with a
    # field equal to the table it already reaches 2.5e-4 (C) and 5.7e-4 (dL/dlam_p) on the shim, so its per-particle bar is 1e-3
    rest = 1e-3 if case == 'icecream' else 1e-4
    bars = {('frame', 'x'): 1e-5, ('frame', 'F'): 1e-5, ('frame', 'v'): rest, ('frame', 'C'): rest}
    bad = {k: e for k, e in errs.items() if not e < bars.get(k, rest)}
    assert not bad, (case, sort, bad, errs)
    assert np.abs(opg['mu']).max() > 0 and np.abs(opg['lam']).max() > 0
    want = pgc.oracle_rows(opg, P, s.get_material_table(), s.p_vol)
    errs['rows'] = pgc.assert_param_grads_close(pg, want, 1e-4, (case, sort))
    return errs


def ring_case(device, sort_every, n_steps=3, T=20, N=400):
    """a T = 20 ring over 3 steps (the backward re-simulates the first chunk), a heterogeneous field, index-matched loss on the last frame: the
    per-particle dL/d(mu, lam) against the oracle.  Sort epochs change the slot order between steps, so a field or gradient gathered in the wrong
    order fails here."""
    rng = np.random.RandomState(31)
    n = 16
    x = rng.uniform(0.38, 0.62, size=(N, 3))
    mat = np.array([(M.ELASTIC, M.ICECREAM)[i % 2] for i in range(N)], dtype=np.int32)
    P = make_particles(x, mat, n)
    mu, lam = random_field(P, rng)
    v0 = (rng.randn(N, 3) * 0.4).astype(np.float32)
    gx = rng.randn(N, 3).astype(np.float32)
    s = _sim(device, P, n, False, T=T)
    s.sort_every, s.store_grids = sort_every, False
    s.set_material_field(mu, lam)
    st = s.get_state(); st['v'][:] = v0; s.set_state(0, st)
    s.enable_grad()
    for _ in range(n_steps):
        s.step(None)
    s.reset_grad()
    z3, z9 = np.zeros((N, 3), np.float32), np.zeros((N, 3, 3), np.float32)
    s.set_grad(gx, z3, z9, z9)
    for _ in range(n_steps):
        s.step_grad(None)
    got = s.get_param_grad()
    o = ParamGradOracle(n, dict(P, mu=mu, lam=lam), gravity=GRAV, boundary=CUBE, precision=64, max_substeps_local=T)
    o.enable_grad()
    o.set_frame(0, x, v0, np.zeros((N, 3, 3)), np.tile(np.eye(3), (N, 1, 1)), P['used'])
    for _ in range(n_steps):
        o.step(None)
    o.reset_grad(); o.set_grad_frame(o.cur_substep_local, gx, z3, z9, z9)
    for _ in range(n_steps):
        o.step_grad(None)
    want = o.get_param_grad()
    # over 30 substeps the fp32 path drifts from fp64 by up to ~6e-3 per particle and ~3e-3 in the row sums, the same with a field equal to the
    # table (measured on the shim and an H100); a field or gradient in the wrong slot order gives errors of order 1
    errs = dict(mu=rel(got['mu_field'], want['mu']), lam=rel(got['lam_field'], want['lam']))
    assert max(errs.values()) < 2e-2, (sort_every, errs)
    errs['rows'] = pgc.assert_param_grads_close(got, pgc.oracle_rows(want, P, s.get_material_table(), s.p_vol), 1e-2, ('ring', sort_every))
    return errs


def _oracle_loss(P, st, seed_g, mu, lam, n_sub=10):
    o = ParamGradOracle(16, dict(P, mu=mu, lam=lam), gravity=GRAV, boundary=CUBE, precision=64, max_substeps_local=20)
    o.set_frame(0, st['x'], st['v'], st['C'], st['F'], st['used'])
    for f in range(n_sub):
        o.substep(f)
    fr = o.get_frame(n_sub)
    return sum(float((seed_g[k].astype(np.float64) * fr[k]).sum()) for k in ('x', 'v', 'C', 'F'))


def central_difference_case(device, n_particles=3):
    """the simulator's per-particle dL/dmu_p and dL/dlam_p over a whole step (10 backward substeps) against central differences of the oracle's
    fp64 forward, for a few particles and along a random direction of the whole field"""
    rng, P, st, seed_g = _scene('mixed', N=200)
    mu, lam = random_field(P, rng)
    s = _sim(device, P, 16, True)
    s.set_material_field(mu, lam)
    g = s.get_state(); g['v'][:] = st['v']; g['F'][:] = st['F']; g['C'][:] = st['C']; s.set_state(0, g)
    s.enable_grad()
    s.step(None)
    s.reset_grad(); s.set_grad(seed_g['x'], seed_g['v'], seed_g['C'], seed_g['F'])
    s.step_grad(None)
    got = s.get_param_grad()
    used = np.where(st['used'] != 0)[0]
    picks = used[np.argsort(-np.abs(got['mu_field'][used]))[:n_particles]]
    out = []
    for p in picks:
        for key, a, b in (('mu', mu, got['mu_field']), ('lam', lam, got['lam_field'])):
            h = 1e-4 * max(abs(a[p]), 1.0)
            ap, am = a.copy(), a.copy(); ap[p] += h; am[p] -= h
            fd = ((_oracle_loss(P, st, seed_g, ap, lam) - _oracle_loss(P, st, seed_g, am, lam)) if key == 'mu' else
                  (_oracle_loss(P, st, seed_g, mu, ap) - _oracle_loss(P, st, seed_g, mu, am))) / (2 * h)
            out.append((key, int(p), fd, float(b[p])))
            assert abs(fd - b[p]) <= 2e-3 * max(abs(fd), 1e-3 * np.abs(b).max()), out[-1]
    dmu, dlam = rng.randn(len(mu)) * mu * 1e-4, rng.randn(len(lam)) * lam * 1e-4
    fd = (_oracle_loss(P, st, seed_g, mu + dmu, lam + dlam) - _oracle_loss(P, st, seed_g, mu - dmu, lam - dlam)) / 2
    an = float((got['mu_field'] * dmu).sum() + (got['lam_field'] * dlam).sum())
    assert abs(fd - an) <= 2e-3 * abs(fd), ('directional', fd, an)
    return out, (fd, an)



def fused_forward_case(device, case='mixed'):
    """forward-only steps on the fused path with a random field (k_p2g_field, then k_fwd<2, false, false> for the inner substeps): the frame after
    two steps against the fp64 oracle, and the same frame as the unfused per-substep path with the same field"""
    rng, P, st, _ = _scene(case)
    mu, lam = random_field(P, rng)
    fr = {}
    for fuse in (True, False):
        s = _sim(device, P, 16, True, pg=False, fuse=fuse)
        s.set_material_field(mu, lam)
        g = s.get_state(); g['v'][:] = st['v']; g['F'][:] = st['F']; g['C'][:] = st['C']; s.set_state(0, g)
        s.step(None); s.step(None)
        fr[fuse] = s.readframe(20)
    if device == 'cpu':
        assert s._lib.fmpm_fwd_path(s._h) & 1, 'the fused forward path runs k_fwd'
    o = ParamGradOracle(16, dict(P, mu=mu, lam=lam), gravity=GRAV, boundary=CUBE, precision=64, max_substeps_local=20)
    o.set_frame(0, st['x'], st['v'], st['C'], st['F'], st['used'])
    for f in range(20):
        o.substep(f)
    want = o.get_frame(20)
    errs = {k: rel(fr[True][k], want[k]) for k in ('x', 'v', 'C', 'F')}
    errs.update({('unfused', k): rel(fr[True][k], fr[False][k]) for k in ('x', 'v', 'C', 'F')})
    bars = dict(x=1e-5, F=1e-5, v=2e-4, C=2e-4)
    bad = {k: e for k, e in errs.items() if not e < bars[k if isinstance(k, str) else k[1]]}
    assert not bad, (bad, errs)
    return errs


def injector_case(device, fuse, sort_every=1, n_steps=3, T=20):
    """an AgentInjector pouring MILK into COFFEE (param_grad_case.latteart_case) with a random field on both liquids (mu_p > 0): the injected
    particles scatter through k_p2g_injected_field (fused steps, fuse=True, with k_g2p2g_field) or the per-substep kernels (fuse=False); a T = 20
    ring over 3 steps.  Per-particle dL/d(mu, lam) and their row sums against the oracle (measured on the shim: 5e-5 per particle, 3e-4 in the row
    sums; the liquids are better conditioned than ring_case's elastic / plastic body)."""
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
    mu = rng.uniform(20.0, 300.0, len(x)).astype(np.float32).astype(np.float64)
    lam = (P['lam'] * rng.uniform(0.5, 2.0, len(x))).astype(np.float32).astype(np.float64)
    kw = dict(ckpt_dest='cpu', device='cpu') if device == 'cpu' else dict(ckpt_dest='gpu')
    env = TaichiEnv(quality=n_grid / 64, max_substeps_local=T, gravity=(0.0, -20.0, 0.0), horizon=n_steps, **kw)
    env.simulator.use_graphs, env.simulator.fuse_g2p2g, env.simulator.sort_every = False, fuse, sort_every
    env.simulator.store_grids = fuse
    env.simulator.param_grad = True
    np.random.seed(5)
    env.setup_agent(cfg)
    env.particle_bodies.get = lambda: P
    env.setup_boundary(**bnd)
    env.setup_loss(loss_cls=LatteArtLoss, type='diff', target=tgt, weights={'chamfer': 1.0})
    env.build()
    sim = env.simulator
    sim.set_material_field(mu, lam)
    rv = env.agent.effectors[0].random_vector_np
    env.set_state(env.get_state()['state'], grad_enabled=True)
    env.apply_agent_action_p(action_p)
    for i in range(n_steps):
        env.step(actions[i])
    env.get_final_loss()
    env.reset_grad(); env.get_final_loss_grad()
    for i in range(n_steps - 1, -1, -1):
        env.step_grad(actions[i])
    got = sim.get_param_grad()
    o = ParamGradOracle(n_grid, dict(P, mu=mu, lam=lam), gravity=(0, -20, 0), boundary=bnd, precision=64, max_substeps_local=T)
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
    want = o.get_param_grad()
    milk = np.arange(n_milk)
    assert np.abs(want['mu'][milk]).max() > 0, 'the injected particles carry a gradient'
    errs = dict(mu=rel(got['mu_field'], want['mu']), lam=rel(got['lam_field'], want['lam']),
                mu_milk=rel(got['mu_field'][milk], want['mu'][milk]), lam_milk=rel(got['lam_field'][milk], want['lam'][milk]))
    assert max(errs.values()) < 2e-4, (fuse, errs)
    errs['rows'] = pgc.assert_param_grads_close(got, pgc.oracle_rows(want, P, sim.get_material_table(), sim.p_vol), 1e-3, ('injector', fuse))
    return errs


def knn_smoother(x, k=16, passes=3):
    """the Sobolev preconditioner of identification_case: per-particle values averaged over each particle's k nearest neighbours in the reference
    configuration x (itself included), `passes` times"""
    from scipy.spatial import cKDTree
    _, nb = cKDTree(x).query(x, k)

    def smooth(g):
        for _ in range(passes):
            g = g[nb].mean(1)
        return g
    return smooth


def identification_case(device, n_grid=16, N=1200, iters=20, lr=0.05, n_steps=2, seed=0):
    """a stiff core (mu and lam x 4 within 0.08 of the centre) inside a soft ELASTIC block, recovered from the recorded end positions of the thrown,
    spinning block (index-matched loss after n_steps steps).  The unknowns are per particle: the log of a stiffness scale s_p (mu_p = s_p mu,
    lam_p = s_p lam, a fixed Poisson ratio), started at 2 everywhere, fitted by torch.optim.Adam with dL/dlog s_p = s_p (mu dL/dmu_p + lam dL/dlam_p)
    from get_param_grad()['mu_field' / 'lam_field'], preconditioned by knn_smoother (a Sobolev gradient: positions alone do not pin a value on each
    particle, the smoothed gradient descends the same loss).  Returns per iteration the field error sqrt(mean(log(s_p / s*_p)^2)) and the mean s
    of the core and of the shell, before every iteration and after the last."""
    import torch
    rng = np.random.RandomState(seed)
    x = rng.uniform((0.35, 0.32, 0.35), (0.65, 0.5, 0.65), size=(N, 3))
    P = make_particles(x, M.ELASTIC, n_grid)
    c = x.mean(0)
    core = np.abs(x - c).max(1) < 0.08
    s_t = np.where(core, 4.0, 1.0)
    s = _sim(device, P, n_grid, True, T=10 * n_steps + 10)
    st0 = s.get_state()
    st0['v'] = (np.array([0.0, -1.5, 0.0]) + 6.0 * np.cross(np.array([0.3, 1.0, 0.2]), x - c)).astype(np.float32)
    smooth = knn_smoother(x)

    def rollout(sv):
        s.set_material_field(sv * P['mu'], sv * P['lam'])
        s.cur_substep_global = 0
        s.set_state(0, st0)
        for _ in range(n_steps):
            s.step(None)
        return s.get_state()['x'].astype(np.float64)
    s.enable_grad()
    tgt = rollout(s_t)
    logs = torch.full((N,), float(np.log(2.0)), dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([logs], lr=lr, eps=1e-30)   # the gradients are ~1e-8: keep Adam's eps below them
    hist = []
    z3, z9 = np.zeros((N, 3), np.float32), np.zeros((N, 3, 3), np.float32)
    for it in range(iters + 1):
        sv = torch.exp(logs.detach()).numpy()
        hist.append((float(np.sqrt((np.log(sv / s_t) ** 2).mean())), float(sv[core].mean()), float(sv[~core].mean())))
        if it == iters:
            break
        xT = rollout(sv)
        s.reset_grad()
        s.set_grad((2.0 * (xT - tgt)).astype(np.float32), z3, z9, z9)
        for _ in range(n_steps):
            s.step_grad(None)
        g = s.get_param_grad()
        opt.zero_grad()
        logs.grad = torch.tensor(smooth((g['mu_field'] * P['mu'] + g['lam_field'] * P['lam']) * sv))
        opt.step()
    return hist
