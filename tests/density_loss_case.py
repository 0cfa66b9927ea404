"""Scenes for the density-loss tests (DensityMatchingLoss, fmpm_loss_density / fmpm_loss_density_grad): the same bodies run on an H100
(tests/test_density_loss_gpu.py) and on the CPU execution-model shim (tests/test_density_loss.py), against the fp64 reference
(tests/density_loss_ref.py) and the fp64 oracle."""
import numpy as np
import torch

import density_loss_ref as dref
from conftest import make_particles
from fluidlab_b200 import macros as M

KERNEL_CASES = ['sorted', 'unsorted', 'aged', 'unused', 'two_mat', 'frozen', 'empty_mask', 'null_target', 'null_sdf']


def rel_max(got, want):
    """max |got - want| relative to the largest entry of want"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def _sim(device, n, P, T=20, param_grad=True):
    from fluidlab_b200 import MPMSimulator
    s = MPMSimulator(dim=3, quality=n / 64, gravity=(0.0, -10.0, 0.0), horizon=50, max_substeps_local=T, max_substeps_global=100000,
                     ckpt_dest='gpu' if device is None else 'cpu', device=device, sort_every=0)
    s.use_graphs, s.param_grad = False, param_grad
    s.setup_boundary(type='cube', lower=(0.05, 0.05, 0.05), upper=(0.95, 0.95, 0.95))
    s.build(None, None, [], P)
    return s


def particle_mass(P, p_vol):
    """the f32 mass the simulator gives every particle (p_vol * rho of its row, MPM:174)"""
    return (np.float32(p_vol) * np.asarray(P['rho'], np.float32)).astype(np.float64)


def sphere_sdf(n, c, r):
    ax = (np.arange(n) + 0.0) / n
    X, Y, Z = np.meshgrid(ax, ax, ax, indexing='ij')
    return (np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r).reshape(-1)


def deposit_matches_p2g(device):
    """one material, every particle used: the reference deposit equals the grid mass of k_p2g; returns the relative error"""
    rng = np.random.RandomState(1)
    n, N = 16, 500
    P = make_particles(rng.uniform(0.2, 0.8, size=(N, 3)), M.ELASTIC, n)
    s = _sim(device, n, P, param_grad=False)
    s.sort_frame(0)
    s.phase('clear_grid', 0); s.phase('p2g', 0, 1)
    _, m, _ = s.read_grid()
    st = s.get_state()
    x = st['x'].astype(np.float64)
    want = dref.deposit(x, particle_mass(P, s.p_vol), dref.selection(x, st['used'], P['mat'], M.ELASTIC, n), n)
    return rel_max(m, want)


def kernel_case(device, case):
    """one frame: the loss, the x adjoint and dL/drho of the kernels against the reference (fresh sort, no sort, a sort with the particles moved
    since, 15 % unused slots, two materials with the mask on one, particles frozen at the grid edge, an empty mask, NULL target / sdf)"""
    rng = np.random.RandomState(KERNEL_CASES.index(case) + 3)
    n, N = 16, 400
    x = rng.uniform(0.3, 0.7, size=(N, 3))
    if case == 'frozen':
        x[:60] = rng.uniform(0.915, 0.99, size=(60, 3))   # int(x / dx - 0.5) > n - 3: the stencil leaves the grid
        x[60:90, 1] = rng.uniform(0.87, 0.9, size=30)      # next to the edge, still inside
    mat = np.where(np.arange(N) % 2 == 0, M.WATER, M.ELASTIC) if case == 'two_mat' else np.full(N, M.ELASTIC)
    used = (rng.rand(N) > 0.15).astype(np.int32) if case == 'unused' else np.ones(N, np.int32)
    P = make_particles(x, mat, n, used=used)
    s = _sim(device, n, P)
    if case != 'unsorted':
        s.sort_frame(0)
    if case == 'aged':   # positions move after the sort: the slots of a cell no longer sit together
        s._pa[0, 0, :, :3] += torch.from_numpy(rng.uniform(-0.6 / n, 0.6 / n, size=(N, 3)).astype(np.float32)).to(s._pa.device)
    st = s.get_state()
    xs = st['x'].astype(np.float64)
    mp = particle_mass(P, s.p_vol)
    row_mask = 0 if case == 'empty_mask' else s.material_row_mask(M.ELASTIC)
    sel = dref.selection(xs, st['used'], P['mat'], M.ELASTIC, n) & (row_mask != 0)
    tgt = None if case == 'null_target' else np.maximum(dref.deposit(xs + 0.04, mp, sel, n) + 2e-4 * rng.rand(n ** 3), 0.0).astype(np.float32)
    sdf = None if case == 'null_sdf' else sphere_sdf(n, (0.5, 0.45, 0.55), 0.15).astype(np.float32)
    wd, ws = 100.0, 0.5
    L, gx, dm = dref.adjoint(xs, mp, sel, n, tgt, sdf, wd, ws)
    dev = s.device
    to = lambda a: None if a is None else torch.from_numpy(a).to(dev)
    scratch = torch.zeros(n ** 3, dtype=torch.float32, device=dev)
    out = torch.zeros(1, dtype=torch.float32, device=dev)
    s.density_loss(scratch, to(tgt), to(sdf), wd, ws, row_mask, out, 0)
    s.reset_grad()
    s.add_x_grad_density(scratch, to(tgt), to(sdf), wd, ws, row_mask, 0)
    got_gx = s.get_grad()['x']
    got_gx = got_gx.cpu().numpy() if torch.is_tensor(got_gx) else np.asarray(got_gx)
    got_rho = s.get_param_grad()['rho']
    table = s.get_material_table()
    pv = float(np.float32(s.p_vol))
    want_rho = np.array([dm[np.asarray(P['mat']) == m].sum() * pv for m in table['mat']])
    scale_rho = np.array([np.abs(dm[np.asarray(P['mat']) == m]).sum() * pv for m in table['mat']])
    got_L = float(out.cpu()[0])
    assert abs(got_L - L) <= 1e-5 * abs(L), (case, got_L, L)
    if case == 'empty_mask':
        assert not got_gx.any() and not got_rho.any(), case
        return
    assert not got_gx[~sel].any(), (case, 'an adjoint on a particle that deposits nothing')
    assert rel_max(got_gx, gx) < 1e-4, (case, rel_max(got_gx, gx))
    assert (np.abs(got_rho - want_rho) <= 1e-4 * np.maximum(np.abs(want_rho), scale_rho)).all(), (case, got_rho, want_rho)


def _oracle(n, P, grav, bnd, v0, n_steps, T):
    from param_grad_ref import ParamGradOracle
    o = ParamGradOracle(n, P, gravity=grav, boundary=bnd, precision=64, max_substeps_local=T)
    N = len(P['x'])
    o.enable_grad()
    o.set_frame(0, P['x'], v0, np.zeros((N, 3, 3)), np.tile(np.eye(3), (N, 1, 1)), P['used'])
    for _ in range(n_steps):
        o.step(None)
    return o


def env_scene(n=32, N=2000, seed=5):
    rng = np.random.RandomState(seed)
    x = rng.uniform((0.38, 0.3, 0.38), (0.62, 0.45, 0.62), size=(N, 3))
    P = make_particles(x, M.ELASTIC, n)
    c = x.mean(0)
    v0 = (np.array([0.0, -1.0, 0.0]) + 4.0 * np.cross(np.array([0.2, 1.0, 0.3]), x - c)).astype(np.float32).astype(np.float64)
    return P, v0


def env_case(device, n_steps=3, T=40):
    """TaichiEnv with DensityMatchingLoss over every step (temporal_range_type='all'), target = the deposits of an oracle run with another v0,
    both terms weighted.  Returns the step losses, dL/d(x0, v0, C0, F0) and dL/drho of the product next to the reference's (the oracle's fp64
    forward and backward seeded per step with the reference's x adjoint) and the direct mass term of dL/drho."""
    from fluidlab_b200 import TaichiEnv, DensityMatchingLoss
    n = 32
    P, v0 = env_scene(n)
    N = len(P['x'])
    grav = (0.0, -10.0, 0.0)
    bnd = dict(type='cube', lower=(0.05, 0.05, 0.05), upper=(0.95, 0.95, 0.95))
    wd, ws = 20.0, 0.5
    pv = float(np.float32((0.5 / n) ** 2))
    mp = (np.float32(pv) * np.asarray(P['rho'], np.float32)).astype(np.float64)
    op = _oracle(n, P, grav, bnd, v0 + np.array([0.4, 0.2, -0.3]), n_steps, T)
    tgt = []
    for i in range(n_steps):
        xp = op.get_frame(10 * (i + 1))['x']
        tgt.append(dref.deposit(xp, mp, dref.selection(xp, P['used'], P['mat'], M.ELASTIC, n), n).astype(np.float32))
    sdf = sphere_sdf(n, (0.55, 0.35, 0.45), 0.1).astype(np.float32)

    kw = dict(ckpt_dest='cpu', device='cpu') if device == 'cpu' else dict(ckpt_dest='gpu')
    env = TaichiEnv(quality=n / 64, max_substeps_local=T, gravity=grav, horizon=n_steps, **kw)
    env.simulator.use_graphs, env.simulator.param_grad = False, True
    env.particle_bodies.get = lambda: P
    env.setup_boundary(**bnd)
    env.setup_loss(loss_cls=DensityMatchingLoss, matching_mat=M.ELASTIC, temporal_range_type='all', weights={'density': wd, 'sdf': ws},
                   target=np.stack(tgt), target_sdf=sdf)
    env.build()
    st = env.get_state()['state']; st['v'] = v0.astype(np.float32)
    env.set_state(st, grad_enabled=True)
    for _ in range(n_steps):
        env.step()
    got_losses = env.loss.step_loss.cpu().numpy().astype(np.float64)
    env.get_final_loss()
    env.reset_grad(); env.get_final_loss_grad()
    for _ in range(n_steps):
        env.step_grad()
    g = env.simulator.get_grad()
    got_g = {k: (g[k].cpu().numpy() if torch.is_tensor(g[k]) else np.asarray(g[k])) for k in 'xvCF'}
    got_rho = float(env.simulator.get_param_grad()['rho'][0])

    def ref_losses(mass_p, P_):
        o = _oracle(n, P_, grav, bnd, v0, n_steps, T)
        out, direct = [], 0.0
        for i in range(n_steps):
            xf = o.get_frame(10 * (i + 1))['x']
            L, gx, dm = dref.adjoint(xf, mass_p, dref.selection(xf, P_['used'], P_['mat'], M.ELASTIC, n), n, tgt[i], sdf, wd, ws)
            out.append(L); direct += dm.sum()
        return o, out, direct
    o, want_losses, direct = ref_losses(mp, P)
    o.reset_grad()
    for i in range(n_steps - 1, -1, -1):
        f = o.cur_substep_local
        xf = o.get_frame(f)['x']
        _, gx, _ = dref.adjoint(xf, mp, dref.selection(xf, P['used'], P['mat'], M.ELASTIC, n), n, tgt[i], sdf, wd, ws)
        gf = o.get_grad_frame(f)
        o.set_grad_frame(f, gf['x'] + gx, gf['v'], gf['C'], gf['F'])
        o.step_grad(None)
    want_g = o.get_grad_frame(0)
    # dL/drho by central differences through the oracle's fp64 forward (the mass enters the dynamics and the deposit)
    rho = float(P['rho'][0]); h = 1e-5 * rho
    fd = []
    for r in (rho + h, rho - h):
        Pr = dict(P); Pr['rho'] = np.full(N, r); Pr['mass'] = np.full(N, (0.5 / n) ** 2 * r)
        fd.append(sum(ref_losses(Pr['mass'], Pr)[1]))
    fd_rho = (fd[0] - fd[1]) / (2 * h)
    return dict(got_losses=got_losses, want_losses=np.array(want_losses), got_g=got_g, want_g=want_g, got_rho=got_rho, fd_rho=fd_rho,
                direct_rho=direct * pv)


def sysid_density_case(device, n_grid=32, N=8000, iters=20, lr=0.06, gamma=0.85, n_steps=2, seed=0, subsample=False):
    """tests/param_grad_case.py::sysid_case without particle correspondence: the recording is the density volumes of the true run's particles
    after a random permutation (subsample=True: a random half of them with twice the mass), the loss DensityMatchingLoss on the last step.
    Returns the relative parameter error max(|mu/mu* - 1|, |lam/lam* - 1|) before every iteration and after the last."""
    from fluidlab_b200 import MPMSimulator, DensityMatchingLoss
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
    st0['v'] = (np.array([0.0, -1.5, 0.0]) + 6.0 * np.cross(np.array([0.3, 1.0, 0.2]), x - c)).astype(np.float32)
    true = s.get_material_table()
    mu_t, lam_t = float(true['mu'][0]), float(true['lam'][0])
    m_p = float(np.float32(s.p_vol) * np.float32(true['rho'][0]))

    def rollout():
        s.cur_substep_global = 0
        s.set_state(0, st0)
        for _ in range(n_steps):
            s.step(None)
    s.enable_grad()
    rollout()
    rec = s.get_state()['x'][rng.permutation(N)]
    mass = m_p
    if subsample:
        rec, mass = rec[:N // 2], 2.0 * m_p
    target = DensityMatchingLoss.density_from_points(rec, mass, n_grid)
    loss = DensityMatchingLoss(M.ELASTIC, target=target, max_loss_steps=1, weights={'density': 1.0 / m_p ** 2}, temporal_range_type='all')
    loss.build(s)
    logp = torch.tensor([np.log(mu_t * 1.3), np.log(lam_t * 0.7)], dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([logp], lr=lr)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma)
    errs = []
    for _ in range(iters):
        mu, lam = (float(v) for v in torch.exp(logp.detach()))
        errs.append(max(abs(mu / mu_t - 1), abs(lam / lam_t - 1)))
        s.set_material_table(mu=[mu], lam=[lam])
        rollout()
        s.reset_grad()
        loss.get_final_loss_grad()   # the seed of the recorded (last) frame
        loss.compute_step_loss_grad(0, s.cur_substep_local)
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
