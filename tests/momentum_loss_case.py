"""Scenes for the momentum-loss tests (MomentumMatchingLoss, fmpm_loss_momentum / fmpm_loss_momentum_grad): the same bodies run on an H100
(tests/test_momentum_loss_gpu.py) and on the CPU execution-model shim (tests/test_momentum_loss.py), against the fp64 reference
(tests/momentum_loss_ref.py) and the fp64 oracle."""
import numpy as np
import torch

import density_loss_case as dlc
import density_loss_ref as dref
import momentum_loss_ref as mref
from conftest import make_particles
from fluidlab_b200 import macros as M

# the density loss's cases, plus a NULL momentum target (m* given, P* = 0) and w_momentum = 0 (then the density loss's values)
KERNEL_CASES = dlc.KERNEL_CASES + ['null_momentum', 'no_momentum_weight']
rel_max = dlc.rel_max


def _np(a):
    return a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)


def pack_target(m_star, p_star, G):
    """(G, 4) float32 (P*, m*) as the kernels read it; None when both are None"""
    if m_star is None and p_star is None:
        return None
    t = np.zeros((G, 4), np.float32)
    if p_star is not None:
        t[:, :3] = p_star
    if m_star is not None:
        t[:, 3] = m_star
    return t


def _set_vc(s, rng, N, c_scale=8.0):
    st = s.get_state()
    st['v'] = rng.uniform(-1.0, 1.0, size=(N, 3)).astype(np.float32)
    st['C'] = (c_scale * rng.randn(N, 3, 3)).astype(np.float32)
    s.set_state(0, st)


def deposit_matches_p2g(device):
    """one material with mu = lam = 0, every particle used, C != 0: the reference's (P, m) equals k_p2g's (momentum, mass) accumulator;
    returns the larger relative error"""
    rng = np.random.RandomState(1)
    n, N = 16, 500
    P = make_particles(rng.uniform(0.2, 0.8, size=(N, 3)), M.ELASTIC, n)
    s = dlc._sim(device, n, P, param_grad=False)
    s.set_material_table(mu=[0.0], lam=[0.0])
    _set_vc(s, rng, N)
    s.sort_frame(0)
    s.phase('clear_grid', 0); s.phase('p2g', 0, 1)
    pm, m, _ = s.read_grid()
    st = s.get_state()
    x = st['x'].astype(np.float64)
    sel = dref.selection(x, st['used'], P['mat'], M.ELASTIC, n)
    want_p, want_m = mref.deposit(x, st['v'], st['C'], dlc.particle_mass(P, s.p_vol), sel, n)
    return max(rel_max(pm, want_p), rel_max(m, want_m))


def kernel_case(device, case):
    """one frame: the loss, the x, v and C adjoints and dL/drho of the kernels against the reference (the density loss's cases with random v and
    C, a NULL momentum target, w_momentum = 0); with w_momentum = 0 also against the density kernels"""
    rng = np.random.RandomState(KERNEL_CASES.index(case) + 11)
    n, N = 16, 400
    x = rng.uniform(0.3, 0.7, size=(N, 3))
    if case == 'frozen':
        x[:60] = rng.uniform(0.915, 0.99, size=(60, 3))   # int(x / dx - 0.5) > n - 3: the stencil leaves the grid
        x[60:90, 1] = rng.uniform(0.87, 0.9, size=30)      # next to the edge, still inside
    mat = np.where(np.arange(N) % 2 == 0, M.WATER, M.ELASTIC) if case == 'two_mat' else np.full(N, M.ELASTIC)
    used = (rng.rand(N) > 0.15).astype(np.int32) if case == 'unused' else np.ones(N, np.int32)
    P = make_particles(x, mat, n, used=used)
    s = dlc._sim(device, n, P)
    _set_vc(s, rng, N)
    if case != 'unsorted':
        s.sort_frame(0)
    if case == 'aged':   # positions move after the sort: the slots of a cell no longer sit together
        s._pa[0, 0, :, :3] += torch.from_numpy(rng.uniform(-0.6 / n, 0.6 / n, size=(N, 3)).astype(np.float32)).to(s._pa.device)
    st = s.get_state()
    xs, vs, Cs = (st[k].astype(np.float64) for k in ('x', 'v', 'C'))
    mp = dlc.particle_mass(P, s.p_vol)
    G = n ** 3
    row_mask = 0 if case == 'empty_mask' else s.material_row_mask(M.ELASTIC)
    sel = dref.selection(xs, st['used'], P['mat'], M.ELASTIC, n) & (row_mask != 0)
    t_m = None if case == 'null_target' else np.maximum(dref.deposit(xs + 0.04, mp, sel, n) + 2e-4 * rng.rand(G), 0.0).astype(np.float32)
    t_p = None
    if case not in ('null_target', 'null_momentum'):
        t_p = (mref.deposit(xs + 0.04, vs[::-1] + 0.3, 0.5 * Cs, mp, sel, n)[0] + 1e-4 * rng.randn(G, 3)).astype(np.float32)
    sdf = None if case == 'null_sdf' else dlc.sphere_sdf(n, (0.5, 0.45, 0.55), 0.15).astype(np.float32)
    wd, ws, wm = 100.0, 0.5, (0.0 if case == 'no_momentum_weight' else 60.0)
    L, gx, gv, gC, dm = mref.adjoint(xs, vs, Cs, mp, sel, n, t_m, t_p, sdf, wd, ws, wm)
    dev = s.device
    to = lambda a: None if a is None else torch.from_numpy(a).to(dev)
    tgt = to(pack_target(t_m, t_p, G))
    field = torch.zeros((G, 4), dtype=torch.float32, device=dev)
    out = torch.zeros(1, dtype=torch.float32, device=dev)
    s.momentum_loss(field, tgt, to(sdf), wd, ws, wm, row_mask, out, 0)
    s.reset_grad()
    s.add_grad_momentum(field, tgt, to(sdf), wd, ws, wm, row_mask, 0)
    g = {k: _np(v) for k, v in s.get_grad().items()}
    got_rho = s.get_param_grad()['rho']
    table = s.get_material_table()
    pv = float(np.float32(s.p_vol))
    want_rho = np.array([dm[np.asarray(P['mat']) == m].sum() * pv for m in table['mat']])
    scale_rho = np.array([np.abs(dm[np.asarray(P['mat']) == m]).sum() * pv for m in table['mat']])
    got_L = float(out.cpu()[0])
    assert abs(got_L - L) <= 1e-5 * abs(L), (case, got_L, L)
    if case == 'empty_mask':
        assert not any(g[k].any() for k in 'xvCF') and not got_rho.any(), case
        return
    for k in 'xvC':
        assert not g[k][~sel].any(), (case, k, 'an adjoint on a particle that deposits nothing')
    assert not g['F'].any(), (case, 'the loss does not depend on F')
    for k, want in (('x', gx), ('v', gv), ('C', gC)):
        if wm == 0.0 and k != 'x':
            assert not g[k].any(), (case, k)
            continue
        assert rel_max(g[k], want) < 1e-4, (case, k, rel_max(g[k], want))
    assert (np.abs(got_rho - want_rho) <= 1e-4 * np.maximum(np.abs(want_rho), scale_rho)).all(), (case, got_rho, want_rho)
    if wm == 0.0:   # the density loss's kernels on the same frame
        mass = torch.zeros(G, dtype=torch.float32, device=dev)
        out_d = torch.zeros(1, dtype=torch.float32, device=dev)
        s.density_loss(mass, to(t_m), to(sdf), wd, ws, row_mask, out_d, 0)
        s.reset_grad()
        s.add_x_grad_density(mass, to(t_m), to(sdf), wd, ws, row_mask, 0)
        gx_d = _np(s.get_grad()['x'])
        assert abs(float(out_d.cpu()[0]) - got_L) <= 1e-5 * abs(L), (float(out_d.cpu()[0]), got_L)
        assert rel_max(g['x'], gx_d) < 1e-4, rel_max(g['x'], gx_d)


def env_case(device, n_steps=3, T=40):
    """TaichiEnv with MomentumMatchingLoss over every step (temporal_range_type='all') on density_loss_case's rotating ELASTIC block; targets:
    the (P, m) deposits of an oracle run with another v0, every term weighted.  Returns the step losses, dL/d(x0, v0, C0, F0) and dL/drho of the
    product next to the reference's (the oracle's fp64 forward and backward seeded per step with the reference's x, v and C adjoints) and the
    direct mass term of dL/drho."""
    from fluidlab_b200 import TaichiEnv, MomentumMatchingLoss
    n = 32
    P, v0 = dlc.env_scene(n)
    N = len(P['x'])
    grav = (0.0, -10.0, 0.0)
    bnd = dict(type='cube', lower=(0.05, 0.05, 0.05), upper=(0.95, 0.95, 0.95))
    wd, ws, wm = 20.0, 0.5, 5.0
    pv = float(np.float32((0.5 / n) ** 2))
    mp = (np.float32(pv) * np.asarray(P['rho'], np.float32)).astype(np.float64)

    def sel_of(fr, P_):
        return dref.selection(fr['x'], P_['used'], P_['mat'], M.ELASTIC, n)
    op = dlc._oracle(n, P, grav, bnd, v0 + np.array([0.4, 0.2, -0.3]), n_steps, T)
    t_p, t_m = [], []
    for i in range(n_steps):
        fr = op.get_frame(10 * (i + 1))
        pm, m = mref.deposit(fr['x'], fr['v'], fr['C'], mp, sel_of(fr, P), n)
        t_p.append(pm.astype(np.float32)); t_m.append(m.astype(np.float32))
    sdf = dlc.sphere_sdf(n, (0.55, 0.35, 0.45), 0.1).astype(np.float32)

    kw = dict(ckpt_dest='cpu', device='cpu') if device == 'cpu' else dict(ckpt_dest='gpu')
    env = TaichiEnv(quality=n / 64, max_substeps_local=T, gravity=grav, horizon=n_steps, **kw)
    env.simulator.use_graphs, env.simulator.param_grad = False, True
    env.particle_bodies.get = lambda: P
    env.setup_boundary(**bnd)
    env.setup_loss(loss_cls=MomentumMatchingLoss, matching_mat=M.ELASTIC, temporal_range_type='all',
                   weights={'density': wd, 'sdf': ws, 'momentum': wm}, target=np.stack(t_m), target_sdf=sdf, target_momentum=np.stack(t_p))
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
    got_g = {k: _np(g[k]) for k in 'xvCF'}
    got_rho = float(env.simulator.get_param_grad()['rho'][0])

    def frame_adjoint(fr, i, mass_p, P_):
        return mref.adjoint(fr['x'], fr['v'], fr['C'], mass_p, sel_of(fr, P_), n, t_m[i], t_p[i], sdf, wd, ws, wm)

    def ref_losses(mass_p, P_):
        o = dlc._oracle(n, P_, grav, bnd, v0, n_steps, T)
        out, direct = [], 0.0
        for i in range(n_steps):
            L, _, _, _, dm = frame_adjoint(o.get_frame(10 * (i + 1)), i, mass_p, P_)
            out.append(L); direct += dm.sum()
        return o, out, direct
    o, want_losses, direct = ref_losses(mp, P)
    o.reset_grad()
    for i in range(n_steps - 1, -1, -1):
        f = o.cur_substep_local
        _, gx, gv, gC, _ = frame_adjoint(o.get_frame(f), i, mp, P)
        gf = o.get_grad_frame(f)
        o.set_grad_frame(f, gf['x'] + gx, gf['v'] + gv, gf['C'] + gC, gf['F'])
        o.step_grad(None)
    want_g = o.get_grad_frame(0)
    # dL/drho by central differences through the oracle's fp64 forward (the mass enters the dynamics and both deposits)
    rho = float(P['rho'][0]); h = 1e-5 * rho
    fd = []
    for r in (rho + h, rho - h):
        Pr = dict(P); Pr['rho'] = np.full(N, r); Pr['mass'] = np.full(N, (0.5 / n) ** 2 * r)
        fd.append(sum(ref_losses(Pr['mass'], Pr)[1]))
    fd_rho = (fd[0] - fd[1]) / (2 * h)
    return dict(got_losses=got_losses, want_losses=np.array(want_losses), got_g=got_g, want_g=want_g, got_rho=got_rho, fd_rho=fd_rho,
                direct_rho=direct * pv)


def fused_frame_case(device, n=16, N=600):
    """the loss on the step-end frame of a forward-only step (fused path: k_fwd, or k_g2p2g where k_fwd does not run) and of the same step on
    the stored-grid path of grad mode, each against the reference on its own state, and the two against each other"""
    from fluidlab_b200 import MPMSimulator
    rng = np.random.RandomState(4)
    x = rng.uniform(0.35, 0.65, size=(N, 3))
    P = make_particles(x, M.ELASTIC, n)
    v0 = (np.array([0.0, -1.0, 0.0]) + 4.0 * np.cross(np.array([0.2, 1.0, 0.3]), x - x.mean(0))).astype(np.float32)
    G = n ** 3
    t_p = (0.01 * rng.randn(G, 3)).astype(np.float32)
    t_m = (0.001 * rng.rand(G)).astype(np.float32)
    wd, ws, wm = 50.0, 0.0, 80.0
    res = {}
    for grad in (False, True):
        s = MPMSimulator(dim=3, quality=n / 64, gravity=(0.0, -10.0, 0.0), horizon=50, max_substeps_local=20, max_substeps_global=100000,
                         ckpt_dest='gpu' if device is None else 'cpu', device=device)
        s.use_graphs, s.fuse_g2p2g = False, True
        s.setup_boundary(type='cube', lower=(0.1, 0.1, 0.1), upper=(0.9, 0.9, 0.9))
        s.build(None, None, [], P)
        if grad:
            s.enable_grad()
            assert s._can_fuse() and s._storing()
        else:
            assert s._can_fuse() and not s.grad_enabled
        st = s.get_state(); st['v'] = v0; s.set_state(0, st)
        s.step(None)
        f = s.cur_substep_local
        dev = s.device
        field = torch.zeros((G, 4), dtype=torch.float32, device=dev)
        out = torch.zeros(1, dtype=torch.float32, device=dev)
        s.momentum_loss(field, torch.from_numpy(pack_target(t_m, t_p, G)).to(dev), None, wd, ws, wm, s.material_row_mask(M.ELASTIC), out, f)
        fr = s.readframe(f)
        sel = dref.selection(fr['x'], fr['used'], P['mat'], M.ELASTIC, n)
        want = mref.adjoint(fr['x'], fr['v'], fr['C'], dlc.particle_mass(P, s.p_vol), sel, n, t_m, t_p, None, wd, ws, wm)[0]
        res[grad] = (float(out.cpu()[0]), want, float(np.abs(fr['C']).max()))
    return res


def sysid_viscosity_case(device, n_grid=32, N=8000, iters=20, lr=0.06, gamma=0.8, n_steps=2, seed=0, w_momentum=True):
    """Viscosity identification without particle correspondence: a MILK_VIS block in shear (v_x grows with y, v_z with x) falls into a box,
    mu starts 30 % high, and 20 Adam iterations on log mu fit it against the (P*, m*) volumes of the true run's particles after a random
    permutation (momentum_from_points with the recording's v and C), MomentumMatchingLoss on the last step.  w_momentum=False: the same fit
    with the density term alone.  Returns |mu / mu* - 1| before every iteration and after the last."""
    from fluidlab_b200 import MPMSimulator, MomentumMatchingLoss
    rng = np.random.RandomState(seed)
    x = rng.uniform((0.35, 0.32, 0.35), (0.65, 0.5, 0.65), size=(N, 3))
    P = make_particles(x, M.MILK_VIS, n_grid)
    s = MPMSimulator(dim=3, quality=n_grid / 64, gravity=(0.0, -10.0, 0.0), horizon=50, max_substeps_local=10 * n_steps + 10, max_substeps_global=100000,
                     ckpt_dest='gpu' if device is None else 'cpu', device=device)
    s.use_graphs = device is None
    s.setup_boundary(type='cube', lower=(0.3, 0.3, 0.3), upper=(0.7, 0.7, 0.7))
    s.param_grad = True
    s.build(None, None, [], P)
    st0 = s.get_state()
    c = x.mean(0)
    st0['v'] = np.stack([8.0 * (x[:, 1] - c[1]), np.full(N, -1.5), -6.0 * (x[:, 0] - c[0])], 1).astype(np.float32)
    true = s.get_material_table()
    mu_t = float(true['mu'][0])
    m_p = float(np.float32(s.p_vol) * np.float32(true['rho'][0]))

    def rollout():
        s.cur_substep_global = 0
        s.set_state(0, st0)
        for _ in range(n_steps):
            s.step(None)
    s.enable_grad()
    rollout()
    rec = s.get_state()
    perm = rng.permutation(N)
    p_star, m_star = MomentumMatchingLoss.momentum_from_points(rec['x'][perm], rec['v'][perm], m_p, n_grid, affine=rec['C'][perm])
    w = {'density': 1.0 / m_p ** 2}
    if w_momentum:
        w['momentum'] = 1.0 / m_p ** 2
    loss = MomentumMatchingLoss(M.MILK_VIS, target=m_star, target_momentum=p_star, max_loss_steps=1, weights=w, temporal_range_type='all')
    loss.build(s)
    logmu = torch.tensor([np.log(mu_t * 1.3)], dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([logmu], lr=lr)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma)
    errs = []
    for _ in range(iters):
        mu = float(torch.exp(logmu.detach())[0])
        errs.append(abs(mu / mu_t - 1))
        s.set_material_table(mu=[mu])
        rollout()
        s.reset_grad()
        loss.get_final_loss_grad()   # the seed of the recorded (last) frame
        loss.compute_step_loss_grad(0, s.cur_substep_local)
        for _ in range(n_steps):
            s.step_grad(None)
        g = s.get_param_grad()
        opt.zero_grad()
        logmu.grad = torch.tensor([g['mu'][0] * mu], dtype=torch.float64)
        opt.step()
        sched.step()
    errs.append(abs(float(torch.exp(logmu.detach())[0]) / mu_t - 1))
    return errs
