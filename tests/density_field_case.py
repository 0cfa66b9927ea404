"""Scenes for the per-particle density tests (MPMSimulator.set_density_field): the same bodies run on an H100 (tests/test_density_field_gpu.py)
and on the CPU execution-model shim (tests/test_density_field.py), each against the fp64 oracle, which takes a mass per particle.  The oracle's
unreduced per-particle dL/dmass (tests/param_grad_ref.py, ParamGradOracle.pg['mass']) times p_vol is the reference for
get_param_grad()['rho_field']; its row sums (param_grad_case.oracle_rows) for the row keys.  The loss references (density_loss_ref,
momentum_loss_ref) take a mass per particle too."""
import numpy as np

from conftest import make_particles
from fluidlab_b200 import macros as M
from param_grad_ref import ParamGradOracle
import density_loss_ref as dref
import material_field_case as mfc
import momentum_loss_ref as mref
import param_grad_case as pgc

rel = pgc.rel
CUBE, GRAV = mfc.CUBE, mfc.GRAV
CASE_MATS = dict(mfc.CASE_MATS, water=[M.WATER])


def random_rho(P, rng, spread=4.0, n=16):
    """per-particle rho log-uniform over x lo .. spread of each particle's row value, fp32-representable.  lo = 1 / spread, but at least
    (n / 64)^2: the time step is fixed (2e-4), and a particle's wave speed grows as 1 / sqrt(rho), so dt c / dx grows as n / sqrt(rho).  The
    bound keeps it at or below that of the row value on the reference's 64^3 grid; beyond it the fp64 oracle's own run diverges (ICECREAM
    with rho / 4 on 64^3 leaves the grid)."""
    lo = max(1.0 / spread, (n / 64.0) ** 2)
    r = np.asarray(P['rho'], np.float64) * np.exp(rng.uniform(np.log(lo), np.log(spread), len(P['rho'])))
    return r.astype(np.float32).astype(np.float64)


def particle_mass(rho, p_vol):
    """the f32 mass the simulator gives a particle of density rho: f32(p_vol) * f32(rho) (MPM:174)"""
    return (np.float32(p_vol) * np.asarray(rho, np.float32)).astype(np.float64)


def _scene(case, N=300, n=16, seed=11):
    """material_field_case._scene with the WATER case; N is the particle count at n = 16 and grows with n (N n / 16)"""
    N = N * n // 16
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


def _row_mass_grad(s):
    import torch
    return None if s._gmat is None else s._gmat[:, 2].to(torch.float64).cpu().numpy()


def equals_table_case(device, case, sort, with_field, n=16):
    """a density field equal to every particle's row rho reproduces the run without it (states, state adjoint, row keys), with the private
    (mu, lam) field (with_field False) and with a random user field (True)"""
    rng, P, st, seed_g = _scene(case, n=n)
    fld = mfc.random_field(P, rng) if with_field else None
    res = {}
    for use_rho in (False, True):
        s = mfc._sim(device, P, n, sort)
        if fld is not None:
            s.set_material_field(*fld)
        if use_rho:
            s.set_density_field(P['rho'])
        res[use_rho] = mfc._run_one_substep_grad(s, st, seed_g)
    (fa, ga, pa), (fb, gb, pb) = res[False], res[True]
    for k in ('x', 'v', 'C', 'F'):   # unordered scatter reductions differ from run to run: v and C by up to 1.3e-5 with a random (mu, lam) field
        assert rel(fb[k], fa[k]) < (1e-5 if k in 'xF' else 1e-4), ('state', k, rel(fb[k], fa[k]))
        assert rel(gb[k], ga[k]) < 1e-3, ('state adjoint', k, rel(gb[k], ga[k]))
    for k in ('mu', 'lam', 'rho', 'gravity'):
        assert rel(pb[k], pa[k]) < 1e-3, ('row key', k, pb[k], pa[k])
    np.testing.assert_allclose(pb['rho_field'].sum(), pb['rho'].sum(), rtol=1e-9)
    assert 'rho_field' not in pa
    assert ('mu_field' in pb) == with_field, 'the private field stays invisible'


def heterogeneous_case(device, case, sort, with_field=False, fuse=False, n=16):
    """random per-particle rho (and with_field: a random (mu, lam) field) against the fp64 oracle: the frame after one step, one backward
    substep's state adjoint and per-particle dL/drho (p_vol * ParamGradOracle.pg['mass']), the row sums against oracle_rows, and the rows'
    dL/dmass accumulator exactly 0 while the field is bound.  fuse (with sort): the stored-grid fused path (k_g2p2g_field_mass).  Returns the
    errors."""
    rng, P, st, seed_g = _scene(case, n=n)
    rho = random_rho(P, rng, n=n)
    fld = mfc.random_field(P, rng) if with_field else None
    s = mfc._sim(device, P, n, sort, fuse=fuse)
    if fld is not None:
        s.set_material_field(*fld)
    s.set_density_field(rho)
    fr, g, pg = mfc._run_one_substep_grad(s, st, seed_g)
    assert not _row_mass_grad(s).any(), 'the rows\' dL/dmass is not written while a density field is bound'
    Pf = dict(P, mass=particle_mass(rho, s.p_vol))
    if fld is not None:
        Pf.update(mu=fld[0], lam=fld[1])
    o = ParamGradOracle(n, Pf, gravity=GRAV, boundary=CUBE, precision=64, max_substeps_local=20)
    o.set_frame(0, st['x'], st['v'], st['C'], st['F'], st['used'])
    for f in range(10):
        o.substep(f)
    want_fr = o.get_frame(10)
    o.reset_grad(); o.set_grad_frame(10, seed_g['x'], seed_g['v'], seed_g['C'], seed_g['F'])
    o.substep_grad(9)
    og, opg = o.get_grad_frame(9), o.get_param_grad()
    pv = float(np.float32(s.p_vol))
    errs = {('frame', k): rel(fr[k], want_fr[k]) for k in ('x', 'v', 'C', 'F')}
    errs.update({('adjoint', k): rel(g[k], og[k]) for k in ('x', 'v', 'C', 'F')})
    errs[('field', 'rho')] = rel(pg['rho_field'], opg['mass'] * pv)
    if fld is not None:
        errs[('field', 'mu')] = rel(pg['mu_field'], opg['mu'])
        errs[('field', 'lam')] = rel(pg['lam_field'], opg['lam'])
    rest = 1e-3 if case == 'icecream' else 1e-4   # the bars of the (mu, lam) field (tests/material_field_case.py::heterogeneous_case)
    # per-particle dL/drho: the masses span x16 and the comparison is relative to the largest term; the mixed scene measured up to 1.04e-4 on
    # the shim and 1.85e-4 on an H100 (every other scene below 1e-4), so 5e-4 (a slot-order or row mistake gives errors of order 1)
    bars = {('frame', 'x'): 1e-5, ('frame', 'F'): 1e-5, ('frame', 'v'): rest, ('frame', 'C'): rest, ('field', 'rho'): max(rest, 5e-4)}
    bad = {k: e for k, e in errs.items() if not e < bars.get(k, rest)}
    assert not bad, (case, sort, with_field, bad, errs)
    assert np.abs(opg['mass']).max() > 0
    want = pgc.oracle_rows(opg, P, s.get_material_table(), s.p_vol)
    errs['rows'] = pgc.assert_param_grads_close(pg, want, rest, (case, sort, with_field))
    return errs


def ring_case(device, sort_every, n_steps=3, T=20, N=400, n=16):
    """a T = 20 ring over 3 steps, a heterogeneous rho, index-matched loss on the last frame: per-particle dL/drho against the oracle.  Sort
    epochs change the slot order between steps, so a mass field or gradient gathered in the wrong order fails here."""
    rng = np.random.RandomState(31)
    N = N * n // 16
    x = rng.uniform(0.38, 0.62, size=(N, 3))
    mat = np.array([(M.ELASTIC, M.ICECREAM)[i % 2] for i in range(N)], dtype=np.int32)
    P = make_particles(x, mat, n)
    rho = random_rho(P, rng, n=n)
    v0 = (rng.randn(N, 3) * 0.4).astype(np.float32)
    gx = rng.randn(N, 3).astype(np.float32)
    s = mfc._sim(device, P, n, False, T=T)
    s.sort_every, s.store_grids = sort_every, False
    s.set_density_field(rho)
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
    o = ParamGradOracle(n, dict(P, mass=particle_mass(rho, s.p_vol)), gravity=GRAV, boundary=CUBE, precision=64, max_substeps_local=T)
    o.enable_grad()
    o.set_frame(0, x, v0, np.zeros((N, 3, 3)), np.tile(np.eye(3), (N, 1, 1)), P['used'])
    for _ in range(n_steps):
        o.step(None)
    o.reset_grad(); o.set_grad_frame(o.cur_substep_local, gx, z3, z9, z9)
    for _ in range(n_steps):
        o.step_grad(None)
    want = o.get_param_grad()
    # the (mu, lam) field's ring bar: fp32 drifts from fp64 by up to ~6e-3 per particle over 30 substeps; a wrong slot order gives order 1
    errs = dict(rho=rel(got['rho_field'], want['mass'] * float(np.float32(s.p_vol))))
    assert max(errs.values()) < 2e-2, (sort_every, errs)
    errs['rows'] = pgc.assert_param_grads_close(got, pgc.oracle_rows(want, P, s.get_material_table(), s.p_vol), 1e-2, ('ring', sort_every))
    return errs


def _oracle_loss(P, st, seed_g, mass, n, n_sub=10):
    o = ParamGradOracle(n, dict(P, mass=mass), gravity=GRAV, boundary=CUBE, precision=64, max_substeps_local=20)
    o.set_frame(0, st['x'], st['v'], st['C'], st['F'], st['used'])
    for f in range(n_sub):
        o.substep(f)
    fr = o.get_frame(n_sub)
    return sum(float((seed_g[k].astype(np.float64) * fr[k]).sum()) for k in ('x', 'v', 'C', 'F'))


def central_difference_case(device, n_particles=3, n=16):
    """the simulator's per-particle dL/drho_p over a whole step against central differences of the oracle's fp64 forward, for a few particles
    and along a random direction of the whole field"""
    rng, P, st, seed_g = _scene('mixed', N=200, n=n)
    rho = random_rho(P, rng, n=n)
    s = mfc._sim(device, P, n, True)
    s.set_density_field(rho)
    g = s.get_state(); g['v'][:] = st['v']; g['F'][:] = st['F']; g['C'][:] = st['C']; s.set_state(0, g)
    s.enable_grad()
    s.step(None)
    s.reset_grad(); s.set_grad(seed_g['x'], seed_g['v'], seed_g['C'], seed_g['F'])
    s.step_grad(None)
    got = s.get_param_grad()['rho_field']
    pv = float(np.float32(s.p_vol))
    used = np.where(st['used'] != 0)[0]
    picks = used[np.argsort(-np.abs(got[used]))[:n_particles]]
    out = []
    for p in picks:
        h = 1e-4 * rho[p]
        rp, rm = rho.copy(), rho.copy(); rp[p] += h; rm[p] -= h
        fd = (_oracle_loss(P, st, seed_g, pv * rp, n) - _oracle_loss(P, st, seed_g, pv * rm, n)) / (2 * h)
        out.append((int(p), fd, float(got[p])))
        assert abs(fd - got[p]) <= 2e-3 * max(abs(fd), 1e-3 * np.abs(got).max()), out[-1]
    d = rng.randn(len(rho)) * rho * 1e-4
    fd = (_oracle_loss(P, st, seed_g, pv * (rho + d), n) - _oracle_loss(P, st, seed_g, pv * (rho - d), n)) / 2
    an = float((got * d).sum())
    assert abs(fd - an) <= 2e-3 * abs(fd), ('directional', fd, an)
    return out, (fd, an)


def fused_forward_case(device, case='mixed', n=16):
    """forward-only steps on the fused path with a random rho (k_p2g_field_mass, then k_fwd<3, false, false> for the inner substeps): the frame
    after two steps against the fp64 oracle and the per-substep path"""
    rng, P, st, _ = _scene(case, n=n)
    rho = random_rho(P, rng, n=n)
    fr = {}
    for fuse in (True, False):
        s = mfc._sim(device, P, n, True, pg=False, fuse=fuse)
        s.set_density_field(rho)
        g = s.get_state(); g['v'][:] = st['v']; g['F'][:] = st['F']; g['C'][:] = st['C']; s.set_state(0, g)
        s.step(None); s.step(None)
        fr[fuse] = s.readframe(20)
    if device == 'cpu':
        assert s._lib.fmpm_fwd_path(s._h) & 1, 'the fused forward path runs k_fwd'
    o = ParamGradOracle(n, dict(P, mass=particle_mass(rho, s.p_vol)), gravity=GRAV, boundary=CUBE, precision=64, max_substeps_local=20)
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


def rigid_case(device, n_grid=16):
    """water, an elastic blob and a MAT_RIGID cube, a random rho on every particle: one step on the fused stored-grid path, where the rigid body's
    particles scatter through k_p2g_rigid_field_mass after the shape matching, against the fp64 oracle (which also matches the body's shape by
    particle count, not mass)"""
    rng = np.random.RandomState(17)
    k = n_grid // 16   # particle counts grow with the grid
    xw = rng.uniform((0.32, 0.32, 0.32), (0.68, 0.42, 0.68), size=(500 * k, 3))
    xa = rng.uniform((0.38, 0.45, 0.38), (0.50, 0.55, 0.50), size=(200 * k, 3))
    xe = rng.uniform((0.54, 0.45, 0.52), (0.62, 0.55, 0.60), size=(150 * k, 3))
    x = np.concatenate([xw, xa, xe])
    mat = np.concatenate([np.full(len(xw), M.WATER), np.full(len(xa), M.RIGID), np.full(len(xe), M.ELASTIC)])
    bid = np.concatenate([np.zeros(len(xw)), np.ones(len(xa)), np.full(len(xe), 2)]).astype(np.int32)
    P = make_particles(x, mat, n_grid)
    P['body_id'] = bid; P['bodies'] = {'n': 3}
    N = len(x)
    rho = random_rho(P, rng, n=n_grid)
    v0 = (rng.randn(N, 3) * 0.3).astype(np.float32)
    s = mfc._sim(device, P, n_grid, True, pg=False, fuse=True)
    s.set_density_field(rho)
    st = s.get_state(); st['v'][:] = v0; s.set_state(0, st)
    s.enable_grad()
    s.step(None)
    assert s._can_fuse()
    got = s.get_state()
    o = ParamGradOracle(n_grid, dict(P, mass=particle_mass(rho, s.p_vol)), gravity=GRAV, boundary=CUBE, precision=64, max_substeps_local=20)
    o.set_bodies(bid, 3)
    o.set_frame(0, x, v0, np.zeros((N, 3, 3)), np.tile(np.eye(3), (N, 1, 1)), P['used'])
    for f in range(10):
        o.substep(f)
    want = o.get_frame(10)
    errs = {k: rel(got[k], want[k]) for k in ('x', 'v', 'F')}
    assert errs['x'] < 1e-5 and errs['F'] < 1e-5 and errs['v'] < 1e-4, errs
    return errs


def injector_case(device, fuse, sort_every=1, n_steps=3, T=20, n_grid=16):
    """material_field_case.injector_case with a random rho instead of the (mu, lam) field: the injected MILK particles scatter through
    k_p2g_injected_field_mass (fused) or the per-substep kernels; per-particle dL/drho and its row sums against the oracle"""
    from fluidlab_b200 import TaichiEnv, LatteArtLoss
    n_coffee, n_milk, flux = 400 * n_grid // 16, 120, 2
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
    rho = random_rho(P, rng, n=n_grid)
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
    sim.set_density_field(rho)
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
    o = ParamGradOracle(n_grid, dict(P, mass=particle_mass(rho, sim.p_vol)), gravity=(0, -20, 0), boundary=bnd, precision=64, max_substeps_local=T)
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
    pv = float(np.float32(sim.p_vol))
    milk = np.arange(n_milk)
    assert np.abs(want['mass'][milk]).max() > 0, 'the injected particles carry a gradient'
    errs = dict(rho=rel(got['rho_field'], want['mass'] * pv), rho_milk=rel(got['rho_field'][milk], want['mass'][milk] * pv))
    assert max(errs.values()) < 2e-4, (fuse, errs)
    # the row keys rho and gravity: mu and lam of these mu = 0 liquids come from the private (mu, lam) field, whose dL/dmu at mu = 0 rests on
    # the fp32 polar rotation of a near-isotropic F (as for the table's rows) and is no part of the density field
    rows = pgc.oracle_rows(want, P, sim.get_material_table(), sim.p_vol)
    errs['rows'] = {k: float((np.abs(np.asarray(got[k]) - rows[k]) / np.maximum(np.abs(rows[k]), np.maximum(rows['scale'][k], 1e-30))).max())
                    for k in ('rho', 'gravity')}
    assert max(errs['rows'].values()) < 1e-3, ('injector', fuse, errs['rows'])
    return errs


def loss_kernel_case(device, n=16, N=400, seed=3):
    """the density and momentum losses' deposits and adjoints with a random rho on one frame, against density_loss_ref / momentum_loss_ref with a
    per-particle mass: the loss, dL/d(x, v, C) and the direct per-particle dL/drho (p_vol times the references' dL/dm)"""
    import torch
    rng = np.random.RandomState(seed)
    x = rng.uniform(0.3, 0.7, size=(N, 3))
    mat = np.array([(M.ELASTIC, M.WATER)[i % 2] for i in range(N)], dtype=np.int32)
    used = (rng.rand(N) > 0.1).astype(np.int32)
    P = make_particles(x, mat, n, used=used)
    rho = random_rho(P, rng, n=n)
    s = mfc._sim(device, P, n, False)
    s.set_density_field(rho)
    v = (rng.randn(N, 3) * 0.5).astype(np.float32)
    Cm = (rng.randn(N, 3, 3) * 4.0).astype(np.float32)
    st = s.get_state(); st['v'][:] = v; st['C'][:] = Cm; s.set_state(0, st)
    x32 = s.readframe(0)['x'].astype(np.float64)
    mp = particle_mass(rho, s.p_vol)
    pv = float(np.float32(s.p_vol))
    mask = s.material_row_mask(M.ELASTIC)
    sel = dref.selection(x32, used, mat, M.ELASTIC, n)
    G = n ** 3
    dev = s.device
    tm = (rng.rand(G) * 2e-4).astype(np.float32)
    tp = (rng.randn(G, 3) * 1e-4).astype(np.float32)
    sdf = rng.randn(G).astype(np.float32)
    wd, ws, wm = 30.0, 0.5, 20.0
    errs = {}
    # density
    want_m = dref.deposit(x32, mp, sel, n)
    L, gx, dm = dref.adjoint(x32, mp, sel, n, tm, sdf, wd, ws)
    mass_dev, out = torch.zeros(G, dtype=torch.float32, device=dev), torch.zeros(1, dtype=torch.float32, device=dev)
    tmd, sdfd = torch.from_numpy(tm).to(dev), torch.from_numpy(sdf).to(dev)
    s.density_loss(mass_dev, tmd, sdfd, wd, ws, mask, out, f=0)
    errs['density_loss'] = abs(float(out[0]) - L) / abs(L)
    s.density_loss(mass_dev, None, None, 1.0, 0.0, mask, out, f=0)
    errs['density_deposit'] = rel(mass_dev.cpu().numpy(), want_m)
    s.reset_grad()
    s.add_x_grad_density(mass_dev, tmd, sdfd, wd, ws, mask, f=0)
    got_g, got_pg = s.get_grad(), s.get_param_grad()
    errs['density_gx'] = rel(_np(got_g['x']), gx)
    errs['density_rho'] = rel(got_pg['rho_field'], dm * pv)
    assert not _row_mass_grad(s).any()
    # momentum
    tgt4 = torch.from_numpy(np.concatenate([tp, tm[:, None]], 1)).to(dev)
    want_pm, want_m2 = mref.deposit(x32, v.astype(np.float64), Cm.astype(np.float64), mp, sel, n)
    L2, gx2, gv2, gC2, dm2 = mref.adjoint(x32, v.astype(np.float64), Cm.astype(np.float64), mp, sel, n, tm, tp, sdf, wd, ws, wm)
    fld = torch.zeros((G, 4), dtype=torch.float32, device=dev)
    out.zero_()
    s.momentum_loss(fld, tgt4, sdfd, wd, ws, wm, mask, out, f=0)
    errs['momentum_loss'] = abs(float(out[0]) - L2) / abs(L2)
    s.momentum_loss(fld, None, None, 1.0, 0.0, 0.0, mask, out, f=0)
    f = fld.cpu().numpy().astype(np.float64)
    errs['momentum_deposit_P'] = rel(f[:, :3], np.asarray(want_pm).reshape(-1, 3))
    errs['momentum_deposit_m'] = rel(f[:, 3], np.asarray(want_m2).reshape(-1))
    s.reset_grad()
    s.add_grad_momentum(fld, tgt4, sdfd, wd, ws, wm, mask, f=0)
    got_g, got_pg = s.get_grad(), s.get_param_grad()
    errs['momentum_gx'] = rel(_np(got_g['x']), gx2)
    errs['momentum_gv'] = rel(_np(got_g['v']), gv2)
    errs['momentum_gC'] = rel(_np(got_g['C']), gC2)
    errs['momentum_rho'] = rel(got_pg['rho_field'], dm2 * pv)
    assert not _row_mass_grad(s).any()
    bad = {k: e for k, e in errs.items() if not e < 1e-4}
    assert not bad, (bad, errs)
    return errs


def _np(a):
    import torch
    return a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)


def env_case(device, n=16, N=600, n_steps=3, T=40, seed=5):
    """TaichiEnv with DensityMatchingLoss over every step and a random rho: the step losses against the oracle's fp64 forward with the
    reference loss, and dL/drho_p (the direct mass terms of the loss included) against central differences of that fp64 pipeline, for a few
    particles and along a random direction"""
    from fluidlab_b200 import TaichiEnv, DensityMatchingLoss
    rng = np.random.RandomState(seed)
    x = rng.uniform((0.38, 0.3, 0.38), (0.62, 0.45, 0.62), size=(N, 3))
    P = make_particles(x, M.ELASTIC, n)
    c = x.mean(0)
    v0 = (np.array([0.0, -1.0, 0.0]) + 4.0 * np.cross(np.array([0.2, 1.0, 0.3]), x - c)).astype(np.float32).astype(np.float64)
    rho = random_rho(P, rng, n=n)
    grav = (0.0, -10.0, 0.0)
    bnd = dict(type='cube', lower=(0.05, 0.05, 0.05), upper=(0.95, 0.95, 0.95))
    wd, ws = 20.0, 0.5
    pv = float(np.float32((0.5 / n) ** 2))

    def oracle_run(mass, v):
        o = ParamGradOracle(n, dict(P, mass=mass), gravity=grav, boundary=bnd, precision=64, max_substeps_local=T)
        o.set_frame(0, P['x'], v, np.zeros((N, 3, 3)), np.tile(np.eye(3), (N, 1, 1)), P['used'])
        for f in range(10 * n_steps):
            o.substep(f)
        return [o.get_frame(10 * (i + 1))['x'] for i in range(n_steps)]
    mp = particle_mass(rho, (0.5 / n) ** 2)
    tgt = []
    for xp in oracle_run(mp, v0 + np.array([0.4, 0.2, -0.3])):
        tgt.append(dref.deposit(xp, mp, dref.selection(xp, P['used'], P['mat'], M.ELASTIC, n), n).astype(np.float32))
    sdf = rng.randn(n ** 3).astype(np.float32) * 0.05

    def ref_loss(mass):
        out = 0.0
        for i, xf in enumerate(oracle_run(mass, v0)):
            out += dref.adjoint(xf, mass, dref.selection(xf, P['used'], P['mat'], M.ELASTIC, n), n, tgt[i], sdf, wd, ws)[0]
        return out

    kw = dict(ckpt_dest='cpu', device='cpu') if device == 'cpu' else dict(ckpt_dest='gpu')
    env = TaichiEnv(quality=n / 64, max_substeps_local=T, gravity=grav, horizon=n_steps, **kw)
    env.simulator.use_graphs, env.simulator.param_grad = False, True
    env.particle_bodies.get = lambda: P
    env.setup_boundary(**bnd)
    env.setup_loss(loss_cls=DensityMatchingLoss, matching_mat=M.ELASTIC, temporal_range_type='all', weights={'density': wd, 'sdf': ws},
                   target=np.stack(tgt), target_sdf=sdf)
    env.build()
    env.simulator.set_density_field(rho)
    st = env.get_state()['state']; st['v'] = v0.astype(np.float32)
    env.set_state(st, grad_enabled=True)
    for _ in range(n_steps):
        env.step()
    got_loss = float(env.loss.step_loss.cpu().numpy().astype(np.float64).sum())
    env.get_final_loss()
    env.reset_grad(); env.get_final_loss_grad()
    for _ in range(n_steps):
        env.step_grad()
    got = env.simulator.get_param_grad()['rho_field']
    want_loss = ref_loss(mp)
    assert abs(got_loss - want_loss) <= 1e-4 * abs(want_loss), (got_loss, want_loss)
    out = []
    for p in np.argsort(-np.abs(got))[:3]:
        h = 1e-4 * rho[p]
        rp, rm = rho.copy(), rho.copy(); rp[p] += h; rm[p] -= h
        fd = (ref_loss(pv * rp) - ref_loss(pv * rm)) / (2 * h)
        out.append((int(p), fd, float(got[p])))
        assert abs(fd - got[p]) <= 5e-3 * max(abs(fd), 1e-3 * np.abs(got).max()), out[-1]
    d = rng.randn(N) * rho * 1e-4
    fd = (ref_loss(pv * (rho + d)) - ref_loss(pv * (rho - d))) / 2
    an = float((got * d).sum())
    assert abs(fd - an) <= 5e-3 * abs(fd), ('directional', fd, an)
    return out, (fd, an)


def identification_case(device, n_grid=16, N=1200, iters=20, lr=0.03, n_steps=2, seed=0):
    """a dense core (rho x 3 within 0.08 of the centre) inside an ELASTIC block, recovered from the block's per-step grid mass (a
    DensityMatchingLoss-style recording: the true run's density deposit after every step).  The unknowns are per particle: log rho_p, started
    uniform at the block's mean true density, fitted by torch.optim.Adam with dL/dlog rho_p = rho_p dL/drho_p from
    get_param_grad()['rho_field'], preconditioned by material_field_case.knn_smoother.  Returns per iteration the field error
    sqrt(mean(log(rho_p / rho*_p)^2)) and the mean rho of the core and of the shell, before every iteration and after the last."""
    import torch
    rng = np.random.RandomState(seed)
    x = rng.uniform((0.35, 0.32, 0.35), (0.65, 0.5, 0.65), size=(N, 3))
    P = make_particles(x, M.ELASTIC, n_grid)
    c = x.mean(0)
    core = np.abs(x - c).max(1) < 0.08
    r_t = np.where(core, 3.0, 1.0) * float(P['rho'][0])
    s = mfc._sim(device, P, n_grid, True, T=10 * n_steps + 10)
    st0 = s.get_state()
    st0['v'] = (np.array([0.0, -1.5, 0.0]) + 6.0 * np.cross(np.array([0.3, 1.0, 0.2]), x - c)).astype(np.float32)
    smooth = mfc.knn_smoother(x)
    G = n_grid ** 3
    dev = s.device
    mask = s.material_row_mask(M.ELASTIC)
    mass_dev = torch.zeros(G, dtype=torch.float32, device=dev)
    out = torch.zeros(1, dtype=torch.float32, device=dev)

    def rollout(rv, record=None):
        s.set_density_field(rv)
        s.cur_substep_global = 0
        s.set_state(0, st0)
        for i in range(n_steps):
            s.step(None)
            if record is not None:
                s.density_loss(mass_dev, None, None, 1.0, 0.0, mask, out)
                record.append(mass_dev.clone())
    s.enable_grad()
    tgt = []
    rollout(r_t, tgt)
    logr = torch.full((N,), float(np.log(r_t.mean())), dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([logr], lr=lr, eps=1e-30)
    hist = []
    for it in range(iters + 1):
        rv = torch.exp(logr.detach()).numpy()
        hist.append((float(np.sqrt((np.log(rv / r_t) ** 2).mean())), float(rv[core].mean()), float(rv[~core].mean())))
        if it == iters:
            break
        rollout(rv)
        s.reset_grad()
        for i in range(n_steps - 1, -1, -1):
            s.add_x_grad_density(mass_dev, tgt[i], None, 1.0, 0.0, mask)
            s.step_grad(None)
        g = s.get_param_grad()['rho_field']
        opt.zero_grad()
        logr.grad = torch.tensor(smooth(g * rv))
        opt.step()
    return hist
