"""Scenes for the plastic yield limit tests (MPMSimulator.set_plastic_limits / set_plastic_field): the same bodies run on an H100
(tests/test_plastic_limits_gpu.py) and on the CPU execution-model shim (tests/test_plastic_limits.py), each against the fp64 oracle with the
same per-particle limits.  The oracle's per-particle dL/dlo, dL/dhi (tests/plastic_grad_ref.py) are the reference for get_param_grad()'s
`theta_c_field` = -dL/dlo and `theta_s_field` = dL/dhi, and their row sums for the row keys `theta_c` / `theta_s`."""
import numpy as np

from conftest import make_particles
from fluidlab_b200 import macros as M
from plastic_grad_ref import NEAR, PLASTIC, PlasticGradOracle, THETA_C, THETA_S, limits
import material_field_case as mfc
import param_grad_case as pgc

rel = pgc.rel
CUBE, GRAV = mfc.CUBE, mfc.GRAV
CYLINDER = dict(type='cylinder', xz_radius=0.2, xz_center=(0.5, 0.5), y_range=(0.3, 0.7))
CASE_MATS = {'icecream': [M.ICECREAM], 'plastic_demo': [M.PLASTIC_DEMO], 'mixed': [M.ICECREAM, M.ELASTIC, M.WATER, M.PLASTIC_DEMO]}
KEYS = ('x', 'v', 'C', 'F')


def random_theta(n, rng):
    """theta_c, theta_s log-uniform over x 1/4 .. 4 of the defaults, fp32-representable"""
    tc = THETA_C * np.exp(rng.uniform(np.log(0.25), np.log(4.0), n))
    ts = THETA_S * np.exp(rng.uniform(np.log(0.25), np.log(4.0), n))
    return tc.astype(np.float32).astype(np.float64), ts.astype(np.float32).astype(np.float64)


def _scene(case, N=300, n=16, seed=11):
    """density_field_case._scene with the plastic cases (N grows with n)"""
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


def _sim(device, P, n, sort, T=20, pg=True, fuse=False, boundary=CUBE):
    from fluidlab_b200 import MPMSimulator
    s = MPMSimulator(dim=3, quality=n / 64, gravity=GRAV, horizon=50, max_substeps_local=T, max_substeps_global=1000,
                     ckpt_dest='gpu' if device is None else 'cpu', device=device, sort_every=1 if sort else 0)
    s.use_graphs, s.store_grids, s.fuse_g2p2g, s.param_grad = device is None, sort, fuse, pg
    s.setup_boundary(**boundary)
    s.build(None, None, [], P)
    return s


def _oracle(P, n, lo=None, hi=None, boundary=CUBE, T=20, **fields):
    return PlasticGradOracle(n, dict(P, **fields), lo=lo, hi=hi, gravity=GRAV, boundary=boundary, precision=64, max_substeps_local=T)


def _rows(P, table):
    """the simulator's row of every particle (material rows are matched on (material, f32 rho))"""
    r = np.zeros(len(P['mat']), np.int64)
    for i, (m, rh) in enumerate(zip(table['mat'], table['rho'])):
        r[(np.asarray(P['mat']) == m) & (np.asarray(P['rho']).astype(np.float32).astype(np.float64) == rh)] = i
    return r


def _theta_rows(og, row, nrows):
    """the oracle's per-particle dL/dlo, dL/dhi as get_param_grad()'s row keys theta_c / theta_s, with the sums of the magnitudes as scale"""
    out = {}
    for k, a in (('theta_c', -og['lo']), ('theta_s', og['hi'])):
        out[k] = np.bincount(row, weights=a, minlength=nrows)
        out[k + '_scale'] = np.bincount(row, weights=np.abs(a), minlength=nrows)
    return out


def _assert_theta_rows(got, want, bar, what):
    errs = {k: float((np.abs(got[k] - want[k]) / np.maximum(np.abs(want[k]), np.maximum(want[k + '_scale'], 1e-30))).max())
            for k in ('theta_c', 'theta_s')}
    assert max(errs.values()) < bar, (what, errs, {k: got[k] for k in errs}, want)
    return errs


def _oracle_loss(P, st, seed_g, n, lo, hi, boundary, n_sub=10):
    o = _oracle(P, n, lo, hi, boundary=boundary)
    o.set_frame(0, st['x'], st['v'], st['C'], st['F'], st['used'])
    for f in range(n_sub):
        o.substep(f)
    fr = o.get_frame(n_sub)
    return sum(float((seed_g[k].astype(np.float64) * fr[k]).sum()) for k in KEYS)


def reference_central_difference_case(case, boundary, per_row, n=16):
    """the fp64 reference dL/dtheta (PlasticGradOracle over the 10 backward substeps of one step) against central differences of the oracle's
    fp64 forward along a direction: one value per material row (per_row) or a random value per particle.  No device."""
    rng, P, st, seed_g = _scene(case, N=200, n=n)
    N = len(P['x'])
    if per_row:
        u, row = np.unique(P['mat'], return_inverse=True)
        tc_r, ts_r = random_theta(len(u), rng)
        tc, ts = tc_r[row], ts_r[row]
        dc, ds = (rng.randn(len(u)) * tc_r)[row], (rng.randn(len(u)) * ts_r)[row]
    else:
        tc, ts = random_theta(N, rng)
        dc, ds = rng.randn(N) * tc, rng.randn(N) * ts
    bnd = CUBE if boundary == 'cube' else CYLINDER
    lo, hi = 1.0 - tc, 1.0 + ts
    o = _oracle(P, n, lo, hi, boundary=bnd)
    o.set_frame(0, st['x'], st['v'], st['C'], st['F'], st['used'])
    for f in range(10):
        o.substep(f)
    o.reset_grad(); o.set_grad_frame(10, seed_g['x'], seed_g['v'], seed_g['C'], seed_g['F'])
    for f in range(9, -1, -1):
        o.substep_grad(f)
    g = o.get_param_grad()
    an = float((-g['lo'] * dc).sum() + (g['hi'] * ds).sum())   # dL/dtheta_c = -dL/dlo, dL/dtheta_s = dL/dhi
    assert np.abs(g['lo']).max() > 0 and np.abs(g['hi']).max() > 0, 'both limits are active in the scene'
    # the clamp is piecewise linear in the limits: a step of 1e-5 theta crosses no kink in these scenes (1e-4 does in the mixed one, 5e-4
    # relative; 1e-2 in every one, 0.2 .. 0.7 %), and a smaller step loses digits to cancellation
    eps = 1e-5
    fd = (_oracle_loss(P, st, seed_g, n, 1.0 - (tc + eps * dc), 1.0 + (ts + eps * ds), bnd)
          - _oracle_loss(P, st, seed_g, n, 1.0 - (tc - eps * dc), 1.0 + (ts - eps * ds), bnd)) / (2 * eps)
    assert abs(fd - an) <= 1e-6 * abs(fd), (case, boundary, per_row, fd, an)   # measured: up to 2e-8 relative
    return fd, an


def defaults_case(device, case, sort, with_field):
    """limits bound at their defaults (set_plastic_limits(), the k_*_field_plastic kernels) against the same fields without them (a density
    field equal to the rows' rho, with_field: and a random user (mu, lam) field; the k_*_field_mass kernels): states, state adjoint and the
    row keys, and against the table run"""
    rng, P, st, seed_g = _scene(case)
    fld = mfc.random_field(P, rng) if with_field else None
    res = {}
    for mode in ('table', 'mass', 'plastic'):
        s = _sim(device, P, 16, sort)
        if mode != 'table':
            if fld is not None:
                s.set_material_field(*fld)
            s.set_density_field(P['rho'])
        if mode == 'plastic':
            s.set_plastic_limits()
            lim = s.get_plastic_limits()
            assert (lim['theta_c'] == THETA_C).all() and (lim['theta_s'] == THETA_S).all()
            assert s._lim_orig is not None and float(s._lim_orig[0, 0]) == np.float32(0.998) and float(s._lim_orig[0, 1]) == np.float32(1.003)
        elif fld is not None and mode == 'table':
            s.set_material_field(*fld)
        res[mode] = mfc._run_one_substep_grad(s, st, seed_g)
        if mode == 'plastic':   # the plastic particles with an axis of F~ at the backward substep within fp32's reach of a default limit
            f9 = s.readframe(9)
            Ft = (np.eye(3)[None] + s.dt * np.asarray(f9['C'], np.float64)) @ np.asarray(f9['F'], np.float64)
            sig = np.linalg.svd(Ft, compute_uv=False)
            near = (np.abs(sig - 0.998).min(1) < NEAR) | (np.abs(sig - 1.003).min(1) < NEAR)
            keep = ~(near & np.isin(P['cls'], PLASTIC) & (np.asarray(f9['used']) != 0))
    (fa, ga, pa), (fb, gb, pb), (fc, gc, pc) = res['table'], res['mass'], res['plastic']
    # two runs may put such a particle's axis on either side of the limit, which switches its own adjoint (and nothing else's) between the two
    # branches of the clamp's derivative: the adjoint bars leave those particles out
    assert (~keep).sum() <= max(2, len(keep) // 25), ('ambiguous particles', int((~keep).sum()))
    ga, gb, gc = ({k: np.asarray(gx[k])[keep] for k in KEYS} for gx in (ga, gb, gc))
    # the scatter's float reductions are unordered, on the shim's threads as on the GPU, so two runs of one setting differ in the last bits:
    # the bars of the density field's test against the table run (tests/density_field_case.py::equals_table_case), with C and v at 5e-4:
    # two runs of the ICECREAM scene at level 3 alone differ by up to 1.6e-4 in C (measured on the shim)
    for ref, what in ((fb, 'level 3'), (fa, 'table')):
        for k in KEYS:
            assert rel(fc[k], ref[k]) < (1e-5 if k in 'xF' else 5e-4), ('state', what, k, rel(fc[k], ref[k]))
    for ref, what in ((gb, 'level 3'), (ga, 'table')):
        for k in KEYS:
            assert rel(gc[k], ref[k]) < 1e-3, ('state adjoint', what, k, rel(gc[k], ref[k]))
    for ref, what in ((pb, 'level 3'), (pa, 'table')):
        for k in ('mu', 'lam', 'rho', 'gravity'):
            assert rel(pc[k], ref[k]) < 1e-3, ('row key', what, k, pc[k], ref[k])
    assert 'theta_c' in pc and 'theta_c' not in pb and 'theta_c_field' not in pc
    assert ('mu_field' in pc) == with_field


def heterogeneous_case(device, case, sort, fuse=False, n=16, per_row=False):
    """random limits per particle (per_row: per material row) against the fp64 oracle: the frame after one step, one backward substep's state
    adjoint, per-particle dL/dtheta and the row sums, and the rows' dL/d(mu, lam, mass) exactly 0 while the limits are bound.  fuse (with
    sort): the stored-grid fused path (k_g2p2g_field_plastic).  Returns the errors."""
    rng, P, st, seed_g = _scene(case, n=n)
    N = len(P['x'])
    s = _sim(device, P, n, sort, fuse=fuse)
    row = _rows(P, s.get_material_table())
    if per_row:
        tc_r, ts_r = random_theta(len(s.get_material_table()['mat']), rng)
        s.set_plastic_limits(tc_r, ts_r)
        tc, ts = tc_r[row], ts_r[row]
    else:
        tc, ts = random_theta(N, rng)
        s.set_plastic_field(tc, ts)
    fr, g, pg = mfc._run_one_substep_grad(s, st, seed_g)
    assert not s._gmat[:, :3].cpu().numpy().any(), 'the rows\' dL/d(mu, lam, mass) are not written while the limits are bound'
    lo, hi = limits(tc, ts)
    o = _oracle(P, n, lo, hi)
    o.set_frame(0, st['x'], st['v'], st['C'], st['F'], st['used'])
    for f in range(10):
        o.substep(f)
    want_fr = o.get_frame(10)
    o.reset_grad(); o.set_grad_frame(10, seed_g['x'], seed_g['v'], seed_g['C'], seed_g['F'])
    o.substep_grad(9)
    og, opg = o.get_grad_frame(9), o.get_param_grad()
    assert np.abs(opg['lo']).max() > 0 and np.abs(opg['hi']).max() > 0
    # the clamp's derivative jumps where a singular value meets a limit: the particles with an axis within fp32's reach of one at the backward
    # substep (PlasticGradOracle.near_limit) have no reference value for their own adjoint and dL/dtheta, and are left out of the per-particle
    # bars (their adjoint does not reach any other particle's within the substep); the frames, being continuous there, keep every particle
    amb = o.near_limit(o.get_frame(9))
    keep = ~amb
    assert amb.sum() <= max(2, N // 25), ('ambiguous particles', int(amb.sum()))
    gl = s._glim_orig.cpu().numpy()   # the simulator's per-particle (dL/dlo, dL/dhi) in original order, also behind per-row limits
    errs = {('frame', k): rel(fr[k], want_fr[k]) for k in KEYS}
    errs.update({('adjoint', k): rel(np.asarray(g[k])[keep], og[k][keep]) for k in KEYS})
    errs[('field', 'theta_c')] = rel(-gl[keep, 0], -opg['lo'][keep])
    errs[('field', 'theta_s')] = rel(gl[keep, 1], opg['hi'][keep])
    if not per_row:
        assert np.array_equal(pg['theta_c_field'], -gl[:, 0]) and np.array_equal(pg['theta_s_field'], gl[:, 1])
    else:
        assert 'theta_c_field' not in pg
    rest = 1e-3   # the bars of the plastic (mu, lam) field cases (tests/material_field_case.py, density_field_case.py: icecream)
    # per-particle dL/dtheta: W_dd = (U^T gF' V)_dd from an fp32 SVD of a nearly isotropic F~ (every singular value of a plastic particle
    # lies within 1.2e-2 of 1), measured up to 1.4e-3 of the largest on the shim (12 runs of the ICECREAM and PLASTIC_DEMO scenes)
    bars = {('frame', 'x'): 1e-5, ('frame', 'F'): 1e-5, ('field', 'theta_c'): 3e-3, ('field', 'theta_s'): 3e-3}
    bad = {k: e for k, e in errs.items() if not e < bars.get(k, rest)}
    assert not bad, (case, sort, bad, errs)
    # the row keys are the sums of the per-particle values: the reference's, with the simulator's own for the ambiguous particles
    want = dict(lo=np.where(amb, gl[:, 0], opg['lo']), hi=np.where(amb, gl[:, 1], opg['hi']))
    errs['rows'] = _assert_theta_rows(pg, _theta_rows(want, row, len(pg['mu'])), rest, (case, sort))
    errs['mu_lam_rho'] = pgc.assert_param_grads_close(pg, pgc.oracle_rows(opg, P, s.get_material_table(), s.p_vol), rest, (case, sort))
    return errs


def ring_case(device, sort_every, n_steps=3, T=20, N=400, n=16):
    """a T = 20 ring over 3 steps with random per-particle limits, index-matched loss on the last frame: per-particle dL/dtheta against the
    oracle.  Sort epochs change the slot order between steps, so limits or gradients gathered in the wrong order fail here."""
    rng = np.random.RandomState(31)
    N = N * n // 16
    x = rng.uniform(0.38, 0.62, size=(N, 3))
    mat = np.array([(M.ELASTIC, M.ICECREAM)[i % 2] for i in range(N)], dtype=np.int32)
    P = make_particles(x, mat, n)
    tc, ts = random_theta(N, rng)
    v0 = (rng.randn(N, 3) * 0.4).astype(np.float32)
    gx = rng.randn(N, 3).astype(np.float32)
    s = _sim(device, P, n, False, T=T)
    s.sort_every, s.store_grids = sort_every, False
    s.set_plastic_field(tc, ts)
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
    lo, hi = limits(tc, ts)
    o = _oracle(P, n, lo, hi, T=T)
    o.enable_grad()
    o.set_frame(0, x, v0, np.zeros((N, 3, 3)), np.tile(np.eye(3), (N, 1, 1)), P['used'])
    for _ in range(n_steps):
        o.step(None)
    o.reset_grad(); o.set_grad_frame(o.cur_substep_local, gx, z3, z9, z9)
    for _ in range(n_steps):
        o.step_grad(None)
    want = o.get_param_grad()
    # fp32 drifts from fp64 over 30 substeps, and an axis that ends within that drift of a limit is clamped in one run and not in the other,
    # which moves its W_dd in or out of dL/dlo: the largest per-particle error is such a particle (2.9e-2 on the shim, 0.10 on an H100 at
    # 32^3), so the per-particle bar is the fields' 2e-2 on the 99th percentile, the row sums the fields' 1e-2; a wrong slot order gives
    # order 1 on most particles
    errs = {}
    for k, g, w in (('theta_c', got['theta_c_field'], -want['lo']), ('theta_s', got['theta_s_field'], want['hi'])):
        errs[k] = float(np.percentile(np.abs(g - w), 99) / np.abs(w).max())
    assert max(errs.values()) < 2e-2, (sort_every, errs)
    errs['rows'] = _assert_theta_rows(got, _theta_rows(want, _rows(P, s.get_material_table()), len(got['mu'])), 1e-2, ('ring', sort_every))
    return errs


def fused_forward_case(device, case='mixed', n=16):
    """forward-only steps on the fused path with random limits (k_p2g_field_plastic, then k_fwd<4, false, false> for the inner substeps): the
    frame after two steps against the fp64 oracle and the per-substep path"""
    rng, P, st, _ = _scene(case, n=n)
    tc, ts = random_theta(len(P['x']), rng)
    fr = {}
    for fuse in (True, False):
        s = _sim(device, P, n, True, pg=False, fuse=fuse)
        s.set_plastic_field(tc, ts)
        g = s.get_state(); g['v'][:] = st['v']; g['F'][:] = st['F']; g['C'][:] = st['C']; s.set_state(0, g)
        s.step(None); s.step(None)
        fr[fuse] = s.readframe(20)
    if device == 'cpu':
        assert s._lib.fmpm_fwd_path(s._h) & 1, 'the fused forward path runs k_fwd'
    o = _oracle(P, n, *limits(tc, ts))
    o.set_frame(0, st['x'], st['v'], st['C'], st['F'], st['used'])
    for f in range(20):
        o.substep(f)
    want = o.get_frame(20)
    errs = {k: rel(fr[True][k], want[k]) for k in KEYS}
    errs.update({('unfused', k): rel(fr[True][k], fr[False][k]) for k in KEYS})
    bars = dict(x=1e-5, F=1e-5, v=2e-4, C=2e-4)
    bad = {k: e for k, e in errs.items() if not e < bars[k if isinstance(k, str) else k[1]]}
    assert not bad, (bad, errs)
    return errs


def rigid_case(device, n_grid=16):
    """water, an ICECREAM blob and a MAT_RIGID cube with random limits on every particle: one step on the fused stored-grid path, where the rigid
    body's particles scatter through k_p2g_rigid_field_plastic after the shape matching, against the fp64 oracle"""
    rng = np.random.RandomState(17)
    k = n_grid // 16
    xw = rng.uniform((0.32, 0.32, 0.32), (0.68, 0.42, 0.68), size=(500 * k, 3))
    xa = rng.uniform((0.38, 0.45, 0.38), (0.50, 0.55, 0.50), size=(200 * k, 3))
    xe = rng.uniform((0.54, 0.45, 0.52), (0.62, 0.55, 0.60), size=(150 * k, 3))
    x = np.concatenate([xw, xa, xe])
    mat = np.concatenate([np.full(len(xw), M.WATER), np.full(len(xa), M.RIGID), np.full(len(xe), M.ICECREAM)])
    bid = np.concatenate([np.zeros(len(xw)), np.ones(len(xa)), np.full(len(xe), 2)]).astype(np.int32)
    P = make_particles(x, mat, n_grid)
    P['body_id'] = bid; P['bodies'] = {'n': 3}
    N = len(x)
    tc, ts = random_theta(N, rng)
    v0 = (rng.randn(N, 3) * 0.3).astype(np.float32)
    s = _sim(device, P, n_grid, True, pg=False, fuse=True)
    s.set_plastic_field(tc, ts)
    st = s.get_state(); st['v'][:] = v0; s.set_state(0, st)
    s.enable_grad()
    s.step(None)
    assert s._can_fuse()
    got = s.get_state()
    o = _oracle(P, n_grid, *limits(tc, ts))
    o.set_bodies(bid, 3)
    o.set_frame(0, x, v0, np.zeros((N, 3, 3)), np.tile(np.eye(3), (N, 1, 1)), P['used'])
    for f in range(10):
        o.substep(f)
    want = o.get_frame(10)
    errs = {k: rel(got[k], want[k]) for k in ('x', 'v', 'F')}
    assert errs['x'] < 1e-5 and errs['F'] < 1e-5 and errs['v'] < 5e-4, errs   # v: the ICECREAM bar of defaults_case
    return errs


def injector_case(device, fuse, sort_every=1, n_steps=3, T=20, n_grid=16):
    """an AgentInjector pouring ICECREAM onto an ICECREAM1 base, random limits on every particle, a chamfer loss on the injected ICECREAM: the
    injected particles scatter through k_p2g_injected_field_plastic (fused) or the per-substep kernels; per-particle dL/dtheta and its row sums
    against the oracle"""
    from fluidlab_b200 import TaichiEnv, ShapeMatchingLoss
    n_base, n_inj, flux = 400 * n_grid // 16, 120, 2
    rng = np.random.RandomState(21)
    x = np.concatenate([np.tile(M.NOWHERE, (n_inj, 1)), rng.uniform((0.38, 0.36, 0.38), (0.62, 0.45, 0.62), size=(n_base, 3))])
    mat = np.concatenate([np.full(n_inj, M.ICECREAM), np.full(n_base, M.ICECREAM1)])
    used = np.concatenate([np.zeros(n_inj), np.ones(n_base)]).astype(np.int32)
    P = make_particles(x, mat, n_grid, used=used)
    bnd = dict(type='cylinder', xz_radius=0.2, xz_center=(0.5, 0.5), y_range=(0.34, 0.9))
    ebnd = dict(type='cylinder', xz_radius=0.12, xz_center=(0.5, 0.5), y_range=(0.55, 0.55))
    cfg = dict(type='AgentInjector', effectors=[dict(type='Injector', params=dict(radius=0.0075, flux=flux, init_pos=(0.5, 0.5, 0.5), action_dim=3, inject_v=(0.0, -3.0, 0.0),
                                                                                 action_scale_p=(1.0, 1.0, 1.0), action_scale_v=(1.0, 1.0, 1.0), locally_random=True), boundary=ebnd)])
    tgt = [rng.uniform(0.4, 0.6, size=x.shape).astype(np.float32) for _ in range(n_steps)]
    actions = rng.uniform(-0.004, 0.004, size=(n_steps, 3)).astype(np.float32)
    action_p = np.array([0.47, 0.55, 0.52], dtype=np.float32)
    tc, ts = random_theta(len(x), rng)
    kw = dict(ckpt_dest='cpu', device='cpu') if device == 'cpu' else dict(ckpt_dest='gpu')
    env = TaichiEnv(quality=n_grid / 64, max_substeps_local=T, gravity=(0.0, -20.0, 0.0), horizon=n_steps, **kw)
    env.simulator.use_graphs, env.simulator.fuse_g2p2g, env.simulator.sort_every = False, fuse, sort_every
    env.simulator.store_grids = fuse
    env.simulator.param_grad = True
    np.random.seed(5)
    env.setup_agent(cfg)
    env.particle_bodies.get = lambda: P
    env.setup_boundary(**bnd)
    env.setup_loss(loss_cls=ShapeMatchingLoss, matching_mat=M.ICECREAM, temporal_range_type='all', target=tgt, weights={'chamfer': 1.0})
    env.build()
    sim = env.simulator
    sim.set_plastic_field(tc, ts)
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
    o = PlasticGradOracle(n_grid, P, lo=limits(tc, ts)[0], hi=limits(tc, ts)[1], gravity=(0, -20, 0), boundary=bnd, precision=64, max_substeps_local=T)
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
        o.loss_seed(o.cur_substep_local, M.ICECREAM, 1.0, tgt[i]); o.step_grad(actions[i])
    want = o.get_param_grad()
    assert np.abs(want['lo']).max() > 0 and np.abs(want['hi']).max() > 0, 'the limits carry a gradient'
    errs = {}   # the ring case's bars: 30 substeps of a plastic body
    for k, g, w in (('theta_c', got['theta_c_field'], -want['lo']), ('theta_s', got['theta_s_field'], want['hi'])):
        errs[k] = float(np.percentile(np.abs(g - w), 99) / np.abs(w).max())
    assert max(errs.values()) < 2e-2, (fuse, errs)
    errs['rows'] = _assert_theta_rows(got, _theta_rows(want, _rows(P, sim.get_material_table()), len(got['mu'])), 1e-2, ('injector', fuse))
    return errs


def check_records(s, order=None):
    """the field level that what the user set selects (3 with any limits, else 2 with rho, else 1 with (mu, lam), else 0), and the records
    the simulator composed for it: every value the user's field where one is set and the rows' otherwise, in f32 as the kernels read it
    (mass f32(p_vol) f32(rho), lo = f32(1 - theta_c), hi = f32(1 + theta_s)).  order (an _Order): each slot buffer the level reads holds its
    record gathered in that slot order.  Returns the records in original order by buffer name."""
    t, row = s.get_material_table(), s._mrow.cpu().numpy() & 0xff
    fld, rho, lim = s.get_material_field(), s.get_density_field(), s.get_plastic_field()
    if lim is None and s._lim_rows is not None:
        lim = tuple(a[row] for a in s._lim_rows)
    level = 3 if lim is not None else 2 if rho is not None else 1 if fld is not None else 0
    assert s._field_level == level, (s._field_level, level)
    mulam = np.stack(fld if fld is not None else (t['mu'][row].astype(np.float32), t['lam'][row].astype(np.float32)), 1)
    mass = np.float32(s.p_vol) * (rho if rho is not None else t['rho'][row].astype(np.float32))
    want = {}
    if level in (1, 2):
        want['_field_slot'] = mulam
    if level >= 2:
        want['_mass_slot'] = mass
    if level == 3:
        want['_pfield_slot'] = np.concatenate([mulam, np.stack([(1.0 - lim[0]).astype(np.float32), (1.0 + lim[1]).astype(np.float32)], 1)], 1)
    got = {name: rec.cpu().numpy() for rec, buf in s._records for name in want if getattr(s, name) is buf}
    assert sorted(got) == sorted(want), (level, sorted(got))
    for name, w in want.items():
        assert got[name].dtype == np.float32 and np.array_equal(got[name].view(np.int32), w.view(np.int32)), (level, name)
        if order is not None:
            ids = np.arange(len(w)) if order.ids is None else order.ids.cpu().numpy()
            assert s._field_ord is order and np.array_equal(getattr(s, name).cpu().numpy().view(np.int32), w[ids].view(np.int32)), (level, name)
    return got


def composition_case(device, set_order, clear_order):
    """the (mu, lam) field, the density field and the plastic field, all equal to the rows, set one after the other in `set_order` and cleared
    in `clear_order` ('m', 'r', 'l'), one step forward and backward after every change, no reset_grad in between: the row keys mu, lam, rho
    and gravity accumulate what the table run accumulates over the same steps (so nothing accumulated under one binding is lost when the
    next changes), each field key is present exactly while its field is set, and the limit keys while limits are set.  After every change,
    the field level and the slot buffers it reads (check_records), in the slot order of frame 0, the last one the backward pass touched."""
    rng, P, st, seed_g = _scene('mixed', N=200)
    N = len(P['x'])
    tc, ts = np.full(N, THETA_C), np.full(N, THETA_S)
    ops = [('set', k) for k in set_order] + [('clear', k) for k in clear_order]

    def run(s, apply):
        s.enable_grad()
        s.reset_grad()
        bound = set()
        for i in range(len(ops) + 1):
            if i > 0 and apply:
                what, k = ops[i - 1]
                if what == 'set':
                    {'m': lambda: s.set_material_field(P['mu'], P['lam']), 'r': lambda: s.set_density_field(P['rho']),
                     'l': lambda: s.set_plastic_field(tc, ts)}[k]()
                    bound.add(k)
                else:
                    {'m': s.clear_material_field, 'r': s.clear_density_field, 'l': s.clear_plastic_field}[k]()
                    bound.discard(k)
            s.cur_substep_global = 0
            g = s.get_state(); g['v'][:] = st['v']; g['F'][:] = st['F']; g['C'][:] = st['C']; s.set_state(0, g)
            s.step(None)
            s.set_grad(seed_g['x'], seed_g['v'], seed_g['C'], seed_g['F'])
            s.step_grad(None)
            pg = s.get_param_grad()
            if apply:
                assert ('mu_field' in pg) == ('m' in bound) and ('rho_field' in pg) == ('r' in bound), (ops[:i], sorted(pg))
                assert ('theta_c_field' in pg) == ('l' in bound) and ('theta_c' in pg) == ('l' in bound), (ops[:i], sorted(pg))
                check_records(s, s._frame_ord[0])
        return s.get_param_grad()
    want = run(_sim(device, P, 16, True), False)
    got = run(_sim(device, P, 16, True), True)
    errs = {k: rel(got[k], want[k]) for k in ('mu', 'lam', 'rho', 'gravity')}
    assert max(errs.values()) < 1e-3, (set_order, clear_order, errs)
    return errs


def identification_case(device, n_grid=16, N=1200, iters=25, lr=0.15, n_steps=4, seed=0, truth=(6e-3, 1e-3)):
    """an ICECREAM block dropped onto the floor, its true limits theta_c / theta_s (`truth`) recovered from the block's per-step grid mass (the
    true run's density deposit after every step, DensityMatchingLoss's recording).  The unknowns are the block's row limits, fitted in log space
    by torch.optim.Adam from the defaults with dL/dlog theta = theta dL/dtheta from get_param_grad()['theta_c' / 'theta_s'].  Returns per
    iteration (theta_c, theta_s, loss), before every iteration and after the last."""
    import torch
    rng = np.random.RandomState(seed)
    x = rng.uniform((0.35, 0.06, 0.35), (0.65, 0.3, 0.65), size=(N, 3))
    P = make_particles(x, M.ICECREAM, n_grid)
    floor = dict(type='cube', lower=(0.05, 0.05, 0.05), upper=(0.95, 0.95, 0.95))
    s = _sim(device, P, n_grid, True, T=10 * n_steps + 10, boundary=floor)
    st0 = s.get_state()
    c = x.mean(0)
    st0['v'] = (np.array([0.0, -3.0, 0.0]) + 8.0 * np.cross(np.array([0.3, 1.0, 0.2]), x - c)).astype(np.float32)
    G = n_grid ** 3
    dev = s.device
    mask = s.material_row_mask(M.ICECREAM)
    mass_dev = torch.zeros(G, dtype=torch.float32, device=dev)
    out = torch.zeros(1, dtype=torch.float32, device=dev)

    def rollout(th, record=None):
        s.set_plastic_limits([th[0]], [th[1]])
        s.cur_substep_global = 0
        s.set_state(0, st0)
        loss = 0.0
        for i in range(n_steps):
            s.step(None)
            if record is not None:
                s.density_loss(mass_dev, None, None, 1.0, 0.0, mask, out)
                record.append(mass_dev.clone())
            else:
                out.zero_()
                s.density_loss(mass_dev, tgt[i], None, 1.0, 0.0, mask, out)
                loss += float(out[0])
        return loss
    s.enable_grad()
    tgt = []
    rollout(truth, tgt)
    logt = torch.tensor(np.log([THETA_C, THETA_S]), dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([logt], lr=lr)
    hist = []
    for it in range(iters + 1):
        th = torch.exp(logt.detach()).numpy()
        loss = rollout(th)
        hist.append((float(th[0]), float(th[1]), loss))
        if it == iters:
            break
        s.reset_grad()
        for i in range(n_steps - 1, -1, -1):
            s.add_x_grad_density(mass_dev, tgt[i], None, 1.0, 0.0, mask)
            s.step_grad(None)
        g = s.get_param_grad()
        opt.zero_grad()
        logt.grad = torch.tensor([g['theta_c'][0] * th[0], g['theta_s'][0] * th[1]], dtype=torch.float64)
        opt.step()
    return hist
