"""The correspondence-free momentum loss (MomentumMatchingLoss) on an H100: the kernels against the fp64 reference, TaichiEnv end to end
against the oracle, the step-end frame of the fused forward path, central differences at full size (C2: 1M water on 128^3) and a viscosity
identification against a momentum recording."""
import numpy as np
import pytest
import torch

import density_loss_case as dlc
import density_loss_ref as dref
import momentum_loss_case as mlc
import momentum_loss_ref as mref
from fluidlab_b200 import macros as M
from test_density_loss import check_env_case
from test_momentum_loss import check_fused_frame_case
from test_param_grad_gpu import _fd_scene

pytestmark = pytest.mark.gpu


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip('needs an H100')


def test_reference_deposit_equals_the_p2g_accumulator():
    _need_gpu()
    assert mlc.deposit_matches_p2g(None) < 1e-6


@pytest.mark.parametrize('case', mlc.KERNEL_CASES)
def test_momentum_kernels_match_the_reference(case):
    _need_gpu()
    mlc.kernel_case(None, case)


def test_momentum_loss_through_taichi_env_matches_the_oracle():
    _need_gpu()
    check_env_case(mlc.env_case(None))


def test_momentum_loss_reads_the_step_end_frame_of_the_fused_forward_path():
    _need_gpu()
    check_fused_frame_case(mlc.fused_frame_case(None))


def _host_deposit(x, v, C, mass, sel, n, chunk=100_000):
    """mref.deposit over chunks of particles (bounded host memory at 1M particles)"""
    pm, m = np.zeros((n ** 3, 3)), np.zeros(n ** 3)
    for a in range(0, len(x), chunk):
        b = slice(a, a + chunk)
        p_, m_ = mref.deposit(x[b], v[b], C[b], mass, sel[b], n)
        pm += p_; m += m_
    return pm, m


def test_momentum_loss_full_size_central_differences_c2():
    """C2 (1M water, 128^3), compressed to J = 0.94 at the start, one step; targets: the (P, m) deposit of the block shifted by half a cell with
    another velocity field, plus an SDF term.  dL/dlam, dL/drho and the derivative along a smooth v0 direction against central differences of
    the fp32 forward, with L evaluated in fp64 on the host from get_state(); 0.5 % bar"""
    _need_gpu()
    from fluidlab_b200 import MomentumMatchingLoss
    s, base, _ = _fd_scene(M.WATER, 1_000_000, (0.25, 0.30, 0.25), (0.75, 0.54, 0.75), 0, 0.98 * np.eye(3))
    n, N = 128, 1_000_000
    x0 = base['x'].astype(np.float64)
    table = s.get_material_table()
    m_p = float(np.float32(s.p_vol) * np.float32(table['rho'][0]))
    tp = 2 * np.pi
    v_star = 0.3 * np.stack([np.cos(tp * x0[:, 1] * 2), np.sin(tp * x0[:, 2] * 2), np.cos(tp * x0[:, 0] * 3)], 1)
    t_p, t_m = MomentumMatchingLoss.momentum_from_points(x0 + np.array([0.5, -0.5, 0.25]) / n, v_star, m_p, n)
    t_p, t_m = t_p.astype(np.float64), t_m.astype(np.float64)
    sdf = dlc.sphere_sdf(n, (0.5, 0.42, 0.5), 0.2)
    wd, ws, wm = 1.0 / m_p ** 2, 0.1 / m_p, 1.0 / m_p ** 2
    dv = (0.2 * np.stack([np.cos(tp * x0[:, 2] * 2), np.sin(tp * x0[:, 0] * 3), np.cos(tp * x0[:, 1] * 2 + 0.5)], 1)).astype(np.float32)

    def host_loss(rho=None):
        st = s.get_state()
        x = st['x'].astype(np.float64)
        mass = m_p if rho is None else float(np.float32(s.p_vol) * np.float32(rho))
        sel = dref.selection(x, st['used'], np.full(N, M.WATER), M.WATER, n)
        pm, m = _host_deposit(x, st['v'].astype(np.float64), st['C'].astype(np.float64), mass, sel, n)
        return mref.loss(pm, m, t_m, t_p, sdf, wd, ws, wm)

    def run(state, rho=None):
        s.cur_substep_global = 0
        s.set_state(0, state)
        s.step(None)
        return host_loss(rho)
    dev = s.device
    tgt_d = torch.from_numpy(mlc.pack_target(t_m, t_p, n ** 3)).to(dev)
    sdf_d = torch.from_numpy(sdf.astype(np.float32)).to(dev)
    field = torch.zeros((n ** 3, 4), dtype=torch.float32, device=dev)
    s.param_grad = True
    s.enable_grad()
    run(base)
    s.reset_grad()
    s.add_grad_momentum(field, tgt_d, sdf_d, wd, ws, wm, s.material_row_mask(M.WATER))
    s.step_grad(None)
    g = s.get_param_grad()
    gv = s.get_grad()['v']
    gv = gv.cpu().numpy() if torch.is_tensor(gv) else np.asarray(gv)
    s.disable_grad()
    res = {}
    for key, h in (('lam', 0.02 * float(table['lam'][0])), ('rho', 0.02 * float(table['rho'][0]))):
        v = float(table[key][0])
        s.set_material_table(**{key: [v + h]}); lp = run(base, v + h if key == 'rho' else None)
        s.set_material_table(**{key: [v - h]}); lm = run(base, v - h if key == 'rho' else None)
        s.set_material_table(**{key: [v]})
        res[key] = ((lp - lm) / (2 * h), float(g[key][0]))
    h = 0.05
    bp, bm = dict(base), dict(base)
    bp['v'] = base['v'] + h * dv; bm['v'] = base['v'] - h * dv
    res['v0_direction'] = ((run(bp) - run(bm)) / (2 * h), float((gv.astype(np.float64) * dv).sum()))
    print('c2 central differences (fd, analytic):', res)
    for k, (fd, an) in res.items():
        assert an != 0.0 and abs(fd - an) < 5e-3 * abs(an), (k, fd, an, res)


def test_momentum_loss_viscosity_identification():
    """20 Adam iterations on log mu of a MILK_VIS block in shear, started 30 % off, against the (P*, m*) volumes of a permuted recording (no
    particle correspondence): the viscosity error shrinks at least 10x.  The same fit with the density term alone is reported."""
    _need_gpu()
    errs = mlc.sysid_viscosity_case(None)
    dens = mlc.sysid_viscosity_case(None, w_momentum=False)
    print('viscosity sysid: error %.4f -> %.5f (momentum + density), %.4f -> %.5f (density alone)' % (errs[0], errs[-1], dens[0], dens[-1]))
    print('  momentum + density:', ' '.join('%.4f' % e for e in errs))
    print('  density alone:     ', ' '.join('%.4f' % e for e in dens))
    assert errs[-1] <= 0.1 * errs[0], errs
