"""The correspondence-free density loss (DensityMatchingLoss) on an H100: the kernels against the fp64 reference, TaichiEnv end to end
against the oracle, central differences at full size (C2: 1M water on 128^3) and a system identification against a density recording."""
import numpy as np
import pytest
import torch

import density_loss_ref as dref
import density_loss_case as dlc
from fluidlab_b200 import macros as M
from test_density_loss import check_env_case
from test_param_grad_gpu import _fd_scene

pytestmark = pytest.mark.gpu


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip('needs an H100')


def test_reference_deposit_equals_the_p2g_grid_mass():
    _need_gpu()
    assert dlc.deposit_matches_p2g(None) < 1e-6


@pytest.mark.parametrize('case', dlc.KERNEL_CASES)
def test_density_kernels_match_the_reference(case):
    _need_gpu()
    dlc.kernel_case(None, case)


def test_density_loss_through_taichi_env_matches_the_oracle():
    _need_gpu()
    check_env_case(dlc.env_case(None))


def test_density_loss_full_size_central_differences_c2():
    """C2 (1M water, 128^3), compressed to J = 0.94 at the start, one step; target: the deposit of the block shifted by half a cell, plus an SDF
    term.  dL/dlam, dL/drho and the derivative along a smooth v0 direction against central differences of the fp32 forward, with L evaluated
    in fp64 on the host from get_state(); 0.5 % bar"""
    _need_gpu()
    s, base, _ = _fd_scene(M.WATER, 1_000_000, (0.25, 0.30, 0.25), (0.75, 0.54, 0.75), 0, 0.98 * np.eye(3))
    n, N = 128, 1_000_000
    x0 = base['x'].astype(np.float64)
    table = s.get_material_table()
    m_p = float(np.float32(s.p_vol) * np.float32(table['rho'][0]))
    tgt = DensityMatchingLoss_points(x0 + np.array([0.5, -0.5, 0.25]) / n, m_p, n)
    sdf = dlc.sphere_sdf(n, (0.5, 0.42, 0.5), 0.2)
    wd, ws = 1.0 / m_p ** 2, 0.1 / m_p
    tp = 2 * np.pi
    dv = (0.2 * np.stack([np.cos(tp * x0[:, 2] * 2), np.sin(tp * x0[:, 0] * 3), np.cos(tp * x0[:, 1] * 2 + 0.5)], 1)).astype(np.float32)

    def host_loss(rho=None):
        st = s.get_state()
        x = st['x'].astype(np.float64)
        mass = m_p if rho is None else float(np.float32(s.p_vol) * np.float32(rho))
        m = dref.deposit(x, mass, dref.selection(x, st['used'], np.full(N, M.WATER), M.WATER, n), n)
        return dref.loss(m, tgt, sdf, wd, ws)

    def run(state, rho=None):
        s.cur_substep_global = 0
        s.set_state(0, state)
        s.step(None)
        return host_loss(rho)
    dev = s.device
    tgt_d, sdf_d = (torch.from_numpy(a.astype(np.float32)).to(dev) for a in (tgt, sdf))
    scratch = torch.zeros(n ** 3, dtype=torch.float32, device=dev)
    s.param_grad = True
    s.enable_grad()
    run(base)
    s.reset_grad()
    s.add_x_grad_density(scratch, tgt_d, sdf_d, wd, ws, s.material_row_mask(M.WATER))
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


def DensityMatchingLoss_points(x, m, n):
    from fluidlab_b200 import DensityMatchingLoss
    return DensityMatchingLoss.density_from_points(x, m, n).astype(np.float64)


def test_density_loss_system_identification():
    """20 Adam iterations on (log mu, log lam) of an ELASTIC block started 30 % off, against the density volumes of a permuted recording (no
    particle correspondence): the parameter error shrinks at least 10x.  The same run against a 50 % subsample with doubled mass is reported."""
    _need_gpu()
    errs = dlc.sysid_density_case(None)
    sub = dlc.sysid_density_case(None, subsample=True)
    print('density sysid: error %.4f -> %.5f (permuted recording), %.4f -> %.5f (50 %% subsample, doubled mass)' % (errs[0], errs[-1], sub[0], sub[-1]))
    assert errs[-1] <= 0.1 * errs[0], errs
