"""Loss gradients with respect to the material parameters and gravity (MPMSimulator.param_grad) on an H100: the kernels against the fp64
oracle, central differences at full size (C2: 1M water on 128^3, plus a 256k ELASTIC block for dL/dmu), and a system identification."""
import numpy as np
import pytest
import torch

from conftest import make_particles
from fluidlab_b200 import macros as M
import param_grad_case as pgc

pytestmark = pytest.mark.gpu


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip('needs an H100')


@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('case', ['water', 'elastic', 'icecream', 'milk_vis', 'mixed'])
def test_param_grad_substep_grad_matches_oracle(case, sort):
    _need_gpu()
    pgc.substep_case(None, case, sort)


@pytest.mark.parametrize('sort_every', [0, 1])
def test_param_grad_dloss_daction_latteart_like(sort_every):
    _need_gpu()
    pgc.latteart_case(None, sort_every)


def _fd_scene(mat, N, lo, hi, seed, F0):
    from fluidlab_b200 import MPMSimulator
    rs = np.random.RandomState(seed)
    x = rs.uniform(lo, hi, size=(N, 3))
    P = make_particles(x, mat, 128)
    s = MPMSimulator(dim=3, quality=2, gravity=(0.0, -10.0, 0.0), horizon=100, max_substeps_local=50, max_substeps_global=100000, ckpt_dest='gpu')
    s.build(None, None, [], P)
    tp = 2 * np.pi
    v0 = (0.2 * np.stack([np.sin(tp * x[:, 1] * 2), np.cos(tp * x[:, 2] * 3), np.sin(tp * x[:, 0] * 2 + 1.0)], 1)).astype(np.float32)
    w = np.stack([np.cos(tp * (x[:, 0] * 2 + 0.3)), np.sin(tp * (x[:, 1] * 3 + x[:, 0])), np.cos(tp * x[:, 2] * 3)], 1).astype(np.float32)
    base = s.get_state(); base['v'] = v0
    base['F'] = np.tile(np.asarray(F0, np.float32), (N, 1, 1))   # a pre-strained start: the pressure / stress term acts from the first substep on
    return s, base, w


def _fd_check(s, base, w, keys):
    """one step (10 substeps), L = sum w . x_T: dL/d(param) from param_grad against central differences through set_material_table / set_gravity"""
    N = len(w)

    def run():
        s.cur_substep_global = 0
        s.set_state(0, base)
        s.step(None)
        return float((s.get_state()['x'].astype(np.float64) * w).sum())
    s.param_grad = True
    s.enable_grad()
    run()
    s.reset_grad()
    z3, z9 = np.zeros((N, 3), np.float32), np.zeros((N, 3, 3), np.float32)
    s.set_grad(w, z3, z9, z9)
    s.step_grad(None)
    g = s.get_param_grad()
    s.disable_grad()
    table = s.get_material_table()
    out = {}
    for key, h in keys:
        if key == 'gravity_y':
            an = float(g['gravity'][1])
            s.set_gravity((0.0, -10.0 + h, 0.0)); lp = run()
            s.set_gravity((0.0, -10.0 - h, 0.0)); lm = run()
            s.set_gravity((0.0, -10.0, 0.0))
        else:
            an = float(g[key][0]); v = float(table[key][0])
            s.set_material_table(**{key: [v + h]}); lp = run()
            s.set_material_table(**{key: [v - h]}); lm = run()
            s.set_material_table(**{key: [v]})
        fd = (lp - lm) / (2 * h)
        out[key] = (fd, an)
    return out


def test_param_grad_full_size_central_differences_c2():
    """C2 (1M water particles, 128^3, all-liquid kernels), compressed to J = 0.94 at the start so that the pressure matters within one step: dL/dlam,
    dL/drho and dL/dg_y against central differences of the fp32 forward, 0.5 % bar"""
    _need_gpu()
    s, base, w = _fd_scene(M.WATER, 1_000_000, (0.25, 0.30, 0.25), (0.75, 0.54, 0.75), 0, 0.98 * np.eye(3))
    lam, rho = float(s.get_material_table()['lam'][0]), float(s.get_material_table()['rho'][0])
    res = _fd_check(s, base, w, [('lam', 0.02 * lam), ('rho', 0.02 * rho), ('gravity_y', 0.5)])
    for k, (fd, an) in res.items():
        assert an != 0.0 and abs(fd - an) < 5e-3 * abs(an), (k, fd, an, res)


def test_param_grad_full_size_central_differences_elastic():
    """a 256k-particle ELASTIC block on 128^3 (general kernel with the SVD), pre-strained: dL/dmu and dL/dlam against central differences, 0.5 % bar"""
    _need_gpu()
    s, base, w = _fd_scene(M.ELASTIC, 262_144, (0.35, 0.35, 0.35), (0.65, 0.65, 0.65), 1, np.diag([0.97, 1.0, 1.03]))
    t = s.get_material_table()
    res = _fd_check(s, base, w, [('mu', 0.02 * float(t['mu'][0])), ('lam', 0.02 * float(t['lam'][0]))])
    for k, (fd, an) in res.items():
        assert an != 0.0 and abs(fd - an) < 5e-3 * abs(an), (k, fd, an, res)


def test_param_grad_system_identification():
    """20 Adam iterations on (log mu, log lam) of an ELASTIC block started 30 % off: the parameter error shrinks at least 10x"""
    _need_gpu()
    errs = pgc.sysid_case(None)
    assert errs[-1] <= 0.1 * errs[0], errs
