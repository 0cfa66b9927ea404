"""Loss gradients with respect to the material parameters (mu, lam, rho per material row) and gravity, on CPU: the fp64 oracle's parameter
adjoints against central differences through its own forward and against torch.autograd on an independent restatement, the CUDA kernels on
the execution-model shim against the oracle, the x-slab rejection and the C ABI."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'cuda_emu'))
import harness  # noqa: E402

from conftest import make_particles, box_sdf  # noqa: E402
from fluidlab_b200 import macros as M  # noqa: E402
from param_grad_ref import ParamGradOracle  # noqa: E402
import param_grad_case as pgc  # noqa: E402

CUBE = dict(type='cube', lower=(0.32, 0.32, 0.32), upper=(0.68, 0.68, 0.68))
CYL = dict(type='cylinder', xz_radius=0.2, xz_center=(0.5, 0.5), y_range=(0.3, 0.7))


def _scene(mat, rng, n_grid=16, N=120):
    P = make_particles(rng.uniform(0.36, 0.64, size=(N, 3)), mat, n_grid)
    st = dict(x=P['x'].copy(), v=rng.randn(N, 3) * 0.5, C=rng.randn(N, 3, 3) * 5.0, F=np.eye(3)[None] + rng.randn(N, 3, 3) * 0.02, used=P['used'])
    return P, st


def _oracle_loss(P, st, wts, gravity, boundary, n_sub, static=None, grads=False):
    o = ParamGradOracle(16, P, gravity=gravity, boundary=boundary, precision=64, max_substeps_local=10)
    if static is not None:
        o.add_static(*static, friction=0.3)
    o.set_frame(0, st['x'], st['v'], st['C'], st['F'], st['used'])
    for f in range(n_sub):
        o.substep(f)
    fr = o.get_frame(n_sub)
    loss = sum((wts[k] * fr[k]).sum() for k in ('x', 'v', 'C', 'F'))
    if not grads:
        return loss
    o.reset_grad()
    o.set_grad_frame(n_sub, wts['x'], wts['v'], wts['C'], wts['F'])
    for f in reversed(range(n_sub)):
        o.substep_grad(f)
    return loss, o.get_param_grad()


@pytest.mark.parametrize('mat', [M.WATER, M.ELASTIC, M.ICECREAM, M.MILK_VIS])
@pytest.mark.parametrize('boundary', ['cube', 'cylinder', 'cube+static'])
def test_oracle_parameter_adjoints_match_central_differences(mat, boundary):
    """dL/dmu, dL/dlam, dL/dmass (every particle of the scene perturbed together: one material row) and dL/dgravity after 3 substeps, against
    central differences through the oracle's own forward.  'cube+static': a static SDF box under the cloud, so dL/dg also runs through collide."""
    rng = np.random.RandomState(3)
    P, st = _scene(mat, rng)
    bnd = CYL if boundary == 'cylinder' else CUBE
    static = box_sdf((0.12, 0.02, 0.12), 0.3) if boundary == 'cube+static' else None
    if static is not None:   # centre the box at (0.5, 0.4, 0.5) inside the cloud
        T = static[1].copy(); T[:3, 3] -= T[0, 0] * np.array([0.5, 0.4, 0.5]); static = (static[0], T)
    grav = (0.3, -10.0, -0.2)
    wts = {k: rng.randn(*st[k].shape) for k in ('x', 'v', 'C', 'F')}
    _, g = _oracle_loss(P, st, wts, grav, bnd, 3, static, grads=True)
    an = dict(mu=g['mu'].sum(), lam=g['lam'].sum(), mass=g['mass'].sum())
    for key in ('mu', 'lam', 'mass'):
        h = 1e-6 * (abs(float(P[key][0])) or 1.0)   # relative step (a row's mass is ~1e-4)
        Pp, Pm = dict(P), dict(P)
        Pp[key] = P[key] + h; Pm[key] = P[key] - h
        fd = (_oracle_loss(Pp, st, wts, grav, bnd, 3, static) - _oracle_loss(Pm, st, wts, grav, bnd, 3, static)) / (2 * h)
        assert abs(fd - an[key]) <= 2e-5 * max(1.0, abs(fd), abs(an[key])), (key, fd, an[key])
    for d in range(3):
        h = 1e-5
        gp, gm = list(grav), list(grav)
        gp[d] += h; gm[d] -= h
        fd = (_oracle_loss(P, st, wts, gp, bnd, 3, static) - _oracle_loss(P, st, wts, gm, bnd, 3, static)) / (2 * h)
        assert abs(fd - g['gravity'][d]) <= 2e-5 * max(1.0, abs(fd), abs(g['gravity'][d])), ('gravity', d, fd, g['gravity'][d])
    if mat == M.WATER:   # mu = 0: the reference still takes the SVD, so dL/dmu is defined and non-zero
        assert abs(an['mu']) > 1e-6


def test_oracle_parameter_adjoints_match_torch_autograd():
    """the same adjoints against torch.autograd on substep_torch (tests/test_torch_autodiff_crosscheck.py), with mu, lam, mass and gravity as
    leaves: 4 materials, 3 substeps, per particle"""
    from test_torch_autodiff_crosscheck import substep_torch
    rng = np.random.RandomState(71)
    n_grid, N, n_sub = 16, 160, 3
    lower, upper = (0.32, 0.32, 0.32), (0.68, 0.68, 0.68)
    x0 = rng.uniform(0.36, 0.64, size=(N, 3))
    mats = (M.WATER, M.ELASTIC, M.ICECREAM, M.MILK_VIS)
    P = make_particles(x0, np.array([mats[i % 4] for i in range(N)], dtype=np.int32), n_grid)
    v0 = rng.randn(N, 3) * 0.5; C0 = rng.randn(N, 3, 3) * 5.0; F0 = np.eye(3)[None] + rng.randn(N, 3, 3) * 0.02
    wts = {k: rng.randn(*a.shape) for k, a in (('x', x0), ('v', v0), ('C', C0), ('F', F0))}
    grav = (0.2, -10.0, 0.1)
    _, og = _oracle_loss(P, dict(x=x0, v=v0, C=C0, F=F0, used=P['used']), wts, grav, dict(type='cube', lower=lower, upper=upper), n_sub, grads=True)
    t = lambda a: torch.tensor(np.asarray(a, dtype=np.float64), dtype=torch.float64)
    mu, lam, mass, g = (t(a).requires_grad_(True) for a in (P['mu'], P['lam'], P['mass'], grav))
    s = (t(x0), t(v0), t(C0), t(F0))
    for _ in range(n_sub):
        s = substep_torch(*s, mu, lam, mass, torch.tensor(P['cls']), n_grid, g, t(np.float32(lower)), t(np.float32(upper)))
    loss = sum((t(wts[k]) * a).sum() for k, a in zip(('x', 'v', 'C', 'F'), s))
    tg = dict(zip(('mu', 'lam', 'mass', 'gravity'), (a.numpy() for a in torch.autograd.grad(loss, (mu, lam, mass, g)))))
    for k in ('mu', 'lam', 'mass', 'gravity'):
        err = np.abs(tg[k] - og[k]).max() / max(1.0, np.abs(og[k]).max())
        assert err < 1e-7, (k, err)
    assert np.abs(og['mu'][P['mat'] == M.WATER]).max() > 0, 'dL/dmu of a mu = 0 liquid is defined (the reference takes the SVD of every particle)'


@pytest.fixture
def emu():
    L = harness.enable()
    yield L
    harness.disable()


@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('case', ['water', 'elastic', 'icecream', 'milk_vis', 'mixed'])
def test_param_grad_kernels_match_the_oracle_on_the_emulated_device(emu, case, sort):
    """k_particle_grad<kMat, true> (all-liquid variant with its own SVD for water) and k_grid_op_grad<true>: one backward substep against the fp64
    oracle; the state adjoint is the same with param_grad on and off (tests/param_grad_case.py, also run on an H100)"""
    pgc.substep_case('cpu', case, sort)


@pytest.mark.parametrize('sort_every', [0, 1])
def test_param_grad_latteart_ring_matches_the_oracle_on_the_emulated_device(emu, sort_every):
    pgc.latteart_case('cpu', sort_every)


def test_param_grad_reduction_is_order_independent_under_a_shuffled_schedule():
    """the warp / CTA reductions of the parameter gradients under CUEMU_SCHED=shuffle (another thread order inside every block): a missing
    barrier between the shared-memory partial sums and their reader would change the result"""
    import subprocess
    env = dict(os.environ, CUEMU_SCHED='shuffle')
    r = subprocess.run([sys.executable, '-m', 'pytest', os.path.abspath(__file__), '-q', '-p', 'no:cacheprovider',
                        '-k', 'kernels_match_the_oracle and (mixed or water) or latteart_ring_matches and 0'],
                       capture_output=True, text=True, timeout=1500, env=env, cwd=os.path.dirname(HERE))
    tail = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else ''
    assert r.returncode == 0 and '5 passed' in tail, r.stdout[-3000:] + r.stderr[-1000:]


def test_slab_simulator_rejects_param_grad():
    from fluidlab_b200.slab import SlabMPMSimulator
    s = SlabMPMSimulator.__new__(SlabMPMSimulator)
    assert s.param_grad is False
    with pytest.raises(NotImplementedError, match='single-GPU'):
        s.param_grad = True
    s.param_grad = False


def test_slab_backward_entry_points_refuse_bound_parameter_gradients():
    """fmpm_substep_grad_finish / fmpm_substep_grad_slab with FmpmParamGrad bound: a library error, not a double count of the ghost planes"""
    import ctypes as C
    from fluidlab_b200 import _lib
    L = C.CDLL(harness.build_library())
    for name, (res, args) in _lib._PROTOS.items():
        fn = getattr(L, name); fn.restype = res; fn.argtypes = args
    cfg = _lib.FmpmConfig()
    cfg.n_grid, cfg.n_particles, cfg.max_substeps_local, cfg.n_substeps, cfg.n_materials = 16, 8, 10, 10, 1
    h = C.c_void_p()
    assert L.fmpm_create(C.byref(cfg), C.byref(h)) == 0
    N, G = 8, 16 ** 3
    keep = [np.zeros(n, np.float32) for n in (11 * 4 * N * 4, 11 * 2 * N * 4, 11 * N, 2 * 4 * N * 4, 2 * 2 * N * 4, 2 * N, G * 4, G * 4, G * 4, G * 4, 4)]
    blk = [np.zeros(8, np.int32) for _ in range(3)]
    b = _lib.FmpmBuffers()
    b.pa, b.pf, b.pf8, b.ga, b.gf, b.gf8, b.grid_pm, b.grid_v, b.ggrid_v, b.ggrid_pm, b.materials = [a.ctypes.data for a in keep]
    b.blk_flags, b.blk_list, b.blk_count = [a.ctypes.data for a in blk]
    assert L.fmpm_bind(h, C.byref(b)) == 0
    gmat, ggrav = np.zeros(4), np.zeros(3)
    half = _lib.FmpmParamGrad(); half.gmat = gmat.ctypes.data
    assert L.fmpm_set_param_grad(h, C.byref(half)) != 0 and b'both' in L.fmpm_last_error(h)
    pg = _lib.FmpmParamGrad(); pg.gmat, pg.ggrav = gmat.ctypes.data, ggrav.ctypes.data
    assert L.fmpm_set_param_grad(h, C.byref(pg)) == 0
    for fn in (L.fmpm_substep_grad_finish, L.fmpm_substep_grad_slab):
        assert fn(h, 0, 1, 0, None) != 0 and b'parameter gradients' in L.fmpm_last_error(h)
    assert L.fmpm_set_param_grad(h, None) == 0
    assert L.fmpm_set_scene_flags(h, 1) == 0 and L.fmpm_set_scene_flags(h, 2) != 0
    assert L.fmpm_set_gravity(h, (C.c_float * 3)(0.0, -9.8, 0.0)) == 0
    L.fmpm_destroy(h)


def test_param_grad_struct_matches_the_c_header(tmp_path):
    import ctypes as C
    import subprocess
    from fluidlab_b200 import _lib
    src = tmp_path / 'pg.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fluidmpm.h"\nint main(void) { printf("%zu %zu %zu\\n", sizeof(FmpmParamGrad), '
                   'offsetof(FmpmParamGrad, gmat), offsetof(FmpmParamGrad, ggrav)); return 0; }\n')
    subprocess.check_call(['gcc', '-I', os.path.join(os.path.dirname(HERE), 'include'), str(src), '-o', str(tmp_path / 'pg')])
    out = [int(v) for v in subprocess.run([str(tmp_path / 'pg')], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [C.sizeof(_lib.FmpmParamGrad), _lib.FmpmParamGrad.gmat.offset, _lib.FmpmParamGrad.ggrav.offset]


def test_system_identification_recovers_mu_and_lam_on_the_emulated_device(emu):
    """20 Adam iterations on (log mu, log lam) of an ELASTIC block started 30 % off shrink the parameter error at least 10x (tests/param_grad_case.py)"""
    errs = pgc.sysid_case('cpu')
    assert errs[-1] <= 0.1 * errs[0], errs
