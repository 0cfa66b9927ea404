"""The correspondence-free density loss (DensityMatchingLoss, fmpm_loss_density / fmpm_loss_density_grad) on CPU: the fp64 reference against
p2g's own grid mass, torch.autograd and central differences; the kernels on the execution-model shim against the reference (also under a
shuffled thread schedule); TaichiEnv end to end against the fp64 oracle; host-side validation and the C ABI."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'cuda_emu'))
import harness  # noqa: E402

import density_loss_ref as dref  # noqa: E402
import density_loss_case as dlc  # noqa: E402
from fluidlab_b200 import macros as M  # noqa: E402


@pytest.fixture
def emu():
    L = harness.enable()
    yield L
    harness.disable()


def _cloud(seed, N=60, n=8):
    rng = np.random.RandomState(seed)
    x = rng.uniform(0.25, 0.75, size=(N, 3))
    mass = rng.uniform(0.5, 2.0, size=N)
    tgt = rng.rand(n ** 3) * 2.0
    sdf = rng.randn(n ** 3)
    return x, mass, tgt, sdf


def test_reference_adjoints_match_torch_autograd():
    """x adjoint and dL/dm_p of the reference against autograd on an fp64 torch restatement (stencil base held fixed), 1e-10"""
    n = 8
    x, mass, tgt, sdf = _cloud(0, n=n)
    sel = np.ones(len(x), bool); sel[::7] = False
    L, gx, dm = dref.adjoint(x, mass, sel, n, tgt, sdf, 3.0, 0.7)
    xt = torch.tensor(x, requires_grad=True); mt = torch.tensor(mass, requires_grad=True)
    base = torch.trunc(xt.detach() * n - 0.5)
    fx = xt * n - base
    w1 = torch.stack([0.5 * (1.5 - fx) ** 2, 0.75 - (fx - 1.0) ** 2, 0.5 * (fx - 0.5) ** 2], 1)
    m = torch.zeros(n ** 3, dtype=torch.float64)
    s = torch.tensor(sel)
    for i in range(3):
        for j in range(3):
            for k in range(3):
                node = ((base[:, 0].long() + i) * n + base[:, 1].long() + j) * n + base[:, 2].long() + k
                m = m.index_add(0, node[s], (mt * w1[:, i, 0] * w1[:, j, 1] * w1[:, k, 2])[s])
    t, phi = torch.tensor(tgt), torch.tensor(sdf)
    Lt = 3.0 * ((m - t) ** 2).sum() + 0.7 * (m * phi).sum()
    agx, adm = torch.autograd.grad(Lt, (xt, mt))
    assert abs(float(Lt.detach()) - L) <= 1e-12 * abs(L)
    assert dlc.rel_max(gx, agx.numpy()) < 1e-10 and dlc.rel_max(dm, adm.numpy()) < 1e-10


def test_reference_x_adjoint_matches_central_differences():
    n = 8
    x, mass, tgt, sdf = _cloud(1, n=n)
    sel = np.ones(len(x), bool)
    _, gx, _ = dref.adjoint(x, mass, sel, n, tgt, sdf, 2.0, 0.3)
    h = 1e-6
    for p in (0, 11, 42):
        for d in range(3):
            xp, xm = x.copy(), x.copy()
            xp[p, d] += h; xm[p, d] -= h
            fd = (dref.loss(dref.deposit(xp, mass, sel, n), tgt, sdf, 2.0, 0.3) - dref.loss(dref.deposit(xm, mass, sel, n), tgt, sdf, 2.0, 0.3)) / (2 * h)
            assert abs(fd - gx[p, d]) <= 1e-6 * max(1.0, abs(fd)), (p, d, fd, gx[p, d])


def test_density_from_points_is_the_reference_deposit():
    """the product's host helper (targets from point clouds) deposits like the reference, and refuses bad input"""
    from fluidlab_b200 import DensityMatchingLoss
    n = 16
    x = np.random.RandomState(2).uniform(0.0, 1.0, size=(300, 3))   # some points near the faces deposit nothing
    want = dref.deposit(x, 0.25, dref.stencil(x, n)[0], n)
    got = DensityMatchingLoss.density_from_points(x, 0.25, n)
    assert got.dtype == np.float32 and got.shape == (n ** 3,) and dlc.rel_max(got, want) < 1e-6
    with pytest.raises(ValueError, match='finite'):
        DensityMatchingLoss.density_from_points(np.full((2, 3), np.nan), 1.0, n)
    with pytest.raises(ValueError, match='non-negative'):
        DensityMatchingLoss.density_from_points(x, -1.0, n)


def test_reference_deposit_equals_the_p2g_grid_mass_on_the_emulated_device(emu):
    assert dlc.deposit_matches_p2g('cpu') < 1e-6


@pytest.mark.parametrize('case', dlc.KERNEL_CASES)
def test_density_kernels_match_the_reference_on_the_emulated_device(emu, case):
    dlc.kernel_case('cpu', case)


def test_density_kernels_are_order_independent_under_a_shuffled_schedule():
    """the MATCH.ANY groups, the pointer-jumping reduction and the shared-memory hand-off under CUEMU_SCHED=shuffle: a missing __syncwarp would
    change the result"""
    import subprocess
    env = dict(os.environ, CUEMU_SCHED='shuffle')
    r = subprocess.run([sys.executable, '-m', 'pytest', os.path.abspath(__file__), '-q', '-p', 'no:cacheprovider',
                        '-k', 'density_kernels_match_the_reference and (sorted or aged or two_mat or frozen)'],
                       capture_output=True, text=True, timeout=1500, env=env, cwd=os.path.dirname(HERE))
    tail = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else ''
    assert r.returncode == 0 and '5 passed' in tail, r.stdout[-3000:] + r.stderr[-1000:]


def check_env_case(r):
    assert np.all(np.abs(r['got_losses'] - r['want_losses']) <= 1e-4 * np.abs(r['want_losses'])), (r['got_losses'], r['want_losses'])
    for k in 'xvCF':
        assert dlc.rel_max(r['got_g'][k], r['want_g'][k]) < 1e-4, (k, dlc.rel_max(r['got_g'][k], r['want_g'][k]))
    fd, an, direct = r['fd_rho'], r['got_rho'], r['direct_rho']
    assert abs(an - fd) <= 2e-3 * abs(fd), (an, fd)
    assert abs(an - direct - fd) > 10 * 2e-3 * abs(fd), ('the direct mass term of the deposit matters here', an, direct, fd)


def test_density_loss_through_taichi_env_matches_the_oracle_on_the_emulated_device(emu):
    """2k ELASTIC particles on 32^3, 3 steps, loss at every step: step losses against the reference on the oracle's states, dL/d(x0, v0, C0, F0)
    against the oracle's backward seeded with the reference's x adjoint, dL/drho against central differences through the oracle's fp64 forward
    (and without the direct mass term it would not match)"""
    check_env_case(dlc.env_case('cpu'))


def _loss_env(emu_on, **kw):
    from fluidlab_b200 import TaichiEnv, DensityMatchingLoss
    from conftest import make_particles
    n = 16
    P = make_particles(np.random.RandomState(0).uniform(0.4, 0.6, size=(50, 3)), M.WATER, n)
    env = TaichiEnv(quality=n / 64, max_substeps_local=20, horizon=2, ckpt_dest='cpu', device='cpu')
    env.simulator.use_graphs = False
    env.particle_bodies.get = lambda: P
    env.setup_loss(loss_cls=DensityMatchingLoss, matching_mat=M.WATER, weights={'density': 1.0}, temporal_range_type='all', **kw)
    env.build()
    return env


def test_density_loss_rejects_bad_targets(emu):
    G = 16 ** 3
    with pytest.raises(ValueError, match='n_grid'):
        _loss_env(emu, target=np.zeros(G + 1))
    with pytest.raises(ValueError, match='n_grid'):
        _loss_env(emu, target=np.zeros((3, G)))                  # neither one volume nor max_loss_steps = 2
    with pytest.raises(ValueError, match='non-finite'):
        _loss_env(emu, target=np.full(G, np.inf))
    with pytest.raises(ValueError, match='non-finite'):
        _loss_env(emu, target=np.zeros(G), target_sdf=np.full((2, 16, 16, 16), np.nan))
    with pytest.raises(ValueError, match='non-negative'):
        _loss_env(emu, target=-np.ones((16, 16, 16)))
    env = _loss_env(emu, target=np.zeros((2, 16, 16, 16)), target_sdf=np.zeros(G))   # a recording and one SDF for every step
    assert tuple(env.loss.tgt.shape) == (2, G) and tuple(env.loss.sdf.shape) == (1, G)


def test_slab_simulator_refuses_the_density_loss():
    from fluidlab_b200.slab import SlabMPMSimulator
    s = SlabMPMSimulator.__new__(SlabMPMSimulator)
    for fn in (s.density_loss, s.add_x_grad_density):
        with pytest.raises(NotImplementedError, match='single-GPU'):
            fn(None, None, None, 1.0, 0.0, 1, None)


def test_density_loss_c_abi_errors_and_struct_layout(tmp_path):
    """error returns (unbound handle, NULL scratch, no grad buffers, bad g, frame out of range) and FmpmDensityLoss as gcc lays it out"""
    import ctypes as C
    import subprocess
    from fluidlab_b200 import _lib
    L = C.CDLL(harness.build_library())
    for name, (res, args) in _lib._PROTOS.items():
        fn = getattr(L, name); fn.restype = res; fn.argtypes = args
    cfg = _lib.FmpmConfig()
    cfg.n_grid, cfg.n_particles, cfg.max_substeps_local, cfg.n_substeps, cfg.n_materials = 16, 8, 10, 10, 1
    h = C.c_void_p()
    assert L.fmpm_create(C.byref(cfg), C.byref(h)) == 0
    G, N = 16 ** 3, 8
    scratch, out = np.zeros(G, np.float32), np.zeros(1, np.float32)
    l = _lib.FmpmDensityLoss(); l.mass, l.w_density, l.mrow_mask_lo = scratch.ctypes.data, 1.0, 1
    assert L.fmpm_loss_density(h, 0, C.byref(l), out.ctypes.data, None) != 0 and b'fmpm_bind' in L.fmpm_last_error(h)
    keep = [np.zeros(k, np.float32) for k in (11 * 4 * N * 4, 11 * 2 * N * 4, 11 * N, G * 4, G * 4, 4)]
    blk = [np.zeros(8, np.int32) for _ in range(3)]
    b = _lib.FmpmBuffers()
    b.pa, b.pf, b.pf8, b.grid_pm, b.grid_v, b.materials = [a.ctypes.data for a in keep]
    b.blk_flags, b.blk_list, b.blk_count = [a.ctypes.data for a in blk]
    assert L.fmpm_bind(h, C.byref(b)) == 0
    assert L.fmpm_loss_density(h, 11, C.byref(l), out.ctypes.data, None) != 0 and b'out of range' in L.fmpm_last_error(h)
    assert L.fmpm_loss_density_grad(h, 0, 0, C.byref(l), None) != 0 and b'no grad buffers' in L.fmpm_last_error(h)
    nul = _lib.FmpmDensityLoss()
    assert L.fmpm_loss_density(h, 0, C.byref(nul), out.ctypes.data, None) != 0 and b'scratch' in L.fmpm_last_error(h)
    assert L.fmpm_loss_density(h, 0, None, out.ctypes.data, None) != 0
    assert L.fmpm_loss_density(h, 0, C.byref(l), out.ctypes.data, None) == 0 and out[0] == 0.0   # no particle used, no target
    g = [np.zeros(k, np.float32) for k in (2 * 4 * N * 4, 2 * 2 * N * 4, 2 * N, G * 4, G * 4)]
    b.ga, b.gf, b.gf8, b.ggrid_v, b.ggrid_pm = [a.ctypes.data for a in g]
    assert L.fmpm_bind(h, C.byref(b)) == 0
    assert L.fmpm_loss_density_grad(h, 0, 2, C.byref(l), None) != 0 and b'bad index' in L.fmpm_last_error(h)
    assert L.fmpm_loss_density_grad(h, 0, 1, C.byref(l), None) == 0
    L.fmpm_destroy(h)
    src = tmp_path / 'dl.c'
    fields = [f for f, _ in _lib.FmpmDensityLoss._fields_]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fluidmpm.h"\nint main(void) { printf("%zu", sizeof(FmpmDensityLoss)); '
                   + ' '.join(f'printf(" %zu", offsetof(FmpmDensityLoss, {f}));' for f in fields) + ' printf("\\n"); return 0; }\n')
    subprocess.check_call(['gcc', '-I', os.path.join(os.path.dirname(HERE), 'include'), str(src), '-o', str(tmp_path / 'dl')])
    got = [int(v) for v in subprocess.run([str(tmp_path / 'dl')], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(_lib.FmpmDensityLoss)] + [getattr(_lib.FmpmDensityLoss, f).offset for f in fields]
