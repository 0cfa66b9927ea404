"""The correspondence-free momentum loss (MomentumMatchingLoss, fmpm_loss_momentum / fmpm_loss_momentum_grad) on CPU: the fp64 reference
against p2g's own (momentum, mass) accumulator, torch.autograd and central differences; the kernels on the execution-model shim against the
reference (also under a shuffled thread schedule); TaichiEnv end to end against the fp64 oracle; the step-end frame of the fused forward
path; host-side validation, the C ABI and the compiler's register allocation."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'cuda_emu'))
import harness  # noqa: E402

import density_loss_ref as dref  # noqa: E402
import momentum_loss_ref as mref  # noqa: E402
import momentum_loss_case as mlc  # noqa: E402
from fluidlab_b200 import macros as M  # noqa: E402
from test_density_loss import check_env_case  # noqa: E402


@pytest.fixture
def emu():
    L = harness.enable()
    yield L
    harness.disable()


def _cloud(seed, N=60, n=8):
    rng = np.random.RandomState(seed)
    x = rng.uniform(0.25, 0.75, size=(N, 3))
    v = rng.randn(N, 3)
    C = 4.0 * rng.randn(N, 3, 3)
    mass = rng.uniform(0.5, 2.0, size=N)
    G = n ** 3
    return x, v, C, mass, rng.rand(G) * 2.0, rng.randn(G, 3), rng.randn(G)


def test_reference_adjoints_match_torch_autograd():
    """x, v, C and m_p adjoints of the reference against autograd on an fp64 torch restatement (stencil base held fixed), 1e-7"""
    n = 8
    x, v, C, mass, tm, tp, sdf = _cloud(0, n=n)
    sel = np.ones(len(x), bool); sel[::7] = False
    wd, ws, wm = 3.0, 0.7, 2.0
    L, gx, gv, gC, dm = mref.adjoint(x, v, C, mass, sel, n, tm, tp, sdf, wd, ws, wm)
    xt, vt, Ct, mt = (torch.tensor(a, requires_grad=True) for a in (x, v, C, mass))
    base = torch.trunc(xt.detach() * n - 0.5)
    fx = xt * n - base
    w1 = torch.stack([0.5 * (1.5 - fx) ** 2, 0.75 - (fx - 1.0) ** 2, 0.5 * (fx - 0.5) ** 2], 1)
    m = torch.zeros(n ** 3, dtype=torch.float64)
    pm = torch.zeros((n ** 3, 3), dtype=torch.float64)
    s = torch.tensor(sel)
    for i in range(3):
        for j in range(3):
            for k in range(3):
                node = ((base[:, 0].long() + i) * n + base[:, 1].long() + j) * n + base[:, 2].long() + k
                mw = mt * w1[:, i, 0] * w1[:, j, 1] * w1[:, k, 2]
                d = (torch.tensor([i, j, k], dtype=torch.float64) - fx) / n
                u = vt + torch.einsum('pab,pb->pa', Ct, d)
                m = m.index_add(0, node[s], mw[s])
                pm = pm.index_add(0, node[s], (mw[:, None] * u)[s])
    t, tpt, phi = torch.tensor(tm), torch.tensor(tp), torch.tensor(sdf)
    Lt = wd * ((m - t) ** 2).sum() + ws * (m * phi).sum() + wm * ((pm - tpt) ** 2).sum()
    ag = torch.autograd.grad(Lt, (xt, vt, Ct, mt))
    assert abs(float(Lt.detach()) - L) <= 1e-12 * abs(L)
    for got, want in zip((gx, gv, gC, dm), ag):
        assert mlc.rel_max(got, want.numpy()) < 1e-7, mlc.rel_max(got, want.numpy())


def test_reference_adjoints_match_central_differences():
    n = 8
    x, v, C, mass, tm, tp, sdf = _cloud(1, n=n)
    sel = np.ones(len(x), bool)
    args = (tm, tp, sdf, 2.0, 0.3, 1.5)
    _, gx, gv, gC, _ = mref.adjoint(x, v, C, mass, sel, n, *args)

    def L(x_, v_, C_):
        pm, m = mref.deposit(x_, v_, C_, mass, sel, n)
        return mref.loss(pm, m, *args)
    h = 1e-6
    for p in (0, 11, 42):
        for d in range(3):
            for arr, grad, idx in ((x, gx, (p, d)), (v, gv, (p, d)), (C, gC, (p, d, (d + 1) % 3))):
                ap, am = arr.copy(), arr.copy()
                ap[idx] += h; am[idx] -= h
                fp = L(*[ap if a is arr else a for a in (x, v, C)])
                fm = L(*[am if a is arr else a for a in (x, v, C)])
                fd = (fp - fm) / (2 * h)
                assert abs(fd - grad[idx]) <= 1e-6 * max(1.0, abs(fd)), (idx, fd, grad[idx])


def test_momentum_from_points_is_the_reference_deposit():
    """the product's host helper (targets from point clouds) deposits like the reference, with and without the APIC term, and refuses bad
    input"""
    from fluidlab_b200 import MomentumMatchingLoss
    n = 16
    rng = np.random.RandomState(2)
    x = rng.uniform(0.0, 1.0, size=(300, 3))   # some points near the faces deposit nothing
    v, C = rng.randn(300, 3), 3.0 * rng.randn(300, 3, 3)
    ok = dref.stencil(x, n)[0]
    for aff in (None, C):
        want_p, want_m = mref.deposit(x, v, np.zeros_like(C) if aff is None else C, 0.25, ok, n)
        got_p, got_m = MomentumMatchingLoss.momentum_from_points(x, v, 0.25, n, affine=aff)
        assert got_p.dtype == np.float32 and got_p.shape == (n ** 3, 3) and got_m.shape == (n ** 3,)
        assert mlc.rel_max(got_p, want_p) < 1e-6 and mlc.rel_max(got_m, want_m) < 1e-6
    with pytest.raises(ValueError, match='shape'):
        MomentumMatchingLoss.momentum_from_points(x, v[:5], 1.0, n)
    with pytest.raises(ValueError, match='affine'):
        MomentumMatchingLoss.momentum_from_points(x, v, 1.0, n, affine=C[:, :2])
    with pytest.raises(ValueError, match='finite'):
        MomentumMatchingLoss.momentum_from_points(x, np.full_like(v, np.nan), 1.0, n)
    with pytest.raises(ValueError, match='non-negative'):
        MomentumMatchingLoss.momentum_from_points(x, v, -1.0, n)


def test_reference_deposit_equals_the_p2g_accumulator_on_the_emulated_device(emu):
    assert mlc.deposit_matches_p2g('cpu') < 1e-6


@pytest.mark.parametrize('case', mlc.KERNEL_CASES)
def test_momentum_kernels_match_the_reference_on_the_emulated_device(emu, case):
    mlc.kernel_case('cpu', case)


def test_momentum_kernels_are_order_independent_under_a_shuffled_schedule():
    """the MATCH.ANY groups and the shared-memory records under CUEMU_SCHED=shuffle: a missing __syncwarp would change the result"""
    env = dict(os.environ, CUEMU_SCHED='shuffle')
    r = subprocess.run([sys.executable, '-m', 'pytest', os.path.abspath(__file__), '-q', '-p', 'no:cacheprovider',
                        '-k', 'momentum_kernels_match_the_reference and (sorted or aged or two_mat or frozen)'],
                       capture_output=True, text=True, timeout=1500, env=env, cwd=os.path.dirname(HERE))
    tail = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else ''
    assert r.returncode == 0 and '5 passed' in tail, r.stdout[-3000:] + r.stderr[-1000:]


def test_momentum_loss_through_taichi_env_matches_the_oracle_on_the_emulated_device(emu):
    """2k ELASTIC particles on 32^3, 3 steps, loss at every step: step losses against the reference on the oracle's states, dL/d(x0, v0, C0, F0)
    against the oracle's backward seeded with the reference's x, v and C adjoints, dL/drho against central differences through the oracle's
    fp64 forward (and without the direct mass term it would not match)"""
    check_env_case(mlc.env_case('cpu'))


def check_fused_frame_case(res):
    (got_f, want_f, cmax_f), (got_s, want_s, cmax_s) = res[False], res[True]
    assert cmax_f > 0.5 and cmax_s > 0.5, 'the scene must exercise the C planes'
    assert abs(got_f - want_f) <= 1e-5 * abs(want_f) and abs(got_s - want_s) <= 1e-5 * abs(want_s), res
    assert abs(got_f - got_s) <= 1e-4 * abs(got_s), res


def test_momentum_loss_reads_the_step_end_frame_of_the_fused_forward_path_on_the_emulated_device(emu):
    check_fused_frame_case(mlc.fused_frame_case('cpu'))


def _loss_env(emu_on, **kw):
    from fluidlab_b200 import TaichiEnv, MomentumMatchingLoss
    from conftest import make_particles
    n = 16
    P = make_particles(np.random.RandomState(0).uniform(0.4, 0.6, size=(50, 3)), M.WATER, n)
    env = TaichiEnv(quality=n / 64, max_substeps_local=20, horizon=2, ckpt_dest='cpu', device='cpu')
    env.simulator.use_graphs = False
    env.particle_bodies.get = lambda: P
    kw.setdefault('weights', {'density': 1.0, 'momentum': 1.0})
    env.setup_loss(loss_cls=MomentumMatchingLoss, matching_mat=M.WATER, temporal_range_type='all', **kw)
    env.build()
    return env


def test_momentum_loss_rejects_bad_targets(emu):
    G = 16 ** 3
    with pytest.raises(ValueError, match='n_grid'):
        _loss_env(emu, target_momentum=np.zeros(G * 3 + 3))
    with pytest.raises(ValueError, match='n_grid'):
        _loss_env(emu, target_momentum=np.zeros((3, G, 3)))         # neither one volume nor max_loss_steps = 2
    with pytest.raises(ValueError, match='n_grid'):
        _loss_env(emu, target_momentum=np.zeros((3, G)))            # components last
    with pytest.raises(ValueError, match='non-finite'):
        _loss_env(emu, target_momentum=np.full((G, 3), np.inf))
    with pytest.raises(ValueError, match='non-finite'):
        _loss_env(emu, target=np.full(G, np.nan))
    with pytest.raises(ValueError, match='non-negative'):
        _loss_env(emu, target=-np.ones((16, 16, 16)))
    with pytest.raises(ValueError, match='finite'):
        _loss_env(emu, weights={'momentum': np.inf})
    env = _loss_env(emu, target=np.ones(G), target_momentum=np.arange(2 * G * 3, dtype=np.float64).reshape(2, G, 3))
    t4 = env.loss.tgt4.cpu().numpy()
    assert t4.shape == (2, G, 4) and (t4[:, :, 3] == 1.0).all() and (t4[1, :, :3].reshape(-1) == np.arange(G * 3, 2 * G * 3)).all()
    env = _loss_env(emu, target_momentum=np.ones((G, 3)))           # m* = 0, one volume for every step
    assert tuple(env.loss.tgt4.shape) == (1, G, 4) and not env.loss.tgt4[:, :, 3].any()
    assert _loss_env(emu).loss.tgt4 is None                        # neither target: the kernels read 0


def test_slab_simulator_refuses_the_momentum_loss():
    from fluidlab_b200.slab import SlabMPMSimulator
    s = SlabMPMSimulator.__new__(SlabMPMSimulator)
    for fn in (s.momentum_loss, s.add_grad_momentum):
        with pytest.raises(NotImplementedError, match='single-GPU'):
            fn(None, None, None, 1.0, 0.0, 1.0, 1, None)


def test_momentum_loss_c_abi_errors_and_struct_layout(tmp_path):
    """error returns (unbound handle, NULL scratch, NULL loss_out, no grad buffers, bad g, frame out of range) and FmpmMomentumLoss as gcc lays
    it out"""
    import ctypes as C
    from fluidlab_b200 import _lib
    L = C.CDLL(harness.build_library())
    for name, (res, args) in _lib._PROTOS.items():
        fn = getattr(L, name); fn.restype = res; fn.argtypes = args
    cfg = _lib.FmpmConfig()
    cfg.n_grid, cfg.n_particles, cfg.max_substeps_local, cfg.n_substeps, cfg.n_materials = 16, 8, 10, 10, 1
    h = C.c_void_p()
    assert L.fmpm_create(C.byref(cfg), C.byref(h)) == 0
    G, N = 16 ** 3, 8
    scratch, out = np.zeros(G * 4, np.float32), np.zeros(1, np.float32)
    l = _lib.FmpmMomentumLoss(); l.field, l.w_density, l.w_momentum, l.mrow_mask_lo = scratch.ctypes.data, 1.0, 1.0, 1
    assert L.fmpm_loss_momentum(h, 0, C.byref(l), out.ctypes.data, None) != 0 and b'fmpm_bind' in L.fmpm_last_error(h)
    keep = [np.zeros(k, np.float32) for k in (11 * 4 * N * 4, 11 * 2 * N * 4, 11 * N, G * 4, G * 4, 4)]
    blk = [np.zeros(8, np.int32) for _ in range(3)]
    b = _lib.FmpmBuffers()
    b.pa, b.pf, b.pf8, b.grid_pm, b.grid_v, b.materials = [a.ctypes.data for a in keep]
    b.blk_flags, b.blk_list, b.blk_count = [a.ctypes.data for a in blk]
    assert L.fmpm_bind(h, C.byref(b)) == 0
    assert L.fmpm_loss_momentum(h, 11, C.byref(l), out.ctypes.data, None) != 0 and b'out of range' in L.fmpm_last_error(h)
    assert L.fmpm_loss_momentum(h, -1, C.byref(l), out.ctypes.data, None) != 0 and b'out of range' in L.fmpm_last_error(h)
    assert L.fmpm_loss_momentum(h, 0, C.byref(l), None, None) != 0 and b'loss_out' in L.fmpm_last_error(h)
    assert L.fmpm_loss_momentum_grad(h, 0, 0, C.byref(l), None) != 0 and b'no grad buffers' in L.fmpm_last_error(h)
    nul = _lib.FmpmMomentumLoss()
    assert L.fmpm_loss_momentum(h, 0, C.byref(nul), out.ctypes.data, None) != 0 and b'scratch' in L.fmpm_last_error(h)
    assert L.fmpm_loss_momentum(h, 0, None, out.ctypes.data, None) != 0
    assert L.fmpm_loss_momentum(h, 0, C.byref(l), out.ctypes.data, None) == 0 and out[0] == 0.0   # no particle used, no target
    g = [np.zeros(k, np.float32) for k in (2 * 4 * N * 4, 2 * 2 * N * 4, 2 * N, G * 4, G * 4)]
    b.ga, b.gf, b.gf8, b.ggrid_v, b.ggrid_pm = [a.ctypes.data for a in g]
    assert L.fmpm_bind(h, C.byref(b)) == 0
    assert L.fmpm_loss_momentum_grad(h, 0, 2, C.byref(l), None) != 0 and b'bad index' in L.fmpm_last_error(h)
    assert L.fmpm_loss_momentum_grad(h, 11, 0, C.byref(l), None) != 0 and b'out of range' in L.fmpm_last_error(h)
    assert L.fmpm_loss_momentum_grad(h, 0, 0, C.byref(nul), None) != 0 and b'scratch' in L.fmpm_last_error(h)
    assert L.fmpm_loss_momentum_grad(h, 0, 1, C.byref(l), None) == 0
    L.fmpm_destroy(h)
    src = tmp_path / 'ml.c'
    fields = [f for f, _ in _lib.FmpmMomentumLoss._fields_]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fluidmpm.h"\nint main(void) { printf("%zu", sizeof(FmpmMomentumLoss)); '
                   + ' '.join(f'printf(" %zu", offsetof(FmpmMomentumLoss, {f}));' for f in fields) + ' printf("\\n"); return 0; }\n')
    subprocess.check_call(['gcc', '-I', os.path.join(os.path.dirname(HERE), 'include'), str(src), '-o', str(tmp_path / 'ml')])
    got = [int(v) for v in subprocess.run([str(tmp_path / 'ml')], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(_lib.FmpmMomentumLoss)] + [getattr(_lib.FmpmMomentumLoss, f).offset for f in fields]


def test_momentum_kernels_do_not_spill(tmp_path):
    """every instantiation of the new kernels, compiled with the library's own flags for sm_90a: no spill stores or loads (needs nvcc)"""
    from test_sass_budget import BUILD, CSRC, _nvcc
    if _nvcc() is None:
        pytest.skip('nvcc not found')
    cmd = [_nvcc()] + BUILD.FLAGS + ['-Xptxas', '-v', '-cubin', os.path.join(CSRC, 'fmpm_io.cu'), '-o', str(tmp_path / 'io.cubin')]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    spills, name = {}, None
    for line in (r.stdout + r.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m and name is not None and 'k_loss_momentum' in name:
            spills[name] = (int(m.group(1)), int(m.group(2)))
            name = None
    assert len(spills) == 5, sorted(spills)   # the deposit, node<false / true>, grad<false / true>
    assert all(v == (0, 0) for v in spills.values()), spills
