"""Per-particle mu and lam (MPMSimulator.set_material_field, fmpm_set_material_field) on CPU: the CUDA kernels on the execution-model shim against
the fp64 oracle (which takes mu and lam per particle) and against central differences of its forward, the refusals, the C ABI and, with nvcc,
the compile-time budget of the field's k_fwd instantiation."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, 'cuda_emu'))
import harness  # noqa: E402

import material_field_case as mfc  # noqa: E402


@pytest.fixture
def emu():
    L = harness.enable()
    yield L
    harness.disable()


@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('case', ['elastic', 'mixed'])
def test_field_equal_to_the_table_reproduces_the_table_run(emu, case, sort):
    mfc.field_equals_table_case('cpu', case, sort)


@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('case', ['elastic', 'icecream', 'milk_vis', 'mixed', 'mixed-mu0'])
def test_heterogeneous_field_matches_the_oracle_on_the_emulated_device(emu, case, sort):
    """k_p2g_field / k_particle_grad<2, *>: one step forward and one backward substep with random per-particle (mu, lam); 'mixed-mu0' also has
    particles with mu_p = 0 (they still take the SVD that dL/dmu needs)"""
    mfc.heterogeneous_case('cpu', case.replace('-mu0', ''), sort, zero_frac=0.2 if case.endswith('mu0') else 0.0)


@pytest.mark.parametrize('sort_every', [0, 1])
def test_field_gradients_across_sort_epochs_and_the_checkpoint_ring(emu, sort_every):
    mfc.ring_case('cpu', sort_every)


def test_field_gradients_match_central_differences_of_the_oracle(emu):
    mfc.central_difference_case('cpu')


def test_fused_forward_with_a_field_matches_the_oracle(emu):
    """k_fwd<2, false, false> (the forward hot kernel with a field) on the fused forward-only path: two steps against the fp64 oracle and the
    per-substep path"""
    mfc.fused_forward_case('cpu')


def test_fused_stored_grad_path_with_a_field_matches_the_oracle(emu):
    """grad mode on the fused stored-grid path (k_g2p2g_field<true, false>), one backward substep against the fp64 oracle"""
    mfc.heterogeneous_case('cpu', 'mixed', True, fuse=True)


@pytest.mark.parametrize('fuse', [True, False], ids=['fused', 'per-substep'])
def test_injector_with_a_field_matches_the_oracle(emu, fuse):
    """an AgentInjector scene with a field on both liquids: k_p2g_injected_field (fused) and the per-substep kernels over a T = 20 ring"""
    mfc.injector_case('cpu', fuse)


def test_identification_recovers_a_stiff_core_on_the_emulated_device(emu):
    """20 Adam iterations on the per-particle log stiffness scale (started at 2 everywhere; truth 4 in the core, 1 in the shell): the field error
    drops at least 1.5x (measured 1.9x and 1.8x for two seeds), the core's mean rises above 3 and the shell's falls below 1.5"""
    hist = mfc.identification_case('cpu')
    (e0, _, _), (e1, core, shell) = hist[0], hist[-1]
    assert e1 <= e0 / 1.5 and core >= 3.0 and shell <= 1.5, hist


def test_field_kernels_are_order_independent_under_a_shuffled_schedule():
    """the heterogeneous cases under CUEMU_SCHED=shuffle (another thread order inside every block)"""
    env = dict(os.environ, CUEMU_SCHED='shuffle')
    r = subprocess.run([sys.executable, '-m', 'pytest', os.path.abspath(__file__), '-q', '-p', 'no:cacheprovider', '-k', 'heterogeneous and mixed'],
                       capture_output=True, text=True, timeout=1500, env=env, cwd=ROOT)
    tail = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else ''
    assert r.returncode == 0 and '4 passed' in tail, r.stdout[-3000:] + r.stderr[-1000:]


def test_set_material_field_validates_its_arguments(emu):
    import torch
    _, P, st, _ = mfc._scene('elastic', N=64)
    s = mfc._sim('cpu', P, 16, False)
    N = len(P['mu'])
    with pytest.raises(ValueError, match='shape'):
        s.set_material_field(P['mu'][:-1], P['lam'][:-1])
    with pytest.raises(ValueError, match='finite'):
        s.set_material_field(np.full(N, np.nan), P['lam'])
    with pytest.raises(ValueError, match='>= 0'):
        s.set_material_field(-P['mu'], P['lam'])
    assert s.get_material_field() is None
    s.set_material_field(torch.tensor(P['mu']), torch.tensor(P['lam'], dtype=torch.float32))
    mu, lam = s.get_material_field()
    np.testing.assert_array_equal(mu, P['mu'].astype(np.float32))
    s.clear_material_field()
    assert s.get_material_field() is None


def test_clearing_the_field_keeps_its_gradient_in_the_row_keys(emu):
    """clear_material_field between the backward pass and get_param_grad: dL/dmu, dL/dlam of the field stay in the row keys (their row sums)"""
    rng, P, st, seed_g = mfc._scene('mixed')
    s = mfc._sim('cpu', P, 16, True)
    mfc._run_one_substep_grad(s, st, seed_g, mfc.random_field(P, rng))
    bound = s.get_param_grad()
    s.clear_material_field()
    cleared = s.get_param_grad()
    assert 'mu_field' not in cleared and np.abs(bound['mu']).max() > 0
    for k in ('mu', 'lam', 'rho'):
        np.testing.assert_allclose(cleared[k], bound[k], rtol=1e-12, atol=0)


def test_all_liquid_scene_runs_the_general_kernels_with_a_field(emu):
    """a WATER scene has the all-liquid flag; binding a field drops it (the field's mu applies), clearing the field restores it"""
    from fluidlab_b200 import macros as M
    from conftest import make_particles
    rng = np.random.RandomState(2)
    P = make_particles(rng.uniform(0.4, 0.6, (64, 3)), M.WATER, 16)
    s = mfc._sim('cpu', P, 16, False)
    L, h = s._lib, s._h
    assert L.fmpm_fwd_path(h) & 2
    s.set_material_field(np.full(64, 50.0), P['lam'])
    assert not L.fmpm_fwd_path(h) & 2
    assert L.fmpm_set_scene_flags(h, 1) != 0 and b'material field' in L.fmpm_last_error(h)
    s.clear_material_field()
    assert L.fmpm_fwd_path(h) & 2


def test_slab_simulator_refuses_a_field():
    from fluidlab_b200.slab import SlabMPMSimulator
    s = SlabMPMSimulator.__new__(SlabMPMSimulator)
    with pytest.raises(NotImplementedError, match='single-GPU'):
        s.set_material_field(np.zeros(4), np.zeros(4))


def _bare_handle(L, N=8, n=16):
    from fluidlab_b200 import _lib
    cfg = _lib.FmpmConfig()
    cfg.n_grid, cfg.n_particles, cfg.max_substeps_local, cfg.n_substeps, cfg.n_materials = n, N, 10, 10, 1
    h = C.c_void_p()
    assert L.fmpm_create(C.byref(cfg), C.byref(h)) == 0
    G = n ** 3
    keep = [np.zeros(k, np.float32) for k in (11 * 4 * N * 4, 11 * 2 * N * 4, 11 * N, 2 * 4 * N * 4, 2 * 2 * N * 4, 2 * N, G * 4, G * 4, G * 4, G * 4, 4)]
    keep += [np.zeros(8, np.int32) for _ in range(3)] + [np.zeros((3, G, 4), np.float32), np.zeros((3, 8), np.int32)]
    b = _lib.FmpmBuffers()
    b.pa, b.pf, b.pf8, b.ga, b.gf, b.gf8, b.grid_pm, b.grid_v, b.ggrid_v, b.ggrid_pm, b.materials = [a.ctypes.data for a in keep[:11]]
    b.blk_flags, b.blk_list, b.blk_count = [a.ctypes.data for a in keep[11:14]]
    b.grid_pm3, b.blk_flags3 = keep[14].ctypes.data, keep[15].ctypes.data
    assert L.fmpm_bind(h, C.byref(b)) == 0
    return h, keep


def test_library_refusals_with_a_bound_field():
    """all-liquid flag, x-slab mode (both orders), the in-kernel grid_op and parameter gradients without gfield: library errors"""
    from fluidlab_b200 import _lib
    L = C.CDLL(harness.build_library())
    for name, (res, args) in _lib._PROTOS.items():
        fn = getattr(L, name); fn.restype = res; fn.argtypes = args
    h, keep = _bare_handle(L)
    fld, gfld = np.zeros(16, np.float32), np.zeros(16, np.float32)
    mf = _lib.FmpmMaterialField(); mf.field = fld.ctypes.data
    assert L.fmpm_set_scene_flags(h, 1) == 0
    assert L.fmpm_set_material_field(h, C.byref(mf)) != 0 and b'ALL_LIQUID' in L.fmpm_last_error(h)
    assert L.fmpm_set_scene_flags(h, 0) == 0
    sl = _lib.FmpmSlab(); sl.enabled = 1
    assert L.fmpm_set_slab(h, C.byref(sl)) == 0
    assert L.fmpm_set_material_field(h, C.byref(mf)) != 0 and b'x-slab' in L.fmpm_last_error(h)
    sl.enabled = 0
    assert L.fmpm_set_slab(h, C.byref(sl)) == 0
    assert L.fmpm_set_material_field(h, C.byref(mf)) == 0
    sl.enabled = 1
    assert L.fmpm_set_slab(h, C.byref(sl)) != 0 and b'material field' in L.fmpm_last_error(h)
    assert L.fmpm_set_scene_flags(h, 1) != 0
    assert L.fmpm_set_fwd_mask(h, 7) == 0
    assert L.fmpm_substeps_fused(h, 0, 2, None) != 0 and b'grid_op' in L.fmpm_last_error(h)
    assert L.fmpm_set_fwd_mask(h, ~4) == 0
    gmat, ggrav = np.zeros(4), np.zeros(3)
    pg = _lib.FmpmParamGrad(); pg.gmat, pg.ggrav = gmat.ctypes.data, ggrav.ctypes.data
    assert L.fmpm_set_param_grad(h, C.byref(pg)) == 0
    assert L.fmpm_substep_grad(h, 0, 1, 0, None) != 0 and b'gfield' in L.fmpm_last_error(h)
    mf.gfield = gfld.ctypes.data
    assert L.fmpm_set_material_field(h, C.byref(mf)) == 0
    assert L.fmpm_set_material_field(h, None) == 0
    assert L.fmpm_set_scene_flags(h, 1) == 0
    L.fmpm_destroy(h)


def test_material_field_struct_matches_the_c_header(tmp_path):
    from fluidlab_b200 import _lib
    src = tmp_path / 'mf.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fluidmpm.h"\nint main(void) { printf("%zu %zu %zu\\n", sizeof(FmpmMaterialField), '
                   'offsetof(FmpmMaterialField, field), offsetof(FmpmMaterialField, gfield)); return 0; }\n')
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(tmp_path / 'mf')])
    out = [int(v) for v in subprocess.run([str(tmp_path / 'mf')], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [C.sizeof(_lib.FmpmMaterialField), _lib.FmpmMaterialField.field.offset, _lib.FmpmMaterialField.gfield.offset]


def test_set_material_field_is_exported():
    from fluidlab_b200 import _lib
    assert 'fmpm_set_material_field' in _lib.EXPORTS
    nm = subprocess.run(['nm', '-D', '--defined-only', harness.build_library()], capture_output=True, text=True, check=True).stdout
    assert re.search(r'\bT fmpm_set_material_field\b', nm)


def test_field_k_fwd_does_not_spill(tmp_path):
    """k_fwd<2, false, false> (the forward hot kernel with a field) meets the bar of k_fwd<0, false, *>: no spills (CUDA 12.9, sm_90a)"""
    import test_sass_budget as sb
    if sb._nvcc() is None:
        pytest.skip('nvcc not found')
    spills = sb._spills('fmpm_forward.cu', str(tmp_path))
    assert spills['k_fwd<2, false, false>'] == (0, 0), spills['k_fwd<2, false, false>']
