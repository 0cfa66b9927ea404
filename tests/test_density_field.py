"""Per-particle density (MPMSimulator.set_density_field, fmpm_set_mass_field) on CPU: the CUDA kernels on the execution-model shim against the
fp64 oracle (which takes a mass per particle), against central differences of its forward and against the loss references, the host semantics,
the refusals, the C ABI and, with nvcc, the compile-time budget of the mass field's k_fwd instantiation."""
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

import density_field_case as dfc  # noqa: E402
import material_field_case as mfc  # noqa: E402


@pytest.fixture
def emu():
    L = harness.enable()
    yield L
    harness.disable()


@pytest.mark.parametrize('with_field', [False, True], ids=['rho', 'rho+mu-lam'])
@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('case', ['elastic', 'mixed'])
def test_density_field_equal_to_the_rows_reproduces_the_table_run(emu, case, sort, with_field):
    dfc.equals_table_case('cpu', case, sort, with_field)


@pytest.mark.parametrize('with_field', [False, True], ids=['rho', 'rho+mu-lam'])
@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('case', ['elastic', 'icecream', 'milk_vis', 'water', 'mixed'])
def test_heterogeneous_density_matches_the_oracle_on_the_emulated_device(emu, case, sort, with_field):
    """k_p2g_field_mass / k_particle_grad<3, *>: one step forward and one backward substep with a random per-particle rho"""
    dfc.heterogeneous_case('cpu', case, sort, with_field)


@pytest.mark.parametrize('sort_every', [0, 1])
def test_density_gradients_across_sort_epochs_and_the_checkpoint_ring(emu, sort_every):
    dfc.ring_case('cpu', sort_every)


def test_density_gradients_match_central_differences_of_the_oracle(emu):
    dfc.central_difference_case('cpu')


def test_fused_forward_with_a_density_field_matches_the_oracle(emu):
    """k_fwd<3, false, false> on the fused forward-only path: two steps against the fp64 oracle and the per-substep path"""
    dfc.fused_forward_case('cpu')


def test_fused_stored_grad_path_with_a_density_field_matches_the_oracle(emu):
    """grad mode on the fused stored-grid path (k_g2p2g_field_mass<true, false>), one backward substep against the fp64 oracle"""
    dfc.heterogeneous_case('cpu', 'mixed', True, with_field=True, fuse=True)


@pytest.mark.parametrize('fuse', [True, False], ids=['fused', 'per-substep'])
def test_injector_with_a_density_field_matches_the_oracle(emu, fuse):
    dfc.injector_case('cpu', fuse)


def test_rigid_bodies_with_a_density_field_match_the_oracle(emu):
    """k_p2g_rigid_field_mass: a MAT_RIGID cube among water and an elastic blob, all with random rho, on the fused stored-grid path"""
    dfc.rigid_case('cpu')


def test_loss_kernels_with_a_density_field_match_the_references(emu):
    """the density and momentum loss deposits and adjoints (k_loss_mfield_*) and their direct per-particle dL/drho"""
    dfc.loss_kernel_case('cpu')


def test_density_loss_env_gradient_matches_central_differences(emu):
    """TaichiEnv + DensityMatchingLoss over 3 steps: dL/drho_p against central differences of the fp64 pipeline (needs the direct term)"""
    dfc.env_case('cpu')


def test_identification_recovers_a_dense_core_on_the_emulated_device(emu):
    """20 Adam iterations on the per-particle log density from the per-step grid mass of a block with a 3x dense core, started uniform at the
    block's mean density: the field error drops at least 1.2x (measured 1.28x on the shim) and the core's mean ends
    at least 1.5x the shell's (truth 3x; 2.0x measured)"""
    hist = dfc.identification_case('cpu')
    (e0, _, _), (e1, core, shell) = hist[0], hist[-1]
    assert e1 <= e0 / 1.2 and core > 1.5 * shell, hist


def test_density_field_kernels_are_order_independent_under_a_shuffled_schedule():
    """the heterogeneous mixed cases under CUEMU_SCHED=shuffle (another thread order inside every block)"""
    env = dict(os.environ, CUEMU_SCHED='shuffle')
    r = subprocess.run([sys.executable, '-m', 'pytest', os.path.abspath(__file__), '-q', '-p', 'no:cacheprovider', '-k',
                        '(heterogeneous and mixed) or loss_kernels'], capture_output=True, text=True, timeout=1500, env=env, cwd=ROOT)
    tail = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else ''
    assert r.returncode == 0 and '5 passed' in tail, r.stdout[-3000:] + r.stderr[-1000:]


def test_set_density_field_validates_its_arguments(emu):
    import torch
    _, P, _, _ = dfc._scene('elastic', N=64)
    s = mfc._sim('cpu', P, 16, False)
    N = len(P['rho'])
    with pytest.raises(ValueError, match='shape'):
        s.set_density_field(P['rho'][:-1])
    with pytest.raises(ValueError, match='finite'):
        s.set_density_field(np.full(N, np.inf))
    with pytest.raises(ValueError, match='> 0'):
        s.set_density_field(np.zeros(N))
    with pytest.raises(ValueError, match='> 0'):
        s.set_density_field(-np.asarray(P['rho']))
    for v, what in ((1e-46, '> 0'), (1e-44, '> 0'), (1e39, 'finite')):   # finite and > 0 in float64, not rho or p_vol * rho in float32
        with pytest.raises(ValueError, match=what):
            s.set_density_field(np.full(N, v))
    assert s.get_density_field() is None
    s.set_density_field(torch.tensor(P['rho'], dtype=torch.float64))
    np.testing.assert_array_equal(s.get_density_field(), np.asarray(P['rho'], np.float32))
    assert s.get_material_field() is None, 'the private (mu, lam) field stays invisible'
    s.clear_density_field()
    assert s.get_density_field() is None and not s._lib.fmpm_set_material_field(s._h, None)


def test_row_mu_with_only_a_density_field_equals_a_table_run(emu):
    """set_material_table(mu=...) while only rho is bound regathers the private field: the run equals a plain table run with that mu"""
    rng, P, st, seed_g = dfc._scene('elastic')
    res = []
    for use_rho in (True, False):
        s = mfc._sim('cpu', P, 16, True)
        if use_rho:
            s.set_density_field(P['rho'])
        t = s.get_material_table()
        s.set_material_table(mu=t['mu'] * 3.0, lam=t['lam'] * 0.5)
        res.append(mfc._run_one_substep_grad(s, st, seed_g))
    (fa, ga, pa), (fb, gb, pb) = res
    for k in ('x', 'v', 'C', 'F'):
        assert dfc.rel(fa[k], fb[k]) < 1e-5, k
    for k in ('mu', 'lam', 'rho'):
        assert dfc.rel(pa[k], pb[k]) < 1e-3, k
    assert 'mu_field' not in pa


def test_clearing_keeps_the_gradients_in_the_row_keys(emu):
    """clear_material_field with rho still bound falls back to the private field, and clear_density_field then leaves dL/drho to the rows:
    the row keys stay as they were while both fields were bound"""
    rng, P, st, seed_g = dfc._scene('mixed')
    s = mfc._sim('cpu', P, 16, True)
    s.set_material_field(*mfc.random_field(P, rng))
    s.set_density_field(dfc.random_rho(P, rng))
    mfc._run_one_substep_grad(s, st, seed_g)
    bound = s.get_param_grad()
    s.clear_material_field()
    mid = s.get_param_grad()
    assert 'mu_field' not in mid and 'rho_field' in mid and s.get_material_field() is None
    np.testing.assert_allclose(mid['rho_field'], bound['rho_field'], rtol=0, atol=0)
    s.clear_density_field()
    cleared = s.get_param_grad()
    assert 'rho_field' not in cleared and np.abs(bound['rho']).max() > 0
    for k in ('mu', 'lam', 'rho'):
        np.testing.assert_allclose(mid[k], bound[k], rtol=1e-12, atol=0)
        np.testing.assert_allclose(cleared[k], bound[k], rtol=1e-12, atol=0)
    assert not s._lib.fmpm_fwd_path(s._h) & 2


def test_all_liquid_scene_runs_the_general_kernels_with_a_density_field(emu):
    from fluidlab_b200 import macros as M
    from conftest import make_particles
    rng = np.random.RandomState(2)
    P = make_particles(rng.uniform(0.4, 0.6, (64, 3)), M.WATER, 16)
    s = mfc._sim('cpu', P, 16, False)
    L, h = s._lib, s._h
    assert L.fmpm_fwd_path(h) & 2
    s.set_density_field(np.full(64, 2000.0))
    assert not L.fmpm_fwd_path(h) & 2
    s.set_material_field(np.zeros(64), P['lam'])
    s.clear_density_field()
    assert not L.fmpm_fwd_path(h) & 2 and s.get_material_field() is not None
    s.clear_material_field()
    assert L.fmpm_fwd_path(h) & 2


def test_slab_simulator_refuses_a_density_field():
    from fluidlab_b200.slab import SlabMPMSimulator
    s = SlabMPMSimulator.__new__(SlabMPMSimulator)
    with pytest.raises(NotImplementedError, match='single-GPU'):
        s.set_density_field(np.ones(4))


def test_library_refusals_with_a_bound_mass_field():
    """no mass field without a material field; the material field cannot be unbound under it; x-slab mode (both orders), the in-kernel
    grid_op, and parameter gradients without gmass (backward substep and loss gradient) fail"""
    from fluidlab_b200 import _lib
    L = C.CDLL(harness.build_library())
    for name, (res, args) in _lib._PROTOS.items():
        fn = getattr(L, name); fn.restype = res; fn.argtypes = args
    h, keep = mfc_bare_handle(L)
    fld, gfld, mass, gmass = np.zeros(16, np.float32), np.zeros(16, np.float32), np.ones(8, np.float32), np.zeros(8, np.float32)
    mf = _lib.FmpmMaterialField(); mf.field, mf.gfield = fld.ctypes.data, gfld.ctypes.data
    mm = _lib.FmpmMassField(); mm.mass = mass.ctypes.data
    assert L.fmpm_set_mass_field(h, C.byref(mm)) != 0 and b'material field' in L.fmpm_last_error(h)
    sl = _lib.FmpmSlab(); sl.enabled = 1
    assert L.fmpm_set_slab(h, C.byref(sl)) == 0
    assert L.fmpm_set_mass_field(h, C.byref(mm)) != 0 and b'x-slab' in L.fmpm_last_error(h)
    sl.enabled = 0
    assert L.fmpm_set_slab(h, C.byref(sl)) == 0
    assert L.fmpm_set_material_field(h, C.byref(mf)) == 0
    assert L.fmpm_set_mass_field(h, C.byref(mm)) == 0
    sl.enabled = 1
    assert L.fmpm_set_slab(h, C.byref(sl)) != 0 and b'mass field' in L.fmpm_last_error(h)
    assert L.fmpm_set_material_field(h, None) != 0 and b'mass field' in L.fmpm_last_error(h)
    assert L.fmpm_set_fwd_mask(h, 7) == 0
    assert L.fmpm_substeps_fused(h, 0, 2, None) != 0 and b'grid_op' in L.fmpm_last_error(h)
    assert L.fmpm_set_fwd_mask(h, ~4) == 0
    gmat, ggrav = np.zeros(4), np.zeros(3)
    pg = _lib.FmpmParamGrad(); pg.gmat, pg.ggrav = gmat.ctypes.data, ggrav.ctypes.data
    assert L.fmpm_set_param_grad(h, C.byref(pg)) == 0
    assert L.fmpm_substep_grad(h, 0, 1, 0, None) != 0 and b'gmass' in L.fmpm_last_error(h)
    scratch = np.zeros(16 ** 3 * 4, np.float32)
    dl = _lib.FmpmDensityLoss(); dl.mass, dl.w_density, dl.mrow_mask_lo = scratch.ctypes.data, 1.0, 1
    assert L.fmpm_loss_density_grad(h, 0, 0, C.byref(dl), None) != 0 and b'gmass' in L.fmpm_last_error(h)
    ml = _lib.FmpmMomentumLoss(); ml.field, ml.w_density, ml.mrow_mask_lo = scratch.ctypes.data, 1.0, 1
    assert L.fmpm_loss_momentum_grad(h, 0, 0, C.byref(ml), None) != 0 and b'gmass' in L.fmpm_last_error(h)
    mm.gmass = gmass.ctypes.data
    assert L.fmpm_set_mass_field(h, C.byref(mm)) == 0
    assert L.fmpm_set_mass_field(h, None) == 0
    assert L.fmpm_set_material_field(h, None) == 0
    L.fmpm_destroy(h)


def mfc_bare_handle(L):
    import test_material_field as tmf
    return tmf._bare_handle(L)


def test_mass_field_struct_matches_the_c_header(tmp_path):
    from fluidlab_b200 import _lib
    src = tmp_path / 'mm.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fluidmpm.h"\nint main(void) { printf("%zu %zu %zu\\n", sizeof(FmpmMassField), '
                   'offsetof(FmpmMassField, mass), offsetof(FmpmMassField, gmass)); return 0; }\n')
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(tmp_path / 'mm')])
    out = [int(v) for v in subprocess.run([str(tmp_path / 'mm')], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [C.sizeof(_lib.FmpmMassField), _lib.FmpmMassField.mass.offset, _lib.FmpmMassField.gmass.offset]


def test_set_mass_field_is_exported():
    from fluidlab_b200 import _lib
    assert 'fmpm_set_mass_field' in _lib.EXPORTS
    nm = subprocess.run(['nm', '-D', '--defined-only', harness.build_library()], capture_output=True, text=True, check=True).stdout
    assert re.search(r'\bT fmpm_set_mass_field\b', nm)


def test_mass_field_k_fwd_does_not_spill(tmp_path):
    """k_fwd<3, false, false> (the forward hot kernel with mu, lam and mass per slot) meets the bar of k_fwd<0, false, *>: no spills"""
    import test_sass_budget as sb
    if sb._nvcc() is None:
        pytest.skip('nvcc not found')
    spills = sb._spills('fmpm_forward.cu', str(tmp_path))
    assert spills['k_fwd<3, false, false>'] == (0, 0), spills['k_fwd<3, false, false>']
