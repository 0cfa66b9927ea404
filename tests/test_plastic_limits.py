"""Plastic yield limits (MPMSimulator.set_plastic_limits / set_plastic_field, fmpm_set_plastic_field) on CPU: the fp64 reference of dL/dtheta
against central differences of the oracle, the CUDA kernels on the execution-model shim against the fp64 oracle with the same limits, the host
semantics, the refusals, the C ABI and, with nvcc, the compile-time budget of the plastic field's k_fwd instantiation."""
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

import plastic_limits_case as plc  # noqa: E402


@pytest.fixture
def emu():
    L = harness.enable()
    yield L
    harness.disable()


@pytest.mark.parametrize('per_row', [True, False], ids=['rows', 'particles'])
@pytest.mark.parametrize('boundary', ['cube', 'cylinder'])
@pytest.mark.parametrize('case', ['icecream', 'plastic_demo', 'mixed'])
def test_reference_limit_gradient_matches_central_differences_of_the_oracle(case, boundary, per_row):
    plc.reference_central_difference_case(case, boundary, per_row)


@pytest.mark.parametrize('with_field', [False, True], ids=['limits', 'limits+mu-lam'])
@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('case', ['icecream', 'mixed'])
def test_default_limits_reproduce_the_runs_without_them(emu, case, sort, with_field):
    plc.defaults_case('cpu', case, sort, with_field)


@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('case', ['icecream', 'plastic_demo', 'mixed'])
def test_random_limits_match_the_oracle_on_the_emulated_device(emu, case, sort):
    """k_p2g_field_plastic / k_particle_grad<4, *>: one step forward and one backward substep with random per-particle limits"""
    plc.heterogeneous_case('cpu', case, sort)


def test_plastic_field_kernels_are_order_independent_under_a_shuffled_schedule():
    """the random-limit cases under CUEMU_SCHED=shuffle (another thread order inside every block)"""
    env = dict(os.environ, CUEMU_SCHED='shuffle')
    r = subprocess.run([sys.executable, '-m', 'pytest', os.path.abspath(__file__), '-q', '-p', 'no:cacheprovider', '-k',
                        'random_limits_match and mixed'], capture_output=True, text=True, timeout=1500, env=env, cwd=ROOT)
    tail = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else ''
    assert r.returncode == 0 and '2 passed' in tail, r.stdout[-3000:] + r.stderr[-1000:]


def test_random_row_limits_match_the_oracle_on_the_emulated_device(emu):
    plc.heterogeneous_case('cpu', 'mixed', True, per_row=True)


@pytest.mark.parametrize('sort_every', [0, 1])
def test_limit_gradients_across_sort_epochs_and_the_checkpoint_ring(emu, sort_every):
    plc.ring_case('cpu', sort_every)


def test_fused_forward_with_limits_matches_the_oracle(emu):
    """k_fwd<4, false, false> on the fused forward-only path: two steps against the fp64 oracle and the per-substep path"""
    plc.fused_forward_case('cpu')


def test_fused_stored_grad_path_with_limits_matches_the_oracle(emu):
    """grad mode on the fused stored-grid path (k_g2p2g_field_plastic<true, false>), one backward substep against the fp64 oracle"""
    plc.heterogeneous_case('cpu', 'mixed', True, fuse=True)


@pytest.mark.parametrize('fuse', [True, False], ids=['fused', 'per-substep'])
def test_injected_icecream_with_limits_matches_the_oracle(emu, fuse):
    plc.injector_case('cpu', fuse)


def test_rigid_bodies_with_limits_match_the_oracle(emu):
    plc.rigid_case('cpu')


@pytest.mark.parametrize('set_order,clear_order', [('mrl', 'lrm'), ('lrm', 'mlr'), ('rlm', 'rml')])
def test_fields_set_and_cleared_in_any_order_keep_the_gradients(emu, set_order, clear_order):
    plc.composition_case('cpu', set_order, clear_order)


def test_identification_recovers_the_limits_from_grid_mass(emu):
    """an ICECREAM block dropped on the floor: theta_c / theta_s from the per-step grid mass, started at the defaults"""
    hist = plc.identification_case('cpu')
    tc, ts, loss = hist[-1]
    # measured on the shim (16^3, 1200 particles, 25 Adam steps): theta_c 6.07e-3 against 6e-3 (1.2 %), the loss 13x lower; theta_s is weakly
    # observed by a block that is mostly compressed, and moves from 3e-3 only to 2.1e-3 (truth 1e-3)
    assert loss < 0.2 * hist[0][2], hist
    assert abs(tc / 6e-3 - 1) < 0.1 and ts < 0.8 * hist[0][1], hist


def _sim_cpu():
    rng, P, st, seed_g = plc._scene('mixed', N=64)
    return plc._sim('cpu', P, 16, True), P


def test_host_validation_and_field_levels(emu):
    """the refusals, the getters, and the field level and composed records that each set and clear leaves behind"""
    s, P = _sim_cpu()
    N, n = len(P['x']), len(s.get_material_table()['mat'])
    lim = s.get_plastic_limits()
    assert (lim['theta_c'] == 2e-3).all() and (lim['theta_s'] == 3e-3).all() and len(lim['theta_c']) == n
    assert s.get_plastic_field() is None
    for tc, ts, msg in ((np.full(n, np.nan), None, 'finite'), (np.full(n, -1e-3), None, 'theta_c'), (np.full(n, 1.0), None, 'theta_c'),
                        (None, np.full(n, -1e-3), 'theta_s'), (None, np.full(n, np.inf), 'finite'),
                        (np.ones(n + 1) * 1e-3, None, 'hold')):
        with pytest.raises(ValueError, match=msg):
            s.set_plastic_limits(tc, ts)
    with pytest.raises(ValueError, match='shape'):
        s.set_plastic_field(np.full(N - 1, 1e-3), np.full(N - 1, 1e-3))
    with pytest.raises(ValueError, match='theta_c'):
        s.set_plastic_field(np.full(N, 1.5), np.full(N, 1e-3))
    assert s._lim_orig is None and s._field_level == 0, 'a refused call binds nothing'
    s.set_plastic_limits(theta_s=np.full(n, 5e-3))
    assert (s.get_plastic_limits()['theta_c'] == 2e-3).all() and (s.get_plastic_limits()['theta_s'] == 5e-3).all()
    assert s.get_density_field() is None and s.get_material_field() is None
    rec = plc.check_records(s)   # limits alone: level 3 on the rows' mu, lam and mass
    assert s._field_level == 3 and (rec['_pfield_slot'][:, 2] == np.float32(0.998)).all() and (rec['_pfield_slot'][:, 3] == np.float32(1.005)).all()
    import torch
    tc = torch.full((N,), 1e-3, dtype=torch.float64)
    s.set_plastic_field(tc, np.full(N, 4e-3))
    got = s.get_plastic_field()
    assert np.allclose(got[0], 1e-3) and np.allclose(got[1], 4e-3)
    assert float(s._lim_orig[0, 0]) == np.float32(1 - 1e-3) and (plc.check_records(s)['_pfield_slot'][:, 2] == np.float32(1 - 1e-3)).all()
    s.clear_plastic_field()
    assert s.get_plastic_field() is None and s._lim_orig is not None and s._field_level == 3, 'the rows keep the limits bound'
    assert (plc.check_records(s)['_pfield_slot'][:, 3] == np.float32(1.005)).all()
    s.clear_plastic_limits()
    assert s._lim_orig is None and s._field_level == 0 and not s._records and s.get_material_field() is None, 'back to the constant-clamp kernels'
    s.param_grad = True
    s.reset_grad()
    assert 'theta_c' not in s.get_param_grad()


def test_slab_simulator_refuses_limits():
    from fluidlab_b200.slab import SlabMPMSimulator
    s = SlabMPMSimulator.__new__(SlabMPMSimulator)
    with pytest.raises(NotImplementedError, match='single-GPU'):
        s.set_plastic_limits(np.ones(1) * 1e-3)
    with pytest.raises(NotImplementedError, match='single-GPU'):
        s.set_plastic_field(np.ones(4), np.ones(4))


def test_library_refusals_with_a_bound_plastic_field():
    """no plastic field without a mass field; the mass field cannot be unbound under it; x-slab mode (both orders), the all-liquid flag, the
    in-kernel grid_op and parameter gradients without the plastic field's gfield fail"""
    from fluidlab_b200 import _lib
    import test_material_field as tmf
    L = C.CDLL(harness.build_library())
    for name, (res, args) in _lib._PROTOS.items():
        fn = getattr(L, name); fn.restype = res; fn.argtypes = args
    h, keep = tmf._bare_handle(L)
    fld, gfld, mass, gmass = np.zeros(16, np.float32), np.zeros(16, np.float32), np.ones(8, np.float32), np.zeros(8, np.float32)
    pfld, gpfld = np.zeros(32, np.float32), np.zeros(32, np.float32)
    mf = _lib.FmpmMaterialField(); mf.field, mf.gfield = fld.ctypes.data, gfld.ctypes.data
    mm = _lib.FmpmMassField(); mm.mass, mm.gmass = mass.ctypes.data, gmass.ctypes.data
    pf = _lib.FmpmPlasticField(); pf.field = pfld.ctypes.data
    assert L.fmpm_set_plastic_field(h, C.byref(pf)) != 0 and b'mass field' in L.fmpm_last_error(h)
    assert L.fmpm_set_material_field(h, C.byref(mf)) == 0
    assert L.fmpm_set_plastic_field(h, C.byref(pf)) != 0 and b'mass field' in L.fmpm_last_error(h)
    assert L.fmpm_set_mass_field(h, C.byref(mm)) == 0
    assert L.fmpm_set_plastic_field(h, C.byref(pf)) == 0
    sl = _lib.FmpmSlab(); sl.enabled = 1
    assert L.fmpm_set_slab(h, C.byref(sl)) != 0 and b'plastic field' in L.fmpm_last_error(h)
    assert L.fmpm_set_mass_field(h, None) != 0 and b'plastic field' in L.fmpm_last_error(h)
    assert L.fmpm_set_material_field(h, None) != 0
    assert L.fmpm_set_scene_flags(h, _lib.SCENE_ALL_LIQUID_MU0) != 0
    assert L.fmpm_set_fwd_mask(h, 7) == 0
    assert L.fmpm_substeps_fused(h, 0, 2, None) != 0 and b'grid_op' in L.fmpm_last_error(h)
    assert L.fmpm_set_fwd_mask(h, ~4) == 0
    gmat, ggrav = np.zeros(4), np.zeros(3)
    pg = _lib.FmpmParamGrad(); pg.gmat, pg.ggrav = gmat.ctypes.data, ggrav.ctypes.data
    assert L.fmpm_set_param_grad(h, C.byref(pg)) == 0
    assert L.fmpm_substep_grad(h, 0, 1, 0, None) != 0 and b'FmpmPlasticField.gfield' in L.fmpm_last_error(h)
    pf.gfield = gpfld.ctypes.data
    assert L.fmpm_set_plastic_field(h, C.byref(pf)) == 0
    assert L.fmpm_set_plastic_field(h, None) == 0
    assert L.fmpm_set_mass_field(h, None) == 0
    assert L.fmpm_set_material_field(h, None) == 0
    # x-slab mode first: the plastic field is refused in the other call order too
    assert L.fmpm_set_slab(h, C.byref(sl)) == 0
    assert L.fmpm_set_plastic_field(h, C.byref(pf)) != 0 and b'x-slab' in L.fmpm_last_error(h)
    L.fmpm_destroy(h)


def test_plastic_field_struct_matches_the_c_header(tmp_path):
    from fluidlab_b200 import _lib
    src = tmp_path / 'pf.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fluidmpm.h"\nint main(void) { printf("%zu %zu %zu\\n", sizeof(FmpmPlasticField), '
                   'offsetof(FmpmPlasticField, field), offsetof(FmpmPlasticField, gfield)); return 0; }\n')
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(tmp_path / 'pf')])
    out = [int(v) for v in subprocess.run([str(tmp_path / 'pf')], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [C.sizeof(_lib.FmpmPlasticField), _lib.FmpmPlasticField.field.offset, _lib.FmpmPlasticField.gfield.offset]


def test_set_plastic_field_is_exported():
    from fluidlab_b200 import _lib
    assert 'fmpm_set_plastic_field' in _lib.EXPORTS
    nm = subprocess.run(['nm', '-D', '--defined-only', harness.build_library()], capture_output=True, text=True, check=True).stdout
    assert re.search(r'\bT fmpm_set_plastic_field\b', nm)


def test_plastic_field_k_fwd_does_not_spill(tmp_path):
    """k_fwd<4, false, false> (the forward hot kernel with mu, lam, the limits and mass per slot) meets the bar of k_fwd<0, false, *>: no
    spills"""
    import test_sass_budget as sb
    if sb._nvcc() is None:
        pytest.skip('nvcc not found')
    spills = sb._spills('fmpm_forward.cu', str(tmp_path))
    assert spills['k_fwd<4, false, false>'] == (0, 0), spills['k_fwd<4, false, false>']
