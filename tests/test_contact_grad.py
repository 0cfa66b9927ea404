"""Loss gradients with respect to the contact parameters (static friction, rigid friction and softness, wall restitution), on CPU: the fp64
reference (tests/contact_grad_ref.py, built on the oracle) against central differences through the oracle's forward, per collide evaluation
and over whole substeps; the CUDA kernels on the execution-model shim against the reference; the C ABI and its errors; a friction
identification."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'cuda_emu'))
import harness  # noqa: E402

import contact_grad_case as cgc  # noqa: E402

SCENES = list(cgc.SCENES)


@pytest.fixture
def emu():
    L = harness.enable()
    yield L
    harness.disable()


@pytest.mark.parametrize('scene', SCENES)
def test_reference_contact_adjoints_match_central_differences(scene):
    """3 substeps of a 300-particle cloud on a 16^3 grid, random linear loss on (x, v, C, F): dL/d(restitution, static friction, rigid
    friction, rigid softness) of the fp64 reference against central differences through the oracle's fp64 forward.  Softness 0 sits on the reference's
    hit-test switch (any softness > 0 makes every node with sd < 2.3 / softness a hit), where the derivative is not defined: the reference reports
    0 there, by the rule that branch conditions carry no gradient, and no difference quotient is taken."""
    loss, g = cgc.oracle_run(scene, grads=True)
    checked = cgc.checked_params(scene)
    for key, nonzero in checked.items():
        base = cgc.oracle_params(scene)[key]
        if key == 'rigid_softness' and base == 0.0:
            assert g[key] == 0.0
            continue
        h = 1e-6 * max(1.0, abs(base))
        fd = (cgc.oracle_run(scene, {key: base + h}) - cgc.oracle_run(scene, {key: base - h})) / (2 * h)
        assert abs(fd - g[key]) <= 2e-5 * max(1.0, abs(fd), abs(g[key])), (scene, key, fd, g[key])
        if nonzero:
            assert abs(g[key]) > 1e-3, (scene, key, 'the scene does not exercise this parameter', g[key])
        else:
            assert g[key] == 0.0, (scene, key, 'the sticky branch has zero derivative', g[key])


@pytest.mark.parametrize('friction,softness', [(0.5, 50.0), (0.5, 0.0), (8.0, 100.0), (12.0, 50.0)], ids=['soft', 'hard', 'cone', 'sticky'])
def test_collide_parameter_derivatives_match_the_oracle_collide(friction, softness):
    """one Dynamic.collide evaluation per random point around a posed box: the reference's d/dfriction and d/dsoftness (torch.autograd on
    collide_torch with both as leaves, tests/contact_grad_ref.py) against central differences of the oracle's own evaluation
    (orc_sdf_collide_eval_q).  Covers the friction (g > 0) and clamped (g = 0) branches, the soft influence (exp < 1), the hard contact
    (softness 0: no derivative by the reference's min rule) and the sticky branch (friction > 10, zero derivative)."""
    import ctypes as C
    from conftest import box_sdf
    from oracle import oracle as orc
    from contact_grad_ref import _collide
    L = orc.lib()
    L.orc_sdf_collide_eval_q.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_double] + [C.c_void_p] * 4
    vox, T = box_sdf(np.array([0.08, 0.05, 0.11]), 0.2)
    vox = np.ascontiguousarray(vox, dtype=np.float64); T = np.ascontiguousarray(T, dtype=np.float64)
    rng = np.random.RandomState(83)
    K = 400
    c0 = np.array([0.5, 0.5, 0.5])
    io = np.zeros((K, 20)); gout = rng.randn(K, 3)
    for k in range(K):
        q0 = rng.randn(4); q0 /= np.linalg.norm(q0)
        d = rng.randn(3); d /= np.linalg.norm(d)
        io[k] = np.concatenate([c0 + d * rng.uniform(0.03, 0.13), rng.randn(3) * 0.5, c0, c0 + rng.randn(3) * 1e-4, q0, q0])

    def oracle_dot(fr, so):   # gout . out of every point, and the points the collider touches
        out = np.zeros((K, 3))
        for k in range(K):
            L.orc_sdf_collide_eval_q(32, vox.ctypes.data, T.ctypes.data, fr, so, 2e-4, io[k].ctypes.data, out[k].ctypes.data, None, None)
        return (out * gout).sum(1), np.abs(out - io[:, 3:6]).max(1) > 1e-9
    _, hit = oracle_dot(friction, softness)
    assert hit.sum() > 60
    t = lambda a: torch.tensor(a, dtype=torch.float64)
    an = np.zeros((K, 2))
    for k in range(K):
        fr = torch.tensor(friction, dtype=torch.float64, requires_grad=True)
        so = torch.tensor(softness, dtype=torch.float64, requires_grad=True)
        out = _collide((t(vox), t(T)), fr, so, 2e-4, t(io[k:k + 1, 0:3]), t(io[k:k + 1, 3:6]), (t(io[k:k + 1, 6:9]), t(io[k:k + 1, 12:16])),
                       (t(io[k:k + 1, 9:12]), t(io[k:k + 1, 16:20])))
        if out.requires_grad:   # the sticky branch depends on neither parameter
            an[k] = [float(v) for v in torch.autograd.grad((out * t(gout[k:k + 1])).sum(), (fr, so), allow_unused=True, materialize_grads=True)]
    fd = np.zeros((K, 2))
    h = 1e-6 * friction
    fd[:, 0] = (oracle_dot(friction + h, softness)[0] - oracle_dot(friction - h, softness)[0]) / (2 * h)
    if softness > 0.0:
        h = 1e-6 * softness
        fd[:, 1] = (oracle_dot(friction, softness + h)[0] - oracle_dot(friction, softness - h)[0]) / (2 * h)
    # rows whose hit / influence / friction-cone switch lies within the step, or on a medial plane of the box (normal = round-off noise, as in
    # test_oracle_collide_matches_torch_autograd), make the difference quotient meaningless: the bar must hold for 95 % of the points
    err = np.abs(an - fd).max(1) / np.maximum(1.0, np.abs(an).max(1))
    assert (err < 1e-6).mean() > 0.95, np.sort(err)[-20:]
    if friction > 10.0:
        assert np.abs(an).max() == 0.0
    else:
        assert np.abs(an[:, 0]).max() > 1e-3 and (np.abs(an[hit, 0]) == 0).sum() > 0   # friction active somewhere, clamped or absent elsewhere
        assert np.abs(an[:, 1]).max() > 1e-3 if softness > 0.0 else np.abs(an[:, 1]).max() == 0.0


@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('scene', SCENES)
def test_contact_grad_kernels_match_the_oracle_on_the_emulated_device(emu, scene, sort):
    """k_grid_op_grad<true> (statics, grid-level Rigid collide, walls) and k_collide_particle_grad<true> (particle-level Rigid collide): one
    step forward and backward against the fp64 reference (tests/contact_grad_case.py, also run on an H100)"""
    got, _, want = cgc.sim_run(scene, 'cpu', sort)
    cgc.assert_contact_close(got, want, scene)


@pytest.mark.parametrize('sort', [True, False], ids=['sorted-stored', 'unsorted-recompute'])
@pytest.mark.parametrize('scene', ['static', 'rigid_both_s50'])
def test_contact_accumulator_leaves_the_other_gradients_alone_on_the_emulated_device(emu, scene, sort):
    cgc.assert_bound_unbound_agree(scene, 'cpu', sort)


def test_contact_grad_reduction_is_order_independent_under_a_shuffled_schedule():
    """the warp / CTA reductions of the contact gradients under CUEMU_SCHED=shuffle (another thread order inside every block): a missing barrier
    between the shared-memory partial sums and their reader would change the result"""
    import subprocess
    env = dict(os.environ, CUEMU_SCHED='shuffle')
    r = subprocess.run([sys.executable, '-m', 'pytest', os.path.abspath(__file__), '-q', '-p', 'no:cacheprovider',
                        '-k', 'kernels_match_the_oracle and (static or rigid_both_s50 or cylinder)'],
                       capture_output=True, text=True, timeout=1500, env=env, cwd=os.path.dirname(HERE))
    tail = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else ''
    assert r.returncode == 0 and '6 passed' in tail, r.stdout[-3000:] + r.stderr[-1000:]


def _emu_handle():
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
    return L, h, (keep, blk, b)


def test_contact_grad_binding_rules_and_slab_refusal():
    """fmpm_set_contact_grad needs the parameter-gradient accumulators; unbinding those unbinds it; the x-slab backward entry points refuse a
    bound contact accumulator; fmpm_set_restitution refuses a non-finite value"""
    import ctypes as C
    from fluidlab_b200 import _lib
    L, h, keep = _emu_handle()
    gc, gmat, ggrav = np.zeros(8), np.zeros(4), np.zeros(3)
    cg = _lib.FmpmContactGrad(); cg.gcontact = gc.ctypes.data
    assert L.fmpm_set_contact_grad(h, C.byref(cg)) != 0 and b'fmpm_set_param_grad' in L.fmpm_last_error(h)
    pg = _lib.FmpmParamGrad(); pg.gmat, pg.ggrav = gmat.ctypes.data, ggrav.ctypes.data
    assert L.fmpm_set_param_grad(h, C.byref(pg)) == 0
    assert L.fmpm_set_contact_grad(h, C.byref(cg)) == 0
    assert L.fmpm_set_param_grad(h, None) == 0   # unbinds the contact accumulator too
    for fn in (L.fmpm_substep_grad_finish, L.fmpm_substep_grad_slab):
        assert fn(h, 0, 1, 0, None) == 0 or b'parameter gradients' not in L.fmpm_last_error(h)
    assert L.fmpm_set_param_grad(h, C.byref(pg)) == 0 and L.fmpm_set_contact_grad(h, C.byref(cg)) == 0
    for fn in (L.fmpm_substep_grad_finish, L.fmpm_substep_grad_slab):
        assert fn(h, 0, 1, 0, None) != 0 and b'fmpm_set_contact_grad' in L.fmpm_last_error(h)
    assert L.fmpm_set_contact_grad(h, None) == 0 and L.fmpm_set_param_grad(h, None) == 0
    assert L.fmpm_set_restitution(h, 0.5) == 0
    assert L.fmpm_set_restitution(h, float('nan')) != 0 and L.fmpm_set_restitution(h, float('inf')) != 0
    L.fmpm_destroy(h)


def test_contact_grad_struct_matches_the_c_header(tmp_path):
    import ctypes as C
    import subprocess
    from fluidlab_b200 import _lib
    src = tmp_path / 'cg.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fluidmpm.h"\nint main(void) { printf("%zu %zu\\n", sizeof(FmpmContactGrad), '
                   'offsetof(FmpmContactGrad, gcontact)); return 0; }\n')
    subprocess.check_call(['gcc', '-I', os.path.join(os.path.dirname(HERE), 'include'), str(src), '-o', str(tmp_path / 'cg')])
    out = [int(v) for v in subprocess.run([str(tmp_path / 'cg')], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [C.sizeof(_lib.FmpmContactGrad), _lib.FmpmContactGrad.gcontact.offset]


def test_set_contact_params_validates_and_round_trips(emu):
    """wrong counts, NaN and negative values are refused before anything changes; accepted values come back from get_contact_params()"""
    from fluidlab_b200 import TaichiEnv, macros as M
    from conftest import make_particles, box_sdf
    env = TaichiEnv(quality=16 / 64, max_substeps_local=20, horizon=2, ckpt_dest='cpu', device='cpu')
    env.setup_boundary(**cgc.CUBE)
    vox, T = box_sdf((0.12, 0.02, 0.12), 0.3)
    env.add_static(file='box.obj', material=M.CUP, has_dynamics=True, pos=(0.46, 0.36, 0.53), sdf=dict(voxels=vox, T_mesh_to_voxels=T))
    P = make_particles(np.random.RandomState(0).uniform(0.4, 0.6, size=(50, 3)), M.WATER, 16)
    env.particle_bodies.get = lambda: P
    env.build()
    s = env.simulator
    before = s.get_contact_params()
    assert set(before) == {'static_friction', 'restitution'}
    for bad in (dict(static_friction=[0.1, 0.2]), dict(static_friction=[float('nan')]), dict(static_friction=[-0.1]), dict(restitution=float('inf')),
                dict(rigid_friction=0.5)):
        with pytest.raises(ValueError):
            s.set_contact_params(**bad)
    assert s.get_contact_params()['static_friction'].tolist() == before['static_friction'].tolist()
    s.set_contact_params(static_friction=[0.25], restitution=0.3)
    after = s.get_contact_params()
    assert after['static_friction'].tolist() == [0.25] and after['restitution'] == 0.3


def test_slab_simulator_still_rejects_param_grad():
    from fluidlab_b200.slab import SlabMPMSimulator
    s = SlabMPMSimulator.__new__(SlabMPMSimulator)
    with pytest.raises(NotImplementedError, match='single-GPU'):
        s.param_grad = True


def test_static_friction_identification_on_the_emulated_device(emu):
    """gradient steps on the friction of a static box, started at 0.1, recover the 0.3 that produced the target trajectory"""
    hist = cgc.friction_sysid_case('cpu')
    assert abs(hist[-1] - 0.3) < 0.03, hist
