"""ctypes binding of libfluidmpm.so (C ABI in include/fluidmpm.h).

The product path has NO CPU fallback: if the CUDA library is missing or no GPU is visible, loading
fails loudly.  (`tests/` use `oracle/` as the checker; nothing here imports it.)
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("FMPM_LIB", os.path.join(_HERE, "libfluidmpm.so"))   # FMPM_LIB: A/B kernel variants (profiles/ab_variants.sh)
_LIB = None

vp = C.c_void_p
C = C  # re-exported for struct builders (meshes.py)


class FmpmConfig(C.Structure):
    _fields_ = [
        ("n_grid", C.c_int), ("n_particles", C.c_int), ("max_substeps_local", C.c_int), ("n_substeps", C.c_int),
        ("dt", C.c_float), ("dx", C.c_float), ("inv_dx", C.c_float), ("p_vol", C.c_float),
        ("k_stress", C.c_float),
        ("gravity", C.c_float * 3),
        ("boundary_type", C.c_int),
        ("b_lower", C.c_float * 3), ("b_upper", C.c_float * 3),
        ("cyl_center", C.c_float * 2), ("cyl_radius", C.c_float),
        ("restitution", C.c_float),
        ("lock_mask", C.c_int),
        ("n_materials", C.c_int),
        ("device", C.c_int),
        ("scene_flags", C.c_int),
    ]


class FmpmMaterial(C.Structure):
    _fields_ = [("mu", C.c_float), ("lam", C.c_float), ("mass", C.c_float), ("cls", C.c_int)]


class FmpmBuffers(C.Structure):
    _fields_ = [
        ("pa", vp), ("pf", vp), ("pf8", vp),
        ("ga", vp), ("gf", vp), ("gf8", vp),
        ("grid_pm", vp), ("grid_v", vp), ("ggrid_v", vp), ("ggrid_pm", vp),
        ("materials", vp),
        ("scratch_a", vp), ("scratch_f", vp), ("scratch_f8", vp),
        ("sort_keys_in", vp), ("sort_keys_out", vp), ("sort_vals_in", vp), ("sort_vals_out", vp),
        ("sort_tmp", vp), ("sort_tmp_bytes", C.c_ulonglong),
        ("blk_flags", vp), ("blk_list", vp), ("blk_count", vp),
        ("grid_pm_ring", vp), ("grid_v_ring", vp), ("blk_list_ring", vp), ("blk_count_ring", vp),
        ("grid_pm3", vp), ("blk_flags3", vp),
    ]


class FmpmEffector(C.Structure):
    _fields_ = [
        ("pos", vp), ("quat", vp), ("v", vp), ("w", vp),
        ("gpos", vp), ("gquat", vp), ("gv", vp), ("gw", vp),
        ("act", vp), ("gact", vp), ("act_p", vp), ("gact_p", vp),
        ("action_dim", C.c_int),
        ("scale_v", C.c_float * 6), ("scale_p", C.c_float * 6),
        ("boundary_type", C.c_int), ("b_lower", C.c_float * 3), ("b_upper", C.c_float * 3),
        ("cyl_center", C.c_float * 2), ("cyl_radius", C.c_float),
    ]


class FmpmInjector(C.Structure):
    _fields_ = [
        ("kind", C.c_int), ("flux", C.c_int), ("radius", C.c_float),
        ("inject_v", C.c_float * 3), ("inject_p", C.c_float * 3),
        ("random_vector", vp), ("act_range", vp), ("n_act_range", C.c_int), ("randomize_inject_v", C.c_int),
    ]


class FmpmSdfMesh(C.Structure):
    _fields_ = [("voxels", vp), ("res", C.c_int), ("T_mesh_to_voxels", C.c_float * 16), ("friction", C.c_float), ("softness", C.c_float)]


class FmpmColliders(C.Structure):
    _fields_ = [("n_statics", C.c_int), ("statics", FmpmSdfMesh * 4), ("has_rigid", C.c_int), ("collide_type", C.c_int),
                ("rigid", FmpmSdfMesh), ("pos", vp), ("quat", vp), ("gpos", vp), ("gquat", vp), ("collide_y_min", C.c_float)]


class FmpmSlab(C.Structure):
    _fields_ = [("enabled", C.c_int), ("peer_pm_left", vp), ("peer_pm_right", vp), ("peer_flags_left", vp), ("peer_flags_right", vp),
                ("left_lo", C.c_int), ("left_hi", C.c_int),
                ("right_lo", C.c_int), ("right_hi", C.c_int), ("peer_ggv_left", vp), ("peer_ggv_right", vp),
                ("signal", vp), ("peer_signal_left", vp), ("peer_signal_right", vp)]


class FmpmCollector(C.Structure):
    _fields_ = [("boundary_type", C.c_int), ("lower", C.c_float * 3), ("upper", C.c_float * 3), ("cyl_center", C.c_float * 2),
                ("cyl_radius", C.c_float), ("row_mask", C.c_uint)]


class FmpmBodies(C.Structure):
    _fields_ = [("n_bodies", C.c_int), ("info", vp), ("state", vp), ("grad", vp)]


class FmpmParamGrad(C.Structure):
    _fields_ = [("gmat", vp), ("ggrav", vp)]


class FmpmContactGrad(C.Structure):
    _fields_ = [("gcontact", vp)]


class FmpmDensityLoss(C.Structure):
    _fields_ = [("mass", vp), ("target", vp), ("sdf", vp), ("w_density", C.c_float), ("w_sdf", C.c_float), ("mrow_mask_lo", C.c_uint),
                ("reserved", C.c_int)]


class FmpmMomentumLoss(C.Structure):
    _fields_ = [("field", vp), ("target", vp), ("sdf", vp), ("w_density", C.c_float), ("w_sdf", C.c_float), ("w_momentum", C.c_float),
                ("mrow_mask_lo", C.c_uint)]


BODY_STATE_STRIDE, BODY_GRAD_STRIDE = 48, 32
SCENE_ALL_LIQUID_MU0 = 1
FWD_KFWD, FWD_LIQUID, FWD_INLINE, FWD_TMA = 1, 2, 4, 8


# ---- include/fluidsmoke.h
class FsmkConfig(C.Structure):
    _fields_ = [("res", C.c_int), ("max_steps_local", C.c_int), ("q_dim", C.c_int), ("solver_iters", C.c_int), ("dt", C.c_float),
                ("lower_y", C.c_int), ("higher_y", C.c_int), ("low_T", C.c_float), ("inject_v", C.c_float * 3), ("device", C.c_int)]


class FsmkBuffers(C.Structure):
    _fields_ = [(k, vp) for k in ("v", "v_tmp", "div", "p", "q", "is_free", "gv", "gv_tmp", "gdiv", "gp", "gq", "tmp_a", "tmp_b", "acc")]


class FsmkAircon(C.Structure):
    _fields_ = [(k, vp) for k in ("pos", "quat", "s", "r", "gpos", "gquat", "gs", "gr")]


_I, _F, _U = C.c_int, C.c_float, C.c_uint
class FmpmAdamCfg(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("lr", "beta_1", "beta_2", "epsilon", "bias_1", "bias_2", "clip_lo", "clip_hi")] + [
        ("rows", C.c_int), ("cols", C.c_int), ("fix_dim_mask", C.c_uint), ("reserved", C.c_int)]


_PROTOS = {
    "fmpm_set_bodies": (_I, [vp, C.POINTER(FmpmBodies)]),
    "fmpm_collect": (_I, [vp, _I, C.POINTER(FmpmCollector), vp]),
    "fmpm_advect_rigid": (_I, [vp, _I, vp]),
    "fmpm_advect_rigid_grad": (_I, [vp, _I, _I, vp, vp]),
    "fmpm_set_colliders": (_I, [vp, C.POINTER(FmpmColliders)]),
    "fmpm_set_slab": (_I, [vp, C.POINTER(FmpmSlab)]),
    "fmpm_slab_sync": (_I, [vp, vp]),
    "fmpm_substeps_slab": (_I, [vp, _I, _I, _I, vp]),
    "fmpm_set_slab_pull": (_I, [vp, _I]),
    "fmpm_create": (_I, [C.POINTER(FmpmConfig), C.POINTER(vp)]),
    "fmpm_destroy": (None, [vp]),
    "fmpm_bind": (_I, [vp, C.POINTER(FmpmBuffers)]),
    "fmpm_last_error": (C.c_char_p, [vp]),
    "fmpm_sort_workspace_bytes": (C.c_ulonglong, [vp]),
    "fmpm_abi_version": (_I, []),
    "fmpm_clear_grid": (_I, [vp, vp]),
    "fmpm_p2g": (_I, [vp, _I, _I, vp]),
    "fmpm_grid_op": (_I, [vp, _I, _I, vp]),
    "fmpm_g2p": (_I, [vp, _I, vp]),
    "fmpm_substep": (_I, [vp, _I, vp]),
    "fmpm_substep_store": (_I, [vp, _I, vp]),
    "fmpm_g2p2g": (_I, [vp, _I, _I, vp]),
    "fmpm_g2p2g_collect": (_I, [vp, _I, _I, C.POINTER(FmpmCollector), vp]),
    "fmpm_substeps_fused": (_I, [vp, _I, _I, vp]),
    "fmpm_fwd_step": (_I, [vp, _I, _I, vp]),
    "fmpm_fwd_path": (_I, [vp]),
    "fmpm_set_fwd_mask": (_I, [vp, _I]),
    "fmpm_p2g_injected": (_I, [vp, _I, C.POINTER(FmpmInjector), _I, vp, _I, C.POINTER(FmpmCollector), vp]),
    "fmpm_p2g_rigid": (_I, [vp, _I, _I, C.POINTER(FmpmCollector), vp]),
    "fmpm_clear_ring_slot": (_I, [vp, _I, vp]),
    "fmpm_p2g_store": (_I, [vp, _I, vp]),
    "fmpm_grid_op_store": (_I, [vp, _I, vp]),
    "fmpm_g2p_store": (_I, [vp, _I, vp]),
    "fmpm_g2p2g_store": (_I, [vp, _I, C.POINTER(FmpmCollector), vp]),
    "fmpm_substeps_fused_store": (_I, [vp, _I, _I, vp]),
    "fmpm_substep_grad_stored": (_I, [vp, _I, _I, _I, vp]),
    "fmpm_substep_grad_scatter": (_I, [vp, _I, _I, vp]),
    "fmpm_substep_grad_finish": (_I, [vp, _I, _I, _I, vp]),
    "fmpm_substep_grad_slab": (_I, [vp, _I, _I, _I, vp]),
    "fmpm_inject": (_I, [vp, _I, C.POINTER(FmpmInjector), C.POINTER(FmpmEffector), _I, _I, vp, vp]),
    "fmpm_substep_grad": (_I, [vp, _I, _I, _I, vp]),
    "fmpm_g2p_grad_scatter": (_I, [vp, _I, _I, vp]),
    "fmpm_grid_op_grad": (_I, [vp, _I, vp]),
    "fmpm_particle_grad": (_I, [vp, _I, _I, _I, vp]),
    "fmpm_inject_grad": (_I, [vp, _I, _I, C.POINTER(FmpmInjector), C.POINTER(FmpmEffector), _I, vp, vp]),
    "fmpm_write_frame": (_I, [vp, _I, vp, vp, vp, vp, vp, vp, vp, vp]),
    "fmpm_read_frame": (_I, [vp, _I, vp, vp, vp, vp, vp, vp, vp]),
    "fmpm_write_grad": (_I, [vp, _I, vp, vp, vp, vp, vp, vp]),
    "fmpm_read_grad": (_I, [vp, _I, vp, vp, vp, vp, vp, vp]),
    "fmpm_zero_grad": (_I, [vp, _I, vp]),
    "fmpm_copy_frame": (_I, [vp, _I, _I, vp]),
    "fmpm_permute_grad": (_I, [vp, _I, _I, vp, vp, vp]),
    "fmpm_sort": (_I, [vp, _I, vp, vp, vp, vp]),
    "fmpm_read_grid": (_I, [vp, vp, vp, vp, vp]),
    "fmpm_read_grid_grad": (_I, [vp, vp, vp, vp, vp]),
    "fmpm_write_grid_grad": (_I, [vp, vp, vp, vp, vp]),
    "fmpm_effector_step": (_I, [vp, C.POINTER(FmpmEffector), _I, _I, vp, vp]),
    "fmpm_effector_step_grad": (_I, [vp, C.POINTER(FmpmEffector), _I, _I, vp]),
    "fmpm_effector_apply_action_p": (_I, [vp, C.POINTER(FmpmEffector), vp]),
    "fmpm_effector_apply_action_p_grad": (_I, [vp, C.POINTER(FmpmEffector), vp]),
    "fmpm_loss_chamfer": (_I, [vp, _I, vp, vp, _U, _F, vp, vp]),
    "fmpm_loss_chamfer_grad": (_I, [vp, _I, _I, vp, vp, _U, _F, vp]),
    "fmpm_set_param_grad": (_I, [vp, C.POINTER(FmpmParamGrad)]),
    "fmpm_set_gravity": (_I, [vp, C.POINTER(C.c_float)]),
    "fmpm_set_scene_flags": (_I, [vp, _I]),
    "fmpm_set_contact_grad": (_I, [vp, C.POINTER(FmpmContactGrad)]),
    "fmpm_set_restitution": (_I, [vp, _F]),
    "fmpm_loss_density": (_I, [vp, _I, C.POINTER(FmpmDensityLoss), vp, vp]),
    "fmpm_loss_density_grad": (_I, [vp, _I, _I, C.POINTER(FmpmDensityLoss), vp]),
    "fmpm_loss_momentum": (_I, [vp, _I, C.POINTER(FmpmMomentumLoss), vp, vp]),
    "fmpm_loss_momentum_grad": (_I, [vp, _I, _I, C.POINTER(FmpmMomentumLoss), vp]),
}
_PROTOS["fmpm_adam_step"] = (_I, [vp, C.POINTER(FmpmAdamCfg), vp, vp, vp, vp, vp, vp])
EXPORTS = tuple(_PROTOS.keys())
_SMOKE_PROTOS = {
    "fsmk_create": (_I, [C.POINTER(FsmkConfig), C.POINTER(vp)]),
    "fsmk_destroy": (None, [vp]),
    "fsmk_bind": (_I, [vp, C.POINTER(FsmkBuffers)]),
    "fsmk_set_statics": (_I, [vp, _I, C.POINTER(FmpmSdfMesh)]),
    "fsmk_set_aircon": (_I, [vp, C.POINTER(FsmkAircon)]),
    "fsmk_last_error": (C.c_char_p, [vp]),
    "fsmk_step": (_I, [vp, _I, _I, vp]),
    "fsmk_step_grad": (_I, [vp, _I, _I, vp]),
    "fsmk_free_space": (_I, [vp, _I, vp]),
    "fsmk_advect": (_I, [vp, _I, _I, vp]),
    "fsmk_divergence": (_I, [vp, _I, vp]),
    "fsmk_pressure": (_I, [vp, _I, vp]),
    "fsmk_project": (_I, [vp, _I, vp]),
    "fsmk_project_grad": (_I, [vp, _I, vp]),
    "fsmk_pressure_grad": (_I, [vp, _I, vp]),
    "fsmk_divergence_grad": (_I, [vp, _I, vp]),
    "fsmk_advect_grad": (_I, [vp, _I, _I, vp]),
}
SMOKE_EXPORTS = tuple(_SMOKE_PROTOS.keys())


def attach_smoke_protos(L):
    for name, (res, args) in _SMOKE_PROTOS.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    return L


def load():
    """dlopen libfluidmpm.so and attach prototypes.  Raises if the library has not been built."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python fluidlab_b200/csrc/build.py` (nvcc, sm_90a). "
                "fluidlab_b200 has no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in _PROTOS.items():
            fn = getattr(L, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        attach_smoke_protos(L)
        _LIB = L
    return _LIB


class FmpmError(RuntimeError):
    pass


def check(lib, handle, rc, what=""):
    if rc != 0:
        msg = lib.fmpm_last_error(handle)
        raise FmpmError(f"{what}: {msg.decode() if msg else 'error %d' % rc}")
