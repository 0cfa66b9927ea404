"""oracle/oracle.py — TEST INFRASTRUCTURE ONLY.

ctypes driver for the CPU restatement of the reference substep (oracle/mpm_oracle.hpp).  Only
tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module; the product package (fluidlab_b200/) never does.

`OracleSim` mirrors the stepping contract of the reference `MPMSimulator`
(fluidlab/fluidengine/simulators/mpm_simulator.py:721-912): `step`, `step_grad`, frame ring of
`max_substeps_local+1` frames, chunk checkpoint + re-simulation in the backward pass.

PARITY STATUS (see the header of mpm_oracle.hpp): forward pinned to runs of the reference's own kernels on an emulated Taichi API
(tests/test_reference_run.py); `ti.svd` internals and Taichi's autodiff stay unpinned (adjoints: finite differences + torch.autograd).
"""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

MAT_LIQUID, MAT_PLASTO_ELASTIC, MAT_ELASTIC, MAT_RIGID, MAT_PLASTO_ELASTIC_DEMO = 200, 201, 202, 203, 204


class Config(C.Structure):
    _fields_ = [
        ("n_grid", C.c_int), ("n_particles", C.c_int), ("T", C.c_int), ("n_substeps", C.c_int),
        ("dt", C.c_double), ("dx", C.c_double), ("inv_dx", C.c_double), ("p_vol", C.c_double),
        ("gravity", C.c_double * 3),
        ("boundary_type", C.c_int),
        ("b_lower", C.c_double * 3), ("b_upper", C.c_double * 3),
        ("cyl_center", C.c_double * 2), ("cyl_radius", C.c_double),
        ("restitution", C.c_double),
        ("lock_mask", C.c_int),
    ]


class EffectorCfg(C.Structure):
    _fields_ = [
        ("type", C.c_int), ("action_dim", C.c_int),
        ("scale_v", C.c_double * 6), ("scale_p", C.c_double * 6),
        ("boundary_type", C.c_int), ("b_lower", C.c_double * 3), ("b_upper", C.c_double * 3),
        ("cyl_center", C.c_double * 2), ("cyl_radius", C.c_double),
        ("radius", C.c_double), ("flux", C.c_int), ("inject_v", C.c_double * 3), ("inject_p", C.c_double * 3),
        ("locally_random", C.c_int), ("random_length", C.c_int), ("randomize_inject_v", C.c_int),
        ("max_action_steps", C.c_int),
    ]


def build(force=False):
    """Compile liboracle.so with the committed Makefile (g++ -O3 -fopenmp)."""
    so = os.path.join(_HERE, "liboracle.so")
    srcs = [os.path.join(_HERE, f) for f in ("mpm_oracle_capi.cpp", "mpm_oracle.hpp", "smoke_oracle_capi.cpp", "smoke_oracle.hpp", "Makefile")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-B", "liboracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(so):
            build()
        L = C.CDLL(so)
        L.orc_create.restype = C.c_void_p
        L.orc_create.argtypes = [C.POINTER(Config), C.c_int]
        L.orc_loss_value.restype = C.c_double
        L.orc_loss_value.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p]
        L.orc_loss_seed.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p]
        L.orc_get_max_threads.restype = C.c_int
        _LIB = L
    return _LIB


def _d(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def boundary_fields(boundary):
    """boundary: dict(type='cube'|'cylinder', ...) as in fluidlab/fluidengine/boundaries/boundaries.py."""
    b = dict(boundary or {})
    t = b.get("type", "cube")
    out = dict(boundary_type=0, b_lower=(0.05, 0.05, 0.05), b_upper=(0.95, 0.95, 0.95), cyl_center=(0.5, 0.5),
               cyl_radius=0.45, restitution=float(b.get("restitution", 0.0)), lock_mask=0)
    for d in b.get("lock_dims", []):
        out["lock_mask"] |= 1 << int(d)
    # the reference casts boundary parameters to DTYPE_NP (f32) before use (boundaries.py:31-35,99-104)
    f32 = lambda v: tuple(float(np.float32(u)) for u in v)
    if t == "cube":
        out["b_lower"] = f32(b.get("lower", (0.05, 0.05, 0.05)))
        out["b_upper"] = f32(b.get("upper", (0.95, 0.95, 0.95)))
    elif t == "cylinder":
        out["boundary_type"] = 1
        yr = f32(b.get("y_range", (0.05, 0.95)))
        out["b_lower"] = (0.0, yr[0], 0.0)
        out["b_upper"] = (1.0, yr[1], 1.0)
        out["cyl_center"] = f32(b.get("xz_center", (0.5, 0.5)))
        out["cyl_radius"] = float(b.get("xz_radius", 0.45))
    else:
        raise AssertionError(t)
    return out


class OracleSim:
    def __init__(self, n_grid, particles, gravity=(0.0, -10.0, 0.0), boundary=None, max_substeps_local=50,
                 precision=32, dt=2e-4, n_substeps=10):
        """particles: dict with x (N,3), used (N,), mat (N,), cls (N,), mu, lam, mass (N,)."""
        L = lib()
        self.L = L
        self.N = int(len(particles["x"]))
        self.n_grid = int(n_grid)
        self.T = int(max_substeps_local)
        self.n_substeps = n_substeps
        self.precision = precision
        dx = 1.0 / n_grid
        cfg = Config()
        cfg.n_grid, cfg.n_particles, cfg.T, cfg.n_substeps = self.n_grid, self.N, self.T, n_substeps
        cfg.dt, cfg.dx, cfg.inv_dx, cfg.p_vol = dt, dx, float(n_grid), (dx * 0.5) ** 2  # MPM:21-25
        cfg.gravity = (C.c_double * 3)(*gravity)
        bf = boundary_fields(boundary)
        cfg.boundary_type = bf["boundary_type"]
        cfg.b_lower = (C.c_double * 3)(*bf["b_lower"])
        cfg.b_upper = (C.c_double * 3)(*bf["b_upper"])
        cfg.cyl_center = (C.c_double * 2)(*bf["cyl_center"])
        cfg.cyl_radius = bf["cyl_radius"]
        cfg.restitution = bf["restitution"]
        cfg.lock_mask = bf["lock_mask"]
        self.cfg = cfg
        self.h = C.c_void_p(L.orc_create(C.byref(cfg), precision))
        mat = np.ascontiguousarray(particles["mat"], dtype=np.int32)
        cls = np.ascontiguousarray(particles["cls"], dtype=np.int32)
        self.mat = mat
        L.orc_set_particle_info(self.h, _p(mat), _p(cls), _p(_d(particles["mu"])), _p(_d(particles["lam"])), _p(_d(particles["mass"])))
        x = _d(particles["x"])
        used = np.ascontiguousarray(particles["used"], dtype=np.int32)
        self.set_frame(0, x, np.zeros((self.N, 3)), np.zeros((self.N, 3, 3)), np.tile(np.eye(3), (self.N, 1, 1)), used)  # MPM:150-175
        self.cur_substep_global = 0
        self.grad_enabled = False
        self.has_agent = False
        self.n_eff = 0
        self.act_eff = 0  # effector that receives the actions
        self.ckpt = {}
        self.actions_buffer = []

    def __del__(self):
        try:
            self.L.orc_destroy(self.h)
        except Exception:
            pass

    # ---- frame io
    def set_frame(self, f, x, v, Cm, F, used):
        self.L.orc_set_frame(self.h, f, _p(_d(x)), _p(_d(v)), _p(_d(Cm)), _p(_d(F)), _p(np.ascontiguousarray(used, dtype=np.int32)))

    def get_frame(self, f):
        x = np.zeros((self.N, 3)); v = np.zeros((self.N, 3)); Cm = np.zeros((self.N, 3, 3)); F = np.zeros((self.N, 3, 3))
        used = np.zeros((self.N,), dtype=np.int32)
        self.L.orc_get_frame(self.h, f, _p(x), _p(v), _p(Cm), _p(F), _p(used))
        return dict(x=x, v=v, C=Cm, F=F, used=used)

    def set_grad_frame(self, f, gx, gv, gC, gF):
        self.L.orc_set_grad_frame(self.h, f, _p(_d(gx)), _p(_d(gv)), _p(_d(gC)), _p(_d(gF)))

    def get_grad_frame(self, f):
        x = np.zeros((self.N, 3)); v = np.zeros((self.N, 3)); Cm = np.zeros((self.N, 3, 3)); F = np.zeros((self.N, 3, 3))
        self.L.orc_get_grad_frame(self.h, f, _p(x), _p(v), _p(Cm), _p(F))
        return dict(x=x, v=v, C=Cm, F=F)

    def get_grid(self):
        G = self.n_grid ** 3
        vin = np.zeros((G, 3)); m = np.zeros((G,)); vout = np.zeros((G, 3))
        self.L.orc_get_grid(self.h, _p(vin), _p(m), _p(vout))
        return vin, m, vout

    def set_grid(self, vin, m):
        """overwrite grid.v_in / grid.mass (the x-slab tests write the ghost-summed accumulator back, tests/test_slab_cpu.py)"""
        self.L.orc_set_grid(self.h, _p(_d(vin)), _p(_d(m)))

    def get_grid_grad(self):
        G = self.n_grid ** 3
        vin = np.zeros((G, 3)); m = np.zeros((G,)); vout = np.zeros((G, 3))
        self.L.orc_get_grid_grad(self.h, _p(vin), _p(m), _p(vout))
        return vin, m, vout

    def set_grid_grad(self, vin, m, vout):
        self.L.orc_set_grid_grad(self.h, _p(_d(vin)), _p(_d(m)), _p(_d(vout)))

    # ---- agent (single effector agents: AgentInjector / plain pose chain)
    def add_effector(self, type=0, action_dim=3, scale_v=(1, 1, 1), scale_p=(1, 1, 1), boundary=None, radius=0.0, flux=0,
                     inject_v=(0, 0, 0), inject_p=(0, 0, 0), locally_random=True, random_vector=None, act_range=None,
                     max_action_steps=1000, init_pos=(0.5, 0.5, 0.5), init_quat=(1, 0, 0, 0), randomize_inject_v=False):
        ec = EffectorCfg()
        ec.type, ec.action_dim = type, action_dim
        sv = list(scale_v) + [1.0] * (6 - len(scale_v)); sp = list(scale_p) + [1.0] * (6 - len(scale_p))
        ec.scale_v = (C.c_double * 6)(*sv); ec.scale_p = (C.c_double * 6)(*sp)
        bf = boundary_fields(boundary)
        ec.boundary_type = bf["boundary_type"]
        ec.b_lower = (C.c_double * 3)(*bf["b_lower"]); ec.b_upper = (C.c_double * 3)(*bf["b_upper"])
        ec.cyl_center = (C.c_double * 2)(*bf["cyl_center"]); ec.cyl_radius = bf["cyl_radius"]
        ec.radius, ec.flux = radius, flux
        ec.inject_v = (C.c_double * 3)(*inject_v); ec.inject_p = (C.c_double * 3)(*inject_p)
        ec.locally_random = int(locally_random); ec.randomize_inject_v = int(randomize_inject_v)
        rv = _d(random_vector) if random_vector is not None else np.zeros((1, max(flux, 1), 3))
        ec.random_length = rv.shape[0]
        ec.max_action_steps = max_action_steps
        ar = np.ascontiguousarray(act_range if act_range is not None else np.zeros(0), dtype=np.int32)
        ei = self.L.orc_add_effector(self.h, C.byref(ec), _p(rv), _p(ar), len(ar))
        st = np.zeros(8); st[:3] = init_pos; st[3:7] = init_quat
        self.L.orc_effector_set_state(self.h, ei, 0, _p(st))
        self.has_agent = True
        self.n_eff = ei + 1
        self.action_dim = action_dim
        if type != 0 and ei == 0:
            self.L.orc_set_agent(self.h, 2)
        return ei

    def set_collector(self, boundary, mat=-1):
        """collector of AgentPouring (mat=-1: every material) / AgentJetBot (mat=WATER); boundary: create_boundary kwargs."""
        bf = boundary_fields(boundary)
        self.L.orc_set_collector(self.h, int(bf["boundary_type"]), _p(_d(bf["b_lower"])), _p(_d(bf["b_upper"])), _p(_d(bf["cyl_center"])),
                                 C.c_double(bf["cyl_radius"]), int(mat))

    def set_bodies(self, body_id, n_bodies=None):
        """body ids per particle (MPM:177-201); enables shape matching for bodies whose first particle is MAT_RIGID."""
        bid = np.ascontiguousarray(body_id, dtype=np.int32)
        nb = int(bid.max()) + 1 if n_bodies is None else int(n_bodies)
        self.L.orc_set_bodies(self.h, _p(bid), nb)

    # ---- SDF colliders (meshes/static.py, meshes/dynamic.py): voxels (res,res,res), T_mesh_to_voxels (4,4)
    def add_static(self, voxels, T_mesh_to_voxels, friction):
        vox = _d(voxels); T = _d(T_mesh_to_voxels)
        self.L.orc_add_static(self.h, int(vox.shape[0]), _p(vox), _p(T), C.c_double(friction))

    def set_rigid_mesh(self, voxels, T_mesh_to_voxels, friction, softness, collide_type='particle'):
        """mesh of the (single) Rigid effector added with add_effector(type=0); agent becomes AgentRigid."""
        vox = _d(voxels); T = _d(T_mesh_to_voxels)
        ct = {'particle': 0, 'grid': 1, 'both': 2}[collide_type]
        self.L.orc_set_rigid_mesh(self.h, int(vox.shape[0]), _p(vox), _p(T), C.c_double(friction), C.c_double(softness), ct)

    def set_collide_y_min(self, y):
        self.L.orc_set_collide_y_min(self.h, C.c_double(y))

    def set_icecream_agent(self, inject_till):
        """AgentIceCreamDynamic layout: effector 0 = (Ball)Injector (never actuated), effector 1 = Rigid (actuated)."""
        self.L.orc_set_agent_layout(self.h, 0, 1, int(inject_till), 1)
        self.L.orc_set_collide_y_min(self.h, C.c_double(0.25))
        self.act_eff = 1

    def effector_state(self, ei, f):
        st = np.zeros(8)
        self.L.orc_effector_get_state(self.h, ei, f, _p(st))
        return st

    def set_effector_state(self, ei, f, st):
        s = np.zeros(8); s[:len(st)] = st
        self.L.orc_effector_set_state(self.h, ei, f, _p(s))

    def apply_action_p(self, action_p):
        self.L.orc_effector_apply_action_p(self.h, self.act_eff, _p(_d(action_p)))

    def apply_action_p_grad(self):
        self.L.orc_effector_apply_action_p_grad(self.h, self.act_eff)

    def get_action_grad(self, n):
        out = np.zeros((n + 1, self.action_dim))
        self.L.orc_effector_get_action_grad(self.h, self.act_eff, n, _p(out))
        return out

    # ---- stepping contract, MPM:225-252, 721-775
    @property
    def cur_substep_local(self):
        return self.cur_substep_global % self.T

    @property
    def cur_step_local(self):
        return self.cur_substep_local // self.n_substeps

    @property
    def cur_step_global(self):
        return self.cur_substep_global // self.n_substeps

    def enable_grad(self):
        self.grad_enabled = True
        self.cur_substep_global = 0

    def disable_grad(self):
        self.grad_enabled = False
        self.cur_substep_global = 0

    def reset_grad(self):
        self.L.orc_reset_grad(self.h)

    def substep(self, f, none_action=True):
        self.L.orc_substep(self.h, f, self.cur_substep_global, int(none_action))

    def substep_grad(self, f, none_action=True):
        self.L.orc_substep_grad(self.h, f, self.cur_substep_global, int(none_action))

    def step_(self, action=None):
        none_action = action is None
        if not none_action:
            for ei in range(self.n_eff):  # effectors that are not actuated still run their pose chain with a zero action
                a = _d(action) if ei == self.act_eff else np.zeros(6)
                self.L.orc_effector_set_action(self.h, ei, self.cur_step_local, self.cur_step_global, _p(a))
        for _ in range(self.n_substeps):
            self.substep(self.cur_substep_local, none_action)
            self.cur_substep_global += 1

    def step(self, action=None):
        if self.grad_enabled and self.cur_substep_local == 0:
            self.actions_buffer = []
        self.step_(action)
        if self.grad_enabled:
            self.actions_buffer.append(None if action is None else np.array(action, dtype=np.float64))
        if self.cur_substep_local == 0:
            self._memory_to_cache()

    def _memory_to_cache(self):  # MPM:777-852
        if self.grad_enabled:
            start = self.cur_substep_global - self.T
            ck = self.get_frame(0)
            ck["actions"] = list(self.actions_buffer)
            ck["eff"] = [self.effector_state(i, 0) for i in range(self.n_eff)]
            self.ckpt[start] = ck
        self.L.orc_copy_frame(self.h, self.T, 0)

    def _memory_from_cache(self):  # MPM:856-909
        assert self.grad_enabled
        self.L.orc_copy_frame(self.h, 0, self.T)
        self.L.orc_copy_grad(self.h, 0, self.T)
        self.L.orc_reset_grad_till(self.h, self.T)
        start = self.cur_substep_global - self.T
        ck = self.ckpt[start]
        self.set_frame(0, ck["x"], ck["v"], ck["C"], ck["F"], ck["used"])
        for i, st in enumerate(ck["eff"]):
            self.set_effector_state(i, 0, st)
        self.cur_substep_global = start
        for a in ck["actions"]:
            self.step_(a)

    def step_grad(self, action=None):
        if self.cur_substep_local == 0:
            self._memory_from_cache()
        none_action = action is None
        for _ in range(self.n_substeps):
            self.cur_substep_global -= 1
            self.substep_grad(self.cur_substep_local, none_action)
        if not none_action:
            self.L.orc_effector_set_action_grad(self.h, self.act_eff, self.cur_substep_local // self.n_substeps,
                                                self.cur_substep_global // self.n_substeps)

    # ---- loss (losses/shapematching_loss.py:80-93)
    def loss_value(self, f, matching_mat, weight, tgt):
        return self.L.orc_loss_value(self.h, f, int(matching_mat), float(weight), _p(_d(tgt)))

    def loss_seed(self, f, matching_mat, weight, tgt):
        self.L.orc_loss_seed(self.h, f, int(matching_mat), float(weight), _p(_d(tgt)))


def svd3(A, precision=64):
    U = np.zeros((3, 3)); s = np.zeros(3); V = np.zeros((3, 3))
    lib().orc_svd3(_p(_d(A)), _p(U), _p(s), _p(V), precision)
    return U, s, V
