"""ctypes wrapper of the smoke-solver oracle (oracle/smoke_oracle.hpp) — TEST INFRASTRUCTURE ONLY.

Restates fluidlab/fluidengine/simulators/smoke_field.py (SF); see the header of smoke_oracle.hpp for the parity status."""
import ctypes as C
import numpy as np
from .oracle import lib, _p, _d


class SmokeConfig(C.Structure):
    _fields_ = [("n", C.c_int), ("S", C.c_int), ("q_dim", C.c_int), ("solver_iters", C.c_int), ("dt", C.c_double),
                ("lower_y", C.c_int), ("higher_y", C.c_int), ("high_T", C.c_double), ("low_T", C.c_double), ("T_sub", C.c_int),
                ("inject_v", C.c_double * 3), ("mpm_dx", C.c_double)]


_proto_done = False


def _protos(L):
    global _proto_done
    if _proto_done:
        return
    L.orc_smoke_create.restype = C.c_void_p
    L.orc_smoke_create.argtypes = [C.POINTER(SmokeConfig), C.c_int]
    vp = C.c_void_p
    for name, args in dict(orc_smoke_destroy=[vp], orc_smoke_add_static=[vp, C.c_int, vp, vp], orc_smoke_set_aircon=[vp, C.c_int, vp],
                           orc_smoke_get_aircon_grad=[vp, C.c_int, vp], orc_smoke_set_frame=[vp, C.c_int, vp, vp, vp, vp, vp],
                           orc_smoke_get_frame=[vp, C.c_int, vp, vp, vp, vp, vp], orc_smoke_set_grad_frame=[vp, C.c_int, vp, vp, vp, vp, vp],
                           orc_smoke_get_grad_frame=[vp, C.c_int, vp, vp, vp, vp, vp], orc_smoke_get_free=[vp, C.c_int, vp],
                           orc_smoke_step=[vp, C.c_int, C.c_int], orc_smoke_step_grad=[vp, C.c_int, C.c_int], orc_smoke_reset_grad=[vp],
                           orc_smoke_copy_frame=[vp, C.c_int, C.c_int], orc_smoke_copy_grad=[vp, C.c_int, C.c_int],
                           orc_smoke_reset_grad_till_frame=[vp, C.c_int], orc_smoke_set_free=[vp, C.c_int, vp],
                           orc_smoke_free_space=[vp, C.c_int], orc_smoke_advect=[vp, C.c_int, C.c_int], orc_smoke_divergence=[vp, C.c_int],
                           orc_smoke_pressure=[vp, C.c_int], orc_smoke_project=[vp, C.c_int], orc_smoke_project_grad=[vp, C.c_int],
                           orc_smoke_pressure_grad=[vp, C.c_int], orc_smoke_divergence_grad=[vp, C.c_int],
                           orc_smoke_advect_grad=[vp, C.c_int, C.c_int]).items():
        getattr(L, name).argtypes = args
        getattr(L, name).restype = None
    _proto_done = True


class SmokeOracle:
    """SF:14-33 constructor arguments; `lower_y` / `higher_y` are class constants in the reference (60 / 68) and parameters here so that
    small grids can be tested.  Air-conditioner state per substep f: 9-vector (pos 3, quat 4, s, r) as effectors/aircon.py:188-196."""

    def __init__(self, res=128, dt=0.03, solver_iters=500, q_dim=3, max_steps_local=10, max_substeps_local=100, lower_y=60, higher_y=68,
                 inject_v=(-0.3, 0.0, 1.0), precision=32):
        L = lib(); _protos(L)
        self.L, self.n, self.q_dim, self.S = L, int(res), int(q_dim), int(max_steps_local)
        cfg = SmokeConfig()
        cfg.n, cfg.S, cfg.q_dim, cfg.solver_iters, cfg.dt = self.n, self.S, self.q_dim, int(solver_iters), float(dt)
        cfg.lower_y, cfg.higher_y, cfg.high_T, cfg.low_T, cfg.T_sub = int(lower_y), int(higher_y), 1.0, 0.0, int(max_substeps_local)
        cfg.inject_v = (C.c_double * 3)(*inject_v)
        cfg.mpm_dx = 0.0
        self.h = C.c_void_p(L.orc_smoke_create(C.byref(cfg), precision))

    def __del__(self):
        try:
            self.L.orc_smoke_destroy(self.h)
        except Exception:
            pass

    def add_static(self, voxels, T_mesh_to_voxels):
        vox = _d(voxels)
        res = int(round(vox.size ** (1 / 3)))
        self.L.orc_smoke_add_static(self.h, res, _p(vox), _p(_d(T_mesh_to_voxels)))

    def set_aircon(self, f, state9):
        self.L.orc_smoke_set_aircon(self.h, int(f), _p(_d(state9)))

    def aircon_grad(self, f):
        out = np.zeros(9)
        self.L.orc_smoke_get_aircon_grad(self.h, int(f), _p(out))
        return out

    def _alloc(self):
        n, qd = self.n, self.q_dim
        return dict(v=np.zeros((n, n, n, 3)), v_tmp=np.zeros((n, n, n, 3)), div=np.zeros((n, n, n)), p=np.zeros((n, n, n)), q=np.zeros((n, n, n, qd)))

    def get_state(self, s):  # SF:427-436
        st = self._alloc()
        self.L.orc_smoke_get_frame(self.h, int(s), _p(st['v']), _p(st['v_tmp']), _p(st['div']), _p(st['p']), _p(st['q']))
        return st

    def set_state(self, s, st):  # SF:438-439
        self.L.orc_smoke_set_frame(self.h, int(s), _p(_d(st['v'])), _p(_d(st['v_tmp'])), _p(_d(st['div'])), _p(_d(st['p'])), _p(_d(st['q'])))

    def get_grad(self, s):
        st = self._alloc()
        self.L.orc_smoke_get_grad_frame(self.h, int(s), _p(st['v']), _p(st['v_tmp']), _p(st['div']), _p(st['p']), _p(st['q']))
        return st

    def set_grad(self, s, st):
        self.L.orc_smoke_set_grad_frame(self.h, int(s), _p(_d(st['v'])), _p(_d(st['v_tmp'])), _p(_d(st['div'])), _p(_d(st['p'])), _p(_d(st['q'])))

    def is_free(self, s):
        out = np.zeros((self.n,) * 3, dtype=np.int32)
        self.L.orc_smoke_get_free(self.h, int(s), _p(out))
        return out

    def set_free(self, s, mask):
        """overwrite the free-space mask of frame s (e.g. with the one a kernel computed), (n, n, n) or flat"""
        m = np.ascontiguousarray(np.asarray(mask).reshape(-1) != 0, dtype=np.int32)
        assert m.size == self.n ** 3
        self.L.orc_smoke_set_free(self.h, int(s), _p(m))

    # the phases of one step and of its adjoint, in the order step / step_grad run them
    def free_space(self, s):  # SF:190-201
        self.L.orc_smoke_free_space(self.h, int(s))

    def advect(self, s, f):  # SF:203-233: v_tmp[s], q[s+1]
        self.L.orc_smoke_advect(self.h, int(s), int(f))

    def divergence(self, s):  # SF:235-261
        self.L.orc_smoke_divergence(self.h, int(s))

    def pressure(self, s):  # SF:97-106: p[s] -> solver_iters sweeps -> p[s+1]
        self.L.orc_smoke_pressure(self.h, int(s))

    def project(self, s):  # SF:275-289
        self.L.orc_smoke_project(self.h, int(s))

    def project_grad(self, s):
        self.L.orc_smoke_project_grad(self.h, int(s))

    def pressure_grad(self, s):
        self.L.orc_smoke_pressure_grad(self.h, int(s))

    def divergence_grad(self, s):
        self.L.orc_smoke_divergence_grad(self.h, int(s))

    def advect_grad(self, s, f):
        self.L.orc_smoke_advect_grad(self.h, int(s), int(f))

    def step(self, s, f):  # SF:95-110
        self.L.orc_smoke_step(self.h, int(s), int(f))

    def step_grad(self, s, f):  # SF:112-127
        self.L.orc_smoke_step_grad(self.h, int(s), int(f))

    def reset_grad(self):
        self.L.orc_smoke_reset_grad(self.h)

    def copy_frame(self, a, b):
        self.L.orc_smoke_copy_frame(self.h, int(a), int(b))

    def copy_grad(self, a, b):
        self.L.orc_smoke_copy_grad(self.h, int(a), int(b))

    def reset_grad_till_frame(self, s):
        self.L.orc_smoke_reset_grad_till_frame(self.h, int(s))
