"""fp64 reference of the plastic yield limits per particle and of the loss gradients with respect to them, on top of the oracle.

A plasto-elastic particle (MAT_PLASTO_ELASTIC, MAT_PLASTO_ELASTIC_DEMO) takes F[f+1] = U diag(clamp(sig_d, lo_p, hi_p)) V^T with
F~ = (I + dt C[f]) F[f] = U diag(sig) V^T (the reference's svd, oracle.svd3).  The oracle clamps to the reference's constants
[1 - 2e-3, 1 + 3e-3] (MPM:367-376); `PlasticGradOracle` is `ParamGradOracle` with per-particle limits (lo, hi) layered on it:

- forward: after the oracle's substep f it rewrites F[f+1] of the used plasto-elastic particles of frame f with their own limits.  Nothing
  else of substep f reads F[f+1], so the frame is then the reference's substep with those limits.
- backward: the clamp enters the oracle's p2g adjoint (oracle/mpm_oracle.hpp p2g_grad, MPM:266-292) only through
      gU += gF' V Sn,  gV += gF'^T U Sn,  gS_dd += (U^T gF' V)_dd pass_d,  gF~ += backward_svd(gU, gS, gV, U, sig, V)
  with Sn = diag(clamp(sig, lo, hi)), pass_d = 1 where the axis is not clamped and gF' the adjoint of F[f+1], and gF~ reaches the frame's
  adjoint as gC[f] += dt gF~ F[f]^T, gF[f] += (I + dt C[f])^T gF~.  All of it is linear in (gU, gS, gV), so after the oracle's substep_grad(f)
  the difference between the particle's limits and the constants is added to gC[f] and gF[f]: backward_svd (the oracle's own restatement,
  orc_backward_svd) of the differences of Sn and pass.
- limit gradients, with W = U^T gF' V:  dL/dlo_p += W_dd over the axes d clamped at lo_p,  dL/dhi_p += W_dd over the axes clamped at hi_p,
  with the tie rule of the clamp's adjoint (fmpm_backward.cu constitutive_grad, the oracle's p2g_grad): axis d is at lo unless lo < sig_d,
  and at hi when lo < sig_d and not max(sig_d, lo) < hi.

`reclamp` (forward) and `limit_grad` (backward, with the limit gradients) are the two layers as functions of one frame, for tests that run
the oracle one phase at a time (tests/fwd_layout_case.py, tests/bwd_layout_case.py).

With the default limits the layer does nothing and the results are the oracle's.  dL/dtheta_c = -dL/dlo and dL/dtheta_s = dL/dhi for
lo = 1 - theta_c, hi = 1 + theta_s."""
import ctypes as C

import numpy as np

from fluidlab_b200 import macros as M
from oracle import oracle as orc
from param_grad_ref import ParamGradOracle

THETA_C, THETA_S = 2e-3, 3e-3
REF_LO, REF_HI = 1 - 2e-3, 1 + 3e-3   # the oracle's constants, R(1 - 2e-3) and R(1 + 3e-3) in fp64
PLASTIC = (M.MAT_PLASTO_ELASTIC, M.MAT_PLASTO_ELASTIC_DEMO)
# fp32 runs of one step put F within 1.6e-6 of the fp64 oracle's (measured on the shim and an H100; two fp32 runs differ by up to 1.4e-6,
# the scatter's float reductions being unordered), so an axis of F~ within about twice that of a limit can be clamped in one and free in the
# other.  In the 16^3 test scenes 0 .. 5 of 256 particles are that close
NEAR = 3e-6


def limits(theta_c, theta_s):
    """(lo, hi) as the simulator gives them to the kernels: 1 - theta_c and 1 + theta_s in float64, rounded to float32"""
    lo = (1.0 - np.asarray(theta_c, np.float64)).astype(np.float32).astype(np.float64)
    hi = (1.0 + np.asarray(theta_s, np.float64)).astype(np.float32).astype(np.float64)
    return lo, hi


def clamp(s, lo, hi):
    """the clamp and its adjoint's pass mask (1 = not clamped) and side (-1 at lo, +1 at hi, 0 free) under the tie rule above"""
    sn, pas, side = np.zeros(3), np.zeros(3), np.zeros(3, np.int64)
    for d in range(3):
        mx = max(s[d], lo); p1 = lo < s[d]
        sn[d] = min(mx, hi); p2 = mx < hi
        pas[d] = 1.0 if (p1 and p2) else 0.0
        side[d] = -1 if not p1 else (1 if not p2 else 0)
    return sn, pas, side


def backward_svd(gU, gS, gV, U, s, V):
    out = np.zeros(9)
    orc.lib().orc_backward_svd.argtypes = [C.c_void_p] * 7
    a = [np.ascontiguousarray(m, np.float64) for m in (gU, gS, gV, U, s, V)]
    orc.lib().orc_backward_svd(*[C.c_void_p(m.ctypes.data) for m in a], C.c_void_p(out.ctypes.data))
    return out.reshape(3, 3)


def _svd(C, F, dt):
    return orc.svd3((np.eye(3) + np.asarray(C, np.float64) * dt) @ np.asarray(F, np.float64))


def reclamp(Fn, C, F, idx, lo, hi, dt):
    """the forward layer: F[f+1] (`Fn`, rewritten in place) of the particles `idx` of frame f (C, F) clamped with their own limits lo[q], hi[q]"""
    for q in idx:
        U, s, V = _svd(C[q], F[q], dt)
        Fn[q] = U @ np.diag(clamp(s, lo[q], hi[q])[0]) @ V.T


def limit_grad(g, gF1, C, F, idx, lo, hi, own, dt):
    """the backward layer on the oracle's adjoint of frame f (`g`, get_grad_frame's dict with the constants' clamp, rewritten in place) for the
    plasto-elastic particles `idx` of frame f (C, F), from gF1, the adjoint of F[f+1]: the particles with own[q] get the difference between
    their limits and the constants added to g['C'] and g['F'].  Returns dL/dlo and dL/dhi of the particles `idx`"""
    dlo, dhi = np.zeros(len(idx)), np.zeros(len(idx))
    for i, q in enumerate(idx):
        U, s, V = _svd(C[q], F[q], dt)
        W = U.T @ gF1[q] @ V
        sn, pas, side = clamp(s, lo[q], hi[q])
        dlo[i] = W.diagonal()[side < 0].sum()
        dhi[i] = W.diagonal()[side > 0].sum()
        if not own[q]:
            continue
        sn0, pas0, _ = clamp(s, REF_LO, REF_HI)
        dS = np.diag(sn - sn0)
        d = backward_svd(gF1[q] @ V @ dS, np.diag(W.diagonal() * (pas - pas0)), gF1[q].T @ U @ dS, U, s, V)
        g['C'][q] += dt * d @ np.asarray(F[q], np.float64).T
        g['F'][q] += (np.eye(3) + np.asarray(C[q], np.float64) * dt).T @ d
    return dlo, dhi


class PlasticGradOracle(ParamGradOracle):
    def __init__(self, n_grid, particles, lo=None, hi=None, **kw):
        self.cls = np.asarray(particles['cls'])
        super().__init__(n_grid, particles, **kw)
        self.lo = np.broadcast_to(REF_LO if lo is None else lo, (self.N,)).astype(np.float64)
        self.hi = np.broadcast_to(REF_HI if hi is None else hi, (self.N,)).astype(np.float64)
        # the particles whose limits differ from the oracle's constants (only those need the forward and backward layer)
        self.own = np.isin(self.cls, PLASTIC) & ((self.lo != REF_LO) | (self.hi != REF_HI))

    def near_limit(self, fr, tol=NEAR):
        """(N,) bool: the used plasto-elastic particles of frame `fr` with a singular value of F~ within `tol` of one of their limits, where
        the clamp's derivative jumps (the side an fp32 run puts such an axis on is decided by its rounding, not by the model)"""
        out = np.zeros(self.N, bool)
        for q in np.where((fr['used'] != 0) & np.isin(self.cls, PLASTIC))[0]:
            s = _svd(fr['C'][q], fr['F'][q], self.dt)[1]
            out[q] = bool((np.abs(s - self.lo[q]) < tol).any() or (np.abs(s - self.hi[q]) < tol).any())
        return out

    def reset_param_grad(self):
        super().reset_param_grad()
        self.pg['lo'], self.pg['hi'] = np.zeros(self.N), np.zeros(self.N)

    def substep(self, f, none_action=True):
        super().substep(f, none_action)
        if not self.own.any():
            return
        fr = self.get_frame(f)   # (after the substep: an injector's act writes frame f before its p2g)
        own = np.where((fr['used'] != 0) & self.own)[0]
        if not len(own):
            return
        nx = self.get_frame(f + 1)
        reclamp(nx['F'], fr['C'], fr['F'], own, self.lo, self.hi, self.dt)
        self.set_frame(f + 1, nx['x'], nx['v'], nx['C'], nx['F'], nx['used'])

    def substep_grad(self, f, none_action=True):
        gF1 = self.get_grad_frame(f + 1)['F']
        super().substep_grad(f, none_action)
        fr = self.get_frame(f)
        p = np.where((fr['used'] != 0) & np.isin(self.cls, PLASTIC))[0]
        g = self.get_grad_frame(f) if self.own[p].any() else None
        dlo, dhi = limit_grad(g, gF1, fr['C'], fr['F'], p, self.lo, self.hi, self.own, self.dt)
        self.pg['lo'][p] += dlo
        self.pg['hi'][p] += dhi
        if g is not None:
            self.set_grad_frame(f, g['x'], g['v'], g['C'], g['F'])
