"""fp64 reference of the loss gradients with respect to the contact parameters, on top of the oracle.

`ContactGradOracle` is `oracle.OracleSim` whose backward substep also accumulates dL/d(friction of every static, friction and softness of the
Rigid mesh, wall restitution).  The oracle itself is unchanged: after its own `substep_grad(f)` it exposes the state of frame f, the forward
grid of frame f, the adjoint of v_out on that grid and the frame-(f+1) adjoint.  From those this module re-evaluates, in PyTorch fp64, every
contact map the substep applied and lets torch.autograd take the products of each map's parameter derivative with its incoming adjoint:
  * grid_op (MPM:380-398): per node with mass, v = v_in / m + dt g through the statics (in order), the grid-level agent collide
    (collide_type grid / both) and the walls; incoming adjoint = the adjoint of v_out.  The walls reflect an axis with v_out = -restitution v
    (cube, boundaries.py:106-120; cylinder y faces :39-63), not on a locked axis and not in the cylinder's radial kill.
  * g2p (MPM:419-422, collide_type particle / both): per used particle, agent.collide(x + dt v', v') with v' = sum w v_out; incoming adjoint
    = gv[f+1] + dt gx[f+1], which is what the oracle's frame-(f+1) velocity adjoint holds after its substep_grad (g2p_advect_grad adds
    dt gx to it in place before the collide adjoint).
Each collide evaluation is `collide_torch` (tests/test_torch_autodiff_crosscheck.py), the PyTorch restatement of Dynamic.collide
(meshes/dynamic.py:93-121); a static mesh is the same map with the identity pose, softness 0 and no sticky branch (meshes/static.py:82-104).
Branch conditions (the hit test, the sticky switch, the wall tests) carry no gradient; min(exp(-sd softness), 1) passes its adjoint to the
exponential only where it is < 1, as the reference's min does (torch.minimum would split a tie at softness 0).
The tests check these against central differences through the oracle's forward (tests/test_contact_grad.py)."""
import numpy as np
import torch

from oracle import oracle as orc
from test_torch_autodiff_crosscheck import collide_torch

_T = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))


def _collide(mesh, friction, softness, dt, p, v, pose0, pose1):
    """one batch of collide evaluations; pose = (pos (n, 3), quat (n, 4)).  collide_torch evaluates min(exp(-sd s), 1) with torch.minimum;
    with s = 0 every hit row sits on its tie, where the reference passes no adjoint to s: the softness leaf is detached there."""
    vox, T = mesh
    s = softness if softness.detach().item() > 0.0 else softness.detach()
    out, _ = collide_torch(vox, T, friction, s, dt, p, v, pose0[0], pose0[1], pose1[0], pose1[1])
    return out


class ContactGradOracle(orc.OracleSim):
    def __init__(self, n_grid, particles, gravity=(0.0, -10.0, 0.0), boundary=None, max_substeps_local=50, precision=64, dt=2e-4, n_substeps=10):
        super().__init__(n_grid, particles, gravity=gravity, boundary=boundary, max_substeps_local=max_substeps_local, precision=precision, dt=dt,
                         n_substeps=n_substeps)
        self.dt, self.gravity = float(dt), np.asarray(gravity, dtype=np.float64)
        self.bf = orc.boundary_fields(boundary)
        self.statics_ref, self.rigid_ref, self.collide_type, self.y_min = [], None, 0, -1e30
        self.reset_contact_grad()

    # the colliders are recorded for the reference as they are handed to the oracle
    def add_static(self, voxels, T_mesh_to_voxels, friction):
        super().add_static(voxels, T_mesh_to_voxels, friction)
        self.statics_ref.append(((_T(voxels), _T(T_mesh_to_voxels)), float(friction)))

    def set_rigid_mesh(self, voxels, T_mesh_to_voxels, friction, softness, collide_type='particle'):
        super().set_rigid_mesh(voxels, T_mesh_to_voxels, friction, softness, collide_type)
        self.rigid_ref = ((_T(voxels), _T(T_mesh_to_voxels)), float(friction), float(softness))
        self.collide_type = {'particle': 0, 'grid': 1, 'both': 2}[collide_type]

    def set_collide_y_min(self, y):
        super().set_collide_y_min(y)
        self.y_min = float(y)

    def reset_contact_grad(self):
        self.cg = dict(static_friction=np.zeros(4), rigid_friction=0.0, rigid_softness=0.0, restitution=0.0)

    def reset_grad(self):
        super().reset_grad()
        self.reset_contact_grad()

    def get_contact_grad(self):
        """dict(static_friction (4,), rigid_friction, rigid_softness, restitution): the layout of FmpmContactGrad (include/fluidmpm.h)"""
        return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in self.cg.items()}

    def _pose(self, f, n):
        st = self.effector_state(self.act_eff, f)
        return _T(st[:3])[None].expand(n, 3), _T(st[3:7])[None].expand(n, 4)

    def _walls(self, pos, v, r):
        """boundary_v (MPM:397): per component, -r v on a reflected axis, 0 on a killed / locked one, v otherwise (hit tests on the values)"""
        bf, vd = self.bf, v.detach().numpy()
        refl, kill = np.zeros(v.shape, bool), np.zeros(v.shape, bool)
        lo, hi = np.asarray(bf['b_lower']), np.asarray(bf['b_upper'])
        if bf['boundary_type'] == 0:
            refl = ((pos >= hi) & (vd >= 0)) | ((pos <= lo) & (vd <= 0))
        else:
            refl[:, 1] = ((pos[:, 1] > hi[1]) & (vd[:, 1] > 0)) | ((pos[:, 1] < lo[1]) & (vd[:, 1] < 0))
            rn = np.sqrt((pos[:, 0] - bf['cyl_center'][0]) ** 2 + (pos[:, 2] - bf['cyl_center'][1]) ** 2 + 1e-12)
            kill[:, 0] = kill[:, 2] = rn > bf['cyl_radius']
        for d in range(3):
            if bf['lock_mask'] & (1 << d):
                kill[:, d] = True
        refl &= ~kill
        zero = torch.zeros_like(v)
        return torch.where(_T(kill).bool(), zero, torch.where(_T(refl).bool(), -r * v, v))

    def substep_grad(self, f, none_action=True):
        super().substep_grad(f, none_action)
        n, dt, dx = self.n_grid, self.dt, 1.0 / self.n_grid
        leaf = lambda x: torch.tensor(float(x), dtype=torch.float64, requires_grad=True)
        fs = [leaf(fr) for _, fr in self.statics_ref]
        r = leaf(self.bf['restitution'])
        rf, rs = (leaf(self.rigid_ref[1]), leaf(self.rigid_ref[2])) if self.rigid_ref else (None, None)
        vin, m, vout = self.get_grid()
        _, _, gvout = self.get_grid_grad()
        terms = []
        # ---- grid level
        has = np.where(m > 1e-12)[0]
        if len(has):
            pos = np.stack([has // (n * n), (has // n) % n, has % n], 1) * dx
            p = _T(pos)
            v = _T(vin[has] / m[has, None] + dt * self.gravity[None])
            ident = (torch.zeros(len(has), 3, dtype=torch.float64), _T([1.0, 0.0, 0.0, 0.0])[None].expand(len(has), 4))
            for (mesh, _), fr in zip(self.statics_ref, fs):
                v = _collide(mesh, fr, torch.zeros((), dtype=torch.float64), dt, p, v, ident, ident)
            if self.rigid_ref and self.collide_type >= 1:
                sel = _T(pos[:, 1] > self.y_min).bool()[:, None]
                v = torch.where(sel, _collide(self.rigid_ref[0], rf, rs, dt, p, v, self._pose(f, len(has)), self._pose(f + 1, len(has))), v)
            terms.append((self._walls(pos, v, r) * _T(gvout[has])).sum())
        # ---- particle level (g2p)
        if self.rigid_ref and self.collide_type in (0, 2):
            fr_, gf = self.get_frame(f), self.get_grad_frame(f + 1)
            pp = np.where(fr_['used'] != 0)[0]
            if len(pp):
                x = fr_['x'][pp]
                base = (x * n - 0.5).astype(np.int64)
                fx = x * n - base
                w = np.stack([0.5 * (1.5 - fx) ** 2, 0.75 - (fx - 1.0) ** 2, 0.5 * (fx - 0.5) ** 2], 1)
                nv = np.zeros((len(pp), 3))
                for i in range(3):
                    for j in range(3):
                        for k in range(3):
                            g = ((base[:, 0] + i) * n + base[:, 1] + j) * n + base[:, 2] + k
                            nv += (w[:, i, 0] * w[:, j, 1] * w[:, k, 2])[:, None] * vout[g]
                xt = x + dt * nv
                out = _collide(self.rigid_ref[0], rf, rs, dt, _T(xt), _T(nv), self._pose(f, len(pp)), self._pose(f + 1, len(pp)))
                sel = _T(xt[:, 1] > self.y_min)[:, None]
                terms.append((out * sel * _T(gf['v'][pp])).sum())
        if not terms:
            return
        leaves = fs + [r] + ([rf, rs] if self.rigid_ref else [])
        grads = torch.autograd.grad(sum(terms), leaves, allow_unused=True, materialize_grads=True)
        for i in range(len(fs)):
            self.cg['static_friction'][i] += float(grads[i])
        self.cg['restitution'] += float(grads[len(fs)])
        if self.rigid_ref:
            self.cg['rigid_friction'] += float(grads[len(fs) + 1])
            self.cg['rigid_softness'] += float(grads[len(fs) + 2])
