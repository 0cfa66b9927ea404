"""Step losses that seed the backward pass.  Mirrors fluidlab/fluidengine/losses/loss.py (`Loss` :13-78),
losses/shapematching_loss.py (`ShapeMatchingLoss` :13-130: index-matched squared distance, temporal range
curriculum) and losses/latteart_loss.py (`LatteArtLoss`).  Targets stay resident in HBM (the reference
re-uploads the step's target every step, shapematching_loss.py:72-78); the per-step loss and its seed are one
kernel each (fmpm_loss_chamfer / fmpm_loss_chamfer_grad)."""
import pickle as pkl
import numpy as np
import torch
from .macros import MILK, ICECREAM, ICECREAM1


class Loss:
    def __init__(self, max_loss_steps, weights=None, target_file=None, target=None):
        self.weights = weights
        self.target_file = target_file
        self.target = target
        self.inf = 1e8
        self.max_loss_steps = max_loss_steps

    def build(self, sim):
        self.sim = sim
        self.res, self.n_grid, self.dx, self.dim = sim.res, sim.n_grid, sim.dx, sim.dim
        self.agent = sim.agent
        self.n_particles = sim.n_particles
        self.step_loss = torch.zeros((self.max_loss_steps,), dtype=torch.float32, device=sim.device)
        self._step_grad_on = np.zeros(self.max_loss_steps, dtype=bool)
        if self.target_file is not None:
            self.load_target(self.target_file)
        elif self.target is not None:
            self.set_target(self.target)
        self.reset()

    def reset_grad(self):  # loss.py:49-51 (total_loss.grad = 1)
        self._step_grad_on[:] = False

    def load_target(self, path):
        pass

    def clear_loss(self):
        self.step_loss.zero_()
        self.total_loss = 0.0
        self._step_grad_on[:] = False

    def reset(self):
        self.clear_loss()

    def step(self):  # loss.py:72-74
        self.compute_step_loss(self.sim.cur_step_global - 1, self.sim.cur_substep_local)

    def step_grad(self):  # loss.py:76-78
        self.compute_step_loss_grad(self.sim.cur_step_global - 1, self.sim.cur_substep_local)


class ShapeMatchingLoss(Loss):
    def __init__(self, matching_mat, temporal_range_type='expand', temporal_init_range_end=50, plateau_count_limit=5,
                 temporal_expand_speed=50, plateau_thresh=(0.01, 0.5), **kwargs):
        super().__init__(**kwargs)
        self.matching_mat = matching_mat
        self.temporal_range_type = temporal_range_type
        self.temporal_init_range_end = temporal_init_range_end
        self.plateau_count_limit = plateau_count_limit
        self.temporal_expand_speed = temporal_expand_speed
        self.plateau_thresh = list(plateau_thresh)

    def build(self, sim):
        self.chamfer_weight = self.weights['chamfer']
        if self.temporal_range_type == 'last':
            self.temporal_range = [self.max_loss_steps - 1, self.max_loss_steps]
        elif self.temporal_range_type == 'all':
            self.temporal_range = [0, self.max_loss_steps]
        elif self.temporal_range_type == 'expand':
            self.temporal_range = [0, self.temporal_init_range_end]
            self.best_loss = self.inf
            self.plateau_count = 0
        super().build(sim)
        self.row_mask = sim.material_row_mask(self.matching_mat)

    def load_target(self, path):  # shapematching_loss.py:52-57
        target = pkl.load(open(path, 'rb'))
        self.set_target(target['x'])

    def set_target(self, xs):
        """xs: sequence of max_loss_steps arrays (N,3), original particle order."""
        assert self.max_loss_steps == len(xs)
        assert self.n_particles == len(xs[0])
        self.tgt = torch.from_numpy(np.ascontiguousarray(np.stack([np.asarray(a, dtype=np.float32) for a in xs]))).to(self.sim.device)

    def compute_step_loss(self, s, f):  # shapematching_loss.py:64-66, 80-88
        self.sim.chamfer_loss(self.tgt[s], self.row_mask, self.chamfer_weight, self.step_loss[s:s + 1], f)

    def compute_step_loss_grad(self, s, f):  # shapematching_loss.py:68-70
        if self._step_grad_on[s]:
            self.sim.add_x_grad_chamfer(self.tgt[s], self.row_mask, self.chamfer_weight, f)

    def _total(self):
        return float(self.step_loss[self.temporal_range[0]:self.temporal_range[1]].sum().item())

    def get_final_loss(self):  # shapematching_loss.py:95-106
        self.total_loss = self._total()
        self.expand_temporal_range()
        return {'loss': self.total_loss, 'last_step_loss': float(self.step_loss[self.max_loss_steps - 1].item()),
                'temporal_range': self.temporal_range[1]}

    def get_final_loss_grad(self):  # shapematching_loss.py:107-108
        self._step_grad_on[:] = False
        self._step_grad_on[self.temporal_range[0]:self.temporal_range[1]] = True

    def expand_temporal_range(self):  # shapematching_loss.py:110-130
        if self.temporal_range_type == 'expand':
            loss_improved = self.best_loss - self.total_loss
            loss_improved_rate = loss_improved / self.best_loss
            if loss_improved_rate < self.plateau_thresh[0] or loss_improved < self.plateau_thresh[1]:
                self.plateau_count += 1
            else:
                self.plateau_count = 0
            if self.best_loss > self.total_loss:
                self.best_loss = self.total_loss
            if self.plateau_count >= self.plateau_count_limit:
                self.plateau_count = 0
                self.best_loss = self.inf
                self.temporal_range[1] = min(self.max_loss_steps, self.temporal_range[1] + self.temporal_expand_speed)


class DensityMatchingLoss(ShapeMatchingLoss):
    """Correspondence-free shape loss on the simulation grid (DESIGN.md §4): the particles of `matching_mat` deposit their mass m_i on the
    nodes with p2g's weights and the step loss is  w_density sum_i (m_i - m*_i)^2 + w_sdf sum_i m_i phi*_i.  The loss depends on where mass is,
    not on which particle carries it, so the target can be a voxelised observation or a point cloud of any size (density_from_points).

    `target` (m*, mass per node) and `target_sdf` (phi*, world units) are each one volume of n_grid^3 floats used at every step, or
    max_loss_steps volumes (a recording), in read_grid()'s node order (x slowest, z fastest); either may be None (= 0).  weights:
    {'density': w_density, 'sdf': w_sdf}.  The temporal-range curriculum and the call sequence are ShapeMatchingLoss's."""

    def __init__(self, matching_mat, target=None, target_sdf=None, **kwargs):
        if kwargs.get('target_file') is not None:
            raise ValueError('DensityMatchingLoss: pass the target volumes as arrays (target=, target_sdf=)')
        super().__init__(matching_mat, target=target, **kwargs)
        self.target_sdf = target_sdf

    def build(self, sim):
        w = dict(self.weights or {})
        self.w_density, self.w_sdf = float(w.get('density', 0.0)), float(w.get('sdf', 0.0))
        if not (np.isfinite(self.w_density) and np.isfinite(self.w_sdf)):
            raise ValueError('DensityMatchingLoss: the weights must be finite')
        if self.temporal_range_type == 'last':
            self.temporal_range = [self.max_loss_steps - 1, self.max_loss_steps]
        elif self.temporal_range_type == 'all':
            self.temporal_range = [0, self.max_loss_steps]
        elif self.temporal_range_type == 'expand':
            self.temporal_range = [0, self.temporal_init_range_end]
            self.best_loss = self.inf
            self.plateau_count = 0
        self.tgt = self.sdf = None
        Loss.build(self, sim)
        if self.target_sdf is not None:
            self.sdf = self._volumes(self.target_sdf, 'target_sdf')
        self.row_mask = sim.material_row_mask(self.matching_mat)
        self._mass = torch.zeros((self.n_grid ** 3,), dtype=torch.float32, device=sim.device)

    def _volumes(self, vols, name):
        """one volume or max_loss_steps volumes of n_grid^3 finite floats -> a (1 | max_loss_steps, n_grid^3) float32 device tensor"""
        G = self.n_grid ** 3
        a = np.asarray(vols, dtype=np.float64)
        if a.size == G:
            a = a.reshape(1, G)
        elif a.size == self.max_loss_steps * G and a.shape[0] == self.max_loss_steps:
            a = a.reshape(self.max_loss_steps, G)
        else:
            raise ValueError(f'DensityMatchingLoss: {name} must be one volume of n_grid^3 = {G} values or max_loss_steps = {self.max_loss_steps} '
                             f'such volumes (got shape {a.shape})')
        if not np.isfinite(a).all():
            raise ValueError(f'DensityMatchingLoss: {name} has non-finite values')
        return torch.from_numpy(a.astype(np.float32)).to(self.sim.device)

    def set_target(self, target):
        t = self._volumes(target, 'target')
        if (t < 0).any():
            raise ValueError('DensityMatchingLoss: the target mass must be non-negative')
        self.tgt = t

    @staticmethod
    def _at(vols, s):
        return None if vols is None else vols[s if vols.shape[0] > 1 else 0]

    def compute_step_loss(self, s, f):
        self.sim.density_loss(self._mass, self._at(self.tgt, s), self._at(self.sdf, s), self.w_density, self.w_sdf, self.row_mask,
                              self.step_loss[s:s + 1], f)

    def compute_step_loss_grad(self, s, f):
        if self._step_grad_on[s]:
            self.sim.add_x_grad_density(self._mass, self._at(self.tgt, s), self._at(self.sdf, s), self.w_density, self.w_sdf, self.row_mask, f)

    @staticmethod
    def _point_stencil(points, mass, n_grid, name):
        """(kept points, mass, base (P, 3), fx (P, 3), weights (P, 3 offsets, 3 axes)) of p2g's stencil for a point cloud; points whose 3x3x3
        stencil leaves the grid are dropped"""
        x = np.asarray(points, dtype=np.float64).reshape(-1, 3)
        m = np.broadcast_to(np.asarray(mass, dtype=np.float64), (len(x),))
        if not (np.isfinite(x).all() and np.isfinite(m).all()):
            raise ValueError(f'{name}: points and mass must be finite')
        if (m < 0).any():
            raise ValueError(f'{name}: mass must be non-negative')
        g = x * float(n_grid)
        t = g - 0.5
        ok = ((t > -1.0) & (t < n_grid - 2)).all(axis=1)
        g, t, m = g[ok], t[ok], m[ok]
        base = np.trunc(t).astype(np.int64)
        fx = g - base
        w = np.stack([0.5 * (1.5 - fx) ** 2, 0.75 - (fx - 1.0) ** 2, 0.5 * (fx - 0.5) ** 2], axis=1)   # (P, 3 offsets, 3 axes)
        return ok, m, base, fx, w

    @staticmethod
    def density_from_points(points, mass, n_grid):
        """the node masses (n_grid^3 float32, read_grid() order) that a point cloud of any size deposits with the simulator's weights: dx =
        1 / n_grid, stencil base int(x / dx - 0.5) (truncation), quadratic B-spline; points whose 3x3x3 stencil leaves the grid deposit nothing.
        `mass` is one value per point or one for all (a particle's mass is p_vol * rho).  NumPy, fp64 accumulation: not for the hot path."""
        _, m, base, _, w = DensityMatchingLoss._point_stencil(points, mass, n_grid, 'density_from_points')
        out = np.zeros(n_grid ** 3, dtype=np.float64)
        for i in range(3):
            for j in range(3):
                for k in range(3):
                    node = ((base[:, 0] + i) * n_grid + base[:, 1] + j) * n_grid + base[:, 2] + k
                    np.add.at(out, node, m * w[:, i, 0] * w[:, j, 1] * w[:, k, 2])
        return out.astype(np.float32)


class MomentumMatchingLoss(DensityMatchingLoss):
    """Correspondence-free flow loss on the simulation grid (DESIGN.md §4): DensityMatchingLoss's particles also deposit p2g's APIC momentum
    P_i = sum_p m_p w_ip (v_p + C_p d_ip), d_ip = (o_i - fx_p) dx, and the step loss is
    w_density sum_i (m_i - m*_i)^2 + w_sdf sum_i m_i phi*_i + w_momentum sum_i |P_i - P*_i|^2.  It sees how the material moves where the mass
    field barely changes (a filled container, a jet), which is what a PIV or optical-flow recording, or a reference solver, observes.

    `target` (m*) and `target_sdf` (phi*) are DensityMatchingLoss's; `target_momentum` (P*) is one volume of shape (n_grid^3, 3) used at every
    step, or max_loss_steps such volumes, in read_grid()'s node order; None = 0.  From a velocity volume u*, pass P* = m* u*
    (momentum_from_points makes both from a point cloud).  weights: {'density': w_density, 'sdf': w_sdf, 'momentum': w_momentum}."""

    def __init__(self, matching_mat, target=None, target_sdf=None, target_momentum=None, **kwargs):
        super().__init__(matching_mat, target=target, target_sdf=target_sdf, **kwargs)
        self.target_momentum = target_momentum

    def build(self, sim):
        super().build(sim)   # the curriculum, w_density / w_sdf, m* (self.tgt) and phi* (self.sdf), validated and resident
        self.w_momentum = float(dict(self.weights or {}).get('momentum', 0.0))
        if not np.isfinite(self.w_momentum):
            raise ValueError('MomentumMatchingLoss: the weights must be finite')
        pm = None if self.target_momentum is None else self._momentum_volumes(self.target_momentum)
        G = self.n_grid ** 3
        self.tgt4 = None   # (1 | max_loss_steps, G, 4) float32 (P*, m*): the layout of the kernels' target
        if self.tgt is not None or pm is not None:
            S = max(1 if v is None else v.shape[0] for v in (self.tgt, pm))
            self.tgt4 = torch.zeros((S, G, 4), dtype=torch.float32, device=sim.device)
            if pm is not None:
                self.tgt4[:, :, :3] = pm
            if self.tgt is not None:
                self.tgt4[:, :, 3] = self.tgt
        self._mass = torch.zeros((G, 4), dtype=torch.float32, device=sim.device)   # the (P, m) scratch

    def _momentum_volumes(self, vols):
        G, S = self.n_grid ** 3, self.max_loss_steps
        a = np.asarray(vols, dtype=np.float64)
        if a.size == 3 * G and a.shape[-1] == 3:
            a = a.reshape(1, G, 3)
        elif a.size == 3 * S * G and a.shape[0] == S and a.shape[-1] == 3:
            a = a.reshape(S, G, 3)
        else:
            raise ValueError(f'MomentumMatchingLoss: target_momentum must be one volume of n_grid^3 = {G} momenta, shape ({G}, 3), or '
                             f'max_loss_steps = {S} such volumes (got shape {a.shape})')
        if not np.isfinite(a).all():
            raise ValueError('MomentumMatchingLoss: target_momentum has non-finite values')
        return torch.from_numpy(a.astype(np.float32)).to(self.sim.device)

    def compute_step_loss(self, s, f):
        self.sim.momentum_loss(self._mass, self._at(self.tgt4, s), self._at(self.sdf, s), self.w_density, self.w_sdf, self.w_momentum,
                               self.row_mask, self.step_loss[s:s + 1], f)

    def compute_step_loss_grad(self, s, f):
        if self._step_grad_on[s]:
            self.sim.add_grad_momentum(self._mass, self._at(self.tgt4, s), self._at(self.sdf, s), self.w_density, self.w_sdf, self.w_momentum,
                                       self.row_mask, f)

    @staticmethod
    def momentum_from_points(points, velocities, mass, n_grid, affine=None):
        """(P*, m*): the node momenta (n_grid^3, 3) and masses (n_grid^3,) float32, read_grid() order, that a point cloud of any size deposits
        with the simulator's stencil and weights (density_from_points), P_i = sum_p m_p w_ip (v_p + C_p d_ip), d_ip = (o_i - fx_p) dx.
        `velocities` is (P, 3); `affine` (P, 3, 3) adds the APIC term C_p d_ip (None = 0); `mass` is one value per point or one for all.
        NumPy, fp64 accumulation: not for the hot path."""
        x = np.asarray(points, dtype=np.float64).reshape(-1, 3)
        v = np.asarray(velocities, dtype=np.float64)
        if v.shape != x.shape:
            raise ValueError(f'momentum_from_points: velocities must have the points\' shape {x.shape} (got {v.shape})')
        c = np.zeros((len(x), 3, 3)) if affine is None else np.asarray(affine, dtype=np.float64)
        if c.shape != (len(x), 3, 3):
            raise ValueError(f'momentum_from_points: affine must have shape {(len(x), 3, 3)} (got {c.shape})')
        if not (np.isfinite(v).all() and np.isfinite(c).all()):
            raise ValueError('momentum_from_points: velocities and affine must be finite')
        ok, m, base, fx, w = DensityMatchingLoss._point_stencil(x, mass, n_grid, 'momentum_from_points')
        v, c = v[ok], c[ok]
        G = n_grid ** 3
        pm, mm = np.zeros((G, 3)), np.zeros(G)
        for i in range(3):
            for j in range(3):
                for k in range(3):
                    node = ((base[:, 0] + i) * n_grid + base[:, 1] + j) * n_grid + base[:, 2] + k
                    mw = m * w[:, i, 0] * w[:, j, 1] * w[:, k, 2]
                    d = (np.array([i, j, k], dtype=np.float64) - fx) / n_grid
                    np.add.at(mm, node, mw)
                    np.add.at(pm, node, mw[:, None] * (v + np.einsum('pab,pb->pa', c, d)))
        return pm.astype(np.float32), mm.astype(np.float32)


class LatteArtLoss(ShapeMatchingLoss):
    def __init__(self, type='diff', **kwargs):
        super().__init__(matching_mat=MILK, temporal_range_type='all', **kwargs)

    def get_step_loss(self):  # latteart_loss.py:25-33
        cur = float(self.step_loss[self.sim.cur_step_global - 1].item())
        return {'reward': 0.025 * (121.3 - cur), 'loss': 0.025 * cur}

    def get_final_loss(self):  # latteart_loss.py:35-45
        info = super().get_final_loss()
        info['reward'] = float(np.sum((121.3 - self.step_loss.cpu().numpy()) * 0.025))
        return info


class _ScaledShapeLoss(ShapeMatchingLoss):
    """ShapeMatchingLoss with a task's material, curriculum start and reward scaling (the reference repeats the class per task: the data differ, the
    kernels do not).  `type='diff'`: the expanding temporal range used by the gradient-based solver; `'default'`: the whole horizon."""
    MAT, INIT_END, OFFSET, SCALE, STEP_LOSS_SCALE = None, 50, 0.0, 1.0, 1.0

    def __init__(self, type='diff', **kwargs):
        if type == 'diff':
            super().__init__(matching_mat=self.MAT, temporal_init_range_end=self.INIT_END, temporal_range_type='expand', **kwargs)
        else:
            assert type == 'default', type
            super().__init__(matching_mat=self.MAT, temporal_range_type='all', **kwargs)

    def get_step_loss(self):
        cur = float(self.step_loss[self.sim.cur_step_global - 1].item())
        return {'reward': self.SCALE * (self.OFFSET - cur), 'loss': self.STEP_LOSS_SCALE * cur}

    def get_final_loss(self):
        info = super().get_final_loss()
        info['reward'] = float(np.sum((self.OFFSET - self.step_loss.cpu().numpy()) * self.SCALE))
        return info


class IceCreamDynamicLoss(_ScaledShapeLoss):
    """losses/icecreamdynamic_loss.py:14-60: ICECREAM particles against the recorded target, range expanding from 200 steps, reward 0.001 (1700 - loss)"""
    MAT, INIT_END, OFFSET, SCALE, STEP_LOSS_SCALE = ICECREAM, 200, 1700.0, 0.001, 0.001


class IceCreamStaticLoss(_ScaledShapeLoss):
    """losses/icecreamstatic_loss.py:13-55: ICECREAM1 particles, range expanding from 100 steps, reward 0.001 (900 - loss), the step loss unscaled"""
    MAT, INIT_END, OFFSET, SCALE, STEP_LOSS_SCALE = ICECREAM1, 100, 900.0, 0.001, 1.0


class CirculationLoss(Loss):
    """temperature loss of the air-circulation task (losses/circulation_loss.py:14-147): 15 detector cells of the smoke field at height 64;
    the first five should stay hot (|q - 1|), the others reach `target_temp` (|q - 0|).  The per-step value is 15 numbers gathered on the
    device; its seed adds sign(q - target) * weight to the smoke field's q adjoint."""
    DETECTORS = [[25, 85], [35, 85], [15, 85], [25, 75], [25, 95], [25, 42], [35, 42], [15, 42], [25, 32], [25, 52], [107, 65], [115, 65], [99, 65], [107, 45], [107, 85]]

    def __init__(self, type='diff', **kwargs):
        super().__init__(**kwargs)
        self.temporal_range_type = 'all'
        self.target_temp, self.detector_h = 0.0, 64

    def build(self, sim):
        self.temp_weight = self.weights['temp']
        self.temporal_range = [0, self.max_loss_steps]
        self.smoke_field = sim.smoke_field
        assert self.smoke_field is not None, 'CirculationLoss needs a smoke field (losses/loss.py:41-42)'
        n = self.smoke_field.n_grid
        cells = [(x * n + self.detector_h) * n + z for x, z in self.DETECTORS]
        self._cells = torch.tensor(cells, dtype=torch.long, device=sim.device)
        self._target = torch.tensor([1.0] * 5 + [self.target_temp] * 10, dtype=torch.float32, device=sim.device)
        super().build(sim)

    def compute_step_loss(self, s, f):  # circulation_loss.py:85-105: step_loss[s] += w * sum |q[s_local, cell][0] - target|
        q = self.smoke_field._q[self.sim.cur_step_local, 0]
        self.step_loss[s] += self.temp_weight * (q[self._cells] - self._target).abs().sum()

    def compute_step_loss_grad(self, s, f):
        if self._step_grad_on[s]:
            sf = self.smoke_field
            sf._ensure_grad_buffers()
            q = sf._q[self.sim.cur_step_local, 0]
            sf._gq[self.sim.cur_step_local, 0].index_add_(0, self._cells, self.temp_weight * torch.sign(q[self._cells] - self._target))

    def get_final_loss(self):  # circulation_loss.py:118-128
        self.total_loss = float(self.step_loss[self.temporal_range[0]:self.temporal_range[1]].sum().item())
        return {'loss': self.total_loss, 'last_step_loss': float(self.step_loss[self.max_loss_steps - 1].item()), 'temporal_range': self.temporal_range[1]}

    def get_final_loss_grad(self):
        self._step_grad_on[:] = False
        self._step_grad_on[self.temporal_range[0]:self.temporal_range[1]] = True

    def get_step_loss(self):  # circulation_loss.py:136-144
        cur = float(self.step_loss[self.sim.cur_step_global - 1].item())
        return {'reward': 1.0 * (11 - cur), 'loss': 1.0 * cur}
