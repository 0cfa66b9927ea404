"""CUDA-native (H100, sm_90a) MLS-MPM simulator behind the reference's `MPMSimulator` interface.

Host-side mirror of fluidlab/fluidengine/simulators/mpm_simulator.py (MPM): same constructor, `setup_boundary`,
`build`, `step`, `step_grad`, `get_state`, `set_state`, `get_x`, `get_v`, `get_used`, `get_state_RL`, `set_x`,
`set_used`, `reset_grad`, `enable_grad`/`disable_grad`, `cur_*` properties, checkpointed frame ring
(`memory_to_cache` / `memory_from_cache`, MPM:777-912).  All physics runs in libfluidmpm.so (hand-written
sm_90a CUDA, csrc/) through the C ABI of include/fluidmpm.h; torch tensors only own the device memory.

What differs from the reference by design (DESIGN.md):
  * particles are stored cell-sorted in float4 planes; the API translates to original particle order;
  * F_tmp/U/S/V and the per-frame grids are never stored — the backward recomputes them;
  * adjoints live in two ping-pong frames instead of a (T+1)-frame ring: `substep_grad(f)` reads the adjoint of
    frame f+1 and overwrites the adjoint of frame f (losses seed the *current* frame through `add_x_grad_*`);
  * checkpoints stay in HBM ('gpu', default), host RAM ('cpu') or disk ('disk') as torch tensors.
"""
import ctypes as C
import os
import uuid
from types import SimpleNamespace

import numpy as np
import torch

from . import _lib
from .boundaries import create_boundary
from .macros import MU, LAMDA, MAT_CLASS, MAT_RIGID, DTYPE_NP


class _Order:
    """slot <-> particle-id maps of one cell-sort epoch (ids[slot] = pid, inv[pid] = slot); None = identity."""
    __slots__ = ("ids", "inv")

    def __init__(self, ids=None, inv=None):
        self.ids, self.inv = ids, inv

    def ids_ptr(self):
        return None if self.ids is None else self.ids.data_ptr()

    def inv_ptr(self):
        return None if self.inv is None else self.inv.data_ptr()


_IDENTITY = _Order()


class _NPField:
    """Tiny stand-in for the Taichi fields some reference callers read with .to_numpy() (optimizer/recorder.py:59)."""

    def __init__(self, getter):
        self._getter = getter

    def to_numpy(self):
        return self._getter()


def _scene_flags(table):
    """FMPM_SCENE_* bits of a material table: every row a mu = 0 liquid (WATER / MILK / COFFEE ...) lets the fused forward substeps carry
    F = J^(1/3) I as one float (MPM:358-359) and the backward skip the SVD"""
    all_liquid = all(int(r['cls']) == 200 and float(r['mu']) == 0.0 for r in table)
    return _lib.SCENE_ALL_LIQUID_MU0 if all_liquid else 0


class MPMSimulator:
    # per-particle parameters.  What the user set, in original particle order (None = not set): the (mu, lam) field (N, 2) f32
    # (set_material_field), rho (N,) f32 with its f32 mass (set_density_field), the row limits (theta_c, theta_s) (set_plastic_limits) and the
    # per-particle limits (N, 2) f64 (set_plastic_field).  _apply_fields derives the field level of the library's kernels from them and composes
    # the (original order record, fixed slot-order buffer) pairs that level reads (_records), which _sync_field gathers in the slot order
    # `_field_ord`.  The gradient: fp32 slot-order accumulators within one sort epoch, flushed into one fp64 (N, 5) accumulator in original order
    # (_gacc: dL/d(mu, lam, m, lo, hi); _glim_orig is its (lo, hi) part) across epochs.  _lim_orig: while limits are set, the composed
    # (lo, hi) = f32(1 - theta_c), f32(1 + theta_s) of every particle.  _src: whether mu / lam and m came from user fields when the level was
    # last composed.
    _field_user = _rho_user = _mass_user = _lim_rows = _lim_user = _lim_orig = None
    _field_level, _records, _field_ord, _src = 0, (), None, (False, False)
    _field_slot = _gfield = _mass_slot = _gmass = _pfield_slot = _gpfield = _gacc = _glim_orig = None
    _gfield_dirty = False

    def __init__(self, dim, quality, gravity, horizon, max_substeps_local, max_substeps_global, ckpt_dest,
                 device=None, sort_every=1):
        assert dim == 3, 'only dim=3 is implemented (every shipped env uses 3, taichi_env.py:23)'
        self.dim = dim
        self.ckpt_dest = ckpt_dest
        self.sim_id = str(uuid.uuid4())
        self.gravity = tuple(float(g) for g in gravity)

        # MPM:21-31
        self.n_grid = int(64 * quality)
        self.dx = 1 / self.n_grid
        self.inv_dx = float(self.n_grid)
        self.dt = 2e-4
        self.p_vol = (self.dx * 0.5) ** 2
        self.res = (self.n_grid,) * self.dim
        self.max_substeps_local = max_substeps_local
        self.max_substeps_global = max_substeps_global
        self.horizon = horizon
        self.n_substeps = int(2e-3 / self.dt)
        self.max_steps_local = int(self.max_substeps_local / self.n_substeps)

        assert self.n_substeps * self.horizon < self.max_substeps_global
        assert self.max_substeps_local % self.n_substeps == 0

        self.boundary = None
        self.has_particles = False
        self.sort_every = int(sort_every)  # cell-sort period in steps (0 = never)
        self.use_graphs = True             # replay the 10 substeps of an agent-free step as one CUDA graph per local step index
        self.store_grids = 'auto'          # grad mode: keep each ring frame's forward grid in HBM instead of recomputing it in the backward:
                                           # True (raise if the ring does not fit), False, or 'auto' (if it fits); the choice made is `grids_stored`
        self.grids_stored = None
        self.fuse_g2p2g = True             # forward-only steps: the gather of substep f and the scatter of f+1 in one kernel (fmpm_substeps_fused: k_fwd, or k_g2p2g
                                           # with agents / MAT_RIGID bodies).  Frames strictly inside a step then
                                           # hold x, used and F only (all-liquid scenes: x, used, F22); step boundaries are complete.  False: plain substeps
        self.param_grad = False            # grad mode: the backward pass also accumulates dL/d(mu, lam, rho) per material row, dL/dgravity and the
                                           # contact gradients (static / rigid friction, rigid softness, restitution) (get_param_grad)
        if device is None:
            if not torch.cuda.is_available():
                raise RuntimeError('fluidlab_b200.MPMSimulator needs a CUDA device (H100, sm_90a); there is no CPU fallback')
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = torch.device(device)
        self._lib = None
        self._h = None

    # ------------------------------------------------------------------------------------------ build
    def setup_boundary(self, **kwargs):
        self.boundary = create_boundary(**kwargs)

    def build(self, agent, smoke_field, statics, particles):
        if self.boundary is None:
            self.boundary = create_boundary()
        self.n_statics = len(statics) if statics is not None else 0
        self.statics = statics
        self.smoke_field = smoke_field   # built by TaichiEnv.build after the simulator (taichi_env.py:125-126)
        self.agent = agent

        if particles is not None:
            self.has_particles = True
            self.n_particles = len(particles['x'])
            self._setup_device(particles)
        else:
            self.has_particles = False
            self.n_particles = 0
        if self.has_particles:
            self.register_colliders()
        self.actions_buffer = []
        self.ckpt_ram = dict()
        self.ckpt_dir = os.path.join('/tmp', 'fluidlab', self.sim_id)
        self.cur_substep_global = 0
        self.disable_grad()

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _ck(self, rc, what):
        _lib.check(self._lib, self._h, rc, what)

    def _setup_device(self, particles):
        lib = self._lib = _lib.load()
        dev, N, T, G = self.device, self.n_particles, self.max_substeps_local, self.n_grid ** 3
        f32, i32 = torch.float32, torch.int32

        # ---- particle info (MPM:136-175): one material-table row per distinct (material, rho)
        mat = np.asarray(particles['mat']).astype(np.int32)
        rho = np.asarray(particles['rho']).astype(DTYPE_NP)
        rows, mrow = {}, np.zeros(N, dtype=np.int32)
        keys = np.stack([mat.astype(np.float64), rho.astype(np.float64)], 1)
        uniq, inverse = np.unique(keys, axis=0, return_inverse=True)
        assert len(uniq) <= 256, 'more than 256 distinct (material, rho) pairs'
        table = np.zeros(len(uniq), dtype=[('mu', np.float32), ('lam', np.float32), ('mass', np.float32), ('cls', np.int32)])
        for r, (m, rh) in enumerate(uniq):
            m = int(m)
            table[r] = (DTYPE_NP(MU[m]), DTYPE_NP(LAMDA[m]), DTYPE_NP(self.p_vol) * DTYPE_NP(rh), MAT_CLASS[m])  # mass: MPM:174 in f32
            rows[r] = m
        mrow[:] = inverse.reshape(-1)
        self._row_material = rows
        self._row_rho = uniq[:, 1].copy()
        self._table = table
        self._mat_np = mat
        self._body_id_np = np.asarray(particles.get('body_id', np.zeros(N))).astype(np.int32)
        self.n_bodies = int(particles['bodies']['n']) if 'bodies' in particles else 1
        self._bodies_info = particles.get('bodies')
        self._materials = torch.from_numpy(table.view(np.float32).reshape(-1, 4).copy()).to(dev)
        # bodies (MPM:177-201): n_particles counts every slot of the body, mat_cls is that of its first particle.  The body id rides
        # in bits 16..23 of the particle meta word (material row in bits 8..15), see include/fluidmpm.h.
        nb = self.n_bodies
        assert nb == int(self._body_id_np.max()) + 1, 'bodies["n"] must equal max(body_id) + 1 (MPM:179)'
        binfo = np.zeros((nb, 2), dtype=np.int32)
        for b in range(nb):
            sel = np.where(self._body_id_np == b)[0]
            binfo[b] = (len(sel), MAT_CLASS[int(mat[sel[0]])] if len(sel) else 0)
        self._has_rigid_bodies = bool((binfo[:, 1] == MAT_RIGID).any())
        if self._has_rigid_bodies:
            assert nb <= 256, 'at most 256 bodies when MAT_RIGID bodies are present'
            mrow = mrow | (self._body_id_np << 8)
        self._body_info_np = binfo
        self._mrow = torch.from_numpy(mrow).to(dev)

        # ---- device buffers (torch owns the memory, the library only sees pointers)
        self._pa = torch.zeros((T + 1, 4, N, 4), dtype=f32, device=dev)
        self._pf = torch.zeros((T + 1, 2, N, 4), dtype=f32, device=dev)
        self._pf8 = torch.zeros((T + 1, N), dtype=f32, device=dev)
        self._grid_pm = torch.zeros((G, 4), dtype=f32, device=dev)
        self._grid_v = torch.zeros((G, 4), dtype=f32, device=dev)
        self._scratch_a = torch.empty((4, N, 4), dtype=f32, device=dev)
        self._scratch_f = torch.empty((2, N, 4), dtype=f32, device=dev)
        self._scratch_f8 = torch.empty((N,), dtype=f32, device=dev)
        self._sort_bufs = [torch.empty((N,), dtype=i32, device=dev) for _ in range(4)]
        assert self.n_grid % 8 == 0, 'n_grid must be a multiple of 8 (sparse grid blocks are 8x8x8 nodes)'
        nblk = (self.n_grid // 8) ** 3
        self._blk_flags = torch.zeros((nblk,), dtype=i32, device=dev)
        self._blk_list = torch.zeros((nblk,), dtype=i32, device=dev)
        self._blk_count = torch.zeros((1,), dtype=i32, device=dev)
        # forward-only fused substeps with grid_op inlined (csrc/fmpm_forward.cu: k_fwd): three accumulators + their block flags
        self._grid_pm3 = torch.zeros((3, G, 4), dtype=f32, device=dev)
        self._blk_flags3 = torch.zeros((3, nblk), dtype=i32, device=dev)
        self._ga = self._gf = self._gf8 = self._ggrid_v = self._ggrid_pm = None
        self._gmat = self._ggrav = self._gcontact = None   # fp64 parameter-gradient accumulators (param_grad)
        self._pg_bound = False
        self._pm_ring = self._v_ring = self._blk_list_ring = self._blk_count_ring = None
        self._ring_valid = [False] * T
        # API-layout staging
        self._sx = torch.empty((N, 3), dtype=f32, device=dev); self._sv = torch.empty((N, 3), dtype=f32, device=dev)
        self._sC = torch.empty((N, 3, 3), dtype=f32, device=dev); self._sF = torch.empty((N, 3, 3), dtype=f32, device=dev)
        self._sused = torch.empty((N,), dtype=i32, device=dev)

        cfg = _lib.FmpmConfig()
        cfg.n_grid, cfg.n_particles, cfg.max_substeps_local, cfg.n_substeps = self.n_grid, N, T, self.n_substeps
        cfg.dt, cfg.dx, cfg.inv_dx, cfg.p_vol = self.dt, self.dx, self.inv_dx, self.p_vol
        cfg.k_stress = -self.dt * self.p_vol * 4 * self.inv_dx * self.inv_dx  # MPM:343, double then rounded to f32
        cfg.gravity = (C.c_float * 3)(*self.gravity)
        b = self.boundary
        cfg.boundary_type = b.type_id
        cfg.b_lower = (C.c_float * 3)(*[float(v) for v in b.lower]); cfg.b_upper = (C.c_float * 3)(*[float(v) for v in b.upper])
        cfg.cyl_center = (C.c_float * 2)(*[float(v) for v in b.xz_center]); cfg.cyl_radius = float(b.xz_radius)
        cfg.restitution = b.restitution; cfg.lock_mask = b.lock_mask
        cfg.n_materials = len(uniq)
        cfg.device = self.device.index if self.device.index is not None else torch.cuda.current_device()
        cfg.scene_flags = _scene_flags(table)
        h = C.c_void_p()
        rc = lib.fmpm_create(C.byref(cfg), C.byref(h))
        self._h = h
        self._ck(rc, 'fmpm_create')
        self._sort_tmp = torch.empty((int(lib.fmpm_sort_workspace_bytes(h)),), dtype=torch.uint8, device=dev)
        if os.environ.get('FMPM_FWD_MASK'):   # A/B of the forward kernels (profiles/): bit 0 k_fwd, 1 liquid specialisation, 2 inlined grid_op, 3 TMA tiles
            self._ck(lib.fmpm_set_fwd_mask(h, int(os.environ['FMPM_FWD_MASK'])), 'fmpm_set_fwd_mask')
        self._bind()
        if self._has_rigid_bodies:
            self._body_info = torch.from_numpy(self._body_info_np).to(dev)
            self._body_state = torch.zeros((T, self.n_bodies, _lib.BODY_STATE_STRIDE), dtype=f32, device=dev)
            self._body_grad = torch.zeros((self.n_bodies, _lib.BODY_GRAD_STRIDE), dtype=f32, device=dev)
            bd = _lib.FmpmBodies()
            bd.n_bodies, bd.info, bd.state, bd.grad = self.n_bodies, self._body_info.data_ptr(), self._body_state.data_ptr(), self._body_grad.data_ptr()
            self._ck(lib.fmpm_set_bodies(h, C.byref(bd)), 'fmpm_set_bodies')

        # ---- initial frame (init_particles_kernel MPM:150-175): v = 0, F = I, C = 0
        x0 = np.asarray(particles['x']).astype(DTYPE_NP)
        used0 = np.asarray(particles['used']).astype(np.int32)
        self._frame_ord = [_IDENTITY] * (T + 1)
        self._gcur, self._grad_ord = 0, _IDENTITY
        self.setframe(0, x0, np.zeros((N, 3), DTYPE_NP), np.zeros((N, 3, 3), DTYPE_NP),
                      np.tile(np.eye(3, dtype=DTYPE_NP), (N, 1, 1)), used0)
        self.particles_i = SimpleNamespace(mat=_NPField(lambda: self._mat_np.copy()))
        self.particles_ng = SimpleNamespace(used=_NPField(lambda: np.stack([self.get_used(f) for f in range(1)])))

    def _bind(self):
        b = _lib.FmpmBuffers()
        p = lambda t: None if t is None else t.data_ptr()
        b.pa, b.pf, b.pf8 = p(self._pa), p(self._pf), p(self._pf8)
        b.ga, b.gf, b.gf8 = p(self._ga), p(self._gf), p(self._gf8)
        b.grid_pm, b.grid_v, b.ggrid_v, b.ggrid_pm = p(self._grid_pm), p(self._grid_v), p(self._ggrid_v), p(self._ggrid_pm)
        b.materials = p(self._materials)
        b.scratch_a, b.scratch_f, b.scratch_f8 = p(self._scratch_a), p(self._scratch_f), p(self._scratch_f8)
        b.sort_keys_in, b.sort_keys_out, b.sort_vals_in, b.sort_vals_out = [p(t) for t in self._sort_bufs]
        b.sort_tmp, b.sort_tmp_bytes = p(self._sort_tmp), self._sort_tmp.numel()
        b.blk_flags, b.blk_list, b.blk_count = p(self._blk_flags), p(self._blk_list), p(self._blk_count)
        b.grid_pm_ring, b.grid_v_ring = p(self._pm_ring), p(self._v_ring)
        b.blk_list_ring, b.blk_count_ring = p(self._blk_list_ring), p(self._blk_count_ring)
        b.grid_pm3, b.blk_flags3 = p(getattr(self, '_grid_pm3', None)), p(getattr(self, '_blk_flags3', None))
        self._ck(self._lib.fmpm_bind(self._h, C.byref(b)), 'fmpm_bind')

    def register_colliders(self):
        """(re)send the SDF colliders to the library: statics with dynamics (MPM:388-390) and the agent's Rigid mesh
        (agents/agent_rigid.py:21-23).  Called at build and again by AgentRigid.build once its effector owns device arrays."""
        col = _lib.FmpmColliders()
        dyn = [s for s in (self.statics or []) if getattr(s, 'has_dynamics', False)]
        assert len(dyn) <= 4, 'at most 4 colliding statics'
        col.n_statics = len(dyn)
        col.collide_y_min = float(getattr(self.agent, 'collide_y_min', -1e30)) if self.agent is not None else -1e30
        for i, s in enumerate(dyn):
            col.statics[i] = s.device_struct(_lib, self.device)
        rigid = getattr(self.agent, 'rigid', None) if self.agent is not None else None
        if rigid is not None and getattr(rigid, 'pos', None) is not None:
            col.has_rigid = 1
            col.collide_type = {'particle': 0, 'grid': 1, 'both': 2}[self.agent.collide_type]
            col.rigid = rigid.mesh.device_struct(_lib, self.device)
            col.pos, col.quat, col.gpos, col.gquat = rigid.pos.data_ptr(), rigid.quat.data_ptr(), rigid.gpos.data_ptr(), rigid.gquat.data_ptr()
        self._colliders = col  # keep the voxel tensors alive through the mesh objects
        self._ck(self._lib.fmpm_set_colliders(self._h, C.byref(col)), 'fmpm_set_colliders')

    def _ensure_grad_buffers(self):
        if self._ga is None:
            N, G, dev, f32 = self.n_particles, self.n_grid ** 3, self.device, torch.float32
            self._ga = torch.zeros((2, 4, N, 4), dtype=f32, device=dev)
            self._gf = torch.zeros((2, 2, N, 4), dtype=f32, device=dev)
            self._gf8 = torch.zeros((2, N), dtype=f32, device=dev)
            if getattr(self, '_ggrid_v', None) is None:   # x-slab peer mode pre-binds a buffer in symmetric memory (slab.py)
                self._ggrid_v = torch.zeros((G, 4), dtype=f32, device=dev)
            self._ggrid_pm = torch.zeros((G, 4), dtype=f32, device=dev)
            # per-frame forward grids for the backward pass (like the reference's grid ring, MPM:117) when HBM allows:
            # 32 B/node/frame; otherwise substep_grad recomputes the forward grid of each frame
            T = self.max_substeps_local
            need = T * G * 32
            free, _ = torch.cuda.mem_get_info(dev)
            fits = need < 0.35 * free
            if self.store_grids is True and not fits:
                raise RuntimeError(f'store_grids=True: the per-frame grid ring needs {need / 2**30:.1f} GiB, only {free / 2**30:.1f} GiB are free (use "auto" or False)')
            self.grids_stored = bool(self.store_grids) and fits
            if self.grids_stored:
                nblk = (self.n_grid // 8) ** 3
                self._pm_ring = torch.zeros((T, G, 4), dtype=f32, device=dev)
                self._v_ring = torch.zeros((T, G, 4), dtype=f32, device=dev)
                self._blk_list_ring = torch.zeros((T, nblk), dtype=torch.int32, device=dev)
                self._blk_count_ring = torch.zeros((T,), dtype=torch.int32, device=dev)
            self._bind()
        self._sync_param_grad()

    def _sync_param_grad(self):
        """bind the parameter-gradient accumulators to the library while `param_grad` is set, unbind them when it is cleared"""
        want = bool(self.param_grad)
        if want and self._gmat is None:
            self._gmat = torch.zeros((len(self._table), 4), dtype=torch.float64, device=self.device)
            self._ggrav = torch.zeros((3,), dtype=torch.float64, device=self.device)
            self._gcontact = torch.zeros((8,), dtype=torch.float64, device=self.device)   # FmpmContactGrad layout
        if want != self._pg_bound:
            pg, cg = _lib.FmpmParamGrad(), _lib.FmpmContactGrad()
            if want:
                pg.gmat, pg.ggrav = self._gmat.data_ptr(), self._ggrav.data_ptr()
                cg.gcontact = self._gcontact.data_ptr()
            self._ck(self._lib.fmpm_set_param_grad(self._h, C.byref(pg)), 'fmpm_set_param_grad')   # unbinding it also unbinds the contact array
            self._ck(self._lib.fmpm_set_contact_grad(self._h, C.byref(cg)), 'fmpm_set_contact_grad')
            self._pg_bound = want

    def __del__(self):
        try:
            if self._h is not None and self._lib is not None:
                self._lib.fmpm_destroy(self._h)
        except Exception:
            pass

    # ------------------------------------------------------------------------------------------ grads
    def reset_grad(self):  # MPM:203-205
        if not self.has_particles:
            return
        self._ensure_grad_buffers()
        self._ga.zero_(); self._gf.zero_(); self._gf8.zero_()
        if self._gmat is not None:
            self._gmat.zero_(); self._ggrav.zero_(); self._gcontact.zero_()
        for g in (self._gfield, self._gmass, self._gpfield, self._gacc):
            if g is not None:
                g.zero_()
        self._gfield_dirty = False
        self._gcur = 0
        self._grad_ord = self._frame_ord[self.cur_substep_local]

    def enable_grad(self):  # MPM:207-212
        self.grad_enabled = True
        self.cur_substep_global = 0

    def disable_grad(self):  # MPM:214-216
        self.grad_enabled = False
        self.cur_substep_global = 0

    def _ensure_grad_order(self, order):
        """Re-express the current adjoint buffer in the slot order `order` (no-op when it already is)."""
        if self._grad_ord is order:
            return
        src, dst = self._gcur, 1 - self._gcur
        self._ck(self._lib.fmpm_permute_grad(self._h, src, dst, self._grad_ord.ids_ptr(), order.inv_ptr(), self._stream()), 'fmpm_permute_grad')
        self._gcur, self._grad_ord = dst, order

    def add_x_grad_chamfer(self, tgt_dev, row_mask, weight, f=None):
        """Seed of losses/shapematching_loss.py:80-84 (.grad): gx[f] += 2 w (x[f] - tgt) on the current adjoint frame."""
        f = self.cur_substep_local if f is None else f
        self._ensure_grad_order(self._frame_ord[f])
        self._ck(self._lib.fmpm_loss_chamfer_grad(self._h, f, self._gcur, self._grad_ord.ids_ptr(), tgt_dev.data_ptr(), int(row_mask),
                                                  float(weight), self._stream()), 'fmpm_loss_chamfer_grad')

    def chamfer_loss(self, tgt_dev, row_mask, weight, out_dev, f=None):
        """out_dev[0] += w * sum |x[f,p] - tgt[p]|^2 over used particles whose material row is in row_mask."""
        f = self.cur_substep_local if f is None else f
        self._ck(self._lib.fmpm_loss_chamfer(self._h, f, self._frame_ord[f].ids_ptr(), tgt_dev.data_ptr(), int(row_mask), float(weight),
                                             out_dev.data_ptr(), self._stream()), 'fmpm_loss_chamfer')

    @staticmethod
    def _density_args(mass_dev, target_dev, sdf_dev, w_density, w_sdf, row_mask):
        l = _lib.FmpmDensityLoss()
        l.mass = mass_dev.data_ptr()
        l.target = None if target_dev is None else target_dev.data_ptr()
        l.sdf = None if sdf_dev is None else sdf_dev.data_ptr()
        l.w_density, l.w_sdf, l.mrow_mask_lo = float(w_density), float(w_sdf), int(row_mask)
        return l

    def density_loss(self, mass_dev, target_dev, sdf_dev, w_density, w_sdf, row_mask, out_dev, f=None):
        """out_dev[0] += w_density sum_i (m_i - target_i)^2 + w_sdf sum_i m_i sdf_i, m = the grid mass that the used particles of frame f whose
        material row is in row_mask deposit with p2g's weights.  Volumes are float32 (n_grid^3,) on the device in read_grid()'s node order,
        target / sdf None = 0; mass_dev is a float32 (n_grid^3,) scratch that the call overwrites."""
        f = self.cur_substep_local if f is None else f
        self._sync_mass_field(f)
        l = self._density_args(mass_dev, target_dev, sdf_dev, w_density, w_sdf, row_mask)
        self._ck(self._lib.fmpm_loss_density(self._h, f, C.byref(l), out_dev.data_ptr(), self._stream()), 'fmpm_loss_density')

    def add_x_grad_density(self, mass_dev, target_dev, sdf_dev, w_density, w_sdf, row_mask, f=None):
        """Seed of density_loss: gx[f] += dL/dx on the current adjoint frame and, while param_grad is set, dL/drho of the rows (per particle
        while a density field is set) through the deposited mass."""
        f = self.cur_substep_local if f is None else f
        self._ensure_grad_order(self._frame_ord[f])
        self._sync_mass_field(f, grad=True)
        l = self._density_args(mass_dev, target_dev, sdf_dev, w_density, w_sdf, row_mask)
        self._ck(self._lib.fmpm_loss_density_grad(self._h, f, self._gcur, C.byref(l), self._stream()), 'fmpm_loss_density_grad')

    @staticmethod
    def _momentum_args(field_dev, target_dev, sdf_dev, w_density, w_sdf, w_momentum, row_mask):
        l = _lib.FmpmMomentumLoss()
        l.field = field_dev.data_ptr()
        l.target = None if target_dev is None else target_dev.data_ptr()
        l.sdf = None if sdf_dev is None else sdf_dev.data_ptr()
        l.w_density, l.w_sdf, l.w_momentum, l.mrow_mask_lo = float(w_density), float(w_sdf), float(w_momentum), int(row_mask)
        return l

    def momentum_loss(self, field_dev, target_dev, sdf_dev, w_density, w_sdf, w_momentum, row_mask, out_dev, f=None):
        """out_dev[0] += w_density sum_i (m_i - m*_i)^2 + w_sdf sum_i m_i sdf_i + w_momentum sum_i |P_i - P*_i|^2, (P, m) = the APIC momentum and
        the mass that the particles of density_loss deposit with p2g's weights (P_i = sum_p m_p w_ip (v_p + C_p d_ip)).  target_dev is float32
        (n_grid^3, 4) = (P*, m*) and sdf_dev float32 (n_grid^3,) on the device in read_grid()'s node order, None = 0; field_dev is a float32
        (n_grid^3, 4) scratch that the call overwrites."""
        f = self.cur_substep_local if f is None else f
        self._sync_mass_field(f)
        l = self._momentum_args(field_dev, target_dev, sdf_dev, w_density, w_sdf, w_momentum, row_mask)
        self._ck(self._lib.fmpm_loss_momentum(self._h, f, C.byref(l), out_dev.data_ptr(), self._stream()), 'fmpm_loss_momentum')

    def add_grad_momentum(self, field_dev, target_dev, sdf_dev, w_density, w_sdf, w_momentum, row_mask, f=None):
        """Seed of momentum_loss: gx, gv, gC[f] += dL/d(x, v, C) on the current adjoint frame and, while param_grad is set, dL/drho of the rows
        through the deposited mass and momentum (per particle while a density field is set)."""
        f = self.cur_substep_local if f is None else f
        self._ensure_grad_order(self._frame_ord[f])
        self._sync_mass_field(f, grad=True)
        l = self._momentum_args(field_dev, target_dev, sdf_dev, w_density, w_sdf, w_momentum, row_mask)
        self._ck(self._lib.fmpm_loss_momentum_grad(self._h, f, self._gcur, C.byref(l), self._stream()), 'fmpm_loss_momentum_grad')

    def _sync_mass_field(self, f, grad=False):
        """the losses read the particles' mass, per slot from field level 2 on"""
        if self._field_level >= 2:
            self._touch_frame(f, grad)

    def material_row_mask(self, material):
        m = 0
        for r, mat in self._row_material.items():
            if mat == material:
                assert r < 32
                m |= 1 << r
        return m

    # ------------------------------------------------------------------------------------------ physical parameters and their gradients
    def get_material_table(self):
        """the material rows as they are now (one per distinct (material, rho) of the scene): dict of arrays `mat` (material id), `rho`, `mu`, `lam`"""
        t = self._table
        return dict(mat=np.array([self._row_material[r] for r in range(len(t))], dtype=np.int32), rho=self._row_rho.astype(np.float64),
                    mu=t['mu'].astype(np.float64), lam=t['lam'].astype(np.float64))

    def set_material_table(self, mu=None, lam=None, rho=None):
        """overwrite mu, lam and / or rho of every row (arrays aligned with get_material_table()); the mass of a row is p_vol * rho in f32 as at
        build (MPM:174).  Takes effect for the steps that follow; call it between steps, not inside a backward pass over steps taken before.
        While a material field (set_material_field) is set the rows' mu and lam do not enter the dynamics, and while a density field
        (set_density_field) is set the rows' rho does not."""
        mu = None if mu is None else self._per_row('set_material_table', 'mu', mu, finite=True)
        lam = None if lam is None else self._per_row('set_material_table', 'lam', lam, finite=True)
        rho = None if rho is None else self._per_row('set_material_table', 'rho', rho, finite=True)
        if rho is not None and not (rho > 0).all():
            raise ValueError('set_material_table: rho must be positive')
        t = self._table.copy()
        if mu is not None:
            t['mu'] = mu.astype(np.float32)
        if lam is not None:
            t['lam'] = lam.astype(np.float32)
        if rho is not None:
            t['mass'] = DTYPE_NP(self.p_vol) * rho.astype(DTYPE_NP)
            self._row_rho = rho.copy()
        self._table = t
        self._materials.copy_(torch.from_numpy(t.view(np.float32).reshape(-1, 4).copy()))
        # the bound level reads mu, lam (from level 1) or the mass (from level 2) per slot, from the rows where no user field is set
        if (self._field_level >= 1 and self._field_user is None and (mu is not None or lam is not None)) or \
                (self._field_level >= 2 and self._rho_user is None and rho is not None):
            self._apply_fields()
        self._ck(self._lib.fmpm_set_scene_flags(self._h, self._scene_flags()), 'fmpm_set_scene_flags')
        self._graphs = {}   # the forward kernels chosen from the scene flags are baked into the captured graphs

    def _scene_flags(self):
        return 0 if self._field_level else _scene_flags(self._table)   # a bound field always runs the general kernels

    def _per_row(self, what, name, a, finite=False):
        """a float64 copy of `a`, checked to hold one value per row of get_material_table()"""
        n = len(self._table)
        a = np.array(a, dtype=np.float64).reshape(-1)
        if a.shape != (n,) or (finite and not np.isfinite(a).all()):
            raise ValueError(f'{what}: {name} must hold {n} {"finite " if finite else ""}values (one per row of get_material_table())')
        return a

    def _per_particle(self, what, name, a, finite=False):
        """`a` (NumPy, or torch on any device) as a float64 tensor on the device, checked to have one value per particle"""
        N = self.n_particles
        t = (a.detach() if torch.is_tensor(a) else torch.as_tensor(np.asarray(a))).to(self.device, torch.float64)
        if tuple(t.shape) != (N,):
            raise ValueError(f'{what}: {name} must have shape ({N},), got {tuple(t.shape)}')
        if finite and not bool(torch.isfinite(t).all()):
            raise ValueError(f'{what}: {name} must be finite')
        return t

    def set_material_field(self, mu, lam):
        """mu and lam per particle: two arrays of shape (N,) in original particle order (NumPy, or torch on any device), finite, mu >= 0.  While
        a field is set every constitutive evaluation of particle p (forward, recompute and backward) uses (mu[p], lam[p]) instead of its material
        row's; the mass (rho, unless set_density_field is set), the material class and the loss row masks still come from the row.  With
        param_grad, get_param_grad() then also
        returns `mu_field` / `lam_field` (dL/d of every particle's value) and its row keys `mu` / `lam` become the sums of those over each row's
        particles.  Like set_material_table: call it between steps, not inside a backward pass over steps taken before."""
        if not self.has_particles:
            raise RuntimeError('set_material_field: the scene has no particles')
        mu = self._per_particle('set_material_field', 'mu', mu, finite=True)
        lam = self._per_particle('set_material_field', 'lam', lam, finite=True)
        if bool((mu < 0).any()):
            raise ValueError('set_material_field: mu must be >= 0')
        self._field_user = torch.stack([mu, lam], 1).to(torch.float32)
        self._apply_fields()

    def clear_material_field(self):
        """back to the material table's mu and lam.  dL/dmu, dL/dlam accumulated while the field was bound stay in get_param_grad()'s row keys
        `mu` / `lam` (their sums over each row); `mu_field` / `lam_field` are only returned while a field is bound."""
        if self._field_user is None:
            return
        self._field_user = None
        self._apply_fields()

    def get_material_field(self):
        """the bound field as (mu, lam): float32 NumPy arrays (N,) in original particle order, or None without a field"""
        if self._field_user is None:
            return None
        f = self._field_user.cpu().numpy()
        return f[:, 0].copy(), f[:, 1].copy()

    def set_density_field(self, rho):
        """rho per particle: an array of shape (N,) in original particle order (NumPy, or torch on any device), finite, > 0.  While it is set,
        particle p has the mass m_p = p_vol * rho[p] (in f32, as the rows' mass) wherever a mass is read: the forward scatter, the recompute and
        the backward, and the deposits and adjoints of the density and momentum losses.  The material class and the loss row masks still come
        from the row, and set_material_table(rho=...) does not change the dynamics while a density field is set.  It is independent of
        set_material_field.  With param_grad, get_param_grad() then also returns `rho_field` (dL/drho of every particle, the losses' direct mass
        terms included) and its row key `rho` adds the sums of those over each row's particles.  Call it between steps, as set_material_table."""
        if not self.has_particles:
            raise RuntimeError('set_density_field: the scene has no particles')
        t = self._per_particle('set_density_field', 'rho', rho)
        # checked on what the kernels read: rho and the mass p_vol * rho, both in f32 (a finite, positive float64 can round to 0 or inf)
        rho32 = t.to(torch.float32)
        mass32 = torch.tensor(float(DTYPE_NP(self.p_vol)), dtype=torch.float32, device=self.device) * rho32   # MPM:174 in f32
        if not (bool(torch.isfinite(rho32).all()) and bool(torch.isfinite(mass32).all())):
            raise ValueError('set_density_field: rho must be finite, and so must p_vol * rho in float32')
        if not (bool((rho32 > 0).all()) and bool((mass32 > 0).all())):
            raise ValueError('set_density_field: rho must be > 0, and so must p_vol * rho in float32')
        self._rho_user, self._mass_user = rho32, mass32
        self._apply_fields()

    def clear_density_field(self):
        """back to the rows' rho.  dL/drho accumulated while the field was set stays in get_param_grad()'s row key `rho` (its sums over each
        row); `rho_field` is only returned while a density field is set."""
        if self._rho_user is None:
            return
        self._rho_user = self._mass_user = None
        self._apply_fields()

    def get_density_field(self):
        """the bound rho as a float32 NumPy array (N,) in original particle order, or None without a density field"""
        return None if self._rho_user is None else self._rho_user.cpu().numpy().copy()

    # plastic yield limits: a plasto-elastic particle (ICECREAM, ICECREAM1, PLASTIC_DEMO) clamps the singular values of its deformation gradient to
    # [1 - theta_c, 1 + theta_s] (MPM:367-376: theta_c = 2e-3, theta_s = 3e-3)
    THETA_C, THETA_S = 2e-3, 3e-3

    def _limits(self, name, tc, ts):
        """(lo, hi) = f32(1 - theta_c), f32(1 + theta_s) as the kernels read them (float64 tensors in, float32 out), checked"""
        if not (bool(torch.isfinite(tc).all()) and bool(torch.isfinite(ts).all())):
            raise ValueError(f'{name}: theta_c and theta_s must be finite')
        lo, hi = (1.0 - tc).to(torch.float32), (1.0 + ts).to(torch.float32)
        if not (bool((tc >= 0).all()) and bool((tc < 1).all()) and bool((lo > 0).all())):
            raise ValueError(f'{name}: theta_c must be >= 0 and < 1, with 1 - theta_c > 0 in float32')
        if not (bool((ts >= 0).all()) and bool(torch.isfinite(hi).all())):
            raise ValueError(f'{name}: theta_s must be >= 0, with 1 + theta_s finite in float32')
        return lo, hi

    def get_plastic_limits(self):
        """the per-row limits: dict of float64 arrays `theta_c`, `theta_s` aligned with get_material_table() (the defaults 2e-3 / 3e-3 when
        set_plastic_limits was not called)"""
        if self._lim_rows is None:
            n = len(self._table)
            return dict(theta_c=np.full(n, self.THETA_C), theta_s=np.full(n, self.THETA_S))
        return dict(theta_c=self._lim_rows[0].copy(), theta_s=self._lim_rows[1].copy())

    def set_plastic_limits(self, theta_c=None, theta_s=None):
        """overwrite the plastic yield limits of every row (arrays aligned with get_material_table(); None keeps the current value): the particles
        of a plasto-elastic row clamp their singular values to [lo, hi] = [f32(1 - theta_c), f32(1 + theta_s)] (computed in float64, rounded to
        float32), 0 <= theta_c < 1, theta_s >= 0; the rows of other classes never read them.  A per-particle field (set_plastic_field) overrides
        the rows.  With param_grad, get_param_grad() then also returns `theta_c` / `theta_s`, dL/d of each row's limits (the sums over its
        particles, dL/dtheta_c = -dL/dlo).  Call it between steps, as set_material_table."""
        if not self.has_particles:
            raise RuntimeError('set_plastic_limits: the scene has no particles')
        cur = self.get_plastic_limits()
        tc = cur['theta_c'] if theta_c is None else self._per_row('set_plastic_limits', 'theta_c', theta_c)
        ts = cur['theta_s'] if theta_s is None else self._per_row('set_plastic_limits', 'theta_s', theta_s)
        self._limits('set_plastic_limits', torch.from_numpy(tc), torch.from_numpy(ts))
        self._lim_rows = (tc, ts)
        self._apply_fields()

    def clear_plastic_limits(self):
        """back to the default limits of every row.  Without a per-particle field the plasto-elastic particles then run the kernels with the
        constant clamp again, and `theta_c` / `theta_s` leave get_param_grad() (the gradient accumulated for them is dropped)"""
        if self._lim_rows is None:
            return
        self._lim_rows = None
        self._apply_fields()

    def set_plastic_field(self, theta_c, theta_s):
        """the plastic yield limits per particle: two arrays of shape (N,) in original particle order (NumPy, or torch on any device), with the
        rules of set_plastic_limits; they override the rows' limits.  With param_grad, get_param_grad() then also returns `theta_c_field` /
        `theta_s_field` (dL/d of every particle's value), and its row keys `theta_c` / `theta_s` are the sums of those over each row's particles.
        Independent of set_material_field and set_density_field: any of the three can be set and cleared in any order.  Call it between steps."""
        if not self.has_particles:
            raise RuntimeError('set_plastic_field: the scene has no particles')
        tc, ts = self._per_particle('set_plastic_field', 'theta_c', theta_c), self._per_particle('set_plastic_field', 'theta_s', theta_s)
        self._limits('set_plastic_field', tc, ts)
        self._lim_user = torch.stack([tc, ts], 1)
        self._apply_fields()

    def clear_plastic_field(self):
        """back to the rows' limits (set_plastic_limits).  The gradient accumulated while the field was set stays in the row keys `theta_c` /
        `theta_s` while row limits are set; `theta_c_field` / `theta_s_field` are only returned while a field is set."""
        if self._lim_user is None:
            return
        self._lim_user = None
        self._apply_fields()

    def get_plastic_field(self):
        """the per-particle limits as (theta_c, theta_s): float64 NumPy arrays (N,) in original particle order, or None without a field"""
        if self._lim_user is None:
            return None
        t = self._lim_user.cpu().numpy()
        return t[:, 0].copy(), t[:, 1].copy()

    # the library's field levels 1 .. 3, each bound over the one below: its setter and struct, and the slot-order buffer and fp32 gradient
    # accumulator (their shape per particle) it takes
    _FIELD_BINDINGS = (('fmpm_set_material_field', _lib.FmpmMaterialField, '_field_slot', '_gfield', (2,)),
                       ('fmpm_set_mass_field', _lib.FmpmMassField, '_mass_slot', '_gmass', ()),
                       ('fmpm_set_plastic_field', _lib.FmpmPlasticField, '_pfield_slot', '_gpfield', (4,)))

    def _apply_fields(self):
        """Bind what the user set.  The field level is 3 with any limits, else 2 with rho, else 1 with (mu, lam), else 0; every value the level
        reads comes from the user's field where one is set and from the rows otherwise:
          level 1: (mu, lam) per slot (_field_slot);  level 2: and the mass (_mass_slot);  level 3: the mass and the (mu, lam, lo, hi) record
          (_pfield_slot; the kernels of level 3 read no _field_slot, which stays bound because the library nests the levels).
        The gradients accumulated so far are flushed first.  dL/d(mu, lam) and dL/dm move into the rows' accumulator when their source changes
        between the rows and a user field, so that the field keys hold only what was accumulated while the user's field was set; the row keys
        count them either way.  dL/d(lo, hi) is dropped with the last limits."""
        self._flush_field_grad()
        N, dev = self.n_particles, self.device
        if self._gacc is None:
            self._gacc = torch.zeros((N, 5), dtype=torch.float64, device=dev)
            self._glim_orig = self._gacc[:, 3:]
        row = (self._mrow & 0xff).long()
        src = (self._field_user is not None, self._rho_user is not None)
        for c in ([0, 1] if src[0] != self._src[0] else []) + ([2] if src[1] != self._src[1] else []):
            if self._gmat is not None:
                self._gmat[:, c].index_add_(0, row, self._gacc[:, c])
            self._gacc[:, c].zero_()
        self._src = src
        limits = self._lim_rows is not None or self._lim_user is not None
        if not limits:
            self._glim_orig.zero_()
        level = 3 if limits else 2 if src[1] else 1 if src[0] else 0

        for _, _, slot, grad, shape in self._FIELD_BINDINGS[:level]:
            if getattr(self, slot) is None:   # fixed buffers: captured graphs and the library keep their pointers
                setattr(self, slot, torch.empty((N,) + shape, dtype=torch.float32, device=dev))
                setattr(self, grad, torch.zeros((N,) + shape, dtype=torch.float32, device=dev))
        records = []
        if level:
            t = self._table
            mulam = self._field_user if src[0] else torch.from_numpy(np.stack([t['mu'], t['lam']], 1)).to(dev)[row]
        if level in (1, 2):
            records.append((mulam, self._field_slot))
        if level >= 2:
            records.append((self._mass_user if src[1] else torch.from_numpy(t['mass'].copy()).to(dev)[row], self._mass_slot))
        self._lim_orig = None
        if level == 3:
            if self._lim_user is not None:
                lo, hi = self._limits('set_plastic_field', self._lim_user[:, 0], self._lim_user[:, 1])
            else:
                rl, rh = self._limits('set_plastic_limits', torch.from_numpy(self._lim_rows[0]), torch.from_numpy(self._lim_rows[1]))
                lo, hi = rl.to(dev)[row], rh.to(dev)[row]
            self._lim_orig = torch.stack([lo, hi], 1)
            records.append((torch.cat([mulam, self._lim_orig], 1), self._pfield_slot))

        self._ck(self._lib.fmpm_set_scene_flags(self._h, 0), 'fmpm_set_scene_flags')   # (the library binds no material field under the all-liquid flag)
        for lv in range(self._field_level, level, -1):   # down: plastic, then mass, then material
            name = self._FIELD_BINDINGS[lv - 1][0]
            self._ck(getattr(self._lib, name)(self._h, None), name)
        for lv in range(self._field_level + 1, level + 1):   # up: material, then mass, then plastic
            name, struct, slot, grad, _ = self._FIELD_BINDINGS[lv - 1]
            self._ck(getattr(self._lib, name)(self._h, C.byref(struct(getattr(self, slot).data_ptr(), getattr(self, grad).data_ptr()))), name)
        self._field_level, self._records = level, records
        self._ck(self._lib.fmpm_set_scene_flags(self._h, self._scene_flags()), 'fmpm_set_scene_flags')
        self._field_ord = None   # re-gathered before the next launch
        self._graphs = {}   # the kernel choice is baked into the captured graphs

    def _touch_frame(self, f, grad=False):
        """a launch on frame f follows: keep the bound records in its slot order; grad: the launch accumulates parameter gradients into them"""
        if self._field_level:
            self._sync_field(self._frame_ord[f])
            self._gfield_dirty = self._gfield_dirty or (grad and self._pg_bound)

    def _sync_field(self, order):
        """Keep the bound records in the slot order `order` (the frame about to be processed), like _ensure_grad_order keeps the adjoint: the
        gradient accumulated in the old order is flushed first."""
        if not self._field_level or self._field_ord is order:
            return
        self._flush_field_grad()
        ids = None if order.ids is None else order.ids.long()
        for rec, slot in self._records:
            if ids is None:
                slot.copy_(rec)
            else:
                torch.index_select(rec, 0, ids, out=slot)
        self._field_ord = order

    def _flush_field_grad(self):
        """the bound level's fp32 slot-order gradients -> _gacc (scattered through the order they were accumulated in), then zeroed"""
        if not self._gfield_dirty:
            return
        lv = self._field_level
        pairs = [(self._gpfield[:, :2] if lv == 3 else self._gfield, 0)]   # level 3 adds (dL/dmu, dL/dlam, dL/dlo, dL/dhi) to its float4 record
        if lv >= 2:
            pairs.append((self._gmass[:, None], 2))
        if lv == 3:
            pairs.append((self._gpfield[:, 2:], 3))
        ids = self._field_ord.ids
        for g, c in pairs:
            acc = self._gacc[:, c:c + g.shape[1]]
            if ids is None:
                acc += g.double()
            else:
                acc.index_add_(0, ids.long(), g.double())
            g.zero_()
        self._gfield_dirty = False

    def set_gravity(self, g):
        """gravity (3,) for the steps that follow"""
        g = tuple(float(v) for v in g)
        if len(g) != 3:
            raise ValueError('set_gravity: gravity has 3 components')
        self.gravity = g
        if self.has_particles:
            self._ck(self._lib.fmpm_set_gravity(self._h, (C.c_float * 3)(*g)), 'fmpm_set_gravity')
        self._graphs = {}   # gravity is part of the kernel arguments captured in the graphs

    def _colliding_statics(self):
        return [s for s in (self.statics or []) if getattr(s, 'has_dynamics', False)]

    def _rigid_mesh(self):
        rigid = getattr(self.agent, 'rigid', None) if self.agent is not None else None
        return rigid.mesh if rigid is not None else None

    def get_contact_params(self):
        """the contact parameters as they are now: `static_friction` (float64, one per colliding static, in `statics` order), `rigid_friction` and
        `rigid_softness` (only when the agent has a Rigid mesh) and the wall `restitution`"""
        out = dict(static_friction=np.array([s.friction for s in self._colliding_statics()], dtype=np.float64))
        mesh = self._rigid_mesh()
        if mesh is not None:
            out['rigid_friction'], out['rigid_softness'] = float(mesh.friction), float(mesh.softness)
        out['restitution'] = float(self.boundary.restitution)
        return out

    def set_contact_params(self, static_friction=None, rigid_friction=None, rigid_softness=None, restitution=None):
        """overwrite contact parameters for the steps that follow (call it between steps, not inside a backward pass over steps taken before):
        `static_friction` holds one value per colliding static (get_contact_params() order); `rigid_friction` / `rigid_softness` belong to the
        agent's Rigid mesh.  Frictions and the softness must be finite and >= 0.  A rigid friction above 10 selects the reference's sticky branch
        (meshes/dynamic.py:107-108: the contact velocity becomes the collider's), whose derivative with respect to friction is 0."""
        statics, mesh = self._colliding_statics(), self._rigid_mesh()

        def scalar(name, v):
            v = float(v)
            if not np.isfinite(v):
                raise ValueError(f'set_contact_params: {name} must be finite')
            return v
        if static_friction is not None:
            static_friction = np.asarray(static_friction, dtype=np.float64).reshape(-1)
            if static_friction.shape != (len(statics),) or not np.isfinite(static_friction).all() or (static_friction < 0).any():
                raise ValueError(f'set_contact_params: static_friction must hold {len(statics)} finite values >= 0 (one per colliding static)')
        if (rigid_friction is not None or rigid_softness is not None) and mesh is None:
            raise ValueError('set_contact_params: the agent has no Rigid mesh')
        if rigid_friction is not None:
            rigid_friction = scalar('rigid_friction', rigid_friction)
            if rigid_friction < 0:
                raise ValueError('set_contact_params: rigid_friction must be >= 0')
        if rigid_softness is not None:
            rigid_softness = scalar('rigid_softness', rigid_softness)
            if rigid_softness < 0:
                raise ValueError('set_contact_params: rigid_softness must be >= 0')
        if restitution is not None:
            restitution = scalar('restitution', restitution)
        if static_friction is not None:
            for s, fr in zip(statics, static_friction):
                s.friction = float(fr)
        if rigid_friction is not None:
            mesh.friction = rigid_friction
        if rigid_softness is not None:
            mesh.softness = rigid_softness
        if self.has_particles:
            self.register_colliders()
            if restitution is not None:
                self._ck(self._lib.fmpm_set_restitution(self._h, restitution), 'fmpm_set_restitution')
        if restitution is not None:
            self.boundary.restitution = restitution
        self._graphs = {}   # the colliders and the restitution are part of the kernel arguments captured in the graphs

    def get_param_grad(self):
        """dL/d(mu, lam, rho) per material row (float64 arrays aligned with get_material_table()), dL/dgravity (3,) and the contact gradients
        (keys of get_contact_params(): `static_friction`, `rigid_friction` / `rigid_softness` with a Rigid mesh, `restitution`), accumulated by
        every backward substep since the last reset_grad() while `param_grad` was set"""
        if not self.param_grad or self._gmat is None:
            raise RuntimeError('get_param_grad: set MPMSimulator.param_grad = True before reset_grad() and the backward pass')
        g = self._gmat.cpu().numpy()
        out = dict(mu=g[:, 0].copy(), lam=g[:, 1].copy(), rho=g[:, 2] * float(DTYPE_NP(self.p_vol)), gravity=self._ggrav.cpu().numpy().copy())
        if self._gacc is not None:   # the per-particle gradients of the user's fields, and their sums over each row in the row keys
            self._flush_field_grad()
            a = self._gacc.cpu().numpy()
            row = (self._mrow.cpu().numpy() & 0xff).astype(np.int64)
            rows = lambda w: np.bincount(row, weights=w, minlength=len(g))
            grho = a[:, 2] * float(DTYPE_NP(self.p_vol))   # dL/drho = p_vol dL/dm
            if self._field_user is not None:
                out['mu_field'], out['lam_field'] = a[:, 0].copy(), a[:, 1].copy()
            if self._rho_user is not None:
                out['rho_field'] = grho
            out['mu'], out['lam'], out['rho'] = out['mu'] + rows(a[:, 0]), out['lam'] + rows(a[:, 1]), out['rho'] + rows(grho)
            if self._field_level == 3:   # dL/dtheta_c = -dL/dlo, dL/dtheta_s = dL/dhi
                if self._lim_user is not None:
                    out['theta_c_field'], out['theta_s_field'] = -a[:, 3], a[:, 4].copy()
                out['theta_c'], out['theta_s'] = rows(-a[:, 3]), rows(a[:, 4])
        c = self._gcontact.cpu().numpy()
        out['static_friction'] = c[:len(self._colliding_statics())].copy()
        if self._rigid_mesh() is not None:
            out['rigid_friction'], out['rigid_softness'] = float(c[4]), float(c[5])
        out['restitution'] = float(c[6])
        return out

    def get_grad(self, which=('x', 'v', 'C', 'F')):
        """Adjoint of the current frame in original particle order (numpy), for tests / diagnostics."""
        N, dev, f32 = self.n_particles, self.device, torch.float32
        gx = torch.empty((N, 3), dtype=f32, device=dev); gv = torch.empty((N, 3), dtype=f32, device=dev)
        gC = torch.empty((N, 3, 3), dtype=f32, device=dev); gF = torch.empty((N, 3, 3), dtype=f32, device=dev)
        self._ck(self._lib.fmpm_read_grad(self._h, self._gcur, gx.data_ptr(), gv.data_ptr(), gC.data_ptr(), gF.data_ptr(),
                                          self._grad_ord.ids_ptr(), self._stream()), 'fmpm_read_grad')
        out = dict(x=gx, v=gv, C=gC, F=gF)
        return {k: out[k].cpu().numpy() for k in which}

    def set_grad(self, gx, gv, gC, gF):
        """Overwrite the adjoint of the current frame (original particle order)."""
        self._ensure_grad_buffers()
        dev, f32 = self.device, torch.float32
        t = [torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).to(dev) for a in (gx, gv, gC, gF)]
        self._grad_ord = self._frame_ord[self.cur_substep_local]
        self._ck(self._lib.fmpm_write_grad(self._h, self._gcur, t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(),
                                           self._grad_ord.ids_ptr(), self._stream()), 'fmpm_write_grad')

    # ------------------------------------------------------------------------------------------ indices, MPM:225-252
    def f_global_to_f_local(self, f_global):
        return f_global % self.max_substeps_local

    def f_local_to_s_local(self, f_local):
        return f_local // self.n_substeps

    def f_global_to_s_local(self, f_global):
        return self.f_local_to_s_local(self.f_global_to_f_local(f_global))

    def f_global_to_s_global(self, f_global):
        return f_global // self.n_substeps

    @property
    def cur_substep_local(self):
        return self.f_global_to_f_local(self.cur_substep_global)

    @property
    def cur_step_local(self):
        return self.f_global_to_s_local(self.cur_substep_global)

    @property
    def cur_step_global(self):
        return self.f_global_to_s_global(self.cur_substep_global)

    # ------------------------------------------------------------------------------------------ substeps
    def sort_frame(self, f):
        """Cell-sort frame f in place (new slot order for the frames written from now on)."""
        N, dev = self.n_particles, self.device
        old = self._frame_ord[f]
        new = _Order(torch.empty((N,), dtype=torch.int32, device=dev), torch.empty((N,), dtype=torch.int32, device=dev))
        self._ck(self._lib.fmpm_sort(self._h, f, old.ids_ptr(), new.ids.data_ptr(), new.inv.data_ptr(), self._stream()), 'fmpm_sort')
        self._frame_ord[f] = new

    def substep(self, f, is_none_action):  # MPM:515-533
        if not is_none_action:
            self.agent.collect(f)   # collector agents: particles leave at frame f, before p2g (agents/agent_pouring.py:31-41)
        if self.has_particles:
            self._touch_frame(f)
            if self._storing():
                self._ck(self._lib.fmpm_substep_store(self._h, f, self._stream()), 'fmpm_substep_store')
                self._ring_valid[f] = True
            else:
                self._ck(self._lib.fmpm_substep(self._h, f, self._stream()), 'fmpm_substep')
                self._ring_valid[f] = False
            self._frame_ord[f + 1] = self._frame_ord[f]
        if not is_none_action:
            # agent.act writes frame f+1 of particles that are unused at f, so running it after g2p is equivalent
            # to the reference order (MPM:521); agent.move was folded into agent.set_action (pose chain kernel).
            self.agent.act(f, self.cur_substep_global)

    def _next_slot_map(self, f):
        """int32[N]: slot in frame f+1 of the particle in slot s of frame f; None when both frames share one order."""
        a, b = self._frame_ord[f], self._frame_ord[f + 1]
        if a is b:
            return None
        ids = a.ids if a.ids is not None else torch.arange(self.n_particles, dtype=torch.int64, device=self.device)
        if b.inv is None:
            return ids.to(torch.int32)
        return b.inv[ids.long()].to(torch.int32).contiguous()

    def _can_fuse(self):
        """g2p2g fusion of steps without an agent: forward-only (fmpm_substeps_fused) and, in grad mode, the stored-grid path
        (fmpm_substeps_fused_store); not the recompute path (csrc/fmpm_forward.cu: k_g2p2g).  Particles of MAT_RIGID bodies go through
        the gather half only; their scatter follows the body's shape matching (fmpm_advect_rigid -> fmpm_p2g_rigid)."""
        if not bool(getattr(self, 'fuse_g2p2g', False)) or self.agent is not None:
            return False
        return (not self.grad_enabled) or self._storing()

    def _can_fuse_injector(self):
        """steps WITH an agent: the fused g2p2g kernels (particle-level agent.collide and the collector's test compiled in where the agent has
        them) plus a tiny scatter of the particles an injector activates; forward-only and, in grad mode, the stored-grid path.  Covers every
        agent of agents.py, with or without MAT_RIGID bodies (their particles scatter after the body's shape matching: fmpm_p2g_rigid)."""
        if not (bool(getattr(self, 'fuse_g2p2g', False)) and self.agent is not None and self.has_particles):
            return False
        return (not self.grad_enabled) or self._storing()

    def _fused_step_with_injector(self):
        """10 substeps with an agent, in the reference's order (MPM:515-533: agent.act [collector part] -> substep kernels -> agent.act [injector
        part writes frame f+1]): collect(f0), p2g(f0), then per substep grid_op(f) -> g2p2g(f) [collector test on the new position inside;
        plain g2p for the last substep] -> agent.act(f) -> scatter of the particles it activated into the grid of f+1.
        Grad mode: the same with the per-frame grid ring (slot = frame; slot f+1 is cleared before g2p2g fills it, every frame is complete)."""
        L, h, st = self._lib, self._h, self._stream
        n = self.n_substeps
        inj = getattr(self.agent, 'injector', None)
        col = getattr(self.agent, '_collector', None)
        colp = None if col is None else C.byref(col)
        store = self._storing()
        f0 = self.cur_substep_local
        self.agent.collect(f0)
        if store:
            self._ck(L.fmpm_clear_ring_slot(h, f0, st()), 'fmpm_clear_ring_slot')
            self._ck(L.fmpm_p2g_store(h, f0, st()), 'fmpm_p2g_store')
        else:
            self._ck(L.fmpm_p2g(h, f0, 1, st()), 'fmpm_p2g')
        for i in range(n):
            f = f0 + i
            last = i + 1 == n
            if store:
                self._ck(L.fmpm_grid_op_store(h, f, st()), 'fmpm_grid_op_store')
                if last:
                    self._ck(L.fmpm_g2p_store(h, f, st()), 'fmpm_g2p_store')
                else:
                    self._ck(L.fmpm_clear_ring_slot(h, f + 1, st()), 'fmpm_clear_ring_slot')
                    self._ck(L.fmpm_g2p2g_store(h, f, colp, st()), 'fmpm_g2p2g_store')
            else:
                self._ck(L.fmpm_grid_op(h, f, 1, st()), 'fmpm_grid_op')
                self._ck(L.fmpm_g2p(h, f, st()) if last else L.fmpm_g2p2g_collect(h, f, 0, colp, st()), 'fmpm_g2p2g')
            if self._has_rigid_bodies:   # shape matching fixes x[f+1] of the bodies' particles (MPM:428-505), then their scatter of frame f+1
                self._ck(L.fmpm_advect_rigid(h, f, st()), 'fmpm_advect_rigid')
                if not last:
                    self._ck(L.fmpm_p2g_rigid(h, f + 1, (f + 1) if store else -1, colp, st()), 'fmpm_p2g_rigid')
            self._frame_ord[f + 1] = self._frame_ord[f]
            self._ring_valid[f] = store
            act_id = None if inj is None else inj.act_id[f]
            self.agent.act(f, self.cur_substep_global)
            if not last and inj is not None and inj.act_id[f + 1] != act_id:
                self._ck(L.fmpm_p2g_injected(h, f + 1, C.byref(inj._inj), act_id, self._frame_ord[f + 1].inv_ptr(), (f + 1) if store else -1, colp, st()),
                         'fmpm_p2g_injected')
            self.cur_substep_global += 1

    def _fused_substeps(self, f0):
        if self._storing():
            self._ck(self._lib.fmpm_substeps_fused_store(self._h, f0, self.n_substeps, self._stream()), 'fmpm_substeps_fused_store')
        else:
            self._ck(self._lib.fmpm_substeps_fused(self._h, f0, self.n_substeps, self._stream()), 'fmpm_substeps_fused')

    def _storing(self):
        if not (self.grad_enabled and self.store_grids):
            return False
        self._ensure_grad_buffers()
        return self._pm_ring is not None

    def _graph_substeps(self):
        """Forward substeps of one step (p2g / grid_op / g2p x n_substeps, no agent) as a captured CUDA graph, one per
        local step index (frame pointers are baked into the kernel arguments).  Returns False if capture is unavailable."""
        if not hasattr(self, '_graphs'):
            self._graphs = {}
        s_local = self.cur_step_local
        f0 = self.cur_substep_local
        store = self._storing()
        key = (s_local, store, self._can_fuse())
        g = self._graphs.get(key)
        if g is None:
            try:
                fn = self._lib.fmpm_substep_store if store else self._lib.fmpm_substep
                g = torch.cuda.CUDAGraph()
                torch.cuda.synchronize(self.device)
                with torch.cuda.graph(g):
                    if self._can_fuse():
                        self._fused_substeps(f0)
                    else:
                        for i in range(self.n_substeps):
                            self._ck(fn(self._h, f0 + i, self._stream()), 'fmpm_substep')
                self._graphs[key] = g
            except _lib.FmpmError:
                raise   # a library error inside the capture is a real bug, not "graphs unavailable"
            except RuntimeError as ex:   # stream capture unsupported / invalidated: fall back to per-substep launches, and say so once
                import warnings
                warnings.warn(f'MPMSimulator: CUDA-graph capture failed ({ex}); falling back to per-substep launches')
                self.use_graphs = False
                return False
        g.replay()
        for i in range(self.n_substeps):
            self._frame_ord[f0 + i + 1] = self._frame_ord[f0]
            self._ring_valid[f0 + i] = store
        return True

    def substep_grad(self, f, is_none_action):  # MPM:535-552
        if self.has_particles:
            self._sync_param_grad()
            self._ensure_grad_order(self._frame_ord[f])
            self._touch_frame(f, grad=True)
            gin, gout = self._gcur, 1 - self._gcur
            if self._has_rigid_bodies:   # advect_grad, MPM:436-447 (needs v[f+1], which lives in the slot order of frame f+1)
                nxt = self._next_slot_map(f)
                self._ck(self._lib.fmpm_advect_rigid_grad(self._h, f, gin, None if nxt is None else nxt.data_ptr(), self._stream()), 'fmpm_advect_rigid_grad')
            if self._pm_ring is not None and self._ring_valid[f]:
                self._ck(self._lib.fmpm_substep_grad_stored(self._h, f, gin, gout, self._stream()), 'fmpm_substep_grad_stored')
            else:
                self._ck(self._lib.fmpm_substep_grad(self._h, f, gin, gout, self._stream()), 'fmpm_substep_grad')
            if not is_none_action:
                self.agent.act_grad(f, self.cur_substep_global, gin)
            self._gcur = gout

    # ------------------------------------------------------------------------------------------ io, MPM:555-719
    def _to_dev(self, arr, staging, dtype):
        a = np.ascontiguousarray(arr, dtype=dtype)
        staging.copy_(torch.from_numpy(a).reshape(staging.shape), non_blocking=False)
        return staging

    def setframe(self, f, x, v, Cm, F, used):
        """x,v,C,F,used: numpy arrays or torch tensors in original particle order (MPM:566-575)."""
        def dev(a, st, dt):
            if torch.is_tensor(a):   # pinned host tensors: an asynchronous H2D copy on the compute stream (the host may refill them only after the frame was written)
                st.copy_(a.reshape(st.shape), non_blocking=bool(a.device.type == 'cpu' and a.is_pinned())); return st
            return self._to_dev(a, st, dt)
        sx, sv, sC, sF = dev(x, self._sx, np.float32), dev(v, self._sv, np.float32), dev(Cm, self._sC, np.float32), dev(F, self._sF, np.float32)
        su = dev(used, self._sused, np.int32)
        self._ck(self._lib.fmpm_write_frame(self._h, f, sx.data_ptr(), sv.data_ptr(), sC.data_ptr(), sF.data_ptr(), su.data_ptr(),
                                            self._mrow.data_ptr(), None, self._stream()), 'fmpm_write_frame')
        self._frame_ord[f] = _IDENTITY

    def readframe_torch(self, f, want=('x', 'v', 'C', 'F', 'used')):
        """Device tensors (staging buffers, valid until the next read) in original particle order."""
        p = lambda k, t: t.data_ptr() if k in want else None
        self._ck(self._lib.fmpm_read_frame(self._h, f, p('x', self._sx), p('v', self._sv), p('C', self._sC), p('F', self._sF), p('used', self._sused),
                                           self._frame_ord[f].ids_ptr(), self._stream()), 'fmpm_read_frame')
        out = dict(x=self._sx, v=self._sv, C=self._sC, F=self._sF, used=self._sused)
        return {k: out[k] for k in want}

    def readframe(self, f, want=('x', 'v', 'C', 'F', 'used')):
        """numpy arrays (fresh allocations, like MPM:618-623).  Each array is the view of a freshly allocated PINNED host tensor
        (torch's caching host allocator recycles the blocks), filled by one batch of async D2H copies + one synchronisation —
        no staging copy on the host."""
        dev = self.readframe_torch(f, want)
        host = {k: torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for k, t in dev.items()}
        for k, t in dev.items():
            host[k].copy_(t, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return {k: h.numpy() for k, h in host.items()}

    def get_state(self):  # MPM:611-631
        f = self.cur_substep_local
        state = {}
        if self.has_particles:
            state.update(self.readframe(f))
        if self.agent is not None:
            state['agent'] = self.agent.get_state(f)
        if self.smoke_field is not None:
            state['smoke_field'] = self.smoke_field.get_state(self.cur_step_local)
        return state

    def set_state(self, f_global, state):  # MPM:633-644
        f = self.f_global_to_f_local(f_global)
        staged = isinstance(state, MPMSimulator._StagedState)
        if staged and self.device.type == 'cuda':   # uploaded earlier on the copy stream (stage_state_async): order the frame write after that upload
            torch.cuda.current_stream(self.device).wait_event(state.ready)
        if self.has_particles:
            self.setframe(f, state['x'], state['v'], state['C'], state['F'], state['used'])
        if staged and self.device.type == 'cuda':   # its device buffers may be refilled once this frame write has run
            ev = torch.cuda.Event(); ev.record(torch.cuda.current_stream(self.device))
            state.slot['consumed'] = ev
        if self.agent is not None:
            self.agent.set_state(f, state['agent'])
        if self.smoke_field is not None:
            self.smoke_field.set_state(self.f_local_to_s_local(f), state['smoke_field'])

    def get_x(self, f=None):
        f = self.cur_substep_local if f is None else f
        if not self.has_particles:
            return np.zeros((0, self.dim), dtype=DTYPE_NP)
        return self.readframe(f, ('x',))['x']

    def get_v(self, f):
        if not self.has_particles:
            return np.zeros((0, self.dim), dtype=DTYPE_NP)
        return self.readframe(f, ('v',))['v']

    def get_used(self, f=None):
        f = self.cur_substep_local if f is None else f
        if not self.has_particles:
            return np.zeros((0,), dtype=np.int32)
        return self.readframe(f, ('used',))['used']

    # ---- pipelined state upload: set_state's H2D copies taken off the compute stream
    class _StagedState(dict):
        """result of stage_state_async: the state dict set_state takes, with x, v, C, F, used already on (or on their way to) the device"""
        ready = None
        slot = None

    def stage_state_async(self, state):
        """Start uploading a host state (the dict get_state returns; pinned tensors make the copies asynchronous) into one of two device staging sets on
        a COPY stream and return at once: a later `set_state(f, staged)` writes the frame from those buffers, so the 100 B per particle of an episode's
        initial state cross PCIe while the previous episode is still stepping (envs reset to states they know in advance).  The returned dict
        is valid until the second-next stage_state_async call."""
        assert self.has_particles
        dev, N = self.device, self.n_particles
        keys = (('x', (N, 3), torch.float32), ('v', (N, 3), torch.float32), ('C', (N, 3, 3), torch.float32), ('F', (N, 3, 3), torch.float32), ('used', (N,), torch.int32))
        out = MPMSimulator._StagedState({k: v for k, v in state.items() if k not in ('x', 'v', 'C', 'F', 'used')})
        if dev.type != 'cuda':   # (the CPU execution-model shim of tests/: nothing is asynchronous there)
            for k, shp, dt in keys:
                out[k] = torch.as_tensor(np.asarray(state[k]) if not torch.is_tensor(state[k]) else state[k]).to(dt).reshape(shp).clone()
            out.slot = {'consumed': None}
            return out
        if not hasattr(self, '_stage_sets'):
            self._stage_sets = [dict(dev={k: torch.empty(shp, dtype=dt, device=dev) for k, shp, dt in keys}, consumed=None) for _ in range(2)]
            self._stage_next = 0
        if getattr(self, '_copy_stream', None) is None:
            self._copy_stream = torch.cuda.Stream(device=dev)
        st = self._stage_sets[self._stage_next]; self._stage_next ^= 1
        with torch.cuda.stream(self._copy_stream):
            if st['consumed'] is not None:
                self._copy_stream.wait_event(st['consumed'])   # the frame write that last read this set has run
            for k, shp, dt in keys:
                a = state[k]
                a = a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))
                st['dev'][k].copy_(a.reshape(shp), non_blocking=bool(a.device.type == 'cpu' and a.is_pinned()))
            ready = torch.cuda.Event(); ready.record(self._copy_stream)
        out.update(st['dev'])
        out.ready, out.slot = ready, st
        return out

    # ---- pipelined state read-back: the same data as get_state_RL, without stalling the simulation
    class _PendingState:
        """result of get_state_RL_async: `.result()` blocks until the copies have landed and returns the dict get_state_RL would have returned (numpy
        views of pinned host buffers, valid until the second-next get_state_RL_async call)"""
        def __init__(self, event, host, extra):
            self._event, self._host, self._extra = event, host, extra

        def result(self):
            self._event.synchronize()
            out = {k: h.numpy() for k, h in self._host.items()}
            out.update(self._extra)
            return out

    def get_state_RL_async(self):
        """get_state_RL (MPM:683-696) as a pipeline stage: frame -> API-layout staging (one of two sets) on the compute stream, then the D2H copies
        into pinned host buffers on a COPY stream, so the next `step()` runs while x, v, used (28 B per particle) cross PCIe.  Callers that
        need the observation before choosing the next action (closed-loop RL) call `.result()` at once — that is get_state_RL; open-loop
        consumers (trajectory optimisation, logging, rendering) call it one step later and never wait.  Ring frames are not rewritten for
        max_substeps_local substeps, and a staging set is reused only after its previous copies have completed."""
        assert self.has_particles
        dev, N = self.device, self.n_particles
        if dev.type != 'cuda':   # (the CPU execution-model shim of tests/: nothing is asynchronous there)
            done = SimpleNamespace(synchronize=lambda: None)
            r = self.get_state_RL()
            return MPMSimulator._PendingState(done, {k: torch.from_numpy(r[k]) for k in ('x', 'v', 'used')}, {k: v for k, v in r.items() if k not in ('x', 'v', 'used')})
        if not hasattr(self, '_rl_sets'):
            f32, i32 = torch.float32, torch.int32
            mk = lambda: dict(x=torch.empty((N, 3), dtype=f32, device=dev), v=torch.empty((N, 3), dtype=f32, device=dev), used=torch.empty((N,), dtype=i32, device=dev))
            mh = lambda: dict(x=torch.empty((N, 3), dtype=f32, pin_memory=True), v=torch.empty((N, 3), dtype=f32, pin_memory=True), used=torch.empty((N,), dtype=i32, pin_memory=True))
            self._rl_sets = [dict(dev=mk(), host=mh(), done=None) for _ in range(2)]
            self._rl_next = 0
            if getattr(self, '_copy_stream', None) is None:
                self._copy_stream = torch.cuda.Stream(device=dev)
        st = self._rl_sets[self._rl_next]; self._rl_next ^= 1
        cur = torch.cuda.current_stream(dev)
        if st['done'] is not None:
            cur.wait_event(st['done'])           # the copies that last read this staging set have finished
        f = self.cur_substep_local
        d = st['dev']
        self._ck(self._lib.fmpm_read_frame(self._h, f, d['x'].data_ptr(), d['v'].data_ptr(), None, None, d['used'].data_ptr(),
                                           self._frame_ord[f].ids_ptr(), self._stream()), 'fmpm_read_frame')
        ready = torch.cuda.Event(); ready.record(cur)
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(ready)
            for k in ('x', 'v', 'used'):
                st['host'][k].copy_(d[k], non_blocking=True)
            done = torch.cuda.Event(); done.record(self._copy_stream)
        st['done'] = done
        extra = {}
        if self.agent is not None:
            extra['agent'] = self.agent.get_state(f)
        if self.smoke_field is not None:
            extra['smoke_field'] = self.smoke_field.get_state(self.cur_step_local)
        return MPMSimulator._PendingState(done, st['host'], extra)

    def get_state_RL(self):  # MPM:683-696
        f = self.cur_substep_local
        state = {}
        if self.has_particles:
            state.update(self.readframe(f, ('x', 'v', 'used')))
        if self.agent is not None:
            state['agent'] = self.agent.get_state(f)
        if self.smoke_field is not None:
            state['smoke_field'] = self.smoke_field.get_state(self.cur_step_local)
        return state

    # ---- observation bridge (SURVEY.md 8f rank 4): what envs/fluid_env.py:99-125 builds from get_state_RL, subsampled ON THE DEVICE
    def build_obs_index(self, n_obs_ptcls_per_body=200, bodies=None):
        """particle ids FluidEnv._get_obs keeps: per body `particle_ids[::max(1, n // n_obs_ptcls_per_body)]` (fluid_env.py:104-112)."""
        if bodies is None:
            bodies = getattr(self, '_bodies_info', None)
        if not self.has_particles or bodies is None or 'particle_ids' not in bodies:
            bodies = {'n': 1, 'n_particles': [self.n_particles], 'particle_ids': [np.arange(self.n_particles)]}
        ids = []
        for b in range(int(bodies['n'])):
            pid = np.asarray(bodies['particle_ids'][b])
            ids.append(pid[::max(1, int(bodies['n_particles'][b]) // int(n_obs_ptcls_per_body))])
        self._obs_ids = [torch.from_numpy(np.ascontiguousarray(i, dtype=np.int64)).to(self.device) for i in ids]
        return ids

    def get_obs_RL(self, n_obs_ptcls_per_body=200):
        """The observation vector of FluidEnv._get_obs (fluid_env.py:99-125) — per body x, v, used of the kept particles, then the agent
        state, then the smoke field's v / q[::10, 60:68, ::10] — assembled on the device and copied to the host as ONE small array
        (the reference moves the whole x, v, used state across PCIe every step, README.md:62).  Returns float32 numpy."""
        f = self.cur_substep_local
        parts = []
        if self.has_particles:
            if getattr(self, '_obs_ids', None) is None or getattr(self, '_obs_n', None) != n_obs_ptcls_per_body:
                self.build_obs_index(n_obs_ptcls_per_body); self._obs_n = n_obs_ptcls_per_body
            st = self.readframe_torch(f, ('x', 'v', 'used'))
            for ids in self._obs_ids:
                parts += [st['x'][ids].reshape(-1), st['v'][ids].reshape(-1), st['used'][ids].to(torch.float32).reshape(-1)]
        if self.agent is not None:
            for e in self.agent.effectors:
                parts.append(torch.cat([e.pos[f], e.quat[f]]) if not hasattr(e, 's') else torch.cat([e.pos[f], e.quat[f], e.s[f:f + 1], e.r[f:f + 1]]))
                if hasattr(e, 'act_id'):
                    parts.append(torch.tensor([float(e.act_id[f])], dtype=torch.float32, device=self.device))
        if self.smoke_field is not None:
            sf, n = self.smoke_field, self.smoke_field.n_grid
            s_loc = self.cur_step_local
            v = sf._v[s_loc, :, :3].reshape(n, n, n, 3)[::10, 60:68, ::10]
            q = sf._q[s_loc].reshape(sf.q_dim, n, n, n).permute(1, 2, 3, 0)[::10, 60:68, ::10]
            parts += [v.reshape(-1), q.reshape(-1)]
        dev = torch.cat(parts) if parts else torch.zeros(0, dtype=torch.float32, device=self.device)
        host = torch.empty(dev.shape, dtype=torch.float32, pin_memory=True)
        host.copy_(dev, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return host.numpy()

    def get_state_render_device(self, f):
        """x (N,3) float32 and used (N,) int32 of frame f in original particle order as DEVICE tensors (staging buffers, valid until the next
        read) — `torch.utils.dlpack.to_dlpack(t)` / `__dlpack__` hands them to a renderer without the GPU -> CPU -> GPU round trip the
        reference's renderers make (renderers/gl_renderer.py:172-177, README.md:62)."""
        r = self.readframe_torch(f, ('x', 'used'))
        return SimpleNamespace(x=r['x'], used=r['used'])

    def get_state_render(self, f):  # MPM:705-707
        r = self.readframe(f, ('x', 'used'))
        return SimpleNamespace(x=r['x'], used=r['used'])

    def set_x(self, f, x):  # MPM:577-581
        st = self.readframe(f)
        self.setframe(f, x, st['v'], st['C'], st['F'], st['used'])

    def set_used(self, f, used):  # MPM:583-586
        st = self.readframe(f)
        self.setframe(f, st['x'], st['v'], st['C'], st['F'], used)

    def copy_frame(self, source, target):  # MPM:588-595
        self._ck(self._lib.fmpm_copy_frame(self._h, source, target, self._stream()), 'fmpm_copy_frame')
        self._frame_ord[target] = self._frame_ord[source]

    # ------------------------------------------------------------------------------------------ step, MPM:721-775
    def step(self, action=None):
        if self.grad_enabled:
            if self.cur_substep_local == 0:
                self.actions_buffer = []
        self.step_(action)
        if self.grad_enabled:
            self.actions_buffer.append(action)
        if self.cur_substep_local == 0:
            self.memory_to_cache()

    def step_(self, action=None):
        is_none_action = action is None
        if not is_none_action:
            self.agent.set_action(s=self.cur_step_local, s_global=self.cur_step_global, n_substeps=self.n_substeps, action=action)
        if self.smoke_field is not None:   # smoke simulates at step level, not substep (MPM:744-747)
            self.smoke_field.step(s=self.cur_step_local, f=self.cur_substep_local)
        if self.has_particles and self.sort_every > 0 and self.cur_step_global % self.sort_every == 0:
            self.sort_frame(self.cur_substep_local)
        if self.has_particles:
            self._touch_frame(self.cur_substep_local)   # every substep of the step runs in this slot order
        if self.use_graphs and is_none_action and self.has_particles and self._graph_substeps():
            self.cur_substep_global += self.n_substeps
        elif not is_none_action and self._can_fuse_injector():
            self._fused_step_with_injector()
        elif is_none_action and self.has_particles and self._can_fuse():
            f0 = self.cur_substep_local
            store = self._storing()
            self._fused_substeps(f0)
            for i in range(self.n_substeps):
                self._frame_ord[f0 + i + 1] = self._frame_ord[f0]
                self._ring_valid[f0 + i] = store
            self.cur_substep_global += self.n_substeps
        else:
            for _ in range(self.n_substeps):
                self.substep(self.cur_substep_local, is_none_action)
                self.cur_substep_global += 1
        assert self.cur_substep_global <= self.max_substeps_global

    def step_grad(self, action=None):
        if self.cur_substep_local == 0:
            self.memory_from_cache()
        is_none_action = action is None
        for _ in range(self.n_substeps - 1, -1, -1):
            self.cur_substep_global -= 1
            self.substep_grad(self.cur_substep_local, is_none_action)
        if self.smoke_field is not None:   # MPM:765-767
            self.smoke_field.step_grad(s=self.cur_step_local, f=self.cur_substep_local)
        if not is_none_action:
            self.agent.set_action_grad(s=self.cur_substep_local // self.n_substeps, s_global=self.cur_substep_global // self.n_substeps,
                                       n_substeps=self.n_substeps, action=action)

    # ------------------------------------------------------------------------------------------ checkpoint ring, MPM:777-912
    def _ckpt_device(self):
        return {'gpu': self.device, 'cpu': torch.device('cpu'), 'disk': torch.device('cpu')}[self.ckpt_dest]

    def memory_to_cache(self):
        T = self.max_substeps_local
        if self.grad_enabled:
            ckpt_start_step = self.cur_substep_global - T
            ckpt_name = f'{ckpt_start_step:06d}'
            d = self._ckpt_device()
            ckpt = {'actions': list(self.actions_buffer)}
            if self.has_particles:
                o = self._frame_ord[0]
                ckpt.update(pa=self._pa[0].to(d, copy=True), pf=self._pf[0].to(d, copy=True), pf8=self._pf8[0].to(d, copy=True),
                            ids=None if o.ids is None else o.ids.to(d, copy=True), inv=None if o.inv is None else o.inv.to(d, copy=True))
            if self.agent is not None:
                ckpt['agent'] = self.agent.get_ckpt()
            if self.smoke_field is not None:
                ckpt['smoke_field'] = self.smoke_field.get_ckpt()
            if self.ckpt_dest == 'disk':
                os.makedirs(self.ckpt_dir, exist_ok=True)
                torch.save(ckpt, os.path.join(self.ckpt_dir, f'{ckpt_name}.pt'))
            else:
                self.ckpt_ram[ckpt_name] = ckpt
        # restart from frame 0 in memory
        if self.has_particles:
            self.copy_frame(T, 0)
        if self.smoke_field is not None:
            self.smoke_field.copy_frame(self.max_steps_local, 0)
        if self.agent is not None:
            self.agent.copy_frame(T, 0)

    def memory_from_cache(self):
        assert self.grad_enabled
        T = self.max_substeps_local
        # reference: copy_frame(0,T); copy_grad(0,T); reset_grad_till_frame(T).  The adjoint ping-pong frame already
        # *is* "the adjoint of the current frame", so only the agent's per-frame adjoints need the shuffle.
        if self.smoke_field is not None:
            self.smoke_field.copy_frame(0, self.max_steps_local)
            self.smoke_field.copy_grad(0, self.max_steps_local)
            self.smoke_field.reset_grad_till_frame(self.max_steps_local)
        if self.agent is not None:
            self.agent.copy_frame(0, T)
            self.agent.copy_grad(0, T)
            self.agent.reset_grad_till_frame(T)
        ckpt_start_step = self.cur_substep_global - T
        ckpt_name = f'{ckpt_start_step:06d}'
        if self.ckpt_dest == 'disk':
            ckpt = torch.load(os.path.join(self.ckpt_dir, f'{ckpt_name}.pt'), weights_only=False)
        else:
            ckpt = self.ckpt_ram[ckpt_name]
        if self.has_particles:
            self._pa[0].copy_(ckpt['pa']); self._pf[0].copy_(ckpt['pf']); self._pf8[0].copy_(ckpt['pf8'])
            self._frame_ord[0] = _IDENTITY if ckpt['ids'] is None else _Order(ckpt['ids'].to(self.device, copy=True), ckpt['inv'].to(self.device, copy=True))
        if self.agent is not None:
            self.agent.set_ckpt(ckpt['agent'])
        if self.smoke_field is not None:
            self.smoke_field.set_ckpt(ckpt=ckpt['smoke_field'])
        # now that the first frame is loaded, a forward pass fills up the rest of the ring
        self.cur_substep_global = ckpt_start_step
        for action in ckpt['actions']:
            self.step_(action)

    # ------------------------------------------------------------------------------------------ x-slab hooks (fluidlab_b200/slab.py)
    # The slab orchestration only talks to its local simulator through these (and step-level methods), so the same orchestration
    # can be driven on CPU by an oracle-backed stand-in in tests/test_slab_cpu.py.
    def slab_positions(self, f):
        """(x coordinate, alive mask) of every slot of frame f, in the slot order of the frame (device views, no copy)."""
        return self._pa[f, 0, :, 0], (self._pa[f, 0, :, 3].view(torch.int32) & 1) != 0

    def slab_grid_acc(self, f):
        """live (G,4) (momentum, mass) accumulator of substep f (double-buffered by substep parity in peer mode)."""
        g = self._grid_pm
        return g[f & 1] if g.dim() == 3 else g

    def slab_grid_acc_commit(self, f, acc):
        pass   # `acc` is the live buffer

    def slab_grid_adj(self, f):
        """live (G,4) adjoint of grid.v_out."""
        return self._ggrid_v

    def slab_grid_adj_commit(self, f, adj):
        pass

    def slab_flag_blocks(self, f, flagger):
        b = self._blk_flags
        flagger(b[f & 1] if b.dim() == 2 else b)

    def slab_snapshot_frame(self, f):
        """everything needed to put ring frame f back later (state planes + its slot order): the chunk checkpoint of a sharded run"""
        o = self._frame_ord[f]
        return dict(pa=self._pa[f].clone(), pf=self._pf[f].clone(), pf8=self._pf8[f].clone(), order=o, mrow=self._mrow.clone())

    def slab_restore_frame(self, f, snap):
        self._pa[f].copy_(snap['pa']); self._pf[f].copy_(snap['pf']); self._pf8[f].copy_(snap['pf8'])
        self._frame_ord[f] = snap['order']
        self._mrow.copy_(snap['mrow'])

    def slab_adjoint_moves_to_frame(self, f):
        pass   # the adjoint ping-pong buffer always holds "the adjoint of the current frame": nothing is indexed by frame here

    def slab_substep_grad_p2g(self, f):
        """backward substep f, part 1: recompute the (momentum, mass) scatter of frame f (ghost sum follows)."""
        self._ensure_grad_order(self._frame_ord[f])
        self._ck(self._lib.fmpm_p2g(self._h, f, 0, self._stream()), 'fmpm_p2g')

    def slab_substep_grad_scatter(self, f):
        """part 2: grid_op of frame f + g2p.grad scatter of the v_out adjoint (ghost sum of that adjoint follows)."""
        self._ck(self._lib.fmpm_substep_grad_scatter(self._h, f, self._gcur, self._stream()), 'fmpm_substep_grad_scatter')

    def slab_substep_grad_finish(self, f):
        """part 3: grid_op.grad (leaves the accumulators clear) + the particle side; the adjoint of frame f becomes current."""
        gin, gout = self._gcur, 1 - self._gcur
        self._ck(self._lib.fmpm_substep_grad_finish(self._h, f, gin, gout, self._stream()), 'fmpm_substep_grad_finish')
        self._gcur = gout

    def slab_substep_grad_one_call(self, f):
        """parts 1-3 with the neighbour handshakes in between, one library call (peer exchange + sync='signal')"""
        self._ensure_grad_order(self._frame_ord[f])
        gin, gout = self._gcur, 1 - self._gcur
        self._ck(self._lib.fmpm_substep_grad_slab(self._h, f, gin, gout, self._stream()), 'fmpm_substep_grad_slab')
        self._gcur = gout

    def read_grad_torch(self):
        """current adjoint frame in original particle order: dict of fresh device tensors x,v (N,3), C,F (N,3,3)."""
        N, dev, f32 = self.n_particles, self.device, torch.float32
        g = dict(x=torch.empty((N, 3), dtype=f32, device=dev), v=torch.empty((N, 3), dtype=f32, device=dev),
                 C=torch.empty((N, 3, 3), dtype=f32, device=dev), F=torch.empty((N, 3, 3), dtype=f32, device=dev))
        self._ck(self._lib.fmpm_read_grad(self._h, self._gcur, g['x'].data_ptr(), g['v'].data_ptr(), g['C'].data_ptr(), g['F'].data_ptr(),
                                          self._grad_ord.ids_ptr(), self._stream()), 'fmpm_read_grad')
        return g

    def write_grad_torch(self, g):
        """overwrite the current adjoint frame from device tensors in original particle order (it is then IN original order)."""
        self._ensure_grad_buffers()
        t = [g[k].to(self.device, torch.float32).contiguous() for k in ('x', 'v', 'C', 'F')]
        self._grad_ord = _IDENTITY
        self._ck(self._lib.fmpm_write_grad(self._h, self._gcur, t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(),
                                           self._grad_ord.ids_ptr(), self._stream()), 'fmpm_write_grad')

    # ------------------------------------------------------------------------------------------ phase-level access (tests, profiling)
    def read_grid(self):
        G, dev, f32 = self.n_grid ** 3, self.device, torch.float32
        vin = torch.empty((G, 3), dtype=f32, device=dev); m = torch.empty((G,), dtype=f32, device=dev); vout = torch.empty((G, 3), dtype=f32, device=dev)
        self._ck(self._lib.fmpm_read_grid(self._h, vin.data_ptr(), m.data_ptr(), vout.data_ptr(), self._stream()), 'fmpm_read_grid')
        return vin.cpu().numpy(), m.cpu().numpy(), vout.cpu().numpy()

    def read_grid_grad(self):
        G, dev, f32 = self.n_grid ** 3, self.device, torch.float32
        vin = torch.empty((G, 3), dtype=f32, device=dev); m = torch.empty((G,), dtype=f32, device=dev); vout = torch.empty((G, 3), dtype=f32, device=dev)
        self._ck(self._lib.fmpm_read_grid_grad(self._h, vin.data_ptr(), m.data_ptr(), vout.data_ptr(), self._stream()), 'fmpm_read_grid_grad')
        return vin.cpu().numpy(), m.cpu().numpy(), vout.cpu().numpy()

    def phase(self, name, f, *args):
        """Run one kernel phase by name ('clear_grid','p2g','grid_op','g2p','g2p_grad_scatter','grid_op_grad','particle_grad')."""
        s = self._stream()
        L, h = self._lib, self._h
        if name != 'clear_grid' and 0 <= f < len(self._frame_ord):   # (the library reports a bad frame)
            self._touch_frame(f, grad=name == 'particle_grad')
        if name == 'clear_grid': rc = L.fmpm_clear_grid(h, s)
        elif name == 'p2g': rc = L.fmpm_p2g(h, f, int(args[0]) if args else 1, s)
        elif name == 'grid_op': rc = L.fmpm_grid_op(h, f, int(args[0]) if args else 0, s)
        elif name == 'g2p':
            rc = L.fmpm_g2p(h, f, s); self._frame_ord[f + 1] = self._frame_ord[f]
        elif name == 'g2p2g':
            rc = L.fmpm_g2p2g(h, f, 0, s); self._frame_ord[f + 1] = self._frame_ord[f]
        elif name == 'g2p_grad_scatter': rc = L.fmpm_g2p_grad_scatter(h, f, self._gcur, s)
        elif name == 'grid_op_grad': rc = L.fmpm_grid_op_grad(h, f, s)
        elif name == 'particle_grad':
            rc = L.fmpm_particle_grad(h, f, self._gcur, 1 - self._gcur, s); self._gcur = 1 - self._gcur
        else: raise KeyError(name)
        self._ck(rc, name)
