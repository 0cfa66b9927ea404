"""Spatial-slab sharding of the MLS-MPM substep across the GPUs of one node (SURVEY.md §8e).

The reference is single-device (no collective anywhere); this is new design.  One process per GPU
(`torch.distributed`, backend nccl; gloo on CPU for the host-logic tests):

  * the grid's x node planes are cut into `world` contiguous slabs (boundaries multiples of 8 = sparse-block size);
    rank r owns the particles whose stencil-centre plane `int(x*inv_dx - 0.5) + 1` lies in [bounds[r], bounds[r+1]);
  * the ghost region of the (momentum, mass) accumulator — `halo` node planes either side of a slab boundary — must hold the
    sum of both neighbours' contributions.  Default (`exchange='peer'`): the reduction is FUSED INTO p2g: each rank maps its
    neighbours' accumulators (symmetric memory) and p2g's vector reductions (REDG.F32x4) for nodes on shared planes go to the
    local grid AND, over NVLink peer memory, to the neighbour's grid (p2g also sets the neighbour's sparse-block flags); the accumulator is double-buffered by substep parity so
    a fast neighbour can never scatter into a buffer that is still being consumed, and one device-side signal-pad barrier
    per substep (symmetric memory) is the only synchronisation.  Fallback (`exchange='nccl'`): one in-place NCCL all-reduce of the ghost planes per boundary
    over a 2-rank communicator.  grid_op then runs redundantly on the ghosts, so g2p needs no second exchange.  The backward pass mirrors it:
    g2p.grad's scatter of the v_out adjoint reduces into the neighbour's adjoint grid over peer memory as well (second barrier per substep);
  * at step boundaries particles whose centre plane left the slab migrate to the neighbour (100 B records + material row
    + global id).  The leaver census is asynchronous (all-reduce -> pinned host, read one step later), so steps without
    leavers never synchronise the host.  `halo` = 4 planes tolerates 3 cells of drift over the two steps between a
    census and its migration (|v| < 3 dx / (20 dt) = 2.9 m/s at 256^3, 11.7 m/s at 64^3); raise `halo` for faster flows.

Backward (`SlabMPMSimulator.step_grad`, SURVEY.md §8e "Backward"): per substep the forward scatter of frame f is recomputed with the same
ghost sum as in the forward pass, g2p's adjoint scatters the v_out adjoint onto owned + ghost planes, ONE more ghost sum (all-reduce of
the 2*halo planes per slab boundary) completes it, and grid_op.grad runs redundantly on the ghosts so the particle side (p2g.grad) needs
no further exchange.  At step boundaries `migrate_grad` sends the adjoint of every migrated particle back to the rank and slot it left.
Trajectories longer than the ring are handled like the single-GPU path (MPM:777-912): every chunk's first frame (+ global ids, material
rows, pending leaver census) is checkpointed in HBM when the chunk starts, and the backward pass re-runs a chunk forward — ghost sums and
migrations included, in lockstep on all ranks — before walking it backwards.

The orchestration talks to the local simulator only through `MPMSimulator`'s step-level methods and its `slab_*` hooks, so
tests/test_slab_cpu.py drives this same code on CPU (gloo, world_size 2) with an oracle-backed stand-in and checks forward AND backward
against the single-domain oracle.
"""
import numpy as np
import torch
import torch.distributed as dist


def slab_bounds(lo_plane, hi_plane, world, align=8):
    """`world`+1 plane indices cutting [lo_plane, hi_plane) into slabs with boundaries on multiples of `align`."""
    assert lo_plane % align == 0 and hi_plane % align == 0 and hi_plane > lo_plane
    nblk = (hi_plane - lo_plane) // align
    assert nblk >= 2 * world, 'slabs must be at least two blocks (16 planes) wide'
    cuts = [lo_plane + align * int(round(nblk * r / world)) for r in range(world + 1)]
    return cuts


class GhostExchange:
    """Sums the ghost planes of a (G,4) accumulator with the neighbouring slabs: one in-place all-reduce per slab boundary
    over a 2-rank communicator, restricted to the `2*halo` planes around the boundary (contiguous: x is the slowest index)."""

    def __init__(self, n_grid, bounds, rank, world, halo=8, group=None):
        self.n, self.bounds, self.rank, self.world, self.halo = n_grid, list(bounds), rank, world, halo
        self.plane = n_grid * n_grid
        self.regions = []  # (boundary index, first_plane, last_plane_exclusive, pair process group)
        if world > 1:
            # every rank creates every pair group, in the same order (torch.distributed requirement)
            pgs = [dist.new_group([i, i + 1]) for i in range(world - 1)]
            # even boundaries first, then odd ones: a globally consistent collective order, no deadlock
            for i in list(range(0, world - 1, 2)) + list(range(1, world - 1, 2)):
                if rank in (i, i + 1):
                    b = self.bounds[i + 1]
                    self.regions.append((i, b - halo, b + halo, pgs[i]))

    def bytes_per_exchange(self):
        return sum((hi - lo) * self.plane * 16 for _, lo, hi, _ in self.regions)

    def exchange_sum(self, grid):
        """grid: (G,4) float32 tensor (cuda for nccl, cpu for gloo).  In place: ghost regions become the 2-rank sums."""
        for _, lo, hi, pg in self.regions:
            dist.all_reduce(grid[lo * self.plane:hi * self.plane], group=pg)

    def flag_ghost_blocks(self, blk_flags):
        """mark the 8^3 blocks covering the ghost regions active so grid_op computes (and clears) them on both ranks."""
        nb = self.n // 8
        f = blk_flags.view(nb, nb, nb)
        for _, lo, hi, _ in self.regions:
            f[lo // 8:(hi + 7) // 8] = 1


class _Done:
    def synchronize(self):
        pass


class SymmetricMemoryPeers:
    """Buffers every rank can address directly: torch.distributed._symmetric_memory (CUDA: each rank's allocation is mapped into every
    other rank's address space over NVLink) + its device-side signal-pad barrier.  `alloc` returns (local tensor, [base pointer of rank r's
    copy in THIS process]).  tests/test_cuda_emu_mpm.py substitutes a POSIX-shared-memory implementation to drive the same kernels on CPU."""

    def __init__(self, group, device):
        import torch.distributed._symmetric_memory as symm_mem
        self._symm_mem, self.group, self.device = symm_mem, group if group is not None else dist.group.WORLD, device
        self._handles = []

    def alloc(self, shape, dtype):
        buf = self._symm_mem.empty(tuple(shape), dtype=dtype, device=self.device)
        buf.zero_()
        hdl = self._symm_mem.rendezvous(buf, self.group)
        self._handles.append(hdl)
        return buf, list(hdl.buffer_ptrs)

    def barrier(self):
        self._handles[0].barrier(channel=0)   # device-side: everything the ranks enqueued before it (incl. their peer reductions) has completed


def centre_plane(x, inv_dx):
    return (x[:, 0] * inv_dx - 0.5).to(torch.int32) + 1


def migrate(state, lo, hi, rank, world, inv_dx, group=None, record=None):
    """Move particles whose centre plane left [lo, hi) to the neighbouring rank.

    state: dict of tensors in slot order — x (N,3), v (N,3), C (N,3,3), F (N,3,3) float32; used, mrow, gid (N,) int32.
    Modified in place (leavers become unused, arrivals fill unused slots).  Returns (n_sent, n_received).
    One host synchronisation per call (counts); called once per step (10 substeps).
    record: optional dict that receives {'sent': {peer: slots}, 'recv': {peer: slots}} — what `migrate_grad` needs to send the
    adjoint of every arrival back to the slot its particle left (the backward pass over x-slabs, SURVEY.md §8e)."""
    if record is not None:
        record['sent'], record['recv'] = {}, {}
    if world == 1:
        return 0, 0
    x, used = state['x'], state['used']
    N = x.shape[0]
    cp = centre_plane(x, inv_dx)
    alive = used != 0
    masks = {}
    if rank > 0:
        masks[rank - 1] = alive & (cp < lo)
    if rank < world - 1:
        masks[rank + 1] = alive & (cp >= hi)

    def pack(idx):
        return torch.cat([state['x'][idx], state['v'][idx], state['C'][idx].reshape(-1, 9), state['F'][idx].reshape(-1, 9),
                          state['mrow'][idx].view(torch.float32).reshape(-1, 1), state['gid'][idx].view(torch.float32).reshape(-1, 1)], 1)
    send = {}
    for peer, m in masks.items():
        idx = torch.nonzero(m).reshape(-1)
        send[peer] = pack(idx).contiguous()
        if record is not None:
            record['sent'][peer] = idx.clone()
        used[idx] = 0
        state['x'][idx] = -100.0  # NOWHERE (configs/macros.py:216)
    # exchange counts, then payloads
    cnt_send = {p: torch.tensor([send[p].shape[0]], dtype=torch.int64, device=x.device) for p in send}
    cnt_recv = {p: torch.zeros(1, dtype=torch.int64, device=x.device) for p in send}
    ops = []
    for p in send:
        ops.append(dist.P2POp(dist.isend, cnt_send[p], p, group)); ops.append(dist.P2POp(dist.irecv, cnt_recv[p], p, group))
    for w in dist.batch_isend_irecv(ops):
        w.wait()
    n_in = {p: int(cnt_recv[p].item()) for p in send}
    recv = {p: torch.empty((n_in[p], 26), dtype=torch.float32, device=x.device) for p in send}
    ops = []
    for p in send:
        if send[p].shape[0] > 0:
            ops.append(dist.P2POp(dist.isend, send[p], p, group))
        if n_in[p] > 0:
            ops.append(dist.P2POp(dist.irecv, recv[p], p, group))
    if ops:
        for w in dist.batch_isend_irecv(ops):
            w.wait()
    total_in = sum(n_in.values())
    if total_in > 0:
        rows = torch.cat([recv[p] for p in sorted(recv)], 0)
        free = torch.nonzero(used == 0).reshape(-1)
        assert free.numel() >= total_in, f'rank {rank}: slab capacity exhausted ({free.numel()} free slots, {total_in} arrivals)'
        dst = free[:total_in]
        if record is not None:
            o = 0
            for p in sorted(recv):
                record['recv'][p] = dst[o:o + n_in[p]].clone(); o += n_in[p]
        state['x'][dst] = rows[:, 0:3]; state['v'][dst] = rows[:, 3:6]
        state['C'][dst] = rows[:, 6:15].reshape(-1, 3, 3); state['F'][dst] = rows[:, 15:24].reshape(-1, 3, 3)
        state['mrow'][dst] = rows[:, 24].contiguous().view(torch.int32); state['gid'][dst] = rows[:, 25].contiguous().view(torch.int32)
        used[dst] = 1
    return sum(s.shape[0] for s in send.values()), total_in


def migrate_grad(gstate, record, group=None):
    """Adjoint of `migrate` on the particle adjoints: gstate = dict x (N,3), v (N,3), C (N,3,3), F (N,3,3) in the slot order AFTER the
    migration that filled `record`; on return it is in the slot order BEFORE it.  The adjoint rows of every arrival travel back to the
    rank and slot the particle left (its slot here held a parked particle before: zero adjoint), no counts need to be exchanged.
    Unused slots are assumed to carry zero adjoint (the loss only reads used particles)."""
    sent, recvd = record.get('sent', {}), record.get('recv', {})
    if not sent and not recvd:
        return

    def pack(idx):
        return torch.cat([gstate['x'][idx], gstate['v'][idx], gstate['C'][idx].reshape(-1, 9), gstate['F'][idx].reshape(-1, 9)], 1).contiguous()
    dev = gstate['x'].device
    out = {p: pack(idx) for p, idx in recvd.items() if idx.numel() > 0}
    back = {p: torch.empty((idx.numel(), 24), dtype=torch.float32, device=dev) for p, idx in sent.items() if idx.numel() > 0}
    ops = [dist.P2POp(dist.isend, out[p], p, group) for p in out] + [dist.P2POp(dist.irecv, back[p], p, group) for p in back]
    if ops:
        for w in dist.batch_isend_irecv(ops):
            w.wait()
    for p, idx in recvd.items():
        if idx.numel() > 0:
            for k in ('x', 'v', 'C', 'F'):
                gstate[k][idx] = 0
    for p, rows in back.items():
        idx = sent[p]
        gstate['x'][idx] = rows[:, 0:3]; gstate['v'][idx] = rows[:, 3:6]
        gstate['C'][idx] = rows[:, 6:15].reshape(-1, 3, 3); gstate['F'][idx] = rows[:, 15:24].reshape(-1, 3, 3)


class SlabMPMSimulator:
    """Forward MLS-MPM over x-slabs: one local `MPMSimulator` per rank + ghost exchange + migration."""

    def __init__(self, quality, gravity, particles, gid, bounds, capacity, boundary=None, max_substeps_local=50, device=None, group=None, halo=4,
                 exchange='peer', migrate=True, sim_factory=None, peer_factory=None, sync='signal', sort_every=1, use_graphs=True, migrate_every=1, statics=None):
        from .macros import NOWHERE
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.group = group
        self.migrate_enabled = bool(migrate)   # False: diagnostics only (particles must then stay inside their ghost range)
        # census + migration period in steps.  A particle may sit up to (2 * migrate_every) steps of drift outside its slab (the census is read one
        # period late): `halo` - 1 cells must cover that (|v_x| < (halo - 1) dx / (20 dt * 2 * migrate_every)); the census also counts particles
        # that left the halo and the next step raises instead of computing with incomplete ghost sums.
        self.migrate_every = max(1, int(migrate_every))
        self.halo = int(halo)
        self.sort_every = int(sort_every)      # cell-sort period in steps (the kernels tolerate an aged sort; arrivals of a migration land in free slots)
        self.use_graphs = bool(use_graphs)     # sync='signal': the one-call step (fmpm_substeps_slab) is replayed as a CUDA graph per local step index
        self._graphs = {}
        n_loc = len(particles['x'])
        assert capacity >= n_loc
        pad = capacity - n_loc
        P = dict(particles)
        P['x'] = np.concatenate([np.asarray(particles['x'], dtype=np.float64), np.tile(np.array(NOWHERE), (pad, 1))])
        for k in ('mat', 'rho', 'body_id'):
            P[k] = np.concatenate([np.asarray(particles[k]), np.full(pad, np.asarray(particles[k])[0] if n_loc else 0)])
        P['used'] = np.concatenate([np.asarray(particles['used']).astype(np.int32), np.zeros(pad, np.int32)])
        if sim_factory is None:
            from .simulator import MPMSimulator
            self.sim = MPMSimulator(dim=3, quality=quality, gravity=gravity, horizon=10 ** 5, max_substeps_local=max_substeps_local,
                                    max_substeps_global=10 ** 7, ckpt_dest='gpu', device=device, sort_every=1)
            if boundary is not None:
                self.sim.setup_boundary(**boundary)
            # static SDF colliders (meshes/static.py, applied in grid_op MPM:388-390): every rank evaluates them on the nodes it converts, shared planes included —
            # no pose, no exchange; Rigid effectors / agents and MAT_RIGID bodies stay single-GPU
            self.sim.build(None, None, statics if statics is not None else [], P)
        else:   # tests: a stand-in with MPMSimulator's step-level methods and slab_* hooks (tests/test_slab_cpu.py)
            self.sim = sim_factory(quality=quality, gravity=gravity, particles=P, boundary=boundary, max_substeps_local=max_substeps_local)
            exchange = 'nccl' if exchange == 'peer' else exchange   # "nccl" = the all-reduce exchange, whatever the backend
        dev = self.sim.device
        self.gid = torch.from_numpy(np.concatenate([np.asarray(gid, dtype=np.int32), np.full(pad, -1, np.int32)])).to(dev)
        self.bounds = list(bounds)
        self.lo, self.hi = self.bounds[self.rank], self.bounds[self.rank + 1]
        self.ghost = GhostExchange(self.sim.n_grid, self.bounds, self.rank, self.world, halo=halo, group=group)
        self.n_migrated = 0
        self.exchange = exchange if self.world > 1 else 'none'
        self._peer_factory = peer_factory if peer_factory is not None else SymmetricMemoryPeers
        # 'signal' (default): a handshake with the two NEIGHBOURS only, inside the library (fmpm_slab_sync: a one-thread kernel posting /
        #            polling epochs in peer memory, bounded in time), and the whole step in one C call (fmpm_substeps_slab) replayed as a
        #            CUDA graph: no host work and no global barrier per substep.
        # 'barrier': one device-side barrier over ALL ranks per substep (symmetric-memory signal pads), four library calls per substep.
        assert sync in ('barrier', 'signal')
        self.sync = sync if exchange == 'peer' else 'barrier'
        self.pull = False
        if self.exchange == 'peer':
            self._setup_peer(halo)
        self._census_host = None
        self._census_event = None
        self._records = {}      # global step index -> what migrate() did before that step (for step_grad)
        self._gid_before = {}   # global step index -> slot -> global id map before that migration
        self._chunks = {}       # first global substep of a chunk -> checkpoint taken when the chunk started (grad mode)
        self._replaying = False

    def _setup_peer(self, halo):
        """Double-buffer the accumulator in PEER-ADDRESSABLE memory (symmetric memory: every rank's buffer is mapped into every other
        rank's address space over NVLink), and register the neighbours' pointers with the library.  The v_out adjoint gets a (single)
        peer-addressable buffer as well, so the backward ghost reduction is fused into g2p.grad's scatter the same way.
        Falls back to the NCCL ghost all-reduce if symmetric memory cannot be set up on this system."""
        import ctypes as C
        from . import _lib
        sim = self.sim
        G = sim.n_grid ** 3
        nblk = (sim.n_grid // 8) ** 3
        try:
            peers = self._peer_factory(self.group, sim.device)
            buf, ptrs = peers.alloc((2, G, 4), torch.float32)
            fbuf, fptrs = peers.alloc((2, nblk), torch.int32)
            gbuf, gptrs = peers.alloc((G, 4), torch.float32)
            sbuf, sptrs = peers.alloc((8,), torch.int32)
        except Exception as e:  # pragma: no cover - depends on the driver / fabric
            if self.rank == 0:
                print(f'[fluidlab_b200.slab] symmetric memory unavailable ({type(e).__name__}: {e}); using the NCCL ghost all-reduce')
            self.exchange = 'nccl'
            return
        sim._grid_pm = buf
        sim._blk_flags = fbuf
        sim._ggrid_v = gbuf          # kept by MPMSimulator._ensure_grad_buffers
        sim._bind()
        self._peers = peers
        self._signal = sbuf
        slab = _lib.FmpmSlab()
        slab.enabled = 1
        slab.signal = sbuf.data_ptr()
        lo, hi = self.bounds[self.rank], self.bounds[self.rank + 1]
        if self.rank > 0:
            slab.peer_pm_left = int(ptrs[self.rank - 1]); slab.peer_flags_left = int(fptrs[self.rank - 1]); slab.peer_ggv_left = int(gptrs[self.rank - 1])
            slab.peer_signal_left = int(sptrs[self.rank - 1])
            slab.left_lo, slab.left_hi = lo - halo, lo + halo
        if self.rank < self.world - 1:
            slab.peer_pm_right = int(ptrs[self.rank + 1]); slab.peer_flags_right = int(fptrs[self.rank + 1]); slab.peer_ggv_right = int(gptrs[self.rank + 1])
            slab.peer_signal_right = int(sptrs[self.rank + 1])
            slab.right_lo, slab.right_hi = hi - halo, hi + halo
        sim._ck(sim._lib.fmpm_set_slab(sim._h, C.byref(slab)), 'fmpm_set_slab')
        # forward steps of the one-call path: PULL form of the ghost reduction (grid_op reads the neighbours' partial sums of the ghost planes; the
        # scatter kernels stay local) — decided from the bounds every rank knows, so all ranks take the same form: no slab narrower than its two
        # ghost ranges.  FMPM_SLAB_PULL=0: the push form (every ghost-plane reduction issued a second time over NVLink).
        import os
        widths = [self.bounds[r + 1] - self.bounds[r] for r in range(self.world)]
        self.pull = bool(self.sync == 'signal' and min(widths) >= 2 * halo and os.environ.get('FMPM_SLAB_PULL', '1') != '0')
        sim._ck(sim._lib.fmpm_set_slab_pull(sim._h, int(self.pull)), 'fmpm_set_slab_pull')
        if sim.device.type == 'cuda':
            torch.cuda.synchronize(sim.device)
        dist.barrier(group=self.group)

    def _census_async(self):
        """enqueue (no host sync): per-rank leaver counts -> all-gather -> total -> pinned host; read one step later."""
        sim = self.sim
        f = sim.cur_substep_local
        xs, alive = sim.slab_positions(f)
        cp = (xs * sim.inv_dx - 0.5).to(torch.int32) + 1
        out = torch.zeros((), dtype=torch.int64, device=xs.device)
        lost = torch.zeros((), dtype=torch.int64, device=xs.device)   # particles whose stencil left the planes shared with the neighbour
        if self.rank > 0:
            out = out + (alive & (cp < self.lo)).sum(); lost = lost + (alive & (cp < self.lo - (self.halo - 1))).sum()
        if self.rank < self.world - 1:
            out = out + (alive & (cp >= self.hi)).sum(); lost = lost + (alive & (cp >= self.hi + (self.halo - 1))).sum()
        out = (out + (lost << 40)).reshape(1)   # one word: leavers in the low 40 bits, halo violations above
        dist.all_reduce(out, group=self.group)
        if xs.device.type != 'cuda':   # host stand-in (tests): nothing is asynchronous
            self._census_host, self._census_event = out.clone(), _Done()
            return
        if self._census_host is None:
            self._census_host = torch.zeros(1, dtype=torch.int64).pin_memory()
        self._census_host.copy_(out, non_blocking=True)
        ev = torch.cuda.Event(); ev.record(torch.cuda.current_stream(xs.device))
        self._census_event = ev

    def _migrate(self):
        """Particles that left the slab move to the neighbour.  The decision uses the census enqueued one step earlier
        (identical on every rank), so a step without leavers anywhere costs no host synchronisation."""
        sim = self.sim
        need = False
        if self._census_event is not None:
            self._census_event.synchronize()
            word = int(self._census_host[0])
            if word >> 40:
                raise RuntimeError(f'SlabMPMSimulator: {word >> 40} particle(s) drifted beyond the {self.halo}-plane halo between two migrations: raise `halo` or lower '
                                   f'`migrate_every` (now {self.migrate_every})')
            need = (word & ((1 << 40) - 1)) != 0
        if need:
            f = sim.cur_substep_local
            st = sim.readframe_torch(f)
            state = dict(x=st['x'], v=st['v'], C=st['C'], F=st['F'], used=st['used'], mrow=sim._mrow, gid=self.gid)
            rec = {} if sim.grad_enabled else None
            gid_before = self.gid.clone() if sim.grad_enabled else None
            n_out, n_in = migrate(state, self.lo, self.hi, self.rank, self.world, sim.inv_dx, self.group, record=rec)
            if n_out or n_in:
                sim.setframe(f, state['x'], state['v'], state['C'], state['F'], state['used'])
                if rec is not None:
                    self._records[sim.cur_step_global] = rec
                    self._gid_before[sim.cur_step_global] = gid_before
            self.n_migrated += n_out
        self._census_async()

    def _checkpoint_chunk_start(self):
        """grad mode, first step of a chunk: keep what a later re-run of this chunk must start from (the reference checkpoints frame 0 of
        every chunk too, MPM:777-852; here additionally what migration changes — slot -> global id, material rows — and the census that
        decides whether THIS step migrates)"""
        sim = self.sim
        pending = None
        if self._census_event is not None:
            self._census_event.synchronize()
            pending = int(self._census_host[0])
        self._chunks[sim.cur_substep_global] = dict(frame=sim.slab_snapshot_frame(0), gid=self.gid.clone(), census=pending)

    def _replay_chunk(self, start):
        """backward pass at a chunk boundary (MPM:856-912): restore the chunk's first frame and run it forward again, exchanges included"""
        sim = self.sim
        ck = self._chunks[start]
        sim.slab_restore_frame(0, ck['frame'])
        sim.slab_adjoint_moves_to_frame(sim.max_substeps_local)   # copy_grad(0, T) + reset_grad_till_frame(T) of MPM:858-860
        self.gid = ck['gid'].clone()
        if self._census_event is not None:
            self._census_event.synchronize()   # no copy into the host word is in flight any more
        if ck['census'] is None:
            self._census_event = None
        else:
            if self._census_host is None:
                self._census_host = torch.zeros(1, dtype=torch.int64)
            self._census_host[0] = ck['census']
            self._census_event = _Done()
        n_steps = sim.max_substeps_local // sim.n_substeps
        sim.cur_substep_global = start
        self._replaying = True
        try:
            for _ in range(n_steps):
                self.step()
        finally:
            self._replaying = False

    def step(self):
        sim = self.sim
        if sim.grad_enabled and sim.cur_substep_local == 0 and not self._replaying:
            self._checkpoint_chunk_start()
        if self.world > 1 and self.migrate_enabled and (sim.cur_step_global % self.migrate_every == 0 or sim.grad_enabled):
            self._migrate()
        if self.sort_every > 0 and sim.cur_step_global % self.sort_every == 0:
            sim.sort_frame(sim.cur_substep_local)
        fuse = bool(getattr(sim, 'fuse_g2p2g', False)) and not sim.grad_enabled   # forward-only: g2p(f) + p2g(f+1) in one kernel (k_fwd)
        if self.exchange == 'peer' and self.sync == 'signal':   # the whole step in one library call, neighbour handshakes between the phases
            f0 = sim.cur_substep_local
            self._one_call_step(f0, fuse)
            for i in range(sim.n_substeps):
                sim._frame_ord[f0 + i + 1] = sim._frame_ord[f0]
            sim.cur_substep_global += sim.n_substeps
            self._wrap_if_needed()
            return
        for i in range(sim.n_substeps):
            f = sim.cur_substep_local
            if not (fuse and i > 0):
                sim.phase('p2g', f, 1)        # fused mode: the previous iteration's g2p2g already scattered frame f
            if self.exchange == 'peer':
                self._sync_ranks()   # device-side: every rank's p2g (incl. its peer reductions and peer block flags) has completed
            elif self.exchange == 'nccl':
                self._ghost_sum_acc(f)
            sim.phase('grid_op', f, 1)
            if fuse and i + 1 < sim.n_substeps:
                sim.phase('g2p2g', f)
            else:
                sim.phase('g2p', f)
            sim.cur_substep_global += 1
        self._wrap_if_needed()

    def _one_call_step(self, f0, fuse):
        """fmpm_substeps_slab(f0, n_substeps): [p2g | previous k_fwd] -> neighbour handshake -> grid_op -> [k_fwd | g2p] per substep, enqueued by ONE
        library call; replayed from a CUDA graph per (f0, fuse) when the device allows it (frame pointers are baked into the kernel arguments)."""
        sim = self.sim
        call = lambda: sim._ck(sim._lib.fmpm_substeps_slab(sim._h, f0, sim.n_substeps, int(fuse), sim._stream()), 'fmpm_substeps_slab')
        if not (self.use_graphs and getattr(sim, 'use_graphs', False) and sim.device.type == 'cuda'):
            return call()
        key = (f0, bool(fuse), bool(sim.grad_enabled))
        g = self._graphs.get(key)
        if g is None:
            from . import _lib
            try:
                g = torch.cuda.CUDAGraph()
                torch.cuda.synchronize(sim.device)
                with torch.cuda.graph(g):
                    call()
                self._graphs[key] = g
                # the capture did not run the kernels: fall through to a first replay
            except _lib.FmpmError:
                raise
            except RuntimeError as ex:
                import warnings
                warnings.warn(f'SlabMPMSimulator: CUDA-graph capture failed ({ex}); using direct launches')
                self.use_graphs = False
                return call()
        g.replay()

    def _wrap_if_needed(self):
        sim = self.sim
        if sim.cur_substep_local == 0 and not self._replaying:   # ring wrap: frame T becomes frame 0 of the next chunk
            if sim.grad_enabled:
                sim.copy_frame(sim.max_substeps_local, 0)
            else:
                sim.memory_to_cache()

    def sync_error(self):
        """True if a neighbour handshake ever gave up waiting (a peer rank stopped): host-synchronising, for tests / diagnostics"""
        return self.exchange == 'peer' and int(self._signal[3]) != 0

    def _sync_ranks(self):
        if self.sync == 'signal':
            self.sim._ck(self.sim._lib.fmpm_slab_sync(self.sim._h, self.sim._stream()), 'fmpm_slab_sync')
        else:
            self._peers.barrier()

    def _ghost_sum_acc(self, f):
        sim = self.sim
        acc = sim.slab_grid_acc(f)
        self.ghost.exchange_sum(acc)
        sim.slab_grid_acc_commit(f, acc)
        sim.slab_flag_blocks(f, self.ghost.flag_ghost_blocks)

    # ------------------------------------------------------------------------------------------ backward (SURVEY.md §8e)
    @property
    def param_grad(self):
        return False

    @param_grad.setter
    def param_grad(self, on):
        if on:
            raise NotImplementedError('SlabMPMSimulator: parameter gradients are single-GPU only (grid_op.grad runs on the ghost planes of both '
                                      'neighbouring ranks, so those nodes would count twice); use MPMSimulator.param_grad')

    def set_material_field(self, *args, **kwargs):
        raise NotImplementedError('SlabMPMSimulator: per-particle material fields are single-GPU only (migration would have to carry the field, '
                                  'and the slab backward has no parameter gradients); use MPMSimulator.set_material_field')

    def set_density_field(self, *args, **kwargs):
        raise NotImplementedError('SlabMPMSimulator: per-particle density fields are single-GPU only (migration would have to carry the field, '
                                  'and the slab backward has no parameter gradients); use MPMSimulator.set_density_field')

    def set_plastic_limits(self, *args, **kwargs):
        raise NotImplementedError('SlabMPMSimulator: plastic yield limits are single-GPU only (migration would have to carry them, and the slab '
                                  'backward has no parameter gradients); use MPMSimulator.set_plastic_limits')

    def set_plastic_field(self, *args, **kwargs):
        raise NotImplementedError('SlabMPMSimulator: plastic yield limits are single-GPU only (migration would have to carry them, and the slab '
                                  'backward has no parameter gradients); use MPMSimulator.set_plastic_field')

    def density_loss(self, *args, **kwargs):
        raise NotImplementedError('SlabMPMSimulator: the density loss is single-GPU only (a rank deposits only its own particles, the ghost '
                                  'planes would need the neighbours\' sum); use MPMSimulator.density_loss')

    add_x_grad_density = density_loss

    def momentum_loss(self, *args, **kwargs):
        raise NotImplementedError('SlabMPMSimulator: the momentum loss is single-GPU only (a rank deposits only its own particles, the ghost '
                                  'planes would need the neighbours\' sum); use MPMSimulator.momentum_loss')

    add_grad_momentum = momentum_loss

    def enable_grad(self):
        if getattr(self.sim, 'param_grad', False):
            raise NotImplementedError('SlabMPMSimulator: parameter gradients are single-GPU only; clear sim.param_grad')
        self.sim.enable_grad()
        self._records, self._gid_before, self._chunks = {}, {}, {}

    def local_state(self):
        """current frame of this rank in slot order: dict(gid, used, x, v, C, F) of device tensors (staging views: copy to keep)."""
        st = self.sim.readframe_torch(self.sim.cur_substep_local)
        return dict(gid=self.gid, **st)

    def set_final_grad(self, gx, gv=None, gC=None, gF=None):
        """seed the adjoint of the current frame (slot order of `local_state`); missing parts are zero."""
        sim = self.sim
        sim.reset_grad()
        N = gx.shape[0]
        z3 = torch.zeros((N, 3), dtype=torch.float32, device=gx.device); z9 = torch.zeros((N, 3, 3), dtype=torch.float32, device=gx.device)
        sim.write_grad_torch(dict(x=gx, v=z3 if gv is None else gv, C=z9 if gC is None else gC, F=z9 if gF is None else gF))

    def _substep_grad(self, f):
        sim = self.sim
        if self.exchange == 'peer' and self.sync == 'signal':
            sim.slab_substep_grad_one_call(f)
            return
        sim.slab_substep_grad_p2g(f)
        if self.exchange == 'peer':
            self._sync_ranks()
        elif self.exchange == 'nccl':
            self._ghost_sum_acc(f)
        sim.slab_substep_grad_scatter(f)
        if self.exchange == 'peer':
            self._sync_ranks()   # every rank's g2p.grad scatter, incl. its reductions into the neighbours' v_out adjoint, has completed
        elif self.world > 1:        # complete the v_out adjoint on the planes shared with the neighbours
            adj = sim.slab_grid_adj(f)
            self.ghost.exchange_sum(adj)
            sim.slab_grid_adj_commit(f, adj)
        sim.slab_substep_grad_finish(f)

    def step_grad(self):
        """adjoint of the most recent `step()` not yet undone; call in exact reverse order after `set_final_grad`."""
        sim = self.sim
        assert sim.grad_enabled and sim.cur_substep_global >= sim.n_substeps
        if sim.cur_substep_local == 0:   # the step to undo is the last one of the previous chunk: bring that chunk back into the ring
            self._replay_chunk(sim.cur_substep_global - sim.max_substeps_local)
        for _ in range(sim.n_substeps):
            sim.cur_substep_global -= 1
            self._substep_grad(sim.cur_substep_local)
        s = sim.cur_step_global
        rec = self._records.get(s)
        if rec is not None:   # this step began with a migration: send the adjoints of the arrivals back where they came from
            g = sim.read_grad_torch()
            migrate_grad(g, rec, self.group)
            sim.write_grad_torch(g)
            self.gid = self._gid_before[s]

    def gather_grad(self):
        """adjoint of the current frame for all used particles of all ranks, sorted by global id: dict(gid, x, v, C, F) numpy."""
        sim = self.sim
        used = sim.readframe_torch(sim.cur_substep_local, ('used',))['used'] != 0
        g = sim.read_grad_torch()
        rec = torch.cat([self.gid.view(torch.float32).reshape(-1, 1), g['x'], g['v'], g['C'].reshape(-1, 9), g['F'].reshape(-1, 9)], 1)
        r, gid = self._gather_by_gid(rec, used)
        return dict(gid=gid, x=r[:, 1:4], v=r[:, 4:7], C=r[:, 7:16].reshape(-1, 3, 3), F=r[:, 16:25].reshape(-1, 3, 3))

    def gather_state(self):
        """all used particles of all ranks, sorted by global id: dict(gid, x, v, F) numpy (every rank gets the same)."""
        sim = self.sim
        st = sim.readframe_torch(sim.cur_substep_local)
        used = st['used'] != 0
        rec = torch.cat([self.gid.view(torch.float32).reshape(-1, 1), st['x'], st['v'], st['F'].reshape(-1, 9)], 1)
        r, gid = self._gather_by_gid(rec, used)
        return dict(gid=gid, x=r[:, 1:4], v=r[:, 4:7], F=r[:, 7:16].reshape(-1, 3, 3))

    def _gather_by_gid(self, rec, used):
        """rows of the used slots of every rank (column 0 = global id bits), sorted by global id; same result on every rank."""
        rec = torch.where(used.reshape(-1, 1), rec, torch.full_like(rec, float('nan')))
        if self.world > 1:
            cap = torch.tensor([rec.shape[0]], device=rec.device); dist.all_reduce(cap, op=dist.ReduceOp.MAX, group=self.group)
            pad = int(cap.item()) - rec.shape[0]
            if pad:
                rec = torch.cat([rec, torch.full((pad, rec.shape[1]), float('nan'), device=rec.device)], 0)
            out = [torch.empty_like(rec) for _ in range(self.world)]
            dist.all_gather(out, rec, group=self.group)
            rec = torch.cat(out, 0)
        rec = rec.cpu()
        keep = ~torch.isnan(rec[:, 1])
        rec = rec[keep]
        gid = rec[:, 0].contiguous().view(torch.int32).numpy()
        order = np.argsort(gid, kind='stable')
        return rec.numpy()[order], gid[order]
