/* =====================================================================================
 * include/fluidmpm.h — C ABI of libfluidmpm.so, the CUDA-native (H100, sm_90a) MLS-MPM substep.
 *
 * Drop-in boundary for ONE hot path of zhouxian/FluidLab: the differentiable MLS-MPM substep of
 * fluidlab/fluidengine/simulators/mpm_simulator.py (abbrev. MPM below).  The reference binds this
 * path through Taichi kernels called from Python (`MPMSimulator.substep`, MPM:515-533, and
 * `substep_grad`, MPM:535-552); a replacement binds the entry points below through ctypes
 * (see INTEGRATION.md).  Plain pointers and sizes only — no torch types.
 *
 * Conventions
 *  - every function returns 0 on success, non-zero on failure (then fmpm_last_error() explains);
 *    no exceptions cross the ABI; the reference's own error behaviour (Python asserts) lives in
 *    the host layer (fluidlab_b200/).
 *  - all pointers are DEVICE pointers owned by the caller (torch tensors) unless stated;
 *    the library allocates nothing after fmpm_bind().
 *  - all work is enqueued on the `stream` argument (a cudaStream_t passed as void*), no implicit
 *    synchronisation; one handle per GPU; not thread-safe per handle (the reference is
 *    single-threaded, MPM:721-775).
 *  - `f` is a LOCAL frame index in [0, max_substeps_local] (MPM:225-227).
 *
 * Device data layout (see DESIGN.md §3).  N = particle slots, G = n_grid^3, T = max_substeps_local.
 *  state ring  pa : float4[(T+1)][4][N]  plane0=(x0,x1,x2,meta) plane1=(v0,v1,v2,C00)
 *                                         plane2=(C01,C02,C10,C11) plane3=(C12,C20,C21,C22)
 *              pf : float4[(T+1)][2][N]  (F00,F01,F02,F10) (F11,F12,F20,F21)
 *              pf8: float [(T+1)][N]     F22
 *  meta (int bits in plane0.w): bit0 = used (MPM:86-88), bit1 = collected at this substep (fmpm_collect, transient),
 *              bits 8..15 = row of the material table, bits 16..23 = body id (MPM:96-103; used by fmpm_advect_rigid).
 *  grads       ga/gf/gf8 : same planar layout, 2 frames (ping-pong: index 0/1).
 *  grid        grid_pm : float4[G] (momentum xyz, mass)   — MPM:112-114 v_in, mass
 *              grid_v  : float4[G] (v_out xyz, unused)     — MPM:115
 *              ggrid_v : float4[G] adjoint of v_out;  ggrid_pm : float4[G] adjoint of (v_in, mass)
 *              grid_v / ggrid_* are only defined on the ACTIVE 8^3-node blocks of the substep (blocks that received
 *              mass in p2g); grid_pm is all-zero between substeps.  n_grid must be a multiple of 8.
 *  Particles are stored in SLOT order (cell-sorted); `ids[slot]` = original particle index and
 *  `inv[pid]` = slot translate at the API boundary (fmpm_read_frame / fmpm_write_frame).
 * ===================================================================================== */
#ifndef FLUIDMPM_H_
#define FLUIDMPM_H_

#ifdef __cplusplus
extern "C" {
#endif

typedef struct FmpmHandle FmpmHandle;

/* material classes, fluidlab/configs/macros.py:37-41 */
enum { FMPM_MAT_LIQUID = 200, FMPM_MAT_PLASTO_ELASTIC = 201, FMPM_MAT_ELASTIC = 202, FMPM_MAT_RIGID = 203,
       FMPM_MAT_PLASTO_ELASTIC_DEMO = 204 };

/* replaces MPMSimulator.__init__ constants (MPM:14-34) + setup_boundary (MPM:39-40,
 * fluidlab/fluidengine/boundaries/boundaries.py:26-37,95-104) */
typedef struct {
  int n_grid;             /* MPM:21 */
  int n_particles;        /* MPM:54 */
  int max_substeps_local; /* MPM:27 (T) */
  int n_substeps;         /* MPM:30 */
  float dt, dx, inv_dx, p_vol; /* MPM:22-25 */
  float k_stress;         /* -dt*p_vol*4*inv_dx^2 evaluated in double then rounded, MPM:343 */
  float gravity[3];       /* MPM:19 */
  int boundary_type;      /* 0 cube, 1 cylinder */
  float b_lower[3], b_upper[3];
  float cyl_center[2], cyl_radius;
  float restitution;
  int lock_mask;          /* bit d: lock_dims contains d */
  int n_materials;        /* rows in the material table */
  int device;             /* CUDA device ordinal */
  int scene_flags;        /* FMPM_SCENE_* bits: what the host knows about the whole particle set (0 = nothing assumed) */
} FmpmConfig;
/* every row of the material table is a MAT_LIQUID with mu == 0 (WATER, MILK, COFFEE, ...: macros.py:131-201): the forward-only fused
 * substeps then skip the SVD entirely and carry F = J^(1/3) I (MPM:358-359) as one float per particle between step boundaries */
#define FMPM_SCENE_ALL_LIQUID_MU0 1

/* one row per distinct (material, rho): replaces particles_i.{mu,lam,mass,mat_cls} (MPM:96-103,170-175) */
typedef struct { float mu, lam, mass; int cls; } FmpmMaterial;

typedef struct {
  void* pa; void* pf; void* pf8;          /* state ring */
  void* ga; void* gf; void* gf8;          /* grad ping-pong (may be NULL when grads are never used) */
  void* grid_pm; void* grid_v; void* ggrid_v; void* ggrid_pm;
  void* materials;                        /* FmpmMaterial[n_materials] */
  void* scratch_a; void* scratch_f; void* scratch_f8;   /* one spare frame (sort / permute staging) */
  void* sort_keys_in; void* sort_keys_out; void* sort_vals_in; void* sort_vals_out; /* int[N] each */
  void* sort_tmp; unsigned long long sort_tmp_bytes;    /* >= fmpm_sort_workspace_bytes() */
  /* sparse grid: 8x8x8-node blocks.  blk_flags int[(n_grid/8)^3] (zero-initialised by the caller), blk_list int[(n_grid/8)^3],
   * blk_count int[1] (the last two are reserved).  p2g flags the blocks it scatters into and every grid kernel of the substep
   * (grid_op, clears, adjoint grid) scans the flags and visits only those blocks; the last consumer resets them. */
  void* blk_flags; void* blk_list; void* blk_count;
  /* optional per-frame grid ring for the backward pass (all four NULL = recompute the forward grid per backward substep):
   * grid_pm_ring / grid_v_ring float4[T][G] (zero-initialised), blk_list_ring int[T][(n_grid/8)^3] (zero; the per-frame block
   * flags), blk_count_ring int[T] (reserved).
   * fmpm_substep_store(f) leaves the (momentum, mass) and v_out grids of frame f in slot f; fmpm_substep_grad_stored(f) reads them.
   * The reference keeps a grid per frame too (MPM:117), 56 B/node dense; here 32 B/node and only touched blocks are rewritten. */
  void* grid_pm_ring; void* grid_v_ring; void* blk_list_ring; void* blk_count_ring;
  /* optional (both NULL = off): three (momentum, mass) accumulators float4[3][G] + their block flags int[3][(n_grid/8)^3], all zero.
   * With them fmpm_substeps_fused evaluates grid_op inside the fused gather / scatter kernel (one launch per substep; scenes without SDF
   * colliders at grid level): the launch of frame f gathers from accumulator f % 3, scatters frame f+1 into (f+1) % 3 and clears (f+2) % 3.
   * All three are clear again when fmpm_substeps_fused returns. */
  void* grid_pm3; void* blk_flags3;
} FmpmBuffers;

/* effector pose chain, fluidlab/fluidengine/effectors/effector.py:34-51 (fields), :157-161 (move_kernel),
 * :218-260 (set_action / set_velocity / apply_action_p), boundary = boundaries.py:65-78,122-125 impose_x */
typedef struct {
  void* pos; void* quat; void* v; void* w;          /* float[(T+1)*3|4] */
  void* gpos; void* gquat; void* gv; void* gw;      /* adjoints, same shapes */
  void* act; void* gact;                            /* float[max_action_steps*action_dim] */
  void* act_p; void* gact_p;                        /* float[action_dim] */
  int action_dim;
  float scale_v[6], scale_p[6];
  int boundary_type; float b_lower[3], b_upper[3]; float cyl_center[2], cyl_radius;
} FmpmEffector;

/* injector, fluidlab/fluidengine/effectors/injector.py:54-68,80-105 (Injector) and :220-256 (BallInjector) */
typedef struct {
  int kind;                 /* 1 Injector, 2 BallInjector */
  int flux;                 /* particles activated per substep */
  float radius;
  float inject_v[3], inject_p[3];
  const void* random_vector; /* float[random_length*flux*3] */
  const void* act_range;     /* int[n_act_range], original particle ids */
  int n_act_range;
  int randomize_inject_v;    /* injector.py:96-97 (Injector only): v += (2 random_vector - 1) * |inject_v| * 2 */
} FmpmInjector;

/* SDF mesh colliders: fluidlab/fluidengine/meshes/static.py:26-104 (Static.collide, applied in grid_op MPM:388-390) and
 * meshes/dynamic.py:29-121 (Dynamic.collide of the agent's Rigid effector, agents/agent_rigid.py:21-23, applied per particle in
 * g2p MPM:419-422 and/or per node in grid_op MPM:393-395 according to Agent.collide_type, agents/agent.py:17). */
typedef struct {
  const void* voxels;            /* float[res^3], the baked SDF volume (utils/mesh.py:63-87) */
  int res;
  float T_mesh_to_voxels[16];    /* row-major 4x4, already multiplied by inv(T_init) (meshes/mesh.py:121-127) */
  float friction, softness;      /* configs/macros.py:131-141 ; mesh cfg `softness` */
} FmpmSdfMesh;
typedef struct {
  int n_statics; FmpmSdfMesh statics[4];
  int has_rigid; int collide_type;          /* 0 particle, 1 grid, 2 both */
  FmpmSdfMesh rigid;
  const void* pos; const void* quat;        /* the Rigid effector's pose arrays float[(T+1)*3], float[(T+1)*4] */
  void* gpos;                               /* adjoint of pos (may be NULL when grads are never used) */
  void* gquat;                              /* adjoint of quat, float[(T+1)*4] (NULL: not accumulated; needed for 6-DOF actions) */
  float collide_y_min;                      /* the rigid collider only acts where y > this (agents/agent_icecreamdynamic.py:38-43); -1e30 = everywhere */
} FmpmColliders;
int  fmpm_set_colliders(FmpmHandle* h, const FmpmColliders* c);

/* Multi-GPU x-slab mode (no counterpart in the reference, which is single-device; SURVEY.md §8e).  The (momentum, mass)
 * accumulator becomes double-buffered by substep parity (grid_pm = float4[2][G]) and p2g adds every contribution that lands
 * on a ghost plane BOTH to the local grid and, with a vector reduction over NVLink peer memory, to the neighbour's grid
 * (peer_pm_* are the neighbours' grid_pm base pointers mapped into this process, e.g. through CUDA IPC).  After one barrier
 * between the ranks both copies of the ghost region hold the full sums — the ghost all-reduce is fused into the scatter. */
typedef struct {
  int enabled;
  void* peer_pm_left; void* peer_pm_right;   /* float4[2][G] of rank-1 / rank+1, NULL at the ends */
  void* peer_flags_left; void* peer_flags_right; /* the neighbours' blk_flags (int[2][(n_grid/8)^3]): p2g also flags the neighbour's blocks
                                                 it reduces into; in slab mode blk_flags is double-buffered by parity like grid_pm */
  int left_lo, left_hi;                      /* node planes [lo,hi) shared with the left neighbour */
  int right_lo, right_hi;                    /* node planes shared with the right neighbour */
  /* backward pass (optional, NULL = the caller sums the ghost planes of the v_out adjoint itself, e.g. with an all-reduce): the
   * neighbours' ggrid_v (float4[G], single-buffered).  g2p.grad's scatter then adds every contribution on a shared plane to the
   * neighbour's v_out adjoint as well, and grid_op.grad zeroes what it consumed, so the buffer is all-zero between substeps. */
  void* peer_ggv_left; void* peer_ggv_right;
  /* neighbour handshake (optional; NULL = the caller synchronises the ranks itself, e.g. with a symmetric-memory barrier): `signal` is this
   * rank's int[8] in peer-addressable memory — [0] last epoch posted by the left neighbour, [1] by the right one, [2] this rank's epoch
   * counter (device side), [3] error flag (a wait gave up) — peer_signal_* the neighbours' arrays.  fmpm_slab_sync posts this rank's next
   * epoch to both neighbours and waits for theirs: a slab only exchanges with its two neighbours, so no global barrier is needed. */
  void* signal; void* peer_signal_left; void* peer_signal_right;
} FmpmSlab;
int  fmpm_set_slab(FmpmHandle* h, const FmpmSlab* s);
int  fmpm_slab_sync(FmpmHandle* h, void* stream);     /* one tiny kernel: post epoch to the neighbours, spin (bounded) until theirs arrived */
/* the forward substeps f0..f0+n-1 of one x-slab rank in ONE call (no host round trip per phase; CUDA-graph capturable): per substep
 * p2g (or, with fuse != 0, the previous substep's g2p2g) -> fmpm_slab_sync -> grid_op -> g2p / g2p2g.  Needs the handshake arrays. */
int  fmpm_substeps_slab(FmpmHandle* h, int f0, int n, int fuse, void* stream);
/* on != 0: fmpm_substeps_slab uses the PULL form of the ghost reduction — the scatter kernels reduce into this rank's accumulator only and
 * grid_op, after the handshake, adds the neighbours' partial sums of the ghost planes read over NVLink (2 * halo planes of active nodes per
 * boundary instead of a second vector reduction for every scatter on those planes); the ghost blocks are cleared one handshake later, and the
 * call ends with one more handshake.  Needs peer_pm_* and peer_flags_*, disjoint ghost ranges, and the SAME setting on every rank (the ranks
 * handshake n + 1 times per call instead of n).  Default off (push form); the phase-level entry points always use the push form. */
int  fmpm_set_slab_pull(FmpmHandle* h, int on);

/* MAT_RIGID bodies: rigidity enforcement by shape matching (MPM:177-201 body structs, MPM:428-505 advect).
 * The body id of a particle travels in bits 16..23 of its meta word: pass mrow[p] = material_row | (body_id << 8) to
 * fmpm_write_frame.  All pointers are device memory owned by the caller. */
#define FMPM_BODY_STATE_STRIDE 48   /* floats per body per frame: COM_t0[3] COM_t1[3] H[9] U[9] S[3] V[9] R[9] pad[3] */
#define FMPM_BODY_GRAD_STRIDE 32    /* floats per body: gR[9] sum_gx[3] gH[9] gCOM_t0[3] gCOM_t1[3] pad[5] */
typedef struct FmpmBodies {
  int n_bodies;                               /* <= 256 */
  const void* info;                           /* int[n_bodies][2]: n_particles (MPM:199-200), mat_cls (MPM:201) */
  void* state;                                /* float[max_substeps_local][n_bodies][48]: body state of every substep of the ring,
                                                 written by the forward pass and reused by the adjoint (the reference recomputes it, MPM:437-441) */
  void* grad;                                 /* float[n_bodies][32]: adjoint scratch */
} FmpmBodies;
int  fmpm_set_bodies(FmpmHandle* h, const FmpmBodies* b);   /* n_bodies == 0 or NULL pointers: no rigid bodies */

int  fmpm_create(const FmpmConfig* cfg, FmpmHandle** out);
void fmpm_destroy(FmpmHandle* h);
int  fmpm_bind(FmpmHandle* h, const FmpmBuffers* b);
const char* fmpm_last_error(FmpmHandle* h);
unsigned long long fmpm_sort_workspace_bytes(FmpmHandle* h);
int  fmpm_abi_version(void);

/* ---- forward substep, MPM:515-533 (reset_grid .. advect) -------------------------------------- */
int fmpm_clear_grid(FmpmHandle* h, void* stream);                      /* MPM:219-223 */
int fmpm_p2g(FmpmHandle* h, int f, int write_F, void* stream);         /* MPM:254-264 + 331-378 fused */
int fmpm_grid_op(FmpmHandle* h, int f, int clear_pm, void* stream);    /* MPM:380-398 */
int fmpm_g2p(FmpmHandle* h, int f, void* stream);                      /* MPM:304-316 + 400-426 + 497-505 fused */
int fmpm_advect_rigid(FmpmHandle* h, int f, void* stream);             /* MPM:449-505 for MAT_RIGID bodies; after fmpm_g2p (no-op without such bodies) */
int fmpm_substep(FmpmHandle* h, int f, void* stream);                  /* p2g, grid_op(clear), g2p, advect_rigid; grid must be clear on entry */
int fmpm_substep_store(FmpmHandle* h, int f, void* stream);            /* same, but the grids of frame f stay in ring slot f */
/* forward-only fusion (no reference counterpart): g2p of frame f + p2g of frame f+1 in one kernel — v, C and x stay in registers
 * between the gather and the next scatter (104 B instead of 212 B per particle and substep).  write_vc = 0: v and C of frame f+1 are not
 * materialised (particles of MAT_RIGID bodies always get the complete frame: fmpm_advect_rigid(f) reads it, then fmpm_p2g_rigid(f+1) scatters them).  x-slab mode: the scatter half behaves like fmpm_p2g(f+1)
 * (peer reductions into the neighbours' accumulators of parity f+1): synchronise the ranks before fmpm_grid_op(f+1). */
int fmpm_g2p2g(FmpmHandle* h, int f, int write_vc, void* stream);
/* n substeps f0..f0+n-1: p2g(f0), [grid_op, g2p2g] x (n-1), grid_op, g2p(f0+n-1); frames f0 and f0+n are complete */
int fmpm_substeps_fused(FmpmHandle* h, int f0, int n, void* stream);
/* which kernels fmpm_substeps_fused uses for this handle (bit 0: k_fwd instead of k_g2p2g, bit 1: all-liquid specialisation, bit 2: grid_op
 * inlined with the triple-buffered accumulators, bit 3: footprint tiles staged by TMA); `mask` clears bits for A/B measurements
 * (fmpm_set_fwd_mask(h, 0) = the round-1 path: grid_op + k_g2p2g).  Default mask: everything except bit 2 (the in-kernel grid_op was
 * slower than the separate k_grid_op launch; fmpm_set_fwd_mask(h, 7) switches it on). */
/* ONE fused substep of the sequence above: g2p(f) + p2g(f+1) with the kernel fmpm_substeps_fused would pick (grid_op NOT inlined: run
 * fmpm_grid_op(f) before).  full != 0: frame f+1 and F[f+2] are written completely (the last fused substep of a step); full == 0: all-liquid
 * scenes write x, used and F22 only.  For hosts that interleave their own work between the substeps, and for per-kernel timing. */
int fmpm_fwd_step(FmpmHandle* h, int f, int full, void* stream);
int fmpm_fwd_path(FmpmHandle* h);
int fmpm_set_fwd_mask(FmpmHandle* h, int mask);
/* the same in grad mode with per-frame grids (like fmpm_substep_store): every frame is written completely, slot f+1's grids are cleared and
 * refilled by the fused kernel: 148 B instead of 212 B per particle and substep, 3 launches instead of 4 */
int fmpm_substeps_fused_store(FmpmHandle* h, int f0, int n, void* stream);
/* agent.act for injector agents, agents/agent_injector.py:23-32; run after fmpm_g2p of the same f */
int fmpm_inject(FmpmHandle* h, int f, const FmpmInjector* inj, const FmpmEffector* e, int act_id, int rand_row,
                const void* inv, void* stream);

/* collector_act_kernel of AgentPouring / AgentJetBot (agents/agent_pouring.py:31-41, agents/agent_jetbot.py:30-40): used particles of
 * frame f that lie outside the collector boundary (boundaries.py:81-93,128-134 is_out) leave the simulation: used[f] = used[f+1] = 0,
 * x[f+1] = NOWHERE (configs/macros.py:216).  Run BEFORE fmpm_substep(f) (the reference runs agent.act before p2g, MPM:521).  It only
 * clears the `used` bit of frame f and tags the particle (meta bit 1); fmpm_g2p(f) then writes the parked position into frame f+1. */
typedef struct FmpmCollector {
  int boundary_type;                 /* 0 cube, 1 cylinder */
  float lower[3], upper[3];          /* cylinder: [1] = y range */
  float cyl_center[2], cyl_radius;
  unsigned int row_mask;             /* material-table rows that are collected (AgentPouring: all rows; AgentJetBot: the WATER rows) */
} FmpmCollector;
int fmpm_collect(FmpmHandle* h, int f, const FmpmCollector* c, void* stream);

/* ---- g2p2g fusion with agents (declared here because they take an FmpmCollector) ---------------- */
/* with a collector agent: the collector's test (fmpm_collect of frame f+1) is applied to the new position inside the kernel, before its scatter */
int fmpm_g2p2g_collect(FmpmHandle* h, int f, int write_vc, const FmpmCollector* col, void* stream);
/* fused steps with an injector agent (agents/agent_injector.py): after fmpm_g2p2g(f-1) and fmpm_inject(f-1, ...) the few newly activated
 * particles of frame f are scattered separately, before fmpm_grid_op(f) */
int fmpm_p2g_injected(FmpmHandle* h, int f, const FmpmInjector* inj, int act_id, const void* inv, int ring_slot, const FmpmCollector* col /* or NULL */,
                      void* stream);   /* ring_slot: -1, or f in grad mode */
/* the pieces of fmpm_substep_store / fmpm_substeps_fused_store one by one (ring slot = frame), for hosts that interleave agent kernels */
int fmpm_clear_ring_slot(FmpmHandle* h, int f, void* stream);
int fmpm_p2g_store(FmpmHandle* h, int f, void* stream);
int fmpm_grid_op_store(FmpmHandle* h, int f, void* stream);
int fmpm_g2p_store(FmpmHandle* h, int f, void* stream);
int fmpm_p2g_rigid(FmpmHandle* h, int f, int ring_slot, const FmpmCollector* col /* or NULL */, void* stream);   /* fused steps with MAT_RIGID bodies: their particles' scatter of frame f, after fmpm_advect_rigid(f-1) */
int fmpm_g2p2g_store(FmpmHandle* h, int f, const FmpmCollector* col /* or NULL */, void* stream);       /* gathers from slot f, scatters into slot f+1 (cleared before), writes frame f+1 completely */

/* ---- backward substep, MPM:535-552 ------------------------------------------------------------ */
/* gin/gout in {0,1}: grad ping-pong index holding frame f+1 (in) and receiving frame f (out). */
int fmpm_substep_grad(FmpmHandle* h, int f, int gin, int gout, void* stream);
int fmpm_substep_grad_stored(FmpmHandle* h, int f, int gin, int gout, void* stream);  /* uses the grids left by fmpm_substep_store(f) */
/* x-slab backward (no reference counterpart; SURVEY.md 8e): fmpm_substep_grad cut at its two ghost exchanges.  Per rank and substep:
 *   fmpm_p2g(f, 0) -> [ghost sum of the (momentum, mass) planes] -> fmpm_substep_grad_scatter (grid_op + g2p.grad grid scatter)
 *                  -> [ghost sum of the v_out-adjoint planes]    -> fmpm_substep_grad_finish  (grid_op.grad, accumulators cleared, particle side) */
int fmpm_substep_grad_scatter(FmpmHandle* h, int f, int gin, void* stream);
int fmpm_substep_grad_finish(FmpmHandle* h, int f, int gin, int gout, void* stream);
/* the three steps above with the two neighbour handshakes (fmpm_slab_sync) in between, in one call; needs FmpmSlab.peer_ggv_* and .signal */
int fmpm_substep_grad_slab(FmpmHandle* h, int f, int gin, int gout, void* stream);
/* MPM:436-447 advect_grad for MAT_RIGID bodies: call BEFORE fmpm_substep_grad* / fmpm_g2p_grad_scatter of the same f (it rewrites
 * the x and v adjoints of rigid particles in gin in place; no-op without such bodies).  next_slot: int[N], slot in frame f+1 of the
 * particle in slot s of frame f, or NULL when both frames share one slot order (no cell sort between them). */
int fmpm_advect_rigid_grad(FmpmHandle* h, int f, int gin, const void* next_slot, void* stream);
int fmpm_g2p_grad_scatter(FmpmHandle* h, int f, int gin, void* stream);           /* g2p.grad: grid side */
int fmpm_grid_op_grad(FmpmHandle* h, int f, void* stream);                        /* grid_op.grad */
int fmpm_particle_grad(FmpmHandle* h, int f, int gin, int gout, void* stream);    /* advect/g2p/p2g/svd/F_tmp .grad: particle side */
int fmpm_inject_grad(FmpmHandle* h, int f, int gin, const FmpmInjector* inj, const FmpmEffector* e, int act_id,
                     const void* inv, void* stream);

/* ---- gradients with respect to the physics (no reference counterpart: the reference returns dL/dAction only) ----------------------
 * While bound, every backward substep (fmpm_substep_grad, fmpm_substep_grad_stored, and the phases fmpm_grid_op_grad / fmpm_particle_grad)
 * ADDS its share of the loss gradient with respect to the material table and gravity to two caller-owned fp64 device arrays; the caller
 * zeroes them before a backward pass.  Per used, in-grid particle p of row r (P = 2 mu (F~ - R) F~^T + lam J (J - 1) I, A = k_stress P + m C,
 * gA = the adjoint of A, gvp = sum_i w_i (adjoint of v_in)_i):
 *   gmat[r][0] += 2 k_stress gA : ((F~ - R) F~^T)     dL/dmu
 *   gmat[r][1] += k_stress J (J - 1) tr(gA)            dL/dlam
 *   gmat[r][2] += v . gvp + gA : C + sum_i w_i gm_i    dL/dmass (gm = adjoint of the node mass); dL/drho = p_vol * dL/dmass
 * and per node with mass, ggrav += dt * (adjoint of v_in / m + dt g, before the colliders and the boundary).  Partial sums within a substep
 * are fp32, the accumulation across substeps fp64.  The x-slab backward (fmpm_substep_grad_finish / _slab) refuses to run while bound
 * (grid_op.grad visits the ghost planes on both ranks). */
typedef struct FmpmParamGrad {
  void* gmat;    /* double[n_materials][4]: dL/dmu, dL/dlam, dL/dmass, 0 */
  void* ggrav;   /* double[3] */
} FmpmParamGrad;
int fmpm_set_param_grad(FmpmHandle* h, const FmpmParamGrad* g);   /* NULL or both NULL: off (default); exactly one NULL is an error */
/* gravity lives in the by-value kernel parameter block: the new value applies to launches enqueued after this call (a captured CUDA graph
 * keeps the value it was captured with).  The material table itself is caller-owned device memory read at run time: rewrite its rows in place. */
int fmpm_set_gravity(FmpmHandle* h, const float g[3]);
/* FmpmConfig.scene_flags after creation; FMPM_SCENE_ALL_LIQUID_MU0 must be dropped before any row gets mu != 0 or a class other than
 * MAT_LIQUID.  Change it only at a step boundary (frames inside a fused all-liquid step carry F as one float). */
int fmpm_set_scene_flags(FmpmHandle* h, int scene_flags);

/* ---- per-particle mu and lam (no reference counterpart as an input: the reference keeps mu, lam and mass per particle, MPM:96-103) ----------
 * While bound, every constitutive evaluation of the particle in slot s (forward, the backward's recompute and the backward itself; MAT_RIGID,
 * injected and plastic particles included) takes (mu, lam) = field[s] instead of mu and lam of its material row.  The mass, the material class
 * (the liquid / plastic / elastic branch of the constitutive model) and the row masks of the losses still come from the row.  The field is read
 * by slot: the caller keeps it in the slot order of the frames it runs (re-gathered after every fmpm_sort) and keeps the pointer fixed while
 * CUDA graphs captured with it are replayed.
 *  - Binding needs FMPM_SCENE_ALL_LIQUID_MU0 clear, and fmpm_set_scene_flags refuses that flag while a field is bound: the all-liquid kernels
 *    carry F as one float and take mu = 0 for granted, so a field always runs the general instantiations.
 *  - Not in x-slab mode: binding fails while fmpm_set_slab has enabled it, and fmpm_set_slab(enabled) fails while a field is bound.
 *    fmpm_substeps_fused fails with the opt-in in-kernel grid_op (fmpm_set_fwd_mask bit 2) while a field is bound.
 *  - With FmpmParamGrad bound too, the backward substeps do NOT write gmat[r][0..1]: they ADD dL/dmu and dL/dlam of the particle in slot s to
 *    gfield[s] instead (plain read-modify-write adds: one lane owns one slot, no atomics; the caller zeroes gfield and re-orders it with the
 *    field).  dL/dmass still goes to gmat[r][2].  A backward substep with FmpmParamGrad bound and gfield NULL fails. */
typedef struct FmpmMaterialField {
  const void* field;   /* float2[N] (mu, lam) in the CURRENT SLOT ORDER, or NULL = off */
  void* gfield;        /* float2[N] slot-order accumulator of (dL/dmu, dL/dlam), or NULL; used only while FmpmParamGrad is bound */
} FmpmMaterialField;
int fmpm_set_material_field(FmpmHandle* h, const FmpmMaterialField* m);   /* NULL or field NULL: off (default); fails while a mass field is bound */

/* ---- per-particle mass (the reference keeps particles_i.mass per particle, MPM:96-103, set at MPM:174) -------------------------------------
 * While bound, every place the kernels read a particle's mass takes m = mass[s] instead of the mass of its material row: the forward scatter
 * (q = m v, A = k_stress P + m C and the node mass; plain, fused, injected and MAT_RIGID scatter), the backward's recompute and the backward
 * itself, and the deposits and adjoints of the density and momentum losses.  The material class and the losses' row masks stay the row's;
 * MAT_RIGID shape matching weights particles by count and reads no mass.  Same slot-order and pointer rules as FmpmMaterialField.
 *  - Binding needs a bound FmpmMaterialField (a mass field always runs the instantiations with mu, lam AND mass per slot: a caller that only
 *    wants the mass binds a mu, lam field gathered from its rows), and fmpm_set_material_field(NULL) fails while a mass field is bound.  So the
 *    refusals of the material field hold for it too: no x-slab mode (either call order), no in-kernel grid_op.
 *  - With FmpmParamGrad bound too, the backward substeps and the loss gradients (fmpm_loss_density_grad, fmpm_loss_momentum_grad) do NOT write
 *    gmat[r][2]: they ADD dL/dm of the particle in slot s to gmass[s] instead (plain read-modify-write adds, one lane per slot).  A backward
 *    substep or loss gradient with FmpmParamGrad bound and gmass NULL fails. */
typedef struct FmpmMassField {
  const void* mass;   /* float[N] m_p in the CURRENT SLOT ORDER, or NULL = off */
  void* gmass;        /* float[N] slot-order accumulator of dL/dm, used only while FmpmParamGrad is bound */
} FmpmMassField;
int fmpm_set_mass_field(FmpmHandle* h, const FmpmMassField* m);   /* NULL or mass NULL: off (default); fails while a plastic field is bound */

/* ---- per-particle plastic yield limits (the reference clamps plasto-elastic singular values to [1 - 2e-3, 1 + 3e-3], MPM:367-376) ---------
 * While bound, every constitutive evaluation of the particle in slot s takes (mu, lam, lo, hi) = field[s]: mu and lam as FmpmMaterialField,
 * and a particle of a plasto-elastic class (FMPM_MAT_PLASTO_ELASTIC, FMPM_MAT_PLASTO_ELASTIC_DEMO) gets F[f+1] = U diag(clamp(sig, lo, hi)) V^T
 * (liquid, elastic and rigid particles never read lo / hi).  Without it the limits are f32(1 - 2e-3) = 0.998f and f32(1 + 3e-3) = 1.003f.
 * The kernels of this level read the 16-byte record alone, so field[s].xy replaces the material field's entry (which stays bound but unread).
 * Same slot-order and pointer rules as FmpmMaterialField.
 *  - Binding needs a bound FmpmMassField (which needs a bound FmpmMaterialField): the plastic field runs the instantiations with mu, lam, the
 *    limits AND the mass per slot.  fmpm_set_mass_field(NULL) fails while a plastic field is bound.  So the refusals of the material field hold
 *    for it too: no x-slab mode (either call order), no in-kernel grid_op, no FMPM_SCENE_ALL_LIQUID_MU0.
 *  - With FmpmParamGrad bound too, the backward substeps ADD (dL/dmu, dL/dlam, dL/dlo, dL/dhi) of the particle in slot s to gfield[s] (plain
 *    read-modify-write adds, one lane per slot) instead of the material field's gfield, and dL/dm to FmpmMassField.gmass.  With W = U^T gF' V
 *    (gF' the adjoint of F[f+1]) and the tie rule of the clamp's adjoint (axis d is at lo unless lo < sig_d, and at hi when lo < sig_d and
 *    not max(sig_d, lo) < hi), dL/dlo += W_dd over the axes at lo and dL/dhi += W_dd over the axes at hi.  A backward substep with FmpmParamGrad
 *    bound and gfield NULL fails. */
typedef struct FmpmPlasticField {
  const void* field;   /* float4[N] (mu, lam, lo, hi) in the CURRENT SLOT ORDER, 0 < lo <= hi, or NULL = off */
  void* gfield;        /* float4[N] slot-order accumulator of (dL/dmu, dL/dlam, dL/dlo, dL/dhi), used only while FmpmParamGrad is bound */
} FmpmPlasticField;
int fmpm_set_plastic_field(FmpmHandle* h, const FmpmPlasticField* m);   /* NULL or field NULL: off (default) */

/* ---- gradients with respect to the contact parameters --------------------------------------------------------------------------------
 * While bound (and only together with FmpmParamGrad), every backward substep also ADDS the loss gradient with respect to the friction of
 * every colliding static, the friction and softness of the agent's Rigid mesh and the wall restitution to a caller-owned fp64 device array
 * double[8]: [0..3] static friction (order of FmpmColliders.statics), [4] rigid friction, [5] rigid softness, [6] restitution, [7] = 0.
 * Per collide evaluation (grid level in fmpm_grid_op_grad, particle level in the Dynamic.collide pre-pass) with incoming adjoint gout and the
 * names of meshes/dynamic.py:93-121 (rel, n, vn, rt, rtn, infl = min(exp(-sd softness), 1), out = cv + rt2 infl + rel (1 - infl)):
 *   friction += vn sbar / rtn, sbar = sum_k rt_k infl gout_k      when vn < 0, rtn > eps and rtn + vn friction > 0 (else 0; the sticky branch,
 *                                                                  friction > 10 on a Rigid mesh, has zero derivative)
 *   softness += ginfl (-sd) infl, ginfl = gout . (rt2 - rel)       Rigid mesh, hit and exp(-sd softness) < 1 (the hit test carries no gradient)
 * and per node with mass and axis i on which the wall reflects (v_out_i = -restitution v_in_i; not a locked axis, not the cylinder's radial
 * kill):  restitution += -v_in_i gv_out_i.  Partial sums are fp32 within a substep and CTA, the accumulation across substeps fp64; the
 * caller zeroes the array.  The x-slab backward refuses to run while bound. */
typedef struct FmpmContactGrad {
  void* gcontact;   /* double[8] */
} FmpmContactGrad;
int fmpm_set_contact_grad(FmpmHandle* h, const FmpmContactGrad* g);   /* NULL (or gcontact NULL): off; binding needs fmpm_set_param_grad
                                                                         bound, and unbinding that also unbinds this */
/* restitution lives in the by-value kernel parameter block like gravity: the new value applies to launches enqueued after this call.
 * Friction and softness travel with fmpm_set_colliders. */
int fmpm_set_restitution(FmpmHandle* h, float restitution);

/* ---- frame ring / io, MPM:555-609 -------------------------------------------------------------- */
/* API layout: x,v float[N,3]; C,F float[N,3,3]; used int[N]; mrow int[N] (material row); all indexed by
 * ORIGINAL particle id.  ids == NULL means identity order. */
int fmpm_write_frame(FmpmHandle* h, int f, const void* x, const void* v, const void* C, const void* F,
                     const void* used, const void* mrow, const void* ids, void* stream);   /* setframe MPM:566-575 */
int fmpm_read_frame(FmpmHandle* h, int f, void* x, void* v, void* C, void* F, void* used, const void* ids, void* stream); /* readframe MPM:555-564 */
int fmpm_write_grad(FmpmHandle* h, int g, const void* x, const void* v, const void* C, const void* F, const void* ids, void* stream);
int fmpm_read_grad(FmpmHandle* h, int g, void* x, void* v, void* C, void* F, const void* ids, void* stream);
int fmpm_zero_grad(FmpmHandle* h, int g, void* stream);
int fmpm_copy_frame(FmpmHandle* h, int src, int dst, void* stream);                        /* MPM:588-595 */
/* re-express grad buffer gsrc (slot order ids_src) in the slot order whose inverse map is inv_dst -> buffer gdst */
int fmpm_permute_grad(FmpmHandle* h, int gsrc, int gdst, const void* ids_src, const void* inv_dst, void* stream);
/* cell-sort frame f in place: ids_in[slot] -> ids_out / inv_out describe the new order (ids_in may be NULL = identity) */
int fmpm_sort(FmpmHandle* h, int f, const void* ids_in, void* ids_out, void* inv_out, void* stream);
/* grid accessors for phase-level parity tests: float[G,3], float[G], float[G,3] (any may be NULL) */
int fmpm_read_grid(FmpmHandle* h, void* v_in, void* mass, void* v_out, void* stream);
int fmpm_read_grid_grad(FmpmHandle* h, void* gv_in, void* gmass, void* gv_out, void* stream);
int fmpm_write_grid_grad(FmpmHandle* h, const void* gv_in, const void* gmass, const void* gv_out, void* stream);

/* ---- effector chain --------------------------------------------------------------------------- */
/* set_action (effector.py:262-268) for step s / s_global followed by the n_substeps move_kernel calls of that step
 * (effector.py:157-161); `action` is a device float[action_dim]. */
int fmpm_effector_step(FmpmHandle* h, const FmpmEffector* e, int s, int s_global, const void* action, void* stream);
/* adjoint of the above: n_substeps move_kernel.grad (reverse) then set_velocity.grad (effector.py:270-274) */
int fmpm_effector_step_grad(FmpmHandle* h, const FmpmEffector* e, int s, int s_global, void* stream);
int fmpm_effector_apply_action_p(FmpmHandle* h, const FmpmEffector* e, void* stream);       /* effector.py:223-226 */
int fmpm_effector_apply_action_p_grad(FmpmHandle* h, const FmpmEffector* e, void* stream);  /* effector.py:233-234 */

/* ---- index-matched shape loss, fluidlab/fluidengine/losses/shapematching_loss.py:80-93 ---------- */
/* loss_out[0] += weight * sum_{p used, mrow_mask bit set} |x[f,p]-tgt[p]|^2 ; tgt float[N,3] by original id */
int fmpm_loss_chamfer(FmpmHandle* h, int f, const void* ids, const void* tgt, unsigned int mrow_mask_lo,
                      float weight, void* loss_out, void* stream);
/* x-grad of buffer g += 2*weight*(x-tgt) (compute_chamfer_loss_kernel.grad with total_loss.grad = 1) */
int fmpm_loss_chamfer_grad(FmpmHandle* h, int f, int g, const void* ids, const void* tgt, unsigned int mrow_mask_lo,
                           float weight, void* stream);

/* ---- correspondence-free density loss on the simulation grid (DESIGN.md §4) ------------------------------------------------------------
 * m_i = sum_p m_p w_ip over the used particles of frame f whose row is in mrow_mask_lo and whose 3x3x3 stencil is inside the grid (the
 * weights and nodes of p2g), L = w_density sum_i (m_i - m*_i)^2 + w_sdf sum_i m_i phi*_i.  Volumes are float[G] in the node layout of
 * fmpm_read_grid.  The adjoint gbar_i = 2 w_density (m_i - m*_i) + w_sdf phi*_i gives x_p += m_p sum_i gbar_i grad w_ip (the stencil base
 * carries no gradient) and, while fmpm_set_param_grad is bound, gmat[row][2] (dL/dmass) += sum_{p in row} sum_i gbar_i w_ip. */
typedef struct FmpmDensityLoss {
  void* mass;            /* float[G] scratch, overwritten by every call */
  const void* target;    /* float[G] m*, or NULL = 0 */
  const void* sdf;       /* float[G] phi*, or NULL = 0 */
  float w_density, w_sdf;
  unsigned int mrow_mask_lo;
  int reserved;
} FmpmDensityLoss;
int fmpm_loss_density(FmpmHandle* h, int f, const FmpmDensityLoss* l, void* loss_out, void* stream);      /* loss_out[0] += L_s */
int fmpm_loss_density_grad(FmpmHandle* h, int f, int g, const FmpmDensityLoss* l, void* stream);         /* x-adjoint of buffer g (+ gmat); re-deposits frame f */

/* ---- correspondence-free momentum loss on the simulation grid (DESIGN.md §4) -----------------------------------------------------------
 * The particles of fmpm_loss_density also deposit p2g's APIC momentum P_i = sum_p m_p w_ip u_ip, u_ip = v_p + C_p d_ip,
 * d_ip = (o_i - fx_p) dx, and L = w_density sum_i (m_i - m*_i)^2 + w_sdf sum_i m_i phi*_i + w_momentum sum_i |P_i - P*_i|^2.  With
 * a_i = 2 w_density (m_i - m*_i) + w_sdf phi*_i, b_i = 2 w_momentum (P_i - P*_i) and the stencil base held fixed, the adjoint adds
 * v_p += m_p sum_i w_ip b_i, C_p += m_p sum_i w_ip b_i d_ip^T, x_p += m_p sum_i [grad w_ip (a_i + b_i . u_ip) - w_ip C_p^T b_i] to planes
 * 0..3 of the adjoint buffer and, while fmpm_set_param_grad is bound, gmat[row][2] (dL/dmass) += sum_{p in row} sum_i w_ip (a_i + b_i . u_ip). */
typedef struct FmpmMomentumLoss {
  void* field;           /* float4[G] (P, m) scratch, overwritten by every call */
  const void* target;    /* float4[G] (P*, m*), or NULL = 0 */
  const void* sdf;       /* float[G] phi*, or NULL = 0 */
  float w_density, w_sdf, w_momentum;
  unsigned int mrow_mask_lo;
} FmpmMomentumLoss;
int fmpm_loss_momentum(FmpmHandle* h, int f, const FmpmMomentumLoss* l, void* loss_out, void* stream);    /* loss_out[0] += L_s */
int fmpm_loss_momentum_grad(FmpmHandle* h, int f, int g, const FmpmMomentumLoss* l, void* stream);       /* x, v, C adjoint of buffer g (+ gmat); re-deposits frame f */

/* ---- trajectory optimiser step, fluidlab/optimizer/optim.py:22-41 + optimizer/policies.py:152-164 --- */
/* One Adam update of the composite action table (rows = horizon + 1: the action_v rows, then action_p; cols = action_dim), resident on the
 * device: params / m / v are double[rows*cols] (the reference keeps them in float64), grads is float[rows*cols] (agent.get_grad's dtype),
 * trainable is unsigned char[rows] or NULL.  Rows with trainable == 0 and columns in fix_dim_mask see a zero gradient; the first rows-1 rows
 * are clipped to [clip_lo, clip_hi] after the update (policies.py:158-164).  bias_1 / bias_2 = 1 - beta^(iter+1), computed by the caller.
 * Every operation is rounded as NumPy rounds it (no contraction), so the result is bit-identical to the reference's. */
typedef struct FmpmAdamCfg {
  double lr, beta_1, beta_2, epsilon, bias_1, bias_2, clip_lo, clip_hi;
  int rows, cols;
  unsigned int fix_dim_mask;
  int reserved;
} FmpmAdamCfg;
int fmpm_adam_step(FmpmHandle* h, const FmpmAdamCfg* cfg, void* params, void* m, void* v, const void* grads, const void* trainable, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FLUIDMPM_H_ */
