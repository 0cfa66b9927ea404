// fmpm_scatter.cuh — register sliding-window scatter shared by p2g (momentum + mass) and the g2p adjoint
// (v_out adjoint).  See fmpm_forward.cu for the rationale (no native shared-memory float atomics on sm_90a).
//
// Two modes alternate inside a warp:
//   particle mode  lane = particle slot: constitutive math, then `scatter_publish` stages per particle
//                  (q, B, m) + its 27 stencil weights + its cell key into the warp's shared staging area and
//                  derives, with ballots, the bit mask of positions where a new cell starts;
//   node mode      lane = stencil node (a,b,c) (27 of 32 lanes): `window_consume` walks the staged particles
//                  run by run (all particles of a run share one cell, so the inner loop has no branches:
//                  4 LDS.128 + 1 LDS + 8 FFMA pairs per particle) accumulating
//                       acc(a,b,c) += w_abc * ( q + B·(a,b,c) ),   acc.m += w_abc * m
//                  in registers; at a run boundary the window either shifts one cell along z (shuffle, flush of the
//                  finished 3x3 plane) or is flushed entirely — flushes are REDG.E.ADD.F32x4 vector reductions.
#pragma once
#include <cuda_runtime.h>

#define SC_FULL 0xffffffffu

#ifdef FMPM_HOST_EMU   // host build of the CUDA execution-model tests (tests/cuda_emu/): no PTX there
__device__ __forceinline__ void red_add_v4(float4* addr, const float4& v) { atomicAdd(&addr->x, v.x); atomicAdd(&addr->y, v.y); atomicAdd(&addr->z, v.z); atomicAdd(&addr->w, v.w); }
__device__ __forceinline__ float2 ffma2(const float2 a, const float2 b, const float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fmul2(const float2 a, const float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
#else
__device__ __forceinline__ void red_add_v4(float4* addr, const float4& v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// sm_90a has no packed fp32 FMA: a pair is two FFMA / FMUL.  The _rn intrinsics keep each lane an IEEE round-to-nearest
// operation that the compiler may not contract or reassociate, so the arithmetic matches the oracle's scalar fp32 order.
__device__ __forceinline__ float2 ffma2(const float2 a, const float2 b, const float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fmul2(const float2 a, const float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
#endif

// the same under a per-lane predicate: one predicated REDG, no branch / convergence barrier around the flush
#ifdef FMPM_HOST_EMU
__device__ __forceinline__ void red_add_v4_if(const bool p, float4* addr, const float4& v) { if (p) red_add_v4(addr, v); }
#else
__device__ __forceinline__ void red_add_v4_if(const bool p, float4* addr, const float4& v) {
  asm volatile("{\n\t.reg .pred pr;\n\tsetp.ne.s32 pr, %5, 0;\n\t@pr red.global.add.v4.f32 [%0], {%1, %2, %3, %4};\n\t}" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "r"((int)p) : "memory");
}
#endif
#define SC_REC 9           // float4 records per particle: 36-word stride, so the 128-bit stores of lane = particle are bank-conflict free
#define SC_WQ 7            // float4 per particle of stencil weights (27 + 1 pad): 28-word stride, conflict free as well
struct __align__(128) ScatterSmem {   // 128-byte aligned: `rec` doubles as the destination of the TMA footprint tile (k_fwd)
  // per particle: nine Q_ab = (q + a*B[:,0] + b*B[:,1], m) for the (a,b) node columns of the stencil and b2 = (B02,B12,B22,0):
  // a lane (a,b,c) needs only Q_ab + c*B[:,2], i.e. 2 LDS.128 + 1 LDS and 4 FFMA pairs per particle
  float4 rec[32 * SC_REC];
  float4 b2[32];
  float4 w[32 * SC_WQ];      // ((float*)w)[particle*28 + node]: lane = particle writes 7 x STS.128, lane = node reads consecutive words
  int key[32];
};

// cell keys are the packed base coordinates (bx << 20 | by << 10 | bz), n_grid <= 1024
__device__ __forceinline__ int pack_key(const int* b) { return (b[0] << 20) | (b[1] << 10) | b[2]; }

struct Window {
  float2 acc01, acc2m;   // (x,y) and (z,mass) accumulators of this lane's stencil node
  int cur_key;           // packed cell whose 27 nodes the window currently covers (-1 = empty)
  int node;              // linear grid index of this lane's node for cur_key
  float oa, ob, oc; int a, b, c; bool lane_valid; int wrow; int qidx;
  int n, nb; int* flags; // grid size, blocks per dim, active-block flags (nullptr: do not flag)
  // x-slab mode: the neighbours' accumulators (NVLink peer memory) and the node planes shared with them
  float4* peer_l; float4* peer_r; int gl_lo, gl_hi, gr_lo, gr_hi; int plane;
  int* peer_fl; int* peer_fr;
};
__device__ __forceinline__ void window_init(Window& W, const int lane, const int n, int* flags) {
  const int L = lane < 27 ? lane : 26;
  const int a = (L >= 9) + (L >= 18), r = L - 9 * a, b = (r >= 3) + (r >= 6), c = r - 3 * b;   // L = 9 a + 3 b + c without integer divisions
  W.oa = (float)a; W.ob = (float)b; W.oc = (float)c; W.a = a; W.b = b; W.c = c;
  W.lane_valid = lane < 27;
  W.wrow = L; W.qidx = a * 3 + b;
  W.acc01 = make_float2(0.f, 0.f); W.acc2m = make_float2(0.f, 0.f);
  W.cur_key = -1; W.node = 0;
  W.n = n; W.nb = n >> 3; W.flags = flags;
  W.peer_l = W.peer_r = nullptr; W.gl_lo = W.gl_hi = W.gr_lo = W.gr_hi = 0; W.plane = 0; W.peer_fl = W.peer_fr = nullptr;
}
__device__ __forceinline__ void window_set_slab(Window& W, float4* peer_l, float4* peer_r, int gl_lo, int gl_hi, int gr_lo, int gr_hi, int* peer_fl, int* peer_fr) {
  W.peer_l = peer_l; W.peer_r = peer_r; W.gl_lo = gl_lo; W.gl_hi = gl_hi; W.gr_lo = gr_lo; W.gr_hi = gr_hi; W.peer_fl = peer_fl; W.peer_fr = peer_fr;
}
// one vector reduction into the local accumulator and, for nodes on a plane shared with a neighbouring slab, the same
// reduction into that neighbour's accumulator over NVLink (the ghost all-reduce fused into the scatter)
__device__ __forceinline__ void window_flush_node(const Window& W, float4* __restrict__ grid, const float4& v) {
  red_add_v4(grid + W.node, v);
  if (W.peer_r != nullptr && W.plane >= W.gr_lo && W.plane < W.gr_hi) red_add_v4(W.peer_r + W.node, v);
  if (W.peer_l != nullptr && W.plane >= W.gl_lo && W.plane < W.gl_hi) red_add_v4(W.peer_l + W.node, v);
}
// flag the 8^3-node block of this lane's node.  Plain store, no test-before-write: a test waits for the flag load, while the store is
// fire-and-forget (same-address lanes coalesce; ~1e5 32-byte L2 writes per launch against 1.7e6 vector reductions).
__device__ __forceinline__ void window_flag(const Window& W, const int i, const int j, const int k) {
  const int blk = ((i >> 3) * W.nb + (j >> 3)) * W.nb + (k >> 3);
  W.flags[blk] = 1;
  // x-slab mode: the neighbour must visit (and later clear) the blocks this rank reduces into over NVLink
  if (W.peer_fr != nullptr && i >= W.gr_lo && i < W.gr_hi) W.peer_fr[blk] = 1;
  if (W.peer_fl != nullptr && i >= W.gl_lo && i < W.gl_hi) W.peer_fl[blk] = 1;
}
__device__ __forceinline__ void window_flush_all(Window& W, float4* __restrict__ grid) {
  if (W.cur_key >= 0 && W.lane_valid) window_flush_node(W, grid, make_float4(W.acc01.x, W.acc01.y, W.acc2m.x, W.acc2m.y));
  W.acc01 = make_float2(0.f, 0.f); W.acc2m = make_float2(0.f, 0.f);
  W.cur_key = -1;
}
// move the window to cell `key` (warp-uniform).  Blocks are flagged when the window is PLACED on a cell (every node of the
// footprint receives a contribution from the cell's particles), so a z+1 shift only has to look at the new c=2 plane.
__device__ __forceinline__ void window_move(Window& W, const int key, float4* __restrict__ grid) {
  if (W.cur_key >= 0) {
    const float4 v = make_float4(W.acc01.x, W.acc01.y, W.acc2m.x, W.acc2m.y);
    if (key == W.cur_key + 1) {  // next cell of the same z-column: plane c=0 is complete, shift the other two
      if (W.lane_valid && W.c == 0) window_flush_node(W, grid, v);
      float4 t;
      t.x = __shfl_down_sync(SC_FULL, v.x, 1); t.y = __shfl_down_sync(SC_FULL, v.y, 1);
      t.z = __shfl_down_sync(SC_FULL, v.z, 1); t.w = __shfl_down_sync(SC_FULL, v.w, 1);
      const bool z = (W.c == 2) || !W.lane_valid;
      W.acc01 = z ? make_float2(0.f, 0.f) : make_float2(t.x, t.y);
      W.acc2m = z ? make_float2(0.f, 0.f) : make_float2(t.z, t.w);
      W.node += 1; W.cur_key = key;
      if (W.flags && W.c == 2 && W.lane_valid) {
        const int k = (key & 1023) + 2;
        if ((k & 7) == 0) window_flag(W, (key >> 20) + W.a, ((key >> 10) & 1023) + W.b, k);
      }
      return;
    }
    if (W.lane_valid) window_flush_node(W, grid, v);
    W.acc01 = make_float2(0.f, 0.f); W.acc2m = make_float2(0.f, 0.f);
  }
  const int i = (key >> 20) + W.a, j = ((key >> 10) & 1023) + W.b, k = (key & 1023) + W.c;
  W.node = (i * W.n + j) * W.n + k; W.plane = i;
  W.cur_key = key;
  if (W.flags && W.lane_valid) window_flag(W, i, j, k);
}

// lane = particle.  key < 0: the particle contributes nothing (unused / out of grid / beyond N).
// The 32 records are staged in ascending key order (stable rank inside the warp), so the node-mode pass sees every cell of the warp as
// ONE run, and the cells of a z-column one after the other (the window then only shifts by one plane), even when the global cell sort is
// a few substeps old: in falling water half of a warp's particles have crossed into the next column down before the next sort, and an
// order of first appearance would alternate between the two columns — a 27-node flush per run.  MATCH.ANY groups equal
// keys; one short warp-uniform loop over the group leaders counts, per lane, the particles in smaller cells.
// Returns the mask of staged positions at which a new cell run starts.
// ALL 32 lanes must call.
__device__ __forceinline__ unsigned scatter_rank(const int lane, const int key, const int carry_key, int& rank) {
  const bool valid = key >= 0;
  const int skey = valid ? key : 0x7fffffff;   // particles without a cell go last (callers consume the first `cnt` staged positions only)
  const unsigned lt = (1u << lane) - 1u;
  const unsigned same = __match_any_sync(SC_FULL, skey);   // MATCH.ANY: the lanes that share my cell
  const bool leader = (same & lt) == 0u;
  const int gsz = __popc(same);
  unsigned leaders = __ballot_sync(SC_FULL, leader);
  int less = 0;
  while (leaders != 0u) {   // warp-uniform: one pass per distinct cell of the warp (4 ... 10)
    const int L = __ffs(leaders) - 1;
    leaders &= leaders - 1u;
    const int k = __shfl_sync(SC_FULL, skey, L), n = __shfl_sync(SC_FULL, gsz, L);
    less += k < skey ? n : 0;
  }
  rank = less + __popc(same & lt);
  // every valid cell starts a run, except when the smallest one continues the cell the window is already on
  return __reduce_or_sync(SC_FULL, (leader && valid && !(less == 0 && skey == carry_key)) ? (1u << less) : 0u);
}
__device__ __forceinline__ unsigned scatter_publish(ScatterSmem& S, const int lane, const int key, const int carry_key, const float* q,
                                                    const float* B, const float m, const float w[3][3]) {
  int rank;
  const unsigned starts = scatter_rank(lane, key, carry_key, rank);
  const bool valid = key >= 0;
  // Q_ab = q + a*B[:,0] + b*B[:,1] in packed (x,y) / (z,m) pairs
  const float2 c0a = make_float2(B[0], B[3]), c0b = make_float2(B[6], 0.f);
  const float2 c1a = make_float2(B[1], B[4]), c1b = make_float2(B[7], 0.f);
  // (stored as 64-bit halves: an FFMA pair result is a register PAIR, a 128-bit store would first need four MOVs into an aligned quad)
  float2* rec = reinterpret_cast<float2*>(S.rec + rank * SC_REC);
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const float2 fa = make_float2((float)a, (float)a);
    const float2 qa01 = ffma2(fa, c0a, make_float2(q[0], q[1])), qa2m = ffma2(fa, c0b, make_float2(q[2], m));
#pragma unroll
    for (int b = 0; b < 3; b++) {
      const float2 fb = make_float2((float)b, (float)b);
      rec[2 * (a * 3 + b)] = ffma2(fb, c1a, qa01);
      rec[2 * (a * 3 + b) + 1] = ffma2(fb, c1b, qa2m);
    }
  }
  S.b2[rank] = make_float4(B[2], B[5], B[8], 0.f);
  float wn[28];
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++) {
      const float wab = valid ? w[a][0] * w[b][1] : 0.f;
#pragma unroll
      for (int c = 0; c < 3; c++) wn[a * 9 + b * 3 + c] = wab * w[c][2];   // w is all-zero for particles without a cell
    }
  wn[27] = 0.f;
#pragma unroll
  for (int k = 0; k < SC_WQ; k++) S.w[rank * SC_WQ + k] = make_float4(wn[4 * k], wn[4 * k + 1], wn[4 * k + 2], wn[4 * k + 3]);
  S.key[rank] = key;
  return starts;
}

// lane = stencil node.  Consumes the 32 staged particles (positions >= cnt carry zero weights, see scatter_publish) in fixed
// groups of four: 12 LDS of a group are issued first, then 8 independent FFMA pairs (Q_ab + c*B2), and only the two accumulator
// FFMA pairs per particle form a dependent chain; run starts are a rare, warp-uniform branch.
__device__ __forceinline__ void window_consume(Window& W, const ScatterSmem& S, const int cnt, const unsigned starts, float4* __restrict__ grid) {
  const float2 oc2 = make_float2(W.oc, W.oc);
  const int ngroups = (cnt + 3) >> 2;
  const float* wf = reinterpret_cast<const float*>(S.w) + W.wrow;
#pragma unroll 1
  for (int g = 0; g < ngroups; g++) {
    float2 t01[4], t2m[4], w2[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int p = g * 4 + u;
      const float4 Q = S.rec[p * SC_REC + W.qidx], B2 = S.b2[p];
      const float w = wf[p * (4 * SC_WQ)];
      w2[u] = make_float2(w, w);
      t01[u] = ffma2(make_float2(B2.x, B2.y), oc2, make_float2(Q.x, Q.y));
      t2m[u] = ffma2(make_float2(B2.z, B2.w), oc2, make_float2(Q.z, Q.w));
    }
    const unsigned sb = (starts >> (g * 4)) & 15u;
    if (sb == 0u) {
#pragma unroll
      for (int u = 0; u < 4; u++) { W.acc01 = ffma2(w2[u], t01[u], W.acc01); W.acc2m = ffma2(w2[u], t2m[u], W.acc2m); }
    } else {
#pragma unroll
      for (int u = 0; u < 4; u++) {
        if ((sb >> u) & 1u) window_move(W, S.key[g * 4 + u], grid);
        W.acc01 = ffma2(w2[u], t01[u], W.acc01); W.acc2m = ffma2(w2[u], t2m[u], W.acc2m);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Lean variants (a profile of the fused kernel charged more of its warp instructions to the window moves of the four-way unrolled
// group loop above than to the node loop itself): (1) the window no longer flags sparse-grid blocks, the kernel
// flags the blocks of the warp's stencil box once (flag_box); (2) the x-slab peer reductions are compiled in only where asked (kSlab);
// (3) the staged particles are consumed RUN BY RUN: one copy of the move code, then the run's particles four at a time plus a remainder.
// ---------------------------------------------------------------------------------------------------------------
template <bool kSlab>
__device__ __forceinline__ void window_flush_node2(const Window& W, const bool pred, float4* __restrict__ grid, const float4& v) {
  red_add_v4_if(pred, grid + W.node, v);
  if (kSlab) {
    red_add_v4_if(pred && W.peer_r != nullptr && W.plane >= W.gr_lo && W.plane < W.gr_hi, W.peer_r + W.node, v);
    red_add_v4_if(pred && W.peer_l != nullptr && W.plane >= W.gl_lo && W.plane < W.gl_hi, W.peer_l + W.node, v);
  }
}
template <bool kSlab>
__device__ __forceinline__ void window_move2(Window& W, const int key, float4* __restrict__ grid) {
  const float4 v = make_float4(W.acc01.x, W.acc01.y, W.acc2m.x, W.acc2m.y);
  const bool open = W.cur_key >= 0;
  if (open && key == W.cur_key + 1) {  // next cell of the same z-column: plane c=0 is complete, shift the other two
    window_flush_node2<kSlab>(W, W.lane_valid && W.c == 0, grid, v);
    float4 t;
    t.x = __shfl_down_sync(SC_FULL, v.x, 1); t.y = __shfl_down_sync(SC_FULL, v.y, 1);
    t.z = __shfl_down_sync(SC_FULL, v.z, 1); t.w = __shfl_down_sync(SC_FULL, v.w, 1);
    const bool z = (W.c == 2) || !W.lane_valid;
    W.acc01 = z ? make_float2(0.f, 0.f) : make_float2(t.x, t.y);
    W.acc2m = z ? make_float2(0.f, 0.f) : make_float2(t.z, t.w);
    W.node += 1; W.cur_key = key;
    return;
  }
  window_flush_node2<kSlab>(W, open && W.lane_valid, grid, v);
  W.acc01 = make_float2(0.f, 0.f); W.acc2m = make_float2(0.f, 0.f);
  const int i = (key >> 20) + W.a, j = ((key >> 10) & 1023) + W.b, k = (key & 1023) + W.c;
  W.node = (i * W.n + j) * W.n + k; W.plane = i;
  W.cur_key = key;
}
template <bool kSlab>
__device__ __forceinline__ void window_flush_all2(Window& W, float4* __restrict__ grid) {
  window_flush_node2<kSlab>(W, W.cur_key >= 0 && W.lane_valid, grid, make_float4(W.acc01.x, W.acc01.y, W.acc2m.x, W.acc2m.y));
  W.acc01 = make_float2(0.f, 0.f); W.acc2m = make_float2(0.f, 0.f);
  W.cur_key = -1;
}
// one staged particle into this lane's node: acc += w * (Q_ab + c * B2), the two FFMA pairs in this order on every path
__device__ __forceinline__ void window_acc(Window& W, const float4& Q, const float4& B2, const float w, const float2 oc2) {
  const float2 w2 = make_float2(w, w);
  W.acc01 = ffma2(w2, ffma2(make_float2(B2.x, B2.y), oc2, make_float2(Q.x, Q.y)), W.acc01);
  W.acc2m = ffma2(w2, ffma2(make_float2(B2.z, B2.w), oc2, make_float2(Q.z, Q.w)), W.acc2m);
}
// The staged particles are consumed in fixed groups of four (positions 4g .. 4g+3; positions >= cnt carry zero weights).
//  * a group in which no run starts takes the fast path, software-pipelined by half groups with two register sets of two particles: the
//    6 LDS of one half are in flight while the other half is accumulated, so the shared-memory latency overlaps the FFMA chains of the same
//    warp.  Each set always holds the same half, so no loaded value is copied from a "next" register into a "current" one, and the two sets
//    take the 36 registers one prefetched group of four did (two full groups in flight make k_fwd spill at its 80-register bound);
//  * a group in which a run starts goes one particle at a time straight from shared memory, through the ONE copy of the window move code
//    (a copy per unrolled pass, each with four inlined moves, doubled the loop's static code).
// Both paths accumulate every particle in staged order with the same FFMAs, so a warp's window values do not depend on the path taken.
template <bool kSlab>
__device__ __forceinline__ void window_consume2(Window& W, const ScatterSmem& S, const int cnt, const unsigned starts, float4* __restrict__ grid) {
  if (starts == 0u && W.cur_key < 0) return;   // nothing staged and nothing open (a warp of unused slots)
  const float2 oc2 = make_float2(W.oc, W.oc);
  // running pointers to the current group: every LDS of the loop is [pointer + immediate]
  const float* wf = reinterpret_cast<const float*>(S.w) + W.wrow;
  const float4* rq = S.rec + W.qidx;
  const float4* rb = S.b2;
  const int* kp = S.key;
  unsigned st = starts;   // run starts of the current group in the low four bits (warp-uniform: starts comes out of a warp reduction)
  int left = (cnt + 3) >> 2;   // groups left, the current one included
  auto next_group = [&]() { rq += 4 * SC_REC; rb += 4; wf += 16 * SC_WQ; kp += 4; st >>= 4; left--; };
  // set A holds the first half of a group, set B the second half
  float4 QA[2], BA[2], QB[2], BB[2]; float wA[2], wB[2];
  auto load = [&](const int p0, float4* Q, float4* B2, float* w) {   // positions p0, p0 + 1 after the current group's first
#pragma unroll
    for (int u = 0; u < 2; u++) { const int p = p0 + u; Q[u] = rq[p * SC_REC]; B2[u] = rb[p]; w[u] = wf[p * (4 * SC_WQ)]; }
  };
  auto accumulate = [&](const float4* Q, const float4* B2, const float* w) {
#pragma unroll
    for (int u = 0; u < 2; u++) window_acc(W, Q[u], B2[u], w[u], oc2);
  };
#pragma unroll 1
  while (left > 0) {   // warp-uniform
    if ((st & 15u) != 0u) {
#pragma unroll 1
      for (int u = 0; u < 4; u++) {
        if ((st >> u) & 1u) window_move2<kSlab>(W, kp[u], grid);
        window_acc(W, rq[u * SC_REC], rb[u], wf[u * (4 * SC_WQ)], oc2);
      }
      next_group();
      continue;
    }
    // a stretch of groups without run starts
    load(0, QA, BA, wA);
#pragma unroll 1
    for (;;) {
      load(2, QB, BB, wB);
      accumulate(QA, BA, wA);
      const bool more = left > 1 && (st & 0xf0u) == 0u;
      // unconditional, so that set A's registers stay fixed (a predicated reload costs a MOV per register); without a next group it reloads
      // this group's first half, which stays inside the staging area
      load(more ? 4 : 0, QA, BA, wA);
      accumulate(QB, BB, wB);
      next_group();
      if (!more) break;
    }
  }
}
// flag the 8^3-node blocks that the stencils of the warp's particles (bases b, valid where ok) can touch: the blocks of the box
// [min b, max b + 2] per axis (a superset is harmless: flagged blocks are only visited).  ALL 32 lanes must call.
template <bool kSlab>
__device__ __forceinline__ void flag_one(const Window& W, int* __restrict__ flags, const int X, const int Y, const int Z) {
  const int blk = (X * W.nb + Y) * W.nb + Z;
  flags[blk] = 1;
  if (kSlab) {   // the neighbour must visit (and later clear) the blocks this rank reduces into over NVLink
    if (W.peer_fr != nullptr && X * 8 + 7 >= W.gr_lo && X * 8 < W.gr_hi) W.peer_fr[blk] = 1;
    if (W.peer_fl != nullptr && X * 8 + 7 >= W.gl_lo && X * 8 < W.gl_hi) W.peer_fl[blk] = 1;
  }
}
template <bool kSlab>
__device__ __forceinline__ void flag_box(const Window& W, int* __restrict__ flags, const int lane, const bool ok, const int* b) {
  const int x1 = __reduce_max_sync(SC_FULL, ok ? b[0] : -1);
  if (x1 < 0) return;   // warp-uniform
  const int x0 = __reduce_min_sync(SC_FULL, ok ? b[0] : 0x7fffffff);
  const int y0 = __reduce_min_sync(SC_FULL, ok ? b[1] : 0x7fffffff), y1 = __reduce_max_sync(SC_FULL, ok ? b[1] : -1);
  const int z0 = __reduce_min_sync(SC_FULL, ok ? b[2] : 0x7fffffff), z1 = __reduce_max_sync(SC_FULL, ok ? b[2] : -1);
  const int X0 = x0 >> 3, Y0 = y0 >> 3, Z0 = z0 >> 3, ex = ((x1 + 2) >> 3) - X0, ey = ((y1 + 2) >> 3) - Y0, ez = ((z1 + 2) >> 3) - Z0;
  if ((ex | ey | ez) <= 1) {   // the usual case (a cell-sorted warp spans a few cells): at most 2 x 2 x 2 blocks, one predicated store per lane
    const int dx = lane & 1, dy = (lane >> 1) & 1, dz = (lane >> 2) & 1;
    if (lane < 8 && dx <= ex && dy <= ey && dz <= ez) flag_one<kSlab>(W, flags, X0 + dx, Y0 + dy, Z0 + dz);
    return;
  }
  for (int X = X0; X <= X0 + ex; X++)
    for (int Y = Y0; Y <= Y0 + ey; Y++)
      for (int t = lane; t <= ez; t += 32) flag_one<kSlab>(W, flags, X, Y, Z0 + t);
}

// ---------------------------------------------------------------------------------------------------------------
// Per-warp staging of a grid footprint for lane = particle gathers (g2p, per-particle adjoint): the 32 cell-sorted
// particles of a warp normally sit in one z-column of cells, so their stencils cover 9 node columns x (kmax-kmin+3)
// nodes.  The warp loads those with 9 coalesced 128-bit loads per lane into shared memory and every particle then
// gathers its 27 nodes with LDS.128.  Warps whose particles straddle columns (or are unsorted) gather straight from L2.
// ---------------------------------------------------------------------------------------------------------------
#define G2P_ZMAX 32
struct Footprint { bool staged; int bx0, by0, kmin, len; };
__device__ __forceinline__ Footprint footprint_of(const bool ok, const int* b) {  // ALL 32 lanes must call
  Footprint fp; fp.staged = false; fp.bx0 = fp.by0 = fp.kmin = 0; fp.len = 0;
  const unsigned valid = __ballot_sync(SC_FULL, ok);
  if (valid == 0u) return fp;
  const int ref = __ffs(valid) - 1;
  fp.bx0 = __shfl_sync(SC_FULL, b[0], ref); fp.by0 = __shfl_sync(SC_FULL, b[1], ref);
  const bool same = __ballot_sync(SC_FULL, ok && (b[0] != fp.bx0 || b[1] != fp.by0)) == 0u;
  fp.kmin = __reduce_min_sync(SC_FULL, ok ? b[2] : 0x7fffffff);
  const int kmax = __reduce_max_sync(SC_FULL, ok ? b[2] : -1);
  fp.len = kmax - fp.kmin + 3;
  fp.staged = same && fp.len <= G2P_ZMAX;
  return fp;
}
__device__ __forceinline__ void footprint_load(const float4* __restrict__ grid, const int n, const Footprint& fp, float4* tile) {
  const int lane = threadIdx.x & 31;
  if (lane < fp.len) {
#pragma unroll
    for (int c = 0; c < 9; c++) tile[c * G2P_ZMAX + lane] = grid[((fp.bx0 + c / 3) * n + (fp.by0 + c % 3)) * n + fp.kmin + lane];
  }
  __syncwarp();
}

// Separable evaluation of  v' = sum w g,  C' = 4 inv_dx sum w g (o - fx)^T  (MPM:409-416): reduce the three nodes of a
// z-column first (G0 = sum_k wz g, G1 = sum_k wz (k - fz) g), then fold the 9 columns in.  FFMA pairs throughout.
// `col3(c)` returns (by value) the three consecutive v_out nodes of stencil column c = i*3+j for this particle.
struct Col3 { float4 g0, g1, g2; };
template <class ColFn>
__device__ __forceinline__ void g2p_gather_v(const float* fx, const float w[3][3], ColFn col3, float* nv, Mat3& nC, const float c4) {
  const float2 wz0 = make_float2(w[0][2], w[0][2]), wz1 = make_float2(w[1][2], w[1][2]), wz2 = make_float2(w[2][2], w[2][2]);
  const float wd0 = w[0][2] * (0.f - fx[2]), wd1 = w[1][2] * (1.f - fx[2]), wd2 = w[2][2] * (2.f - fx[2]);
  const float2 wzd0 = make_float2(wd0, wd0), wzd1 = make_float2(wd1, wd1), wzd2 = make_float2(wd2, wd2);
  const float2 wzz0 = make_float2(w[0][2], wd0), wzz1 = make_float2(w[1][2], wd1), wzz2 = make_float2(w[2][2], wd2);
  float2 v01 = make_float2(0.f, 0.f), v2c22 = make_float2(0.f, 0.f), c02_12 = make_float2(0.f, 0.f);
  float2 c00_10 = make_float2(0.f, 0.f), c01_11 = make_float2(0.f, 0.f), c20_21 = make_float2(0.f, 0.f);
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) {
      const Col3 c = col3(i * 3 + j);
      const float4 g0 = c.g0, g1 = c.g1, g2 = c.g2;
      float2 G0xy = fmul2(make_float2(g0.x, g0.y), wz0); G0xy = ffma2(make_float2(g1.x, g1.y), wz1, G0xy); G0xy = ffma2(make_float2(g2.x, g2.y), wz2, G0xy);
      float2 G1xy = fmul2(make_float2(g0.x, g0.y), wzd0); G1xy = ffma2(make_float2(g1.x, g1.y), wzd1, G1xy); G1xy = ffma2(make_float2(g2.x, g2.y), wzd2, G1xy);
      float2 Gz = fmul2(make_float2(g0.z, g0.z), wzz0); Gz = ffma2(make_float2(g1.z, g1.z), wzz1, Gz); Gz = ffma2(make_float2(g2.z, g2.z), wzz2, Gz);  // (G0_z, G1_z)
      const float wxy = w[i][0] * w[j][1];
      const float bx = wxy * ((float)i - fx[0]), by = wxy * ((float)j - fx[1]);
      const float2 a2 = make_float2(wxy, wxy);
      v01 = ffma2(a2, G0xy, v01);
      v2c22 = ffma2(a2, Gz, v2c22);
      c02_12 = ffma2(a2, G1xy, c02_12);
      c00_10 = ffma2(make_float2(bx, bx), G0xy, c00_10);
      c01_11 = ffma2(make_float2(by, by), G0xy, c01_11);
      c20_21 = ffma2(make_float2(bx, by), make_float2(Gz.x, Gz.x), c20_21);
    }
  nv[0] = v01.x; nv[1] = v01.y; nv[2] = v2c22.x;
  nC.m[0] = c4 * c00_10.x; nC.m[1] = c4 * c01_11.x; nC.m[2] = c4 * c02_12.x;
  nC.m[3] = c4 * c00_10.y; nC.m[4] = c4 * c01_11.y; nC.m[5] = c4 * c02_12.y;
  nC.m[6] = c4 * c20_21.x; nC.m[7] = c4 * c20_21.y; nC.m[8] = c4 * v2c22.y;
}
// `col(c)` returns a pointer to the three consecutive v_out nodes of stencil column c
template <class ColFn>
__device__ __forceinline__ void g2p_gather(const float* fx, const float w[3][3], ColFn col, float* nv, Mat3& nC, const float c4) {
  g2p_gather_v(fx, w, [&](int c) { const float4* p = col(c); Col3 r; r.g0 = p[0]; r.g1 = p[1]; r.g2 = p[2]; return r; }, nv, nC, c4);
}

