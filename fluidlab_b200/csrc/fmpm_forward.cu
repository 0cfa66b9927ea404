// fmpm_forward.cu — forward MLS-MPM substep kernels for sm_90a (H100).
//
// Reference semantics: fluidlab/fluidengine/simulators/mpm_simulator.py (MPM) substep(), MPM:515-533.
// Reference structure (17 Taichi launches per substep, per-particle float atomics, F_tmp/U/S/V round
// trips through global memory) is NOT followed.  Design:
//
//  * particles live in cell-sorted SLOT order in float4 planes -> every particle load/store is a fully
//    coalesced 128-bit access;
//  * p2g fuses F_tmp + SVD + stress + scatter + F-update (MPM:254-264, 331-378).  The scatter does not
//    issue one atomic per (particle,node,component): shared-memory float atomics are CAS loops on
//    sm_90a (ATOMS.CAST.SPIN), so instead each warp walks its sorted particles with lane = stencil
//    node (27 of 32 lanes), accumulating the node sums of the current cell in REGISTERS.  When the walk
//    moves to the next cell of the z-column the window shifts by one plane through warp shuffles and only
//    the finished 3x3 plane is flushed with one vector reduction (REDG.E.ADD.F32x4: momentum xyz + mass
//    in a single 16-byte L2 atomic).  ~1.5 vector REDs per particle instead of 108 scalar atomics.
//  * grid_op (MPM:380-398) also clears the momentum/mass accumulators for the next substep;
//  * g2p fuses advect_used / process_unused_particles / g2p / advect_kernel (MPM:304-316, 400-426, 497-505).
#include <cstdio>
#include <cstring>
#include "fmpm_common.cuh"

#include "fmpm_scatter.cuh"
#include "fmpm_sdf.cuh"

#ifndef P2G_WARPS
#define P2G_WARPS 4
#endif
#ifndef P2G_ROUNDS
#define P2G_ROUNDS 1   // 32-particle rounds per warp: one round needs no loop-carried window state and no prefetch registers
#endif
#ifndef P2G_MINB
#define P2G_MINB 5   // <=102 registers: 20 warps/SM
#endif

#ifndef P2G_PREFETCH
#define P2G_PREFETCH 1   // (only matters for P2G_ROUNDS > 1) next round's particle data: 0 = not prefetched, 1 = into registers, 2 = prefetch.global.L2 only
#endif

// =============================================================================================
// p2g
// =============================================================================================
struct PRaw { float4 a0, a1, a2, a3, f0, f1; float f8; };
#ifndef FMPM_STREAM_HINTS
#define FMPM_STREAM_HINTS 2   // >= 1: particle planes of frame f are read with ld.global.cs (evict-first); >= 2: F[f+1] is written with st.global.cs
#endif
#if FMPM_STREAM_HINTS
#define P2G_LD(p) __ldcs(p)
#else
#define P2G_LD(p) (*(p))
#endif
// F[f+1] is next read one whole substep (>200 MB of traffic) later: with FMPM_STREAM_HINTS >= 2 it is written evict-first
__device__ __forceinline__ void p2g_store_F(const KParams& P, const int f, const int s, const Mat3& F) {
#if FMPM_STREAM_HINTS >= 2
  __stcs(&P.pf[pf_idx(P, f, 0, s)], make_float4(F.m[0], F.m[1], F.m[2], F.m[3]));
  __stcs(&P.pf[pf_idx(P, f, 1, s)], make_float4(F.m[4], F.m[5], F.m[6], F.m[7]));
  __stcs(&P.pf8[pf8_idx(P, f, s)], F.m[8]);
#else
  store_F(P.pf, P.pf8, P, f, s, F);
#endif
}
__device__ __forceinline__ void p2g_load_raw(const KParams& P, const int f, const long long sl, PRaw& R) {
  if (sl < P.N) {
    const int s = (int)sl;
    R.a0 = P2G_LD(&P.pa[pa_idx(P, f, 0, s)]); R.a1 = P2G_LD(&P.pa[pa_idx(P, f, 1, s)]); R.a2 = P2G_LD(&P.pa[pa_idx(P, f, 2, s)]); R.a3 = P2G_LD(&P.pa[pa_idx(P, f, 3, s)]);
    R.f0 = P2G_LD(&P.pf[pf_idx(P, f, 0, s)]); R.f1 = P2G_LD(&P.pf[pf_idx(P, f, 1, s)]); R.f8 = P2G_LD(&P.pf8[pf8_idx(P, f, s)]);
  } else {
    R.a0 = make_float4(0.f, 0.f, 0.f, 0.f);  // meta = 0 -> unused
  }
}
__device__ __forceinline__ void p2g_prefetch_l2(const KParams& P, const int f, const long long sl) {
#ifndef FMPM_HOST_EMU
  if (sl < P.N) {
    const int s = (int)sl;
    asm volatile("prefetch.global.L2 [%0];" ::"l"(P.pa + pa_idx(P, f, 0, s)));
    asm volatile("prefetch.global.L2 [%0];" ::"l"(P.pa + pa_idx(P, f, 1, s)));
    asm volatile("prefetch.global.L2 [%0];" ::"l"(P.pa + pa_idx(P, f, 2, s)));
    asm volatile("prefetch.global.L2 [%0];" ::"l"(P.pa + pa_idx(P, f, 3, s)));
    asm volatile("prefetch.global.L2 [%0];" ::"l"(P.pf + pf_idx(P, f, 0, s)));
    asm volatile("prefetch.global.L2 [%0];" ::"l"(P.pf + pf_idx(P, f, 1, s)));
    asm volatile("prefetch.global.L2 [%0];" ::"l"(P.pf8 + pf8_idx(P, f, s)));
  }
#endif
}
__device__ __forceinline__ void p2g_unpack(const PRaw& R, PState& st) {
  st.x[0] = R.a0.x; st.x[1] = R.a0.y; st.x[2] = R.a0.z; st.meta = __float_as_int(R.a0.w);
  st.v[0] = R.a1.x; st.v[1] = R.a1.y; st.v[2] = R.a1.z;
  st.C.m[0] = R.a1.w; st.C.m[1] = R.a2.x; st.C.m[2] = R.a2.y; st.C.m[3] = R.a2.z; st.C.m[4] = R.a2.w;
  st.C.m[5] = R.a3.x; st.C.m[6] = R.a3.y; st.C.m[7] = R.a3.z; st.C.m[8] = R.a3.w;
  st.F.m[0] = R.f0.x; st.F.m[1] = R.f0.y; st.F.m[2] = R.f0.z; st.F.m[3] = R.f0.w;
  st.F.m[4] = R.f1.x; st.F.m[5] = R.f1.y; st.F.m[6] = R.f1.z; st.F.m[7] = R.f1.w; st.F.m[8] = R.f8;
}

template <bool kWriteF, bool kSlab>
__global__ void __launch_bounds__(P2G_WARPS * 32, P2G_MINB) k_p2g(const KParams P, const int f) {
  __shared__ ScatterSmem smem[P2G_WARPS];
  const int lane = threadIdx.x & 31, wib = __shfl_sync(SC_FULL, (int)(threadIdx.x >> 5), 0);   // broadcast: dependent code is compiled warp-uniform
  ScatterSmem& S = smem[wib];
  fmpm_pdl_trigger();
  const long long gw = (long long)blockIdx.x * P2G_WARPS + wib;
  const long long slot0 = gw * (32 * P2G_ROUNDS);
  if (slot0 >= P.N) return;
  Window W; window_init(W, lane, P.n, nullptr);   // blocks are flagged once per round (flag_box), not by the window
  fmpm_pdl_wait();
  if (P.epoch != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *P.epoch += 16;   // opens a fused step with lazy grid_op: fresh tags for its k_fwd launches
  if (kSlab) window_set_slab(W, P.peer_l, P.peer_r, P.gl_lo, P.gl_hi, P.gr_lo, P.gr_hi, P.peer_fl, P.peer_fr);
  PRaw R; p2g_load_raw(P, f, slot0 + lane, R);
#pragma unroll 1
  for (int r = 0; r < P2G_ROUNDS; r++) {
    const long long sl = slot0 + r * 32 + lane;
    const long long rem = (long long)P.N - (slot0 + r * 32);
    if (rem <= 0) break;  // warp-uniform
#if P2G_PREFETCH != 1
    if (r > 0) p2g_load_raw(P, f, sl, R);
#endif
    const int cnt = rem < 32 ? (int)rem : 32;
    int key = -1;
    float q[3] = {0.f, 0.f, 0.f}, B[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, m = 0.f;
    float w[3][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    int b[3] = {0, 0, 0}; bool ok = false;
    if (sl < P.N) {
      const int s = (int)sl;
      PState st; p2g_unpack(R, st);
      float fx[3];
      const bool used = st.meta & 1;
      ok = used && base_fx(P, st.x, b, fx);
      if (ok) {
        const float4 mt = __ldg(P.mats + ((st.meta >> 8) & 0xff));
        Constit K; constitutive(P, st, mt.x, mt.y, mt.z, __float_as_int(mt.w), K);
        m = mt.z;
        bspline(fx, w);
        // contribution_i = w_i * (m v + A (o - fx) dx) = w_i * (q + B o),  B = A dx,  q = m v - B fx
#pragma unroll
        for (int i = 0; i < 9; i++) B[i] = K.A.m[i] * P.dx;
#pragma unroll
        for (int i = 0; i < 3; i++) q[i] = m * st.v[i] - (B[i * 3] * fx[0] + B[i * 3 + 1] * fx[1] + B[i * 3 + 2] * fx[2]);
        key = pack_key(b);
        if (kWriteF) p2g_store_F(P, f + 1, s, K.Fn);
      } else if (kWriteF) {
        p2g_store_F(P, f + 1, s, st.F);  // process_unused_particles (MPM:316) / frozen out-of-grid particle
      }
    }
    flag_box<kSlab>(W, P.blk_flags, lane, ok, b);
    const unsigned starts = scatter_publish(S, lane, key, W.cur_key, q, B, m, w);
    // software pipelining: the next round's 100 B/particle are in flight while this round is scattered
#if P2G_PREFETCH == 1
    if (r + 1 < P2G_ROUNDS) p2g_load_raw(P, f, sl + 32, R);
#elif P2G_PREFETCH == 2
    if (r + 1 < P2G_ROUNDS) p2g_prefetch_l2(P, f, sl + 32);
#endif
    __syncwarp();
    window_consume2<kSlab>(W, S, cnt, starts, P.grid_pm);
    __syncwarp();
  }
  window_flush_all2<kSlab>(W, P.grid_pm);
}

// =============================================================================================
// sparse grid: p2g flags the 8^3-node blocks it scatters into (blk_flags); every grid kernel of the substep scans the flag
// array with a grid-stride loop and visits only flagged blocks (no separate compaction launch).
// =============================================================================================
// MPM:380-398 on the active blocks; optionally clears the (momentum, mass) accumulators for the next substep
// and zeroes the v_out adjoint of the same blocks (backward pass).
// v_out of one node from its (momentum, mass) sum: MPM:380-398 with SDF colliders and the agent's grid-level collision
__device__ __forceinline__ float4 grid_op_node_full(const KParams& P, const int f, const int i, const int j, const int k, const float4 pm) {
  float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
  if (pm.w > FMPM_EPS) {
    const float inv_m = 1.f / pm.w;
    float v[3] = {inv_m * pm.x + P.dt * P.gx, inv_m * pm.y + P.dt * P.gy, inv_m * pm.z + P.dt * P.gz};
    const float pos[3] = {(float)i * P.dx, (float)j * P.dx, (float)k * P.dx};
    for (int si = 0; si < P.col.n_statics; si++) {  // statics[i].collide, MPM:388-390
      float o[3]; sdf_collide<false>(P.col.statics[si], false, nullptr, nullptr, nullptr, nullptr, P.dt, pos, v, o, nullptr, nullptr, nullptr, nullptr, nullptr);
      v[0] = o[0]; v[1] = o[1]; v[2] = o[2];
    }
    if (P.col.has_rigid && P.col.collide_type >= 1) {  // agent.collide at grid level, MPM:393-395
      float o[3]; agent_collide<false>(P, f, pos, v, o, nullptr, nullptr, nullptr, nullptr, nullptr);
      v[0] = o[0]; v[1] = o[1]; v[2] = o[2];
    }
    float fac[3];
    boundary_v(P, pos, v, fac);
    out = make_float4(v[0], v[1], v[2], 0.f);
  }
  return out;
}
#ifndef GOP_PER_SM
#define GOP_PER_SM 8   // CTAs of k_grid_op per SM (one resident wave of 256-thread CTAs)
#endif
__global__ void __launch_bounds__(256) k_grid_op(const KParams P, const int f, const int clear_pm, const int zero_ggv, const int reset_flags) {
  const int n = P.n, nb = P.nb, nblk = nb * nb * nb;
  // this CTA owns blocks blockIdx.x + q*gridDim.x; their flags are fetched in parallel (thread q reads flag q) and the CTA
  // then walks the flagged ones (nblk / gridDim.x <= 256 for every supported grid)
  // (A one-CTA-per-block variant without shared memory or barriers was slower: 4096 tiny CTAs cost more to schedule than the flag compaction below.)
  __shared__ int s_act[256];
  __shared__ int s_n;
  if (threadIdx.x == 0) s_n = 0;
  fmpm_pdl_trigger();
  fmpm_pdl_wait();
  __syncthreads();
  {
    const int blk = blockIdx.x + threadIdx.x * gridDim.x;
    if (blk < nblk && P.blk_flags[blk] != 0) s_act[atomicAdd(&s_n, 1)] = blk;
  }
  __syncthreads();
  const int n_act = s_n;
  for (int ai = 0; ai < n_act; ai++) {
    const int blk = s_act[ai];
    const int bx = blk / (nb * nb), by = (blk / nb) % nb, bz = blk % nb;
#pragma unroll
    for (int r = 0; r < 2; r++) {
      const int t = threadIdx.x + r * 256;
      const int i = bx * 8 + (t >> 6), j = by * 8 + ((t >> 3) & 7), k = bz * 8 + (t & 7);
      const int g = (i * n + j) * n + k;
      const float4 pm = P.grid_pm[g];
      P.grid_v[g] = grid_op_node_full(P, f, i, j, k, pm);
      if (clear_pm && (pm.w != 0.f || pm.x != 0.f || pm.y != 0.f || pm.z != 0.f)) P.grid_pm[g] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (zero_ggv) P.ggrid_v[g] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (reset_flags && threadIdx.x == 0) P.blk_flags[blk] = 0;
  }
}

// Warp-per-block variant (GOP_WARP=1, A/B): no shared memory, no block barrier — every warp owns the flags gw, gw + n_warps, ...; a flagged block is 16 nodes per
// lane, converted four at a time (four independent 128-bit loads in flight per lane, rows of 8 nodes = 128 contiguous bytes).
#ifndef GOP_WARP
#define GOP_WARP 0
#endif
__global__ void __launch_bounds__(256) k_grid_op_warp(const KParams P, const int f, const int clear_pm, const int zero_ggv, const int reset_flags) {
  const int n = P.n, nb = P.nb, nblk = nb * nb * nb;
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * 8 + (threadIdx.x >> 5), nw = gridDim.x * 8;
  fmpm_pdl_trigger();
  fmpm_pdl_wait();
  for (int blk = gw; blk < nblk; blk += nw) {
    if (P.blk_flags[blk] == 0) continue;   // warp-uniform
    const int bx = blk / (nb * nb), by = (blk / nb) % nb, bz = blk % nb;
#pragma unroll 1
    for (int r0 = 0; r0 < 16; r0 += 4) {
      float4 pm[4]; int g[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int t = lane + (r0 + u) * 32;
        g[u] = ((bx * 8 + (t >> 6)) * n + by * 8 + ((t >> 3) & 7)) * n + bz * 8 + (t & 7);
        pm[u] = P.grid_pm[g[u]];
      }
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int t = lane + (r0 + u) * 32;
        P.grid_v[g[u]] = grid_op_node_full(P, f, bx * 8 + (t >> 6), by * 8 + ((t >> 3) & 7), bz * 8 + (t & 7), pm[u]);
        if (clear_pm && (pm[u].w != 0.f || pm[u].x != 0.f || pm[u].y != 0.f || pm[u].z != 0.f)) P.grid_pm[g[u]] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (zero_ggv) P.ggrid_v[g[u]] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    __syncwarp();
    if (reset_flags && lane == 0) P.blk_flags[blk] = 0;
  }
}

// ---- x-slab forward steps, PULL form of the ghost reduction (fmpm_substeps_slab) -------------------------------------------------------------
// The push form (k_p2g / k_fwd with kSlab: every vector reduction on a ghost plane issued a second time into the neighbour's accumulator over
// NVLink) doubles the scatter's reductions on 2 * halo planes per slab boundary — two thirds of ALL reductions for the 24-plane slabs of the
// 8-GPU bench.  Here the scatter stays local (kSlab = false) and grid_op,
// which already runs after the neighbour handshake, READS the neighbour's partial sums of the ghost planes over NVLink: 2 * halo planes of
// active nodes x 16 B per boundary and substep instead.  own + peer is one commutative addition, so both ranks compute bit-identical ghost
// nodes.  Clearing: the neighbour reads this rank's ghost planes during ITS grid_op(f), so blocks that hold ghost planes (and their flags)
// are left as they are and cleared one handshake later — by grid_op(f+1), on the other parity buffer (`Po`) — when the neighbour's
// grid_op(f) is known to be complete; fmpm_substeps_slab ends with one more handshake and a k_clear_blocks of the last parity.
__device__ __forceinline__ float4 ld_peer_v4(const float4* p) {
#ifdef FMPM_HOST_EMU
  return *p;
#else
  float4 v;   // never through L1: the line may be there from the previous substep
  asm volatile("ld.volatile.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
#endif
}
__device__ __forceinline__ int ld_peer_flag(const int* p) { return *(const volatile int*)p; }
// Handshake inside the launch (sig != nullptr; opt-in, FMPM_SLAB_FSYNC=1 — parity green on 2 GPUs but SLOWER than the separate one-thread k_slab_sync launch:
// the one resident wave of 444 fat blocks it needs costs the neighbour-independent part more than the launch it saves): block 0 posts this rank's epoch E = sig[2] + 1 to the neighbours (sig[2] is only advanced by
// the LAST block of this launch, so every block reads the same E), the blocks first convert the nodes no neighbour contributes to, and only then wait
// for the neighbours' epochs — once — before they read peer flags / peer ghost planes and clear the other parity's ghost blocks.
__device__ __forceinline__ void grid_op_pull_block(const KParams& P, const int f, const int blk, const bool ghost) {
  const int n = P.n, nb = P.nb;
  const int bx = blk / (nb * nb), by = (blk / nb) % nb, bz = blk % nb;
  const int x0 = bx * 8;
  const bool gl = ghost && P.peer_l != nullptr && x0 < P.gl_hi && x0 + 8 > P.gl_lo, gr = ghost && P.peer_r != nullptr && x0 < P.gr_hi && x0 + 8 > P.gr_lo;
#pragma unroll
  for (int r = 0; r < 2; r++) {
    const int t = threadIdx.x + r * 256;
    const int i = x0 + (t >> 6), j = by * 8 + ((t >> 3) & 7), k = bz * 8 + (t & 7);
    const int g = (i * n + j) * n + k;
    float4 pm = P.grid_pm[g];
    const bool clr = !(gl || gr) && (pm.w != 0.f || pm.x != 0.f || pm.y != 0.f || pm.z != 0.f);
    if (gl && i >= P.gl_lo && i < P.gl_hi) { const float4 q = ld_peer_v4(P.peer_l + g); pm.x += q.x; pm.y += q.y; pm.z += q.z; pm.w += q.w; }
    if (gr && i >= P.gr_lo && i < P.gr_hi) { const float4 q = ld_peer_v4(P.peer_r + g); pm.x += q.x; pm.y += q.y; pm.z += q.z; pm.w += q.w; }
    P.grid_v[g] = grid_op_node_full(P, f, i, j, k, pm);
    if (clr) P.grid_pm[g] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (!(gl || gr) && threadIdx.x == 0) P.blk_flags[blk] = 0;
}
__global__ void __launch_bounds__(256) k_grid_op_pull(const KParams P, const int f, float4* __restrict__ pm_other, int* __restrict__ flags_other,
                                                      int* sig, int* psig_l, int* psig_r) {
  const int n = P.n, nb = P.nb, nblk = nb * nb * nb;
  __shared__ int s_act[256];
  __shared__ int s_gho[256];
  __shared__ int s_clr[256];
  __shared__ int s_n, s_ng, s_nc;
  if (threadIdx.x == 0) { s_n = 0; s_ng = 0; s_nc = 0; }
  const int E = sig ? ((volatile int*)sig)[2] + 1 : 0;
  if (sig && blockIdx.x == 0 && threadIdx.x == 0) {   // my scatter of frame f (the kernels before this one) is complete: tell the neighbours
    FMPM_SYSTEM_FENCE();
    if (psig_l) ((volatile int*)psig_l)[1] = E;   // I am my left neighbour's RIGHT neighbour
    if (psig_r) ((volatile int*)psig_r)[0] = E;
    FMPM_SYSTEM_FENCE();
  }
  __syncthreads();
  {
    const int blk = blockIdx.x + threadIdx.x * gridDim.x;
    if (blk < nblk) {
      const int x0 = (blk / (nb * nb)) * 8;
      const bool ghost = (P.peer_fl != nullptr && x0 < P.gl_hi && x0 + 8 > P.gl_lo) || (P.peer_fr != nullptr && x0 < P.gr_hi && x0 + 8 > P.gr_lo);
      if (ghost) s_gho[atomicAdd(&s_ng, 1)] = blk;                       // its flags (mine | the neighbour's) are read after the handshake
      else if (P.blk_flags[blk] != 0) s_act[atomicAdd(&s_n, 1)] = blk;
      if (flags_other[blk] != 0) s_clr[atomicAdd(&s_nc, 1)] = blk;      // ghost blocks of the previous substep: cleared after the handshake
    }
  }
  __syncthreads();
  const int n_act = s_n, n_gho = s_ng, n_clr = s_nc;
  for (int ai = 0; ai < n_act; ai++) grid_op_pull_block(P, f, s_act[ai], false);
  if (n_gho > 0 || n_clr > 0) {
    if (sig && threadIdx.x == 0) {
      if (psig_l) slab_wait((volatile int*)sig + 0, E, sig + 3);
      if (psig_r) slab_wait((volatile int*)sig + 1, E, sig + 3);
      FMPM_SYSTEM_FENCE();
    }
    __syncthreads();
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    if (threadIdx.x < n_gho) {   // (n_gho <= 256: one candidate per thread at most)
      const int blk = s_gho[threadIdx.x];
      const int x0 = (blk / (nb * nb)) * 8;
      int act = P.blk_flags[blk];
      if (P.peer_fl != nullptr && x0 < P.gl_hi && x0 + 8 > P.gl_lo) act |= ld_peer_flag(P.peer_fl + blk);
      if (P.peer_fr != nullptr && x0 < P.gr_hi && x0 + 8 > P.gr_lo) act |= ld_peer_flag(P.peer_fr + blk);
      if (act != 0) s_act[atomicAdd(&s_n, 1)] = blk;
    }
    __syncthreads();
    const int n_act2 = s_n;
    for (int ai = 0; ai < n_act2; ai++) grid_op_pull_block(P, f, s_act[ai], true);
    for (int ci = 0; ci < n_clr; ci++) {
      const int blk = s_clr[ci];
      const int bx = blk / (nb * nb), by = (blk / nb) % nb, bz = blk % nb;
#pragma unroll
      for (int r = 0; r < 2; r++) {
        const int t = threadIdx.x + r * 256;
        const int i = bx * 8 + (t >> 6), j = by * 8 + ((t >> 3) & 7), k = bz * 8 + (t & 7);
        pm_other[(i * n + j) * n + k] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      if (threadIdx.x == 0) flags_other[blk] = 0;
    }
  }
  if (sig && threadIdx.x == 0) {   // the last block out advances the epoch for the next handshake (sig[4]: blocks done)
    FMPM_SYSTEM_FENCE();
    const int done = atomicAdd(sig + 4, 1);
    if (done == (int)gridDim.x - 1) { sig[4] = 0; ((volatile int*)sig)[2] = E; }
  }
}

// =============================================================================================
// g2p (+ advect_used, process_unused_particles, advect_kernel)
// =============================================================================================
#define G2P_WARPS 4

// no min-blocks bound: ptxas settles at 72 registers (7 CTAs/SM)
__global__ void __launch_bounds__(G2P_WARPS * 32) k_g2p(const KParams P, const int f) {
  __shared__ float4 tiles[G2P_WARPS][9 * G2P_ZMAX];
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  float4* tile = tiles[threadIdx.x >> 5];
  fmpm_pdl_trigger();
  fmpm_pdl_wait();
  float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (s < P.N) a0 = P.pa[pa_idx(P, f, 0, s)];
  const int meta = __float_as_int(a0.w);
  const float x[3] = {a0.x, a0.y, a0.z};
  int b[3]; float fx[3];
  const bool ok = (s < P.N) && (meta & 1) && base_fx(P, x, b, fx);
  Footprint fp = footprint_of(ok, b);
  if (fp.staged) footprint_load(P.grid_v, P.n, fp, tile);
  const bool staged = fp.staged; const int kmin = fp.kmin;
  if (s >= P.N) return;
  if (!ok) {  // unused (MPM:309-316) or frozen: carry the state over unchanged
    if (meta & 2) {  // collected at this substep (fmpm_collect): parked, agents/agent_pouring.py:37-38
      a0.x = a0.y = a0.z = FMPM_NOWHERE; a0.w = __int_as_float(meta & ~3);
    }
    P.pa[pa_idx(P, f + 1, 0, s)] = a0;
    P.pa[pa_idx(P, f + 1, 1, s)] = P.pa[pa_idx(P, f, 1, s)];
    P.pa[pa_idx(P, f + 1, 2, s)] = P.pa[pa_idx(P, f, 2, s)];
    P.pa[pa_idx(P, f + 1, 3, s)] = P.pa[pa_idx(P, f, 3, s)];
    return;
  }
  float w[3][3]; bspline(fx, w);
  float nv[3]; Mat3 nC;
  const float c4 = 4.f * P.inv_dx;
  if (staged) {
    const float4* t0 = tile + (b[2] - kmin);
    g2p_gather(fx, w, [&](int c) { return t0 + c * G2P_ZMAX; }, nv, nC, c4);
  } else {
    const float4* gv = P.grid_v + ((b[0] * P.n + b[1]) * P.n + b[2]);
    const int n = P.n;
    g2p_gather(fx, w, [&](int c) { return gv + ((c / 3) * n + (c % 3)) * n; }, nv, nC, c4);
  }
  if (P.col.has_rigid && P.col.collide_type != 1) {  // agent.collide at particle level (the default), MPM:419-422
    const float xt[3] = {x[0] + P.dt * nv[0], x[1] + P.dt * nv[1], x[2] + P.dt * nv[2]};
    float o[3]; agent_collide<false>(P, f, xt, nv, o, nullptr, nullptr, nullptr, nullptr, nullptr);
    nv[0] = o[0]; nv[1] = o[1]; nv[2] = o[2];
  }
  const float nx[3] = {x[0] + P.dt * nv[0], x[1] + P.dt * nv[1], x[2] + P.dt * nv[2]};  // advect_kernel MPM:505
  store_A(P.pa, P, f + 1, s, nx, meta, nv, nC);
}

// =============================================================================================
// g2p2g: g2p of frame f FUSED with p2g of frame f+1 (forward-only steps without agents; Wang et al. 2020 call the pattern G2P2G).
// A particle's new velocity / affine matrix / position never leave registers between the gather and the next scatter, so an
// intermediate substep moves x + meta (16 B) and F (36 B) in and out: 104 B per particle instead of the 212 B of p2g + g2p, and a
// substep is two launches (grid_op, g2p2g) instead of three.  v and C of the intermediate frames are NOT materialised (kWriteVC =
// false); the step's first p2g and last g2p are the plain kernels, so every step boundary holds a complete frame.
// The scatter's warp-local key ranking (fmpm_scatter.cuh) absorbs the mismatch between the slot order (cells of the last sort)
// and the cells of x[f+1].
// =============================================================================================
// collector boundary test of agents/agent_pouring.py:31-41 / agents/agent_jetbot.py:30-40 (boundaries.py:81-93, 128-134): true = the particle leaves
__device__ __forceinline__ bool collector_takes(const FmpmCollector& c, const int meta, const float* x) {
  const int row = (meta >> 8) & 0xff;
  if (row >= 32 || !((c.row_mask >> row) & 1u)) return false;
  if (c.boundary_type == 0) return x[0] > c.upper[0] || x[1] > c.upper[1] || x[2] > c.upper[2] || x[0] < c.lower[0] || x[1] < c.lower[1] || x[2] < c.lower[2];
  const float rx = x[0] - c.cyl_center[0], rz = x[2] - c.cyl_center[1];
  return x[1] > c.upper[1] || x[1] < c.lower[1] || sqrtf(rx * rx + rz * rz + FMPM_EPS) > c.cyl_radius;
}
// particle of a MAT_RIGID body (body id in meta bits 16..23, FmpmBodies.info = (first, material class) per body)
__device__ __forceinline__ bool rigid_body_slot(const int meta, const int* __restrict__ info, const int nb) {
  const int b = (meta >> 16) & 0xff;
  return (meta & 1) && b < nb && __ldg(info + 2 * b + 1) == FMPM_MAT_RIGID;
}
#ifndef G2P2G_MINB
#define G2P2G_MINB P2G_MINB   // 96 registers at 5 CTAs of 4 warps; A/B other bounds with FMPM_DEFS=-DG2P2G_MINB=... (profiles/ab_variants.sh, PT_FUSED=1)
#endif
// kAgent: particle-level agent.collide and the collector test are compiled in (scenes with a Rigid effector and / or a collector agent)
template <bool kWriteVC, bool kAgent>
__global__ void __launch_bounds__(P2G_WARPS * 32, G2P2G_MINB) k_g2p2g(const KParams P, const int f, const FmpmCollector col, const int has_col,
                                                                              const int* __restrict__ body_info, const int n_bodies) {
  __shared__ ScatterSmem smem[P2G_WARPS];
  static_assert(sizeof(((ScatterSmem*)0)->rec) >= 9 * G2P_ZMAX * sizeof(float4), "the gather tile is staged in the scatter records' storage");
  const int lane = threadIdx.x & 31, wib = __shfl_sync(SC_FULL, (int)(threadIdx.x >> 5), 0);   // broadcast: dependent code is compiled warp-uniform
  ScatterSmem& S = smem[wib];
  float4* tile = S.rec;   // gather tile first, scatter records afterwards (a __syncwarp separates the two uses)
  const long long slot0 = ((long long)blockIdx.x * P2G_WARPS + wib) * 32;
  if (slot0 >= P.N) return;   // warp-uniform
  const long long sl = slot0 + lane;
  const long long rem = (long long)P.N - slot0;
  const int cnt = rem < 32 ? (int)rem : 32;
  Window W; window_init(W, lane, P.n, nullptr);   // blocks are flagged once per warp (flag_box); x-slab forward steps use k_fwd
  // ---- g2p of frame f (MPM:304-316, 400-426, 497-505)
  float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (sl < P.N) a0 = P2G_LD(&P.pa[pa_idx(P, f, 0, (int)sl)]);
  const int meta = __float_as_int(a0.w);
  const float x[3] = {a0.x, a0.y, a0.z};
  int b[3]; float fx[3];
  const bool ok = (sl < P.N) && (meta & 1) && base_fx(P, x, b, fx);
  Footprint fp = footprint_of(ok, b);
  if (fp.staged) footprint_load(P.grid_v, P.n, fp, tile);
  int key = -1;
  int b1[3] = {0, 0, 0}; bool ok1 = false;
  float q[3] = {0.f, 0.f, 0.f}, B[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, m = 0.f;
  float w[3][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
  if (sl < P.N) {
    const int s = (int)sl;
    PState st;
    {  // F[f+1] was written by the p2g / g2p2g of frame f
      const float4 f0 = P2G_LD(&P.pf[pf_idx(P, f + 1, 0, s)]), f1 = P2G_LD(&P.pf[pf_idx(P, f + 1, 1, s)]);
      st.F.m[0] = f0.x; st.F.m[1] = f0.y; st.F.m[2] = f0.z; st.F.m[3] = f0.w; st.F.m[4] = f1.x; st.F.m[5] = f1.y; st.F.m[6] = f1.z; st.F.m[7] = f1.w;
      st.F.m[8] = P2G_LD(&P.pf8[pf8_idx(P, f + 1, s)]);
    }
    if (!ok) {  // unused (MPM:309-316) or frozen: the whole state is carried over unchanged
      if (meta & 2) { a0.x = a0.y = a0.z = FMPM_NOWHERE; a0.w = __int_as_float(meta & ~3); }
      P.pa[pa_idx(P, f + 1, 0, s)] = a0;
      P.pa[pa_idx(P, f + 1, 1, s)] = P.pa[pa_idx(P, f, 1, s)];
      P.pa[pa_idx(P, f + 1, 2, s)] = P.pa[pa_idx(P, f, 2, s)];
      P.pa[pa_idx(P, f + 1, 3, s)] = P.pa[pa_idx(P, f, 3, s)];
      p2g_store_F(P, f + 2, s, st.F);
    } else {
      bspline(fx, w);
      const float c4 = 4.f * P.inv_dx;
      if (fp.staged) {
        const float4* t0 = tile + (b[2] - fp.kmin);
        g2p_gather(fx, w, [&](int c) { return t0 + c * G2P_ZMAX; }, st.v, st.C, c4);
      } else {
        const float4* gv = P.grid_v + ((b[0] * P.n + b[1]) * P.n + b[2]);
        const int n = P.n;
        g2p_gather(fx, w, [&](int c) { return gv + ((c / 3) * n + (c % 3)) * n; }, st.v, st.C, c4);
      }
      if (kAgent && P.col.has_rigid && P.col.collide_type != 1) {  // agent.collide at particle level (the default), MPM:419-422
        const float xt[3] = {x[0] + P.dt * st.v[0], x[1] + P.dt * st.v[1], x[2] + P.dt * st.v[2]};
        float o[3]; agent_collide<false>(P, f, xt, st.v, o, nullptr, nullptr, nullptr, nullptr, nullptr);
        st.v[0] = o[0]; st.v[1] = o[1]; st.v[2] = o[2];
      }
#pragma unroll
      for (int d = 0; d < 3; d++) st.x[d] = x[d] + P.dt * st.v[d];   // advect_kernel MPM:505
      // collector agents act on frame f+1 BEFORE its p2g (MPM:521): a particle that left is tagged (used bit off, bit 1 on), does not
      // scatter, and the next substep's gather parks it — exactly what fmpm_collect(f+1) + k_p2g + k_g2p do on the unfused path
      // a particle of a MAT_RIGID body: its position of frame f+1 is only final after the body's shape matching (fmpm_advect_rigid(f), MPM:428-505),
      // so it leaves here with the complete provisional frame; k_p2g_rigid applies the collector test, scatters it and writes F[f+2] after that pass
      const bool rigid = kAgent && body_info != nullptr && rigid_body_slot(meta, body_info, n_bodies);
      const bool taken = kAgent && has_col && !rigid && collector_takes(col, meta, st.x);
      st.meta = taken ? ((meta & ~1) | 2) : meta;
      // ---- p2g of frame f+1 (MPM:254-264, 331-378)
      float fx1[3];
      ok1 = !taken && !rigid && base_fx(P, st.x, b1, fx1);
      if (kWriteVC || !ok1) store_A(P.pa, P, f + 1, s, st.x, st.meta, st.v, st.C);
      else P.pa[pa_idx(P, f + 1, 0, s)] = make_float4(st.x[0], st.x[1], st.x[2], __int_as_float(st.meta));
      if (ok1) {
        const float4 mt = __ldg(P.mats + ((meta >> 8) & 0xff));
        Constit K; constitutive(P, st, mt.x, mt.y, mt.z, __float_as_int(mt.w), K);
        m = mt.z;
        bspline(fx1, w);
#pragma unroll
        for (int i = 0; i < 9; i++) B[i] = K.A.m[i] * P.dx;
#pragma unroll
        for (int i = 0; i < 3; i++) q[i] = m * st.v[i] - (B[i * 3] * fx1[0] + B[i * 3 + 1] * fx1[1] + B[i * 3 + 2] * fx1[2]);
        key = pack_key(b1);
        p2g_store_F(P, f + 2, s, K.Fn);
      } else if (!rigid) {
        p2g_store_F(P, f + 2, s, st.F);
      }
    }
  }
  flag_box<false>(W, P.blk_flags, lane, ok1, b1);
  __syncwarp();   // every lane is done with the gather tile before the scatter staging is written
  const unsigned starts = scatter_publish(S, lane, key, W.cur_key, q, B, m, w);
  __syncwarp();
  window_consume2<false>(W, S, cnt, starts, P.grid_pm);
  window_flush_all2<false>(W, P.grid_pm);
}

// =============================================================================================
// k_fwd: the forward-only substep kernel of agent-free scenes — g2p(f) [+ grid_op(f) inlined] + p2g(f+1) in ONE launch.
//   kMat == 1  every particle is a mu = 0 liquid (WATER / MILK / COFFEE ...: BASELINE configs C1-C3, C5): no SVD code at all, and because
//              F[f+1] = J^(1/3) I (MPM:358-359) the deformation gradient of the intermediate frames travels as the single float s = F22
//              (plane pf8): F~ = (I + dt C) s is bit-identical to the general product with F = diag(s, s, s).  Intermediate frames then
//              hold x + meta + s: 20 B in and 20 B out per particle and substep instead of the 212 B of p2g + g2p.
//   kInline    grid_op (MPM:380-398: momentum -> velocity, gravity, domain boundary; scenes without SDF colliders at grid level) is
//              evaluated while the warp stages its node footprint, straight from the (momentum, mass) accumulator: grid_v is never written
//              or read and the substep is ONE launch.  The accumulator is triple-buffered by frame (f % 3): this launch gathers from buffer
//              f % 3, scatters frame f+1 into (f+1) % 3 and clears the blocks of (f+2) % 3 that the launch before gathered from.
// The footprint of a warp is the box of nodes its 32 particles touch, up to 4 x 4 node columns x 16 nodes (a fresh sort gives 3 x 3 x ~7;
// the extra column in x and y absorbs the drift between two cell sorts), staged with coalesced 128-bit loads.
// =============================================================================================
#ifndef FWD_MINB
#define FWD_MINB 7   // with FWD_WARPS 3 ptxas settles at 80 registers, so 8 CTAs = 24 warps fit an SM; 6 and 8 time slower on an H100 (DESIGN.md §8)
#endif
#ifndef FWD_AHEAD
#define FWD_AHEAD 0   // > 0: L2 prefetch of the particle lines of the CTA FWD_AHEAD CTAs further on (one resident wave ahead: SMs x 8)
#endif
#ifndef FWD_PERSIST
#define FWD_PERSIST 0   // (off: the loop costs more instructions and spills than the CTA turnover it saves)  1: persistent warps — sm_count x FWD_MINB CTAs, every warp claims 32-slot chunks from a global counter (P.blk_list[0]) until none is
                        // left: no CTA turnover, and the tail of the grid shrinks from a partial wave of CTAs to one chunk.  Not with the lazy grid_op (kInline).
#endif
#ifndef FWD_WARPS
#define FWD_WARPS 3   // warps per CTA of k_fwd
#endif
#define FWD_TILE_COLS 16   // 4 x 4 node columns
// grid_op of one node without SDF colliders (MPM:380-386,398): the same operations, in the same order, as k_grid_op.
// interior: the caller knows that no boundary condition can act on this node (then boundary_v would multiply by 1: skipped)
__device__ __forceinline__ float4 grid_op_node(const KParams& P, const int i, const int j, const int k, const float4 pm, const bool interior = false) {
  float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
  if (pm.w > FMPM_EPS) {
    const float inv_m = 1.f / pm.w;
    float v[3] = {inv_m * pm.x + P.dt * P.gx, inv_m * pm.y + P.dt * P.gy, inv_m * pm.z + P.dt * P.gz};
    if (!interior) {
      const float pos[3] = {(float)i * P.dx, (float)j * P.dx, (float)k * P.dx};
      float fac[3];
      boundary_v(P, pos, v, fac);
    }
    out = make_float4(v[0], v[1], v[2], 0.f);
  }
  return out;
}
// true when no node of the box [i0,i1] x [j0,j1] x [k0,k1] can be touched by the domain boundary (boundaries.py:39-63,106-120): the cube's
// walls / the cylinder's caps and mantle lie strictly outside it and no dimension is locked.  Conservative, warp-uniform.
__device__ __forceinline__ bool box_is_interior(const KParams& P, const int i0, const int i1, const int j0, const int j1, const int k0, const int k1) {
  if (P.lock_mask != 0) return false;
  const float x0 = (float)i0 * P.dx, x1 = (float)i1 * P.dx, y0 = (float)j0 * P.dx, y1 = (float)j1 * P.dx, z0 = (float)k0 * P.dx, z1 = (float)k1 * P.dx;
  if (P.boundary_type == 0)
    return x0 > P.lo[0] && x1 < P.hi[0] && y0 > P.lo[1] && y1 < P.hi[1] && z0 > P.lo[2] && z1 < P.hi[2];
  const float ax = fmaxf(fabsf(x0 - P.cyl_cx), fabsf(x1 - P.cyl_cx)), az = fmaxf(fabsf(z0 - P.cyl_cz), fabsf(z1 - P.cyl_cz));
  return y0 >= P.lo[1] && y1 <= P.hi[1] && sqrtf(ax * ax + az * az + FMPM_EPS) < 0.999f * P.cyl_r;
}
// lazy grid_op: a node's v_out and its tag travel in ONE 16-byte access, which the GPU performs as a single transaction.  The host build of the execution-model
// tests has no such guarantee (a float4 copy may be four moves: a reader could pair a fresh tag with stale components), so there the tag is written last
// and read first, with the ordering x86-TSO provides once the compiler is kept from reordering.
__device__ __forceinline__ float4 ld_tagged(const float4* p) {
#ifdef FMPM_HOST_EMU
  float4 g;
  g.w = *(const volatile float*)&p->w;
  __atomic_thread_fence(__ATOMIC_ACQUIRE);
  g.x = *(const volatile float*)&p->x; g.y = *(const volatile float*)&p->y; g.z = *(const volatile float*)&p->z;
  return g;
#else
  return __ldcg(p);
#endif
}
__device__ __forceinline__ void st_tagged(float4* p, const float4& g) {
#ifdef FMPM_HOST_EMU
  *(volatile float*)&p->x = g.x; *(volatile float*)&p->y = g.y; *(volatile float*)&p->z = g.z;
  __atomic_thread_fence(__ATOMIC_RELEASE);
  *(volatile float*)&p->w = g.w;
#else
  *p = g;
#endif
}
// the rare warp whose particles do not fit one footprint box (no cell sort yet, or a very old one): every lane gathers its own 27 nodes
// from L2.  The node loop stays rolled so that the hot kernel stays small in the instruction cache.
template <bool kInline>
__device__ __forceinline__ void fwd_gather_unstaged(const KParams& P, const float4* __restrict__ pms, const int tagf, const int* b, const float* fx, float* nv, float* nC) {
  const int n = P.n;
  const int cell = (b[0] * n + b[1]) * n + b[2];
  float v[3] = {0.f, 0.f, 0.f}, C[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
  for (int c = 0; c < 27; c++) {
    const int i = c / 9, j = (c / 3) % 3, k = c % 3;
    const int node = cell + (i * n + j) * n + k;
    float4 g = kInline ? ld_tagged(&P.grid_v[node]) : P.grid_v[node];
    if (kInline && __float_as_int(g.w) != tagf) {   // lazy grid_op, see k_fwd
      g = grid_op_node(P, b[0] + i, b[1] + j, b[2] + k, pms[node]);
      g.w = __int_as_float(tagf);
      st_tagged(&P.grid_v[node], g);
    }
    const float d[3] = {(float)i - fx[0], (float)j - fx[1], (float)k - fx[2]};
    float wt = 1.f;
#pragma unroll
    for (int r = 0; r < 3; r++) {   // quadratic B-spline weight of offset o = (i, j, k)[r] (bspline(), MPM:336), selected without indexing a local array
      const int o = r == 0 ? i : (r == 1 ? j : k);
      const float a = 1.5f - fx[r], bb = fx[r] - 1.0f, cc = fx[r] - 0.5f;
      wt *= o == 0 ? 0.5f * a * a : (o == 1 ? 0.75f - bb * bb : 0.5f * cc * cc);
    }
    const float gvv[3] = {g.x, g.y, g.z};
#pragma unroll
    for (int r = 0; r < 3; r++) {
      v[r] += wt * gvv[r];
#pragma unroll
      for (int q = 0; q < 3; q++) C[r * 3 + q] += wt * gvv[r] * d[q];
    }
  }
  const float c4 = 4.f * P.inv_dx;
#pragma unroll
  for (int r = 0; r < 3; r++) nv[r] = v[r];
#pragma unroll
  for (int r = 0; r < 9; r++) nC[r] = c4 * C[r];
}
// kInline (lazy grid_op): P.grid_v is a CACHE of v_out whose w component carries the tag (launch epoch) of the substep it was computed for;
// pms is the (momentum, mass) accumulator of frame f.  A node whose cached tag is not this launch's tag is converted on the spot
// (grid_op_node) and written back with the tag in ONE 16-byte store, so each node is converted by the first warp that needs it (plus the
// few that race with it: they store identical values) instead of by every warp that stages it.  `stride` permutes the CTA -> slot-block
// map (an odd prime not dividing the grid size): neighbouring slot blocks — which share their nodes — then run in different waves.
// frame bases of one k_fwd launch, computed on the host (in the kernel the 64-bit products f * 4 * N ... were ~20 per-lane instructions per warp)
struct FwdFrames { float4* pa_f; float4* pa_n; float4* pf_r; float4* pf_w; float* p8_r; float* p8_w; };
template <int kMat, bool kInline, bool kSlab>
__global__ void __launch_bounds__(FWD_WARPS * 32, FWD_MINB) k_fwd(const KParams P, const FwdFrames FR, const int f, float4* __restrict__ clr, int* __restrict__ clr_flags, const int full,
                                                                            const float4* __restrict__ pms, const int tag_off, const int stride,
                                                                            const __grid_constant__ CUtensorMap tm8, const __grid_constant__ CUtensorMap tm16, const int use_tma) {
  __shared__ ScatterSmem smem[FWD_WARPS];
  __shared__ unsigned long long tbar[FWD_WARPS];   // one mbarrier per warp: completion of its TMA footprint tile
  static_assert(sizeof(((ScatterSmem*)0)->rec) >= FWD_TILE_COLS * 16 * sizeof(float4), "the gather tile is staged in the scatter records' storage");
  const int lane = threadIdx.x & 31, wib = __shfl_sync(SC_FULL, (int)(threadIdx.x >> 5), 0);   // broadcast: dependent code is compiled warp-uniform
  ScatterSmem& S = smem[wib];
  float4* tile = S.rec;   // gather tile first, scatter records afterwards (a __syncwarp separates the two uses)
  const long long gw = (long long)blockIdx.x * FWD_WARPS + wib;
  // the slot block this warp works on; only the lazy grid_op permutes the CTA -> slot-block map (32-bit: the host checks blocks * stride < 2^32) —
  // elsewhere the identity is compiled in (the modulo costs instructions in every warp)
  const long long gws = kInline ? (long long)((blockIdx.x * (unsigned)stride) % gridDim.x) * FWD_WARPS + wib : gw;
  fmpm_pdl_trigger();
  fmpm_pdl_wait();
  const int tagf = kInline ? (*P.epoch + tag_off) : 0;
  // ---- clear duty (kInline): one warp per flagged 8^3-node block of the accumulator that the previous launch gathered from
  if (kInline && clr != nullptr) {
    const int nb = P.nb, nblk = nb * nb * nb, n = P.n;
    const long long nwarps = (long long)gridDim.x * FWD_WARPS;
    for (long long blk = gw; blk < nblk; blk += nwarps) {
      if (clr_flags[blk] != 0) {   // warp-uniform
        const int bx = (int)(blk / (nb * nb)), by = (int)((blk / nb) % nb), bz = (int)(blk % nb);
#pragma unroll 4
        for (int r = 0; r < 16; r++) {
          const int t = lane + r * 32;
          const int i = bx * 8 + (t >> 6), j = by * 8 + ((t >> 3) & 7), k = bz * 8 + (t & 7);
          clr[(i * n + j) * n + k] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        __syncwarp();
        if (lane == 0) clr_flags[blk] = 0;
      }
    }
  }
  constexpr bool kPersist = FWD_PERSIST && !kInline && (kMat == 1 || FWD_PERSIST >= 2);   // (the general instantiation spills 250 B inside the loop: FWD_PERSIST=2 to force it)
  unsigned tph = 0;   // phase of the warp's mbarrier (it completes once per TMA tile)
#ifndef FMPM_HOST_EMU
  if (kPersist && use_tma) {
    if (lane == 0) mbar_init(&tbar[wib], 1);
    __syncwarp();
  }
#endif
#if FWD_PERSIST
  for (;;) {
#endif
  long long slot0 = gws * 32;
  if (kPersist) {   // claim the next chunk of 32 slots
    int chunk = 0;
    if (lane == 0) chunk = atomicAdd(P.blk_list, 1);
    slot0 = (long long)__shfl_sync(SC_FULL, chunk, 0) * 32;
  }
#if FWD_PERSIST
  if (slot0 >= P.N) break;    // warp-uniform
#else
  if (slot0 >= P.N) return;   // warp-uniform
#endif
  const long long sl = slot0 + lane;
  const long long rem = (long long)P.N - slot0;
  const int cnt = rem < 32 ? (int)rem : 32;
  const bool inrange = sl < P.N;
  const int s = (int)sl;
  // plane pointers of this slot: frame f / f+1 of the state planes, frame f+1 / f+2 of F
  const size_t Ns = (size_t)P.N;
#ifdef FWD_DEVICE_PTRS   // A/B (profiles/ab_variants.sh): the earlier form, frame offsets computed per lane in the kernel
  float4* const pa_f = P.pa + (size_t)f * 4 * Ns + s; float4* const pa_n = pa_f + 4 * Ns;
  float4* const pf_r = P.pf + (size_t)(f + 1) * 2 * Ns + s; float4* const pf_w = pf_r + 2 * Ns;
  float* const p8_r = P.pf8 + (size_t)(f + 1) * Ns + s; float* const p8_w = p8_r + Ns;
#else
  float4* const pa_f = FR.pa_f + s; float4* const pa_n = FR.pa_n + s;
  float4* const pf_r = FR.pf_r + s; float4* const pf_w = FR.pf_w + s;
  float* const p8_r = FR.p8_r + s; float* const p8_w = FR.p8_w + s;
#endif
  // ---- particle loads: x + meta of frame f, F[f+1] (written by the p2g / k_fwd of frame f)
  float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 f0 = make_float4(1.f, 0.f, 0.f, 0.f), f1 = make_float4(1.f, 0.f, 0.f, 0.f); float f8 = 1.f;
  if (inrange) {
    a0 = P2G_LD(pa_f);
    f8 = P2G_LD(p8_r);
    if (kMat != 1) { f0 = P2G_LD(pf_r); f1 = P2G_LD(pf_r + Ns); }
  }
#if FWD_AHEAD > 0
  {   // CTAs are dispatched in index order: the one that takes this CTA's place is ~FWD_AHEAD CTAs further on.  Its x / F lines go to L2 now, so that its
      // first loads (the one DRAM latency nothing overlaps) are L2 hits.  One 128-byte line per 8 lanes.
    const long long ahead = (long long)FWD_AHEAD * FWD_WARPS * 32;
    if (sl + ahead < P.N) {
      if ((lane & 7) == 0) prefetch_l2(pa_f + ahead);
      if (lane == 0) prefetch_l2(p8_r + ahead);
      if (kMat != 1 && (lane & 7) == 0) { prefetch_l2(pf_r + ahead); prefetch_l2(pf_r + Ns + ahead); }
    }
  }
#endif
  const int meta = __float_as_int(a0.w);
  const float x[3] = {a0.x, a0.y, a0.z};
  int b[3]; float fx[3];
  const bool ok = inrange && (meta & 1) && base_fx(P, x, b, fx);
  // ---- footprint box of the warp
  const int bx0 = __reduce_min_sync(SC_FULL, ok ? b[0] : 0x7fffffff), bx1 = __reduce_max_sync(SC_FULL, ok ? b[0] : -1);
  const int by0 = __reduce_min_sync(SC_FULL, ok ? b[1] : 0x7fffffff), by1 = __reduce_max_sync(SC_FULL, ok ? b[1] : -1);
  const int bz0 = __reduce_min_sync(SC_FULL, ok ? b[2] : 0x7fffffff), bz1 = __reduce_max_sync(SC_FULL, ok ? b[2] : -1);
  const int nx = bx1 - bx0 + 3, ny = by1 - by0 + 3, nz = bz1 - bz0 + 3;
  const bool any = bx1 >= 0;
  const bool staged = any && nx <= 4 && ny <= 4 && nz <= 16;
  const int tzs = nz <= 8 ? 3 : 4;   // rows of 8 or 16 nodes
#ifndef FMPM_HOST_EMU
  const bool tma = !kInline && use_tma && staged;   // warp-uniform
  if (tma) {
    // The 3x3x3 neighbourhoods of the warp's particles as ONE TMA tile: cp.async.bulk.tensor.4d copies the box (4 components, 8 | 16 nodes in z,
    // 4 in y, 4 in x) at (0, bz0, by0, bx0) of grid_v into the warp's tile (out-of-range nodes arrive as zeros) and completes on the warp's
    // mbarrier; the lanes meanwhile go on with the particle-side arithmetic and wait just before the gather.
    if (lane == 0) {
      if (!kPersist) mbar_init(&tbar[wib], 1);
      else asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the tile overwrites the previous chunk's scatter records (generic-proxy stores)
      mbar_expect_tx(&tbar[wib], (unsigned)((FWD_TILE_COLS << tzs) * sizeof(float4)));
      tma_load_4d(tile, tzs == 3 ? &tm8 : &tm16, &tbar[wib], 0, bz0, by0, bx0);
    }
  } else
#else
  const bool tma = false;
#endif
  if (staged) {
    const int n = P.n, tot = FWD_TILE_COLS << tzs;
    // four rows of 32 slots per batch: all loads of a batch are issued before the first use (one exposed L2 latency per batch)
#pragma unroll 1
    for (int t0 = 0; t0 < tot; t0 += 128) {
      if (((t0 >> tzs) >> 2) >= nx) break;   // warp-uniform: the remaining columns lie outside the box
      float4 g[4]; bool act[4]; int gi[4], gj[4], gk[4];
      bool stale = false;
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int t = t0 + u * 32 + lane;
        const int iz = t & ((1 << tzs) - 1), c = t >> tzs, iy = c & 3, ix = c >> 2;
        act[u] = ix < nx && iy < ny && iz < nz;
        gi[u] = bx0 + ix; gj[u] = by0 + iy; gk[u] = bz0 + iz;
        if (act[u]) g[u] = kInline ? ld_tagged(&P.grid_v[(gi[u] * n + gj[u]) * n + gk[u]]) : P.grid_v[(gi[u] * n + gj[u]) * n + gk[u]];
        if (kInline) stale = stale || (act[u] && __float_as_int(g[u].w) != tagf);
      }
      if (kInline && __any_sync(SC_FULL, stale)) {   // warp-uniform; false for most warps once the first toucher of a node has converted it
        const bool interior = box_is_interior(P, bx0, bx0 + nx - 1, by0, by0 + ny - 1, bz0, bz0 + nz - 1);
#pragma unroll
        for (int u = 0; u < 4; u++)
          if (act[u] && __float_as_int(g[u].w) != tagf) {
            const int node = (gi[u] * n + gj[u]) * n + gk[u];
            g[u] = grid_op_node(P, gi[u], gj[u], gk[u], pms[node], interior);
            g[u].w = __int_as_float(tagf);
            st_tagged(&P.grid_v[node], g[u]);   // v_out and its tag in one 16-byte store
          }
      }
#pragma unroll
      for (int u = 0; u < 4; u++)
        if (act[u]) tile[t0 + u * 32 + lane] = g[u];
    }
    __syncwarp();
  }
#ifndef FMPM_HOST_EMU
  if (tma) __syncwarp();   // the warp's mbarrier was initialised by lane 0
#endif
  int key = -1;
  int b1[3] = {0, 0, 0}; bool ok1 = false;
  float q[3] = {0.f, 0.f, 0.f}, B[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, m = 0.f;
  float w[3][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
  if (inrange) {
    PState st;
    if (!ok) {  // unused (MPM:309-316) or frozen: the whole state is carried over unchanged (these slots always hold complete frames)
      if (meta & 2) { a0.x = a0.y = a0.z = FMPM_NOWHERE; a0.w = __int_as_float(meta & ~3); }
      if (kMat == 1) { f0 = pf_r[0]; f1 = pf_r[Ns]; }
      pa_n[0] = a0; pa_n[Ns] = pa_f[Ns]; pa_n[2 * Ns] = pa_f[2 * Ns]; pa_n[3 * Ns] = pa_f[3 * Ns];
      pf_w[0] = f0; pf_w[Ns] = f1; *p8_w = f8;
    } else {
      // ---- g2p of frame f (MPM:400-426) + advect (MPM:497-505)
      bspline(fx, w);
      const float c4 = 4.f * P.inv_dx;
#ifndef FMPM_HOST_EMU
      if (tma) mbar_wait(&tbar[wib], tph);   // the tile has landed (every gathering lane waits; the others meet them at the __syncwarp before the staging)
#endif
      if (staged) {
        const float4* t0 = tile + ((((b[0] - bx0) << 2) + (b[1] - by0)) << tzs) + (b[2] - bz0);
        g2p_gather_v(fx, w, [&](int c) { const float4* p = t0 + ((((c / 3) << 2) + (c % 3)) << tzs); Col3 r; r.g0 = p[0]; r.g1 = p[1]; r.g2 = p[2]; return r; }, st.v, st.C, c4);
      } else if (kInline) {
        fwd_gather_unstaged<kInline>(P, pms, tagf, b, fx, st.v, st.C.m);
      } else {   // warps that straddle two z-columns (1 in 16 at 8 particles per cell) or are not cell-sorted: 27 gathers per lane from L2
        const float4* gv = P.grid_v + ((b[0] * P.n + b[1]) * P.n + b[2]);
        const int n = P.n;
        g2p_gather(fx, w, [&](int c) { return gv + ((c / 3) * n + (c % 3)) * n; }, st.v, st.C, c4);
      }
#pragma unroll
      for (int d = 0; d < 3; d++) st.x[d] = x[d] + P.dt * st.v[d];
      st.meta = meta;
      // ---- p2g of frame f+1 (MPM:254-264, 331-378)
      float fx1[3];
      ok1 = base_fx(P, st.x, b1, fx1);
      pa_n[0] = make_float4(st.x[0], st.x[1], st.x[2], a0.w);
      if (full || !ok1) {
        pa_n[Ns] = make_float4(st.v[0], st.v[1], st.v[2], st.C.m[0]);
        pa_n[2 * Ns] = make_float4(st.C.m[1], st.C.m[2], st.C.m[3], st.C.m[4]);
        pa_n[3 * Ns] = make_float4(st.C.m[5], st.C.m[6], st.C.m[7], st.C.m[8]);
      }
      if (ok1) {
        const float4 mt = __ldg(P.mats + ((meta >> 8) & 0xff));
        m = mt.z;
        float Bm[9];   // affine = k_stress * stress + m C  (MPM:344), times dx
        if (kMat == 1) {
          float Ft[9];
#pragma unroll
          for (int i = 0; i < 9; i++) Ft[i] = (P.dt * st.C.m[i] + ((i % 4 == 0) ? 1.f : 0.f)) * f8;   // (I + dt C) F with F = f8 I
          const float J = Ft[0] * (Ft[4] * Ft[8] - Ft[5] * Ft[7]) - Ft[1] * (Ft[3] * Ft[8] - Ft[5] * Ft[6]) + Ft[2] * (Ft[3] * Ft[7] - Ft[4] * Ft[6]);
          const float iso = mt.y * J * (J - 1.f);
#pragma unroll
          for (int i = 0; i < 9; i++) Bm[i] = (P.k_stress * ((i % 4 == 0) ? iso : 0.f) + m * st.C.m[i]) * P.dx;
          float sn = (J > 0.f) ? cbrtf(J) : __int_as_float(0x7fc00000);   // pow(J, 1/3): NaN for J < 0 like the reference
          if (J == 0.f) sn = 0.f;
          if (full) { __stcs(pf_w, make_float4(sn, 0.f, 0.f, 0.f)); __stcs(pf_w + Ns, make_float4(sn, 0.f, 0.f, 0.f)); }
          __stcs(p8_w, sn);
        } else {
          st.F.m[0] = f0.x; st.F.m[1] = f0.y; st.F.m[2] = f0.z; st.F.m[3] = f0.w; st.F.m[4] = f1.x; st.F.m[5] = f1.y; st.F.m[6] = f1.z; st.F.m[7] = f1.w; st.F.m[8] = f8;
          Constit K; constitutive(P, st, mt.x, mt.y, mt.z, __float_as_int(mt.w), K);
#pragma unroll
          for (int i = 0; i < 9; i++) Bm[i] = K.A.m[i] * P.dx;
          __stcs(pf_w, make_float4(K.Fn.m[0], K.Fn.m[1], K.Fn.m[2], K.Fn.m[3])); __stcs(pf_w + Ns, make_float4(K.Fn.m[4], K.Fn.m[5], K.Fn.m[6], K.Fn.m[7]));
          __stcs(p8_w, K.Fn.m[8]);
        }
        bspline(fx1, w);
#pragma unroll
        for (int i = 0; i < 9; i++) B[i] = Bm[i];
#pragma unroll
        for (int i = 0; i < 3; i++) q[i] = m * st.v[i] - (B[i * 3] * fx1[0] + B[i * 3 + 1] * fx1[1] + B[i * 3 + 2] * fx1[2]);
        key = pack_key(b1);
      } else {   // left the grid: frozen from now on, with the complete state (F = f8 I for kMat == 1)
        if (kMat == 1) { f0 = make_float4(f8, 0.f, 0.f, 0.f); f1 = f0; }
        pf_w[0] = f0; pf_w[Ns] = f1; *p8_w = f8;
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
          for (int j = 0; j < 3; j++) w[i][j] = 0.f;
      }
    }
  }
  // the window is set up only now: its per-lane fields (node offsets, pointers) would otherwise stay live through the gather and the particle
  // update, where the 80-register bound is tightest
  Window W; window_init(W, lane, P.n, nullptr);   // blocks are flagged once per warp (flag_box), not by the window
  if (kSlab) window_set_slab(W, P.peer_l, P.peer_r, P.gl_lo, P.gl_hi, P.gr_lo, P.gr_hi, P.peer_fl, P.peer_fr);   // x-slab mode: like k_p2g
  flag_box<kSlab>(W, P.blk_flags, lane, ok1, b1);
  __syncwarp();   // every lane is done with the gather tile before the scatter staging is written
  const unsigned starts = scatter_publish(S, lane, key, W.cur_key, q, B, m, w);
  __syncwarp();
  window_consume2<kSlab>(W, S, cnt, starts, P.grid_pm);
  window_flush_all2<kSlab>(W, P.grid_pm);
#if FWD_PERSIST
  if (!kPersist) break;
  if (tma) tph ^= 1u;
  __syncwarp();   // the staging area is the next chunk's gather tile
  }
  if (kPersist && lane == 0) {   // the last warp out resets the chunk counter for the next launch (every other warp has left its loop by then)
    const int done = atomicAdd(P.blk_list + 1, 1);
    if (done == (int)(gridDim.x * FWD_WARPS) - 1) { P.blk_list[0] = 0; P.blk_list[1] = 0; }
  }
#endif
}

// p2g of the few particles an injector has just activated in frame f (fused steps with an injector agent: the g2p2g kernel of the previous
// substep ran before agent.act wrote them, so their contribution to the grid of frame f is added here — flux particles, plain vector
// reductions, no window).  Same arithmetic as k_p2g for one particle; also writes F[f+1] and flags the touched blocks.
// one particle's p2g with plain vector reductions (no window): used for the few particles the fused steps handle outside k_g2p2g
__device__ __forceinline__ void p2g_one_particle(const KParams& P, const int f, const int s, const FmpmCollector& col, const int has_col) {
  PRaw R; p2g_load_raw(P, f, s, R);
  PState st; p2g_unpack(R, st);
  int b[3]; float fx[3];
  if ((st.meta & 1) && has_col && collector_takes(col, st.meta, st.x)) {   // fmpm_collect(f) would have tagged it before p2g(f)
    P.pa[pa_idx(P, f, 0, s)].w = __int_as_float((st.meta & ~1) | 2);
    p2g_store_F(P, f + 1, s, st.F); return;
  }
  if (!((st.meta & 1) && base_fx(P, st.x, b, fx))) { p2g_store_F(P, f + 1, s, st.F); return; }
  const float4 mt = __ldg(P.mats + ((st.meta >> 8) & 0xff));
  Constit K; constitutive(P, st, mt.x, mt.y, mt.z, __float_as_int(mt.w), K);
  const float m = mt.z;
  float w[3][3]; bspline(fx, w);
  float B[9], q[3];
#pragma unroll
  for (int k = 0; k < 9; k++) B[k] = K.A.m[k] * P.dx;
#pragma unroll
  for (int k = 0; k < 3; k++) q[k] = m * st.v[k] - (B[k * 3] * fx[0] + B[k * 3 + 1] * fx[1] + B[k * 3 + 2] * fx[2]);
  const int n = P.n, nb = P.nb;
  for (int a = 0; a < 3; a++) for (int bb = 0; bb < 3; bb++) for (int c = 0; c < 3; c++) {
    const float wt = w[a][0] * w[bb][1] * w[c][2];
    const int gi = b[0] + a, gj = b[1] + bb, gk = b[2] + c;
    const float4 v = make_float4(wt * (q[0] + B[0] * a + B[1] * bb + B[2] * c), wt * (q[1] + B[3] * a + B[4] * bb + B[5] * c),
                                 wt * (q[2] + B[6] * a + B[7] * bb + B[8] * c), wt * m);
    red_add_v4(P.grid_pm + (gi * n + gj) * n + gk, v);
    P.blk_flags[((gi >> 3) * nb + (gj >> 3)) * nb + (gk >> 3)] = 1;
  }
  p2g_store_F(P, f + 1, s, K.Fn);
}
__global__ void k_p2g_injected(const KParams P, const int f, const FmpmInjector inj, const int act_id, const int* __restrict__ inv, const FmpmCollector col,
                               const int has_col) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= inj.flux) return;
  const int pid = ((const int*)inj.act_range)[act_id + i];
  p2g_one_particle(P, f, inv ? inv[pid] : pid, col, has_col);
}
// particles of MAT_RIGID bodies in fused steps: k_g2p2g leaves their scatter out (their position of frame f is only final after the body's
// shape matching, fmpm_advect_rigid(f-1)); this kernel adds it, after that pass and before grid_op(f)
__global__ void __launch_bounds__(128) k_p2g_rigid(const KParams P, const int f, const int* __restrict__ body_info, const int n_bodies, const FmpmCollector col,
                                                    const int has_col) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= P.N) return;
  const int meta = __float_as_int(P.pa[pa_idx(P, f, 0, s)].w);
  if (rigid_body_slot(meta, body_info, n_bodies)) p2g_one_particle(P, f, s, col, has_col);
}

// =============================================================================================
// injector act (agents/agent_injector.py:30-32 -> effectors/injector.py:80-105, 240-256)
// =============================================================================================
__device__ __forceinline__ void quat_rot(const float* q, const float* v, float* o) {  // utils/geom.py:92-97
  float uv[3] = {q[2] * v[2] - q[3] * v[1], q[3] * v[0] - q[1] * v[2], q[1] * v[1] - q[2] * v[0]};
  float uuv[3] = {q[2] * uv[2] - q[3] * uv[1], q[3] * uv[0] - q[1] * uv[2], q[1] * uv[1] - q[2] * uv[0]};
#pragma unroll
  for (int k = 0; k < 3; k++) o[k] = v[k] + 2.f * (q[0] * uv[k] + uuv[k]);
}
__global__ void k_inject(const KParams P, const int f, const FmpmInjector inj, const float* __restrict__ epos,
                         const float* __restrict__ equat, const int act_id, const int rand_row, const int* __restrict__ inv) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= inj.flux) return;
  const int pid = ((const int*)inj.act_range)[act_id + i];
  const int s = inv ? inv[pid] : pid;
  const float* rv = (const float*)inj.random_vector + ((size_t)rand_row * inj.flux + i) * 3;
  const float* pos = epos + f * 3;
  const float* quat = equat + f * 4;
  float x[3], v[3];
  if (inj.kind == 1) {
    float ipr[3]; quat_rot(quat, inj.inject_p, ipr);
#pragma unroll
    for (int k = 0; k < 3; k++) x[k] = (rv[k] * 2.f - 1.f) * inj.radius + pos[k] + ipr[k];
    quat_rot(quat, inj.inject_v, v);
    if (inj.randomize_inject_v) {   // injector.py:96-97; a constant of the pose: the adjoint (k_inject_grad) is unchanged
      const float nv2 = 2.f * sqrtf(inj.inject_v[0] * inj.inject_v[0] + inj.inject_v[1] * inj.inject_v[1] + inj.inject_v[2] * inj.inject_v[2]);
#pragma unroll
      for (int k = 0; k < 3; k++) v[k] += (rv[k] * 2.f - 1.f) * nv2;
    }
  } else {
#pragma unroll
    for (int k = 0; k < 3; k++) { x[k] = rv[k] + pos[k]; v[k] = inj.inject_v[k]; }
  }
  float4 a0 = P.pa[pa_idx(P, f + 1, 0, s)], a1 = P.pa[pa_idx(P, f + 1, 1, s)];
  const int meta = __float_as_int(a0.w) | 1;  // used[f+1, pid] = 1
  P.pa[pa_idx(P, f + 1, 0, s)] = make_float4(x[0], x[1], x[2], __int_as_float(meta));
  P.pa[pa_idx(P, f + 1, 1, s)] = make_float4(v[0], v[1], v[2], a1.w);
}

// =============================================================================================
// host entry points
// =============================================================================================
static int check_bound(FmpmHandle* h, const char* name) {
  if (!h) return 1;
  if (!h->bound) { snprintf(h->err, sizeof(h->err), "%s: fmpm_bind() has not been called", name); return 1; }
  return 0;
}
#define G2P2G_K(a, b) (k_g2p2g<a, b>)   /* a template-id with a comma cannot be a macro argument by itself */
#define G2P2G_K2(k, a, b) (k<a, b>)
#define FWD_K(a, b, c) (k_fwd<a, b, c>)
static FmpmCollector no_collector() { FmpmCollector c; memset(&c, 0, sizeof(c)); return c; }
static int check_frame(FmpmHandle* h, int f, int maxf, const char* name) {
  if (f < 0 || f > maxf) { snprintf(h->err, sizeof(h->err), "%s: frame %d out of range [0,%d]", name, f, maxf); return 1; }
  return 0;
}

extern "C" int fmpm_clear_grid(FmpmHandle* h, void* stream) {
  if (check_bound(h, "fmpm_clear_grid")) return 1;
  const size_t G = (size_t)h->cfg.n_grid * h->cfg.n_grid * h->cfg.n_grid * (h->slab.enabled ? 2 : 1);
  cudaError_t e = cudaMemsetAsync(h->buf.grid_pm, 0, G * sizeof(float4), (cudaStream_t)stream);
  if (e != cudaSuccess) { snprintf(h->err, sizeof(h->err), "fmpm_clear_grid: %s", cudaGetErrorString(e)); return 1; }
  return 0;
}

int fmpm_p2g_impl(FmpmHandle* h, int f, int write_F, int ring_slot, void* stream) {
  if (check_bound(h, "fmpm_p2g") || check_frame(h, f, h->cfg.max_substeps_local - (write_F ? 1 : 0), "fmpm_p2g")) return 1;
  KParams P = make_kparams(h, ring_slot, f);
  if (P.N == 0) return 0;
  const long long warps = ((long long)P.N + 32 * P2G_ROUNDS - 1) / (32 * P2G_ROUNDS);
  const int blocks = (int)((warps + P2G_WARPS - 1) / P2G_WARPS);
  const bool pdl = h->use_pdl != 0;
  if (h->slab.enabled && !h->slab_pull) { if (write_F) FMPM_LAUNCH_PDL(pdl, G2P2G_K2(k_p2g, true, true), blocks, P2G_WARPS * 32, 0, stream, P, f); else FMPM_LAUNCH_PDL(pdl, G2P2G_K2(k_p2g, false, true), blocks, P2G_WARPS * 32, 0, stream, P, f); }
  else { if (write_F) FMPM_LAUNCH_PDL(pdl, G2P2G_K2(k_p2g, true, false), blocks, P2G_WARPS * 32, 0, stream, P, f); else FMPM_LAUNCH_PDL(pdl, G2P2G_K2(k_p2g, false, false), blocks, P2G_WARPS * 32, 0, stream, P, f); }
  FMPM_CHECK_LAUNCH(h, "fmpm_p2g");
  return 0;
}
extern "C" int fmpm_p2g(FmpmHandle* h, int f, int write_F, void* stream) { return fmpm_p2g_impl(h, f, write_F, -1, stream); }

int fmpm_grid_op_impl(FmpmHandle* h, int f, int clear_pm, int zero_ggv, int ring_slot, void* stream) {
  if (check_bound(h, "fmpm_grid_op")) return 1;
  KParams P = make_kparams(h, ring_slot, f);
  if (!P.blk_flags) { snprintf(h->err, sizeof(h->err), "fmpm_grid_op: sparse-grid block flags were not bound"); return 1; }
  if (zero_ggv && !P.ggrid_v) { snprintf(h->err, sizeof(h->err), "fmpm_grid_op: gradient grids were not bound"); return 1; }
  const int nblk = P.nb * P.nb * P.nb;
  int grid = nblk < h->sm_count * GOP_PER_SM ? nblk : h->sm_count * GOP_PER_SM;
  if ((nblk + grid - 1) / grid > 256) grid = (nblk + 255) / 256;  // keep <= 256 blocks per CTA (parallel flag fetch)
  // the flags are consumed (reset) here only when nothing later in the substep needs them: plain forward substeps
  const int reset_flags = (clear_pm && ring_slot < 0) ? 1 : 0;
  if (h->slab_pull) {   // fmpm_substeps_slab, pull form: ghost planes read from the neighbours, the other parity's ghost blocks cleared
    const KParams Po = make_kparams(h, -1, f + 1);
    int* sig = h->slab_fsync ? (int*)h->slab.signal : nullptr;   // handshake inside the launch (fmpm_substeps_slab then skips its k_slab_sync)
    if (sig) {   // blocks that wait for a neighbour must not keep later blocks (with neighbour-independent work) off the SMs: one resident wave (78 registers x 256)
      const int resident = h->sm_count * 3;
      if (grid > resident && (nblk + resident - 1) / resident <= 256) grid = resident;
    }
    FMPM_LAUNCH(k_grid_op_pull, grid, 256, 0, stream, P, f, Po.grid_pm, Po.blk_flags, sig, sig ? (int*)h->slab.peer_signal_left : nullptr,
                sig ? (int*)h->slab.peer_signal_right : nullptr);
    FMPM_CHECK_LAUNCH(h, "fmpm_grid_op(pull)");
    return 0;
  }
#if GOP_WARP
  {
    int gridw = (nblk + 7) / 8;
    if (gridw > h->sm_count * 8) gridw = h->sm_count * 8;
    FMPM_LAUNCH_PDL(h->use_pdl != 0, k_grid_op_warp, gridw, 256, 0, stream, P, f, clear_pm, zero_ggv, reset_flags);
  }
#else
  FMPM_LAUNCH_PDL(h->use_pdl != 0, k_grid_op, grid, 256, 0, stream, P, f, clear_pm, zero_ggv, reset_flags);
#endif
  FMPM_CHECK_LAUNCH(h, "fmpm_grid_op");
  return 0;
}
extern "C" int fmpm_grid_op(FmpmHandle* h, int f, int clear_pm, void* stream) {
  return fmpm_grid_op_impl(h, f, clear_pm, 0, -1, stream);
}

int fmpm_g2p_impl(FmpmHandle* h, int f, int ring_slot, void* stream) {
  if (check_bound(h, "fmpm_g2p") || check_frame(h, f, h->cfg.max_substeps_local - 1, "fmpm_g2p")) return 1;
  KParams P = make_kparams(h, ring_slot);
  if (P.N == 0) return 0;
  FMPM_LAUNCH_PDL(h->use_pdl != 0, k_g2p, (P.N + G2P_WARPS * 32 - 1) / (G2P_WARPS * 32), G2P_WARPS * 32, 0, stream, P, f);
  FMPM_CHECK_LAUNCH(h, "fmpm_g2p");
  return 0;
}

extern "C" int fmpm_g2p(FmpmHandle* h, int f, void* stream) { return fmpm_g2p_impl(h, f, -1, stream); }

// sparse clear of a ring slot: zero the (momentum, mass) nodes of the blocks its previous occupant touched
__global__ void __launch_bounds__(256) k_clear_blocks(const KParams P) {
  const int n = P.n, nb = P.nb, nblk = nb * nb * nb;
  for (int blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
    if (P.blk_flags[blk] == 0) continue;
    const int bx = blk / (nb * nb), by = (blk / nb) % nb, bz = blk % nb;
#pragma unroll
    for (int r = 0; r < 2; r++) {
      const int t = threadIdx.x + r * 256;
      const int i = bx * 8 + (t >> 6), j = by * 8 + ((t >> 3) & 7), k = bz * 8 + (t & 7);
      P.grid_pm[(i * n + j) * n + k] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    if (threadIdx.x == 0) P.blk_flags[blk] = 0;
  }
}
extern "C" int fmpm_substep_store(FmpmHandle* h, int f, void* stream) {
  if (check_bound(h, "fmpm_substep_store")) return 1;
  if (!h->buf.grid_pm_ring || !h->buf.grid_v_ring || !h->buf.blk_list_ring) {
    snprintf(h->err, sizeof(h->err), "fmpm_substep_store: the per-frame grid ring was not bound"); return 1;
  }
  if (check_frame(h, f, h->cfg.max_substeps_local - 1, "fmpm_substep_store")) return 1;
  KParams P = make_kparams(h, f);
  const int nblk = P.nb * P.nb * P.nb;
  const int grid = nblk < h->sm_count * 8 ? nblk : h->sm_count * 8;
  FMPM_LAUNCH(k_clear_blocks, grid, 256, 0, stream, P);  // previous occupant of slot f
  FMPM_CHECK_LAUNCH(h, "fmpm_substep_store(clear)");
  if (fmpm_p2g_impl(h, f, 1, f, stream)) return 1;
  if (fmpm_grid_op_impl(h, f, 0, 0, f, stream)) return 1;
  if (fmpm_g2p_impl(h, f, f, stream)) return 1;
  return fmpm_advect_rigid_impl(h, f, stream);
}

// ---- k_fwd dispatch --------------------------------------------------------------------------------------------
enum { FWD_KFWD = 1, FWD_LIQUID = 2, FWD_INLINE = 4, FWD_TMA = 8 };
// what fmpm_substeps_fused may use for this handle: k_fwd needs an agent-free scene without MAT_RIGID bodies; the inlined grid_op also
// needs the triple-buffered accumulators, no SDF collider at grid level and no x-slab peers (their ghost exchange is per parity buffer)
static int fwd_path(const FmpmHandle* h) {
  int p = 0;
  const bool agent = (h->col.has_rigid != 0) || h->bodies.n_bodies > 0;
  if (!agent) {
    p |= FWD_KFWD;
    if (h->cfg.scene_flags & FMPM_SCENE_ALL_LIQUID_MU0) p |= FWD_LIQUID;
    if (h->tma_ok) p |= FWD_TMA;
    if (h->buf.grid_pm3 && h->buf.blk_flags3 && h->col.n_statics == 0 && !h->slab.enabled) p |= FWD_INLINE;
  }
  p &= h->fwd_mask;
  if (!(p & FWD_KFWD)) p = 0;
  return p;
}
extern "C" int fmpm_fwd_path(FmpmHandle* h) { return h ? fwd_path(h) : 0; }
extern "C" int fmpm_set_fwd_mask(FmpmHandle* h, int mask) { if (!h) return 1; h->fwd_mask = mask; return 0; }

static int fwd_launch(FmpmHandle* h, int f, int path, int full, void* stream, int tag_f0 = 0);
// g2p(f) fused with p2g(f+1): forward-only steps without agents, MAT_RIGID bodies or slabs (see k_g2p2g)
static int g2p2g_impl(FmpmHandle* h, int f, int write_vc, const FmpmCollector* col, void* stream);
extern "C" int fmpm_g2p2g(FmpmHandle* h, int f, int write_vc, void* stream) { return g2p2g_impl(h, f, write_vc, nullptr, stream); }
extern "C" int fmpm_g2p2g_collect(FmpmHandle* h, int f, int write_vc, const FmpmCollector* col, void* stream) { return g2p2g_impl(h, f, write_vc, col, stream); }
static int g2p2g_impl(FmpmHandle* h, int f, int write_vc, const FmpmCollector* col, void* stream) {
  if (check_bound(h, "fmpm_g2p2g") || check_frame(h, f, h->cfg.max_substeps_local - 2, "fmpm_g2p2g")) return 1;
  if (h->bodies.n_bodies > 0 && h->slab.enabled) { snprintf(h->err, sizeof(h->err), "fmpm_g2p2g: MAT_RIGID bodies are not available in x-slab mode"); return 1; }
  // agent-free scenes (and every x-slab scene): k_fwd, general-material instantiation with complete F planes (the callers of this phase-level
  // entry point own the step structure; the lean all-liquid frames are only used inside fmpm_substeps_fused / fmpm_substeps_slab)
  if (col == nullptr && (fwd_path(h) & FWD_KFWD)) return fwd_launch(h, f, FWD_KFWD, write_vc, stream);
  if (h->slab.enabled) { snprintf(h->err, sizeof(h->err), "fmpm_g2p2g: agents / colliders are not available in x-slab mode"); return 1; }
  KParams P = make_kparams(h, -1, f + 1);   // x-slab mode: the scatter goes to the accumulator / block flags / peers of substep parity f+1
  if (P.N == 0) return 0;
  const int blocks = (int)(((long long)P.N + 32 * P2G_WARPS - 1) / (32 * P2G_WARPS));
  const FmpmCollector c = col ? *col : no_collector();
  const int nbod = h->bodies.n_bodies; const int* binfo = nbod > 0 ? (const int*)h->bodies.info : nullptr;
  const bool agent = col != nullptr || (h->col.has_rigid && h->col.collide_type != 1) || nbod > 0;
  if (write_vc) { if (agent) FMPM_LAUNCH(G2P2G_K(true, true), blocks, P2G_WARPS * 32, 0, stream, P, f, c, col ? 1 : 0, binfo, nbod); else FMPM_LAUNCH(G2P2G_K(true, false), blocks, P2G_WARPS * 32, 0, stream, P, f, c, 0, binfo, 0); }
  else { if (agent) FMPM_LAUNCH(G2P2G_K(false, true), blocks, P2G_WARPS * 32, 0, stream, P, f, c, col ? 1 : 0, binfo, nbod); else FMPM_LAUNCH(G2P2G_K(false, false), blocks, P2G_WARPS * 32, 0, stream, P, f, c, 0, binfo, 0); }
  FMPM_CHECK_LAUNCH(h, "fmpm_g2p2g");
  return 0;
}
// the same fusion in grad mode with per-frame grids (fmpm_substep_store): g2p gathers from ring slot f, p2g scatters into ring slot f+1, and
// every frame is written completely (the backward pass reads x, v, C, F of every frame): 148 B instead of 212 B per particle and substep
static int g2p2g_store_impl(FmpmHandle* h, int f, void* stream, const FmpmCollector* col = nullptr) {
  if (check_bound(h, "fmpm_g2p2g(store)") || check_frame(h, f, h->cfg.max_substeps_local - 2, "fmpm_g2p2g(store)")) return 1;
  if (h->slab.enabled) { snprintf(h->err, sizeof(h->err), "fmpm_g2p2g(store): not available in x-slab mode"); return 1; }
  KParams P = make_kparams(h, f + 1);            // scatter target: accumulator + block flags of slot f+1
  P.grid_v = make_kparams(h, f).grid_v;          // gather source: v_out of slot f
  if (P.N == 0) return 0;
  const int blocks = (int)(((long long)P.N + 32 * P2G_WARPS - 1) / (32 * P2G_WARPS));
  const FmpmCollector c = col ? *col : no_collector();
  const int nbod = h->bodies.n_bodies; const int* binfo = nbod > 0 ? (const int*)h->bodies.info : nullptr;
  if (col != nullptr || (h->col.has_rigid && h->col.collide_type != 1) || nbod > 0) FMPM_LAUNCH(G2P2G_K(true, true), blocks, P2G_WARPS * 32, 0, stream, P, f, c, col ? 1 : 0, binfo, nbod);
  else FMPM_LAUNCH(G2P2G_K(true, false), blocks, P2G_WARPS * 32, 0, stream, P, f, c, 0, binfo, 0);
  FMPM_CHECK_LAUNCH(h, "fmpm_g2p2g(store)");
  return 0;
}
// store-mode pieces for fused steps with an injector agent (the host interleaves agent.act between them)
extern "C" int fmpm_clear_ring_slot(FmpmHandle* h, int f, void* stream) {
  if (check_bound(h, "fmpm_clear_ring_slot") || check_frame(h, f, h->cfg.max_substeps_local - 1, "fmpm_clear_ring_slot")) return 1;
  if (!h->buf.grid_pm_ring || !h->buf.blk_list_ring) { snprintf(h->err, sizeof(h->err), "fmpm_clear_ring_slot: the per-frame grid ring was not bound"); return 1; }
  KParams P = make_kparams(h, f);
  const int nblk = P.nb * P.nb * P.nb;
  const int grid = nblk < h->sm_count * 8 ? nblk : h->sm_count * 8;
  FMPM_LAUNCH(k_clear_blocks, grid, 256, 0, stream, P);
  FMPM_CHECK_LAUNCH(h, "fmpm_clear_ring_slot");
  return 0;
}
extern "C" int fmpm_g2p2g_store(FmpmHandle* h, int f, const FmpmCollector* col, void* stream) { return g2p2g_store_impl(h, f, stream, col); }
extern "C" int fmpm_p2g_store(FmpmHandle* h, int f, void* stream) { return fmpm_p2g_impl(h, f, 1, f, stream); }
extern "C" int fmpm_grid_op_store(FmpmHandle* h, int f, void* stream) { return fmpm_grid_op_impl(h, f, 0, 0, f, stream); }
extern "C" int fmpm_g2p_store(FmpmHandle* h, int f, void* stream) { return fmpm_g2p_impl(h, f, f, stream); }
extern "C" int fmpm_substeps_fused_store(FmpmHandle* h, int f0, int n, void* stream) {
  if (check_bound(h, "fmpm_substeps_fused_store")) return 1;
  if (!h->buf.grid_pm_ring || !h->buf.grid_v_ring || !h->buf.blk_list_ring) {
    snprintf(h->err, sizeof(h->err), "fmpm_substeps_fused_store: the per-frame grid ring was not bound"); return 1;
  }
  if (n < 1 || check_frame(h, f0 + n - 1, h->cfg.max_substeps_local - 1, "fmpm_substeps_fused_store")) return 1;
  const int nblk = (h->cfg.n_grid / 8) * (h->cfg.n_grid / 8) * (h->cfg.n_grid / 8);
  const int grid = nblk < h->sm_count * 8 ? nblk : h->sm_count * 8;
  for (int i = 0; i < n; i++) {
    const int f = f0 + i;
    KParams P = make_kparams(h, f);
    FMPM_LAUNCH(k_clear_blocks, grid, 256, 0, stream, P);   // previous occupant of slot f
    FMPM_CHECK_LAUNCH(h, "fmpm_substeps_fused_store(clear)");
    if (i == 0) { if (fmpm_p2g_impl(h, f, 1, f, stream)) return 1; }
    else {
      if (g2p2g_store_impl(h, f - 1, stream)) return 1;
      if (h->bodies.n_bodies > 0 && (fmpm_advect_rigid_impl(h, f - 1, stream) || fmpm_p2g_rigid(h, f, f, nullptr, stream))) return 1;
    }
    if (fmpm_grid_op_impl(h, f, 0, 0, f, stream)) return 1;
  }
  if (fmpm_g2p_impl(h, f0 + n - 1, f0 + n - 1, stream)) return 1;
  return fmpm_advect_rigid_impl(h, f0 + n - 1, stream);
}
// one k_fwd launch: g2p(f) + p2g(f+1).  acc < 0: plain accumulator / grid_v (grid_op ran before); acc >= 0: inlined grid_op, frame f lives in
// accumulator acc % 3
static int fwd_launch(FmpmHandle* h, int f, int path, int full, void* stream, int tag_f0) {
  if (check_frame(h, f, h->cfg.max_substeps_local - 2, "fmpm_substeps_fused(k_fwd)")) return 1;
  const bool inl = (path & FWD_INLINE) != 0, liq = (path & FWD_LIQUID) != 0;
  KParams P = inl ? make_kparams(h, -2 - ((f + 1) % 3)) : make_kparams(h, -1, f + 1);   // scatter target: accumulator + block flags of frame f+1
  float4* clr = nullptr; int* clr_flags = nullptr; const float4* pms = nullptr;
  if (inl) {
    const KParams Ps = make_kparams(h, -2 - (f % 3)), Pc = make_kparams(h, -2 - ((f + 2) % 3));
    pms = Ps.grid_pm;   // the (momentum, mass) accumulator of frame f; P.grid_v is the tagged v_out cache
    clr = Pc.grid_pm; clr_flags = Pc.blk_flags;
  }
  if (P.N == 0) return 0;
  int blocks = (int)(((long long)P.N + 32 * FWD_WARPS - 1) / (32 * FWD_WARPS));
#if FWD_PERSIST
  if (!inl && (liq || FWD_PERSIST >= 2)) {   // persistent warps: one resident set of CTAs, chunks claimed from P.blk_list[0] (a reserved, zero-initialised buffer of FmpmBuffers)
    if (!P.blk_list) { snprintf(h->err, sizeof(h->err), "fmpm_substeps_fused(k_fwd): blk_list (the chunk counter of the persistent kernel) was not bound"); return 1; }
    const int resident = h->sm_count * FWD_MINB;
    if (blocks > resident) blocks = resident;
  }
#endif
  int stride = 1;   // CTA -> slot-block permutation (lazy grid_op): an odd prime that does not divide the grid size
  if (inl && h->fwd_stride != 1) {
    static const int primes[] = {1021, 1031, 2053, 509, 257};
    for (int k = 0; k < 5 && stride == 1; k++) if (blocks > primes[k] && blocks % primes[k] != 0 && (long long)blocks * primes[k] < (1LL << 32)) stride = primes[k];
  }
  const int tag_off = f - tag_f0;
  FwdFrames FR;   // frame f / f+1 of the state planes, frame f+1 / f+2 of F
  {
    const size_t Ns = (size_t)P.N;
    FR.pa_f = P.pa + (size_t)f * 4 * Ns; FR.pa_n = FR.pa_f + 4 * Ns;
    FR.pf_r = P.pf + (size_t)(f + 1) * 2 * Ns; FR.pf_w = FR.pf_r + 2 * Ns;
    FR.p8_r = P.pf8 + (size_t)(f + 1) * Ns; FR.p8_w = FR.p8_r + Ns;
  }
  const bool slab = h->slab.enabled != 0 && !h->slab_pull;   // (never together with the inlined grid_op, see fwd_path; pull form: local scatter)
  const int use_tma = (h->tma_ok && (path & FWD_TMA) && !inl) ? 1 : 0;
#define FWD_GO(a, b, c) FMPM_LAUNCH_PDL(h->use_pdl != 0, FWD_K(a, b, c), blocks, FWD_WARPS * 32, 0, stream, P, FR, f, clr, clr_flags, full, pms, tag_off, stride, h->tm_gv8, h->tm_gv16, use_tma)
  if (liq) { if (inl) FWD_GO(1, true, false); else if (slab) FWD_GO(1, false, true); else FWD_GO(1, false, false); }
  else { if (inl) FWD_GO(0, true, false); else if (slab) FWD_GO(0, false, true); else FWD_GO(0, false, false); }
#undef FWD_GO
  FMPM_CHECK_LAUNCH(h, "fmpm_substeps_fused(k_fwd)");
  return 0;
}
// one fused substep (g2p(f) + p2g(f+1)) with whatever the scene allows short of the inlined grid_op: x-slab steps (fmpm_substeps_slab)
int fmpm_fwd_step_impl(FmpmHandle* h, int f, int full, void* stream) {
  if (check_bound(h, "fmpm_fwd_step")) return 1;
  const int path = fwd_path(h) & ~FWD_INLINE;
  if (path & FWD_KFWD) return fwd_launch(h, f, path, full, stream);
  return fmpm_g2p2g(h, f, 0, stream);
}
extern "C" int fmpm_fwd_step(FmpmHandle* h, int f, int full, void* stream) { return fmpm_fwd_step_impl(h, f, full, stream); }
int fmpm_clear_blocks_launch(FmpmHandle* h, const KParams& P, void* stream) {
  const int nblk = P.nb * P.nb * P.nb;
  const int grid = nblk < h->sm_count * 8 ? nblk : h->sm_count * 8;
  FMPM_LAUNCH(k_clear_blocks, grid, 256, 0, stream, P);
  FMPM_CHECK_LAUNCH(h, "fmpm_substeps_fused(clear)");
  return 0;
}
// n forward substeps f0 .. f0+n-1 with the inner g2p / p2g pairs fused.  Frames f0 and f0+n are complete; the frames in between hold x, used
// and F only (all-liquid scenes: x, used and F22).  The grid must be clear on entry (as for fmpm_substep) and is clear on return.
//   round-1 path            p2g(f0), [grid_op, k_g2p2g] x (n-1), grid_op, g2p(f0+n-1)
//   k_fwd                   p2g(f0), [grid_op, k_fwd]   x (n-1), grid_op, g2p(f0+n-1)
//   k_fwd + inlined grid_op p2g(f0), k_fwd x (n-1), grid_op, clear, g2p(f0+n-1)          (accumulators f % 3)
extern "C" int fmpm_substeps_fused(FmpmHandle* h, int f0, int n, void* stream) {
  if (n < 1) { if (h) snprintf(h->err, sizeof(h->err), "fmpm_substeps_fused: n must be >= 1"); return 1; }
  if (check_bound(h, "fmpm_substeps_fused")) return 1;
  const int path = fwd_path(h);
  if (path & FWD_INLINE) {
    if (fmpm_p2g_impl(h, f0, 1, -2 - (f0 % 3), stream)) return 1;
    for (int i = 0; i + 1 < n; i++)
      if (fwd_launch(h, f0 + i, path, i + 2 == n, stream, f0)) return 1;
    const int fl = f0 + n - 1;
    if (fmpm_grid_op_impl(h, fl, 1, 0, -2 - (fl % 3), stream)) return 1;        // consumes and clears the accumulator of the last frame
    if (n >= 2 && fmpm_clear_blocks_launch(h, make_kparams(h, -2 - ((fl + 2) % 3)), stream)) return 1;   // the one the last k_fwd gathered from
    return fmpm_g2p(h, fl, stream);
  }
  if (fmpm_p2g(h, f0, 1, stream)) return 1;
  for (int i = 0; i + 1 < n; i++) {
    if (fmpm_grid_op(h, f0 + i, 1, stream)) return 1;
    if (path & FWD_KFWD) { if (fwd_launch(h, f0 + i, path, i + 2 == n, stream)) return 1; }
    else if (fmpm_g2p2g(h, f0 + i, 0, stream)) return 1;
    if (h->bodies.n_bodies > 0 && (fmpm_advect_rigid_impl(h, f0 + i, stream) || fmpm_p2g_rigid(h, f0 + i + 1, -1, nullptr, stream))) return 1;
  }
  if (fmpm_grid_op(h, f0 + n - 1, 1, stream) || fmpm_g2p(h, f0 + n - 1, stream)) return 1;
  return fmpm_advect_rigid_impl(h, f0 + n - 1, stream);
}

extern "C" int fmpm_substep(FmpmHandle* h, int f, void* stream) {
  if (fmpm_p2g(h, f, 1, stream)) return 1;
  if (fmpm_grid_op(h, f, 1, stream)) return 1;
  if (fmpm_g2p(h, f, stream)) return 1;
  return fmpm_advect_rigid_impl(h, f, stream);
}

// collector_act_kernel (agents/agent_pouring.py:31-41, agents/agent_jetbot.py:30-40)
__global__ void k_collect(const KParams P, const int f, const FmpmCollector c) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= P.N) return;
  const float4 a0 = P.pa[pa_idx(P, f, 0, s)];
  const int meta = __float_as_int(a0.w);
  const int row = (meta >> 8) & 0xff;
  if (!(meta & 1) || row >= 32 || !((c.row_mask >> row) & 1u)) return;
  bool out = false;
  if (c.boundary_type == 0) {   // boundaries.py:128-134
    out = a0.x > c.upper[0] || a0.y > c.upper[1] || a0.z > c.upper[2] || a0.x < c.lower[0] || a0.y < c.lower[1] || a0.z < c.lower[2];
  } else {                      // boundaries.py:81-93
    out = a0.y > c.upper[1] || a0.y < c.lower[1];
    const float rx = a0.x - c.cyl_center[0], rz = a0.z - c.cyl_center[1];
    out = out || sqrtf(rx * rx + rz * rz + FMPM_EPS) > c.cyl_radius;
  }
  if (out) P.pa[pa_idx(P, f, 0, s)].w = __int_as_float((meta & ~1) | 2);
}
extern "C" int fmpm_collect(FmpmHandle* h, int f, const FmpmCollector* c, void* stream) {
  if (check_bound(h, "fmpm_collect") || check_frame(h, f, h->cfg.max_substeps_local - 1, "fmpm_collect")) return 1;
  if (!c) { snprintf(h->err, sizeof(h->err), "fmpm_collect: null collector"); return 1; }
  KParams P = make_kparams(h);
  if (P.N == 0) return 0;
  FMPM_LAUNCH(k_collect, (P.N + 255) / 256, 256, 0, stream, P, f, *c);
  FMPM_CHECK_LAUNCH(h, "fmpm_collect");
  return 0;
}

// fused steps with an injector agent: scatter the particles that fmpm_inject(f-1, ...) has just activated in frame f (act_id = the injector's
// counter BEFORE that injection).  Call after fmpm_g2p2g(f-1) + fmpm_inject(f-1) and before fmpm_grid_op(f).
extern "C" int fmpm_p2g_injected(FmpmHandle* h, int f, const FmpmInjector* inj, int act_id, const void* inv, int ring_slot, const FmpmCollector* col, void* stream) {
  if (check_bound(h, "fmpm_p2g_injected") || check_frame(h, f, h->cfg.max_substeps_local - 1, "fmpm_p2g_injected")) return 1;
  if (!inj || act_id < 0 || act_id + inj->flux > inj->n_act_range) { snprintf(h->err, sizeof(h->err), "fmpm_p2g_injected: bad injector range"); return 1; }
  if (h->slab.enabled) { snprintf(h->err, sizeof(h->err), "fmpm_p2g_injected: not available in x-slab mode"); return 1; }
  KParams P = make_kparams(h, ring_slot);   // ring_slot >= 0: the accumulator / block flags of that slot of the per-frame ring (grad mode)
  FMPM_LAUNCH(k_p2g_injected, (inj->flux + 31) / 32, 32, 0, stream, P, f, *inj, act_id, (const int*)inv, col ? *col : no_collector(), col ? 1 : 0);
  FMPM_CHECK_LAUNCH(h, "fmpm_p2g_injected");
  return 0;
}
// fused steps with MAT_RIGID bodies: scatter their particles of frame f (after fmpm_advect_rigid(f-1) fixed their positions), before fmpm_grid_op(f)
extern "C" int fmpm_p2g_rigid(FmpmHandle* h, int f, int ring_slot, const FmpmCollector* col, void* stream) {
  if (check_bound(h, "fmpm_p2g_rigid") || check_frame(h, f, h->cfg.max_substeps_local - 1, "fmpm_p2g_rigid")) return 1;
  if (h->bodies.n_bodies == 0) return 0;
  KParams P = make_kparams(h, ring_slot);
  if (P.N == 0) return 0;
  FMPM_LAUNCH(k_p2g_rigid, (P.N + 127) / 128, 128, 0, stream, P, f, (const int*)h->bodies.info, h->bodies.n_bodies, col ? *col : no_collector(), col ? 1 : 0);
  FMPM_CHECK_LAUNCH(h, "fmpm_p2g_rigid");
  return 0;
}
extern "C" int fmpm_inject(FmpmHandle* h, int f, const FmpmInjector* inj, const FmpmEffector* e, int act_id, int rand_row,
                           const void* inv, void* stream) {
  if (check_bound(h, "fmpm_inject") || check_frame(h, f, h->cfg.max_substeps_local - 1, "fmpm_inject")) return 1;
  if (act_id < 0 || act_id + inj->flux > inj->n_act_range) {
    snprintf(h->err, sizeof(h->err), "fmpm_inject: too many particles added (act_id %d + flux %d > %d)", act_id, inj->flux, inj->n_act_range);
    return 2;
  }
  KParams P = make_kparams(h);
  FMPM_LAUNCH(k_inject, (inj->flux + 31) / 32, 32, 0, stream, P, f, *inj, (const float*)e->pos, (const float*)e->quat, act_id, rand_row, (const int*)inv);
  FMPM_CHECK_LAUNCH(h, "fmpm_inject");
  return 0;
}
