// fmpm_backward.cu — adjoint of the MLS-MPM substep for sm_90a (H100).
//
// Reference semantics: MPMSimulator.substep_grad (MPM:535-552): advect_kernel.grad, g2p.grad, grid_op.grad,
// p2g.grad, svd_grad (manual, MPM:266-302), compute_F_tmp.grad, process_unused_particles.grad — the
// Taichi-autodiff generated parts are restated by hand (SURVEY.md Appendix A; validated against finite
// differences through the oracle).  The reference stores F_tmp/U/S/V and a grid per frame; here the forward
// grid of frame f is recomputed (fmpm_p2g(write_F=0) + fmpm_grid_op(clear=0)) and the constitutive scratch
// is recomputed in registers, so the backward reads only the 100 B/particle state ring.
//
// Kernels:
//   k_g2p_grad_scatter : v_out adjoint scatter (same register sliding-window + REDG.F32x4 as p2g)
//   k_grid_op_grad     : per node (v_in, mass) adjoint
//   k_particle_grad    : everything per particle: gathers v_out and the (v_in, mass) adjoint on the 27 nodes,
//                        writes the frame-f adjoint planes once (no read-modify-write, no zeroing).
#include <cstdio>
#include "fmpm_common.cuh"

#include "fmpm_scatter.cuh"
#include "fmpm_sdf.cuh"

#define SC_WARPS 4
#ifndef SC_AHEAD
#define SC_AHEAD 0   // > 0: L2 prefetch of the first plane of the CTA SC_AHEAD CTAs further on
#endif
#ifndef SC_ROUNDS
#define SC_ROUNDS 4   // 32-particle rounds per warp (1 / 2 / 4 can be compared with profiles/ab_variants.sh)
#endif

#ifndef BWD_PREFETCH
#define BWD_PREFETCH 1   // L2 prefetch of the planes k_particle_grad reads late (the adjoint of frame f+1, F): at 128 registers few warps are resident, the kernel
                         // is bound by long-scoreboard stalls and issues its second batch of loads only after the footprint staging; k_g2p_grad_scatter has no such prefetch
                         // (it costs that kernel registers)
#endif
// one 128-byte line per 8 lanes of a float4 plane (the warp's 32 slots are 512 contiguous bytes), lane 0 for a float plane (prefetch_l2: fmpm_common.cuh)
__device__ __forceinline__ void prefetch_planes4(const float4* base, const KParams& P, const int g, const int nplanes, const int s) {
  if (BWD_PREFETCH && (threadIdx.x & 7) == 0)
    for (int k = 0; k < nplanes; k++) prefetch_l2(base + ((size_t)g * nplanes + k) * (size_t)P.N + s);
}
__device__ __forceinline__ void prefetch_plane1(const float* base, const KParams& P, const int g, const int s) {
  if (BWD_PREFETCH && (threadIdx.x & 31) == 0) prefetch_l2(base + (size_t)g * (size_t)P.N + s);
}
// grads in a ping-pong buffer g (0/1): same planar layout as the state ring with frame index g
struct GState { float x[3], v[3]; Mat3 C, F; };
__device__ __forceinline__ void load_grad(const KParams& P, int g, int s, GState& G) {
  PState t; load_A(P.ga, P, g, s, t);
  G.x[0] = t.x[0]; G.x[1] = t.x[1]; G.x[2] = t.x[2]; G.v[0] = t.v[0]; G.v[1] = t.v[1]; G.v[2] = t.v[2]; G.C = t.C;
  load_F(P.gf, P.gf8, P, g, s, G.F);
}

// =============================================================================================
// g2p.grad, grid side:  gv_out[i] += w_i * (gv + 4 inv_dx * gC' (o - fx)),  gv = gv' + dt * gx'
// =============================================================================================
template <bool kSlab>
__global__ void __launch_bounds__(SC_WARPS * 32) k_g2p_grad_scatter(const KParams P, const int f, const int gin) {
  __shared__ ScatterSmem smem[SC_WARPS];
  const int lane = threadIdx.x & 31, wib = __shfl_sync(SC_FULL, (int)(threadIdx.x >> 5), 0);   // broadcast: dependent code is compiled warp-uniform
  ScatterSmem& S = smem[wib];
  const long long gw = (long long)blockIdx.x * SC_WARPS + wib;
  const long long slot0 = gw * (32 * SC_ROUNDS);
  if (slot0 >= P.N) return;
  Window W; window_init(W, lane, P.n, nullptr);
  if (kSlab) window_set_slab(W, P.peer_gl, P.peer_gr, P.gl_lo, P.gl_hi, P.gr_lo, P.gr_hi, nullptr, nullptr);   // x-slab backward: ghost planes also go to the neighbour
#pragma unroll 1
  for (int r = 0; r < SC_ROUNDS; r++) {
    const long long rem = (long long)P.N - (slot0 + r * 32);
    if (rem <= 0) break;
    const int cnt = rem < 32 ? (int)rem : 32;
    const long long sl = slot0 + r * 32 + lane;
    int key = -1;
    float q[3] = {0.f, 0.f, 0.f}, B[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float w[3][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    if (sl < P.N) {
      const int s = (int)sl;
#if SC_AHEAD > 0
      if (r == 0 && sl + (long long)SC_AHEAD * SC_WARPS * 32 * SC_ROUNDS < P.N && (threadIdx.x & 7) == 0)
        prefetch_l2(P.pa + pa_idx(P, f, 0, s + SC_AHEAD * SC_WARPS * 32 * SC_ROUNDS));
#endif
      const float4 a0 = P.pa[pa_idx(P, f, 0, s)];
      const float x[3] = {a0.x, a0.y, a0.z};
      int b[3]; float fx[3];
      if ((__float_as_int(a0.w) & 1) && base_fx(P, x, b, fx)) {
        PState g; load_A(P.ga, P, gin, s, g);  // (gx', gv', gC')
        const float c4 = 4.f * P.inv_dx;
#pragma unroll
        for (int i = 0; i < 9; i++) B[i] = c4 * g.C.m[i];
#pragma unroll
        for (int i = 0; i < 3; i++) q[i] = (g.v[i] + P.dt * g.x[i]) - (B[i * 3] * fx[0] + B[i * 3 + 1] * fx[1] + B[i * 3 + 2] * fx[2]);
        bspline(fx, w);
        key = pack_key(b);
      }
    }
    const unsigned starts = scatter_publish(S, lane, key, W.cur_key, q, B, 0.f, w);
    __syncwarp();
    window_consume2<kSlab>(W, S, cnt, starts, P.ggrid_v);
    __syncwarp();
  }
  window_flush_all2<kSlab>(W, P.ggrid_v);
}

// =============================================================================================
// grid_op.grad (MPM:539): v_out = B(v_in / m + dt g)
// kPG: also dL/dg = dt * sum over nodes with mass of the adjoint of v_in / m + dt g (vb after the collider chain), one fp64 atomic per CTA
// and component; while P.pg_contact is bound also the contact-parameter gradients of the collider chain and the walls (FmpmContactGrad)
// =============================================================================================
template <bool kPG>
__global__ void __launch_bounds__(256) k_grid_op_grad(const KParams P, const int f, const int clear_pm, const int zero_ggv_after) {
  const int n = P.n, nb = P.nb, nblk = nb * nb * nb;
  float gsum[3] = {0.f, 0.f, 0.f};   // kPG only
  float csum[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};   // kPG only: FmpmContactGrad components 0..6
  for (int blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
    if (P.blk_flags[blk] == 0) continue;  // CTA-uniform
    const int bx = blk / (nb * nb), by = (blk / nb) % nb, bz = blk % nb;
#pragma unroll
    for (int r = 0; r < 2; r++) {
      const int t = threadIdx.x + r * 256;
      const int i = bx * 8 + (t >> 6), j = by * 8 + ((t >> 3) & 7), k = bz * 8 + (t & 7);
      const int g = (i * n + j) * n + k;
      const float4 pm = P.grid_pm[g];
      float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
      float pg0[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, pg1[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // effector pose adjoint of this node (grid-level agent collide)
      const bool agent_grid = P.col.has_rigid && P.col.collide_type >= 1;
      if (pm.w > FMPM_EPS) {
        const float inv_m = 1.f / pm.w;
        float v[3] = {inv_m * pm.x + P.dt * P.gx, inv_m * pm.y + P.dt * P.gy, inv_m * pm.z + P.dt * P.gz};
        const float pos[3] = {(float)i * P.dx, (float)j * P.dx, (float)k * P.dx};
        // forward chain statics -> agent -> boundary with the intermediate velocities kept (MPM:388-398)
        float vc[5][3];
        vc[0][0] = v[0]; vc[0][1] = v[1]; vc[0][2] = v[2];
#pragma unroll
        for (int si = 0; si < 4; si++) {
          if (si < P.col.n_statics) sdf_collide<false>(P.col.statics[si], false, nullptr, nullptr, nullptr, nullptr, P.dt, pos, vc[si], vc[si + 1], nullptr, nullptr, nullptr, nullptr, nullptr);
          else { vc[si + 1][0] = vc[si][0]; vc[si + 1][1] = vc[si][1]; vc[si + 1][2] = vc[si][2]; }
        }
        float vl[3] = {vc[4][0], vc[4][1], vc[4][2]};
        if (agent_grid) agent_collide<false>(P, f, pos, vc[4], vl, nullptr, nullptr, nullptr, nullptr, nullptr);
        float fac[3];
        float vw[3]; int hit;   // kPG: the velocity entering the walls and the axes they reflect
        if constexpr (kPG) { vw[0] = vl[0]; vw[1] = vl[1]; vw[2] = vl[2]; }
        boundary_v<kPG>(P, pos, vl, fac, &hit);
        const float4 gv = P.ggrid_v[g];
        if constexpr (kPG) {
          if (hit & 1) csum[6] -= vw[0] * gv.x;
          if (hit & 2) csum[6] -= vw[1] * gv.y;
          if (hit & 4) csum[6] -= vw[2] * gv.z;
        }
        float vb[3] = {gv.x * fac[0], gv.y * fac[1], gv.z * fac[2]};
        if (agent_grid) {
          float o[3], gvv[3] = {0.f, 0.f, 0.f}, gpp[3] = {0.f, 0.f, 0.f};  // node positions are constants: gpp is dropped
          agent_collide<true, kPG>(P, f, pos, vc[4], o, vb, gvv, gpp, pg0, pg1, csum + 4);
          vb[0] = gvv[0]; vb[1] = gvv[1]; vb[2] = gvv[2];
        }
#pragma unroll
        for (int si = 3; si >= 0; si--) {
          if (si < P.col.n_statics) {
            float o[3], gvv[3] = {0.f, 0.f, 0.f}, gpp[3] = {0.f, 0.f, 0.f}, d0[3] = {0.f, 0.f, 0.f}, d1[3] = {0.f, 0.f, 0.f};
            // a static mesh writes gparam[0] (friction) only: softness is a dynamic-mesh parameter
            sdf_collide<true, kPG>(P.col.statics[si], false, nullptr, nullptr, nullptr, nullptr, P.dt, pos, vc[si], o, vb, gvv, gpp, d0, d1, csum + si);
            vb[0] = gvv[0]; vb[1] = gvv[1]; vb[2] = gvv[2];
          }
        }
        if constexpr (kPG) { gsum[0] += vb[0]; gsum[1] += vb[1]; gsum[2] += vb[2]; }
        out.x = vb[0] * inv_m; out.y = vb[1] * inv_m; out.z = vb[2] * inv_m;
        out.w = -(pm.x * vb[0] + pm.y * vb[1] + pm.z * vb[2]) * inv_m * inv_m;
      }
      if (agent_grid && P.col.egpos) reduce_pose_grad(P.col.egpos, P.col.egquat, f, pg0, pg1);
      P.ggrid_pm[g] = out;
      if (zero_ggv_after) P.ggrid_v[g] = make_float4(0.f, 0.f, 0.f, 0.f);   // consumed: all-zero again before any neighbour's next scatter
      if (clear_pm && (pm.w != 0.f || pm.x != 0.f || pm.y != 0.f || pm.z != 0.f)) P.grid_pm[g] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (clear_pm) { __syncthreads(); if (threadIdx.x == 0) P.blk_flags[blk] = 0; }  // recompute path: last consumer of the flags
  }
  if constexpr (kPG) {   // every thread of the CTA gets here (the block loop is CTA-uniform)
    __shared__ float red[10][8];   // gravity 0..2, then the contact components 0..6
#pragma unroll
    for (int c = 0; c < 3; c++) {
      float v = gsum[c];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if ((threadIdx.x & 31) == 0) red[c][threadIdx.x >> 5] = v;
    }
    if (P.pg_contact) {   // kernel-uniform
#pragma unroll
      for (int c = 0; c < 7; c++) {
        float v = csum[c];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) red[3 + c][threadIdx.x >> 5] = v;
      }
    }
    __syncthreads();
    if (threadIdx.x < 3) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < 8; w++) v += red[threadIdx.x][w];
      if (v != 0.f) atomic_add_f64(P.pg_grav + threadIdx.x, (double)P.dt * (double)v);
    } else if (threadIdx.x < 10 && P.pg_contact) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < 8; w++) v += red[threadIdx.x][w];
      if (v != 0.f) atomic_add_f64(P.pg_contact + (threadIdx.x - 3), (double)v);
    }
  }
}

// =============================================================================================
// agent.collide(f, x + dt v', v', dt).grad at particle level (MPM:419-422 inside g2p.grad): pre-pass that rewrites the
// frame-(f+1) adjoint in place so that the two kernels below see the adjoint of the PRE-collision v' and of x_tmp:
//   gx' <- gx' + gxt ,  gv' <- gvpre - dt * gx'     (then gv'+dt*gx' = gvpre + dt*gxt, as the chain rule requires)
// kPG: also dL/d(rigid friction, rigid softness), reduced over the block: one fp64 atomic per block and component into P.pg_contact[4..5]
// =============================================================================================
template <bool kPG>
__global__ void __launch_bounds__(128) k_collide_particle_grad(const KParams P, const int f, const int gin) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  float g0[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, g1[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float gfs[2] = {0.f, 0.f};   // kPG only
  if (s < P.N) {
    const float4 a0 = P.pa[pa_idx(P, f, 0, s)];
    const float x[3] = {a0.x, a0.y, a0.z};
    int b[3]; float fx[3];
    if ((__float_as_int(a0.w) & 1) && base_fx(P, x, b, fx)) {
      float w[3][3]; bspline(fx, w);
      float nv[3]; Mat3 nC;
      const float4* gvp = P.grid_v + ((b[0] * P.n + b[1]) * P.n + b[2]);
      const int n = P.n;
      g2p_gather(fx, w, [&](int c) { return gvp + ((c / 3) * n + (c % 3)) * n; }, nv, nC, 4.f * P.inv_dx);
      float4 gx4 = P.ga[pa_idx(P, gin, 0, s)], gv4 = P.ga[pa_idx(P, gin, 1, s)];
      const float gout[3] = {gv4.x + P.dt * gx4.x, gv4.y + P.dt * gx4.y, gv4.z + P.dt * gx4.z};
      const float xt[3] = {x[0] + P.dt * nv[0], x[1] + P.dt * nv[1], x[2] + P.dt * nv[2]};
      float o[3], gvpre[3] = {0.f, 0.f, 0.f}, gxt[3] = {0.f, 0.f, 0.f};
      agent_collide<true, kPG>(P, f, xt, nv, o, gout, gvpre, gxt, g0, g1, gfs);
      gv4.x = gvpre[0] - P.dt * gx4.x; gv4.y = gvpre[1] - P.dt * gx4.y; gv4.z = gvpre[2] - P.dt * gx4.z;
      gx4.x += gxt[0]; gx4.y += gxt[1]; gx4.z += gxt[2];
      P.ga[pa_idx(P, gin, 0, s)] = gx4; P.ga[pa_idx(P, gin, 1, s)] = gv4;
    }
  }
  if (P.col.egpos) reduce_pose_grad(P.col.egpos, P.col.egquat, f, g0, g1);
  if constexpr (kPG) {   // no thread has returned: the particle test above is an if
    __shared__ float red[2][4];
#pragma unroll
    for (int c = 0; c < 2; c++) {
      float v = gfs[c];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if ((threadIdx.x & 31) == 0) red[c][threadIdx.x >> 5] = v;
    }
    __syncthreads();
    if (threadIdx.x < 2) {
      const float v = red[threadIdx.x][0] + red[threadIdx.x][1] + red[threadIdx.x][2] + red[threadIdx.x][3];
      if (v != 0.f) atomic_add_f64(P.pg_contact + 4 + threadIdx.x, (double)v);
    }
  }
}

// =============================================================================================
// per-particle adjoint
// =============================================================================================
__device__ __forceinline__ float clamp_svd(float a) { return a >= 0.f ? fmaxf(a, 1e-8f) : fminf(a, -1e-8f); }  // MPM:294-302

// adjoint of the constitutive block: given gA (adjoint of `affine`, MPM:344) and gFn (adjoint of F[f+1]),
// returns gFt (adjoint of F_tmp) — p2g.grad constitutive part + svd_grad (MPM:266-292) in a numerically
// stable factored form (identical to the reference formula in exact arithmetic, including its clamp).
__device__ __forceinline__ Mat3 constitutive_grad(const KParams& P, const Constit& K, float mu, float lam, int cls, const Mat3& gA, const Mat3& gFn) {
  Mat3 gP = m3_scale(gA, P.k_stress);
  const float trP = m3_trace(gP);
  float gJ = lam * (2.f * K.J - 1.f) * trP;
  const bool plastic = (cls == FMPM_MAT_PLASTO_ELASTIC) || (cls == FMPM_MAT_PLASTO_ELASTIC_DEMO);
  if (cls == FMPM_MAT_LIQUID) {
    // F_new = I * J^(1/3):  dJ += (1/3) J^(-2/3) tr(gFn)
    const float cb = cbrtf(K.J);
    gJ += (1.f / 3.f) * (cb / K.J) * m3_trace(gFn);
  }
  Mat3 gFt;
  if (!K.need_svd) {
    // J = det(F_tmp): gFt = gJ * cof(F_tmp)
    const float* a = K.Ft.m;
    gFt.m[0] = gJ * (a[4] * a[8] - a[5] * a[7]); gFt.m[1] = gJ * (a[5] * a[6] - a[3] * a[8]); gFt.m[2] = gJ * (a[3] * a[7] - a[4] * a[6]);
    gFt.m[3] = gJ * (a[2] * a[7] - a[1] * a[8]); gFt.m[4] = gJ * (a[0] * a[8] - a[2] * a[6]); gFt.m[5] = gJ * (a[1] * a[6] - a[0] * a[7]);
    gFt.m[6] = gJ * (a[1] * a[5] - a[2] * a[4]); gFt.m[7] = gJ * (a[2] * a[3] - a[0] * a[5]); gFt.m[8] = gJ * (a[0] * a[4] - a[1] * a[3]);
    if (cls == FMPM_MAT_ELASTIC || cls == FMPM_MAT_RIGID) gFt = m3_add(gFt, gFn);
    return gFt;
  }
  const float* s = K.sig;
  Mat3 R = m3_mul_nt(K.U, K.V);
  Mat3 M = m3_sub(K.Ft, R);
  Mat3 gM = m3_scale(m3_mul(gP, K.Ft), 2.f * mu);                      // M̄ = 2μ P̄ F̃
  gFt = m3_add(gM, m3_scale(m3_mul_tn(gP, M), 2.f * mu));              // F̃̄ = M̄ + 2μ P̄ᵀ M
  if (cls == FMPM_MAT_ELASTIC || cls == FMPM_MAT_RIGID) gFt = m3_add(gFt, gFn);
  // R̄ = -M̄ ;  Rr = Uᵀ R̄ V
  Mat3 Rr = m3_scale(m3_mul(m3_mul_tn(K.U, gM), K.V), -1.f);
  Mat3 Wp = m3_zero();
  float sp[3] = {s[0], s[1], s[2]}; float pass[3] = {1.f, 1.f, 1.f};
  if (plastic) {
    Wp = m3_mul(m3_mul_tn(K.U, gFn), K.V);                             // W = Uᵀ F̄' V
#pragma unroll
    for (int d = 0; d < 3; d++) {
      const float lo = 0.998f, hi = 1.003f;
      const float mx = fmaxf(s[d], lo); const bool p1 = lo < s[d];
      const float mn = fminf(mx, hi);   const bool p2 = mx < hi;
      sp[d] = mn; pass[d] = (p1 && p2) ? 1.f : 0.f;
    }
  }
  Mat3 Z;
  Z.m[0] = gJ * s[1] * s[2] + (plastic ? Wp.m[0] * pass[0] : 0.f);
  Z.m[4] = gJ * s[0] * s[2] + (plastic ? Wp.m[4] * pass[1] : 0.f);
  Z.m[8] = gJ * s[0] * s[1] + (plastic ? Wp.m[8] * pass[2] : 0.f);
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) {
      if (i == j) continue;
      const float d = s[j] * s[j] - s[i] * s[i];
      const bool regular = fabsf(d) >= 1e-8f;
      const float kc = 1.f / clamp_svd(d);                 // reference K_ij
      const float inv_sum = regular ? 1.f / (s[i] + s[j]) : (s[j] - s[i]) * kc;   // (σj-σi)/clamp(σj²-σi²)
      float z = (Rr.m[i * 3 + j] - Rr.m[j * 3 + i]) * inv_sum;
      if (plastic) {
        const float wij = Wp.m[i * 3 + j], wji = Wp.m[j * 3 + i];
        const bool ci = pass[i] == 0.f, cj = pass[j] == 0.f;
        if (!ci && !cj) z += wij * (regular ? 1.f : d * kc);
        else if (ci && cj && sp[i] == sp[j]) z += sp[i] * (wij - wji) * inv_sum;
        else z += (wij * (sp[j] * s[j] - sp[i] * s[i]) + wji * (s[i] * sp[j] - sp[i] * s[j])) * kc;
      }
      Z.m[i * 3 + j] = z;
    }
  gFt = m3_add(gFt, m3_mul_nt(m3_mul(K.U, Z), K.V));
  return gFt;
}

#define PG_WARPS 4
#ifndef PG_AHEAD
#define PG_AHEAD 0   // > 0: L2 prefetch of the state planes of the CTA PG_AHEAD CTAs further on (one resident wave ahead: SMs x 4)
#endif
#ifndef PG_MINB_LIQUID
#define PG_MINB_LIQUID 4   // all-liquid instantiation: <= 128 registers (16 warps/SM)
#endif
#ifndef PG_MINB
#define PG_MINB 4   // <= 128 registers (16 warps/SM) at the price of a few hundred bytes of L1-resident spills
#endif

// Adjoint gather on the 27 stencil nodes, column-factored.  With g_i = v_out (forward), a_i = adjoint of v_in, am_i = adjoint
// of mass, delta_i = o_i - fx, Mg = 4 inv_dx gC', Ma = A dx:
//   vp    = sum w g                      (the forward v')
//   gvp   = sum w a ,  S_ao = sum w a (x) o
//   gfx   = -Mg^T vp - Ma^T gvp + sum_i s_i grad(w_i),   s_i = g_i.(gve + Mg delta_i) + a_i.(m v + Ma delta_i) + m am_i
// (SURVEY.md Appendix A g2p.grad + p2g.grad particle side, regrouped so the z-direction is reduced first.)
// kPG: also s_am = sum_i w_i am_i (the mass-adjoint term of dL/dmass)
template <bool kPG, class ColG, class ColA>
__device__ __forceinline__ void adjoint_gather(const float* fx, const float w[3][3], const float dw[3][3], ColG colg, ColA cola,
                                               const float* gve, const Mat3& Mg, const float* mv, const Mat3& Ma, const float m,
                                               float* vp, float* gvp, Mat3& S_ao, float* gfx, float& s_am) {
  float a0[3], b0[3];  // coefficient bases: alpha0 = gve - Mg fx, beta0 = m v - Ma fx
#pragma unroll
  for (int r = 0; r < 3; r++) {
    a0[r] = gve[r] - (Mg.m[r * 3] * fx[0] + Mg.m[r * 3 + 1] * fx[1] + Mg.m[r * 3 + 2] * fx[2]);
    b0[r] = mv[r] - (Ma.m[r * 3] * fx[0] + Ma.m[r * 3 + 1] * fx[1] + Ma.m[r * 3 + 2] * fx[2]);
  }
  vp[0] = vp[1] = vp[2] = 0.f; gvp[0] = gvp[1] = gvp[2] = 0.f; gfx[0] = gfx[1] = gfx[2] = 0.f;
  S_ao = m3_zero();
  float sgx = 0.f, sgy = 0.f, sgz = 0.f;  // sum_i s_i grad(w_i)
  if constexpr (kPG) s_am = 0.f;
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) {
      const float4* cg = colg(i * 3 + j);
      const float4* ca = cola(i * 3 + j);
      const float wxy = w[i][0] * w[j][1], dxw = dw[i][0] * w[j][1], dyw = w[i][0] * dw[j][1];
      float cgb[3], cab[3];
#pragma unroll
      for (int r = 0; r < 3; r++) {
        cgb[r] = a0[r] + Mg.m[r * 3] * (float)i + Mg.m[r * 3 + 1] * (float)j;
        cab[r] = b0[r] + Ma.m[r * 3] * (float)i + Ma.m[r * 3 + 1] * (float)j;
      }
      float G0[3] = {0.f, 0.f, 0.f}, A0[3] = {0.f, 0.f, 0.f}, A1[3] = {0.f, 0.f, 0.f};
      float s_w = 0.f, s_dz = 0.f;  // sum_k s wz[k], sum_k s dwz[k]
      float am_w = 0.f;             // kPG: sum_k am wz[k]
#pragma unroll
      for (int k = 0; k < 3; k++) {
        const float4 g = cg[k], a = ca[k];
        const float kk = (float)k;
        const float sv = g.x * (cgb[0] + Mg.m[2] * kk) + g.y * (cgb[1] + Mg.m[5] * kk) + g.z * (cgb[2] + Mg.m[8] * kk) +
                         a.x * (cab[0] + Ma.m[2] * kk) + a.y * (cab[1] + Ma.m[5] * kk) + a.z * (cab[2] + Ma.m[8] * kk) + m * a.w;
        const float wk = w[k][2];
        s_w = fmaf(sv, wk, s_w); s_dz = fmaf(sv, dw[k][2], s_dz);
        G0[0] = fmaf(wk, g.x, G0[0]); G0[1] = fmaf(wk, g.y, G0[1]); G0[2] = fmaf(wk, g.z, G0[2]);
        A0[0] = fmaf(wk, a.x, A0[0]); A0[1] = fmaf(wk, a.y, A0[1]); A0[2] = fmaf(wk, a.z, A0[2]);
        const float wkk = wk * kk;
        A1[0] = fmaf(wkk, a.x, A1[0]); A1[1] = fmaf(wkk, a.y, A1[1]); A1[2] = fmaf(wkk, a.z, A1[2]);
        if constexpr (kPG) am_w = fmaf(wk, a.w, am_w);
      }
      sgx = fmaf(dxw, s_w, sgx); sgy = fmaf(dyw, s_w, sgy); sgz = fmaf(wxy, s_dz, sgz);
      if constexpr (kPG) s_am = fmaf(wxy, am_w, s_am);
      const float wi = wxy * (float)i, wj = wxy * (float)j;
#pragma unroll
      for (int r = 0; r < 3; r++) {
        vp[r] = fmaf(wxy, G0[r], vp[r]);
        gvp[r] = fmaf(wxy, A0[r], gvp[r]);
        S_ao.m[r * 3 + 0] = fmaf(wi, A0[r], S_ao.m[r * 3 + 0]);
        S_ao.m[r * 3 + 1] = fmaf(wj, A0[r], S_ao.m[r * 3 + 1]);
        S_ao.m[r * 3 + 2] = fmaf(wxy, A1[r], S_ao.m[r * 3 + 2]);
      }
    }
  // gfx = -Mg^T vp - Ma^T gvp + sum s grad w
  gfx[0] = sgx - (Mg.m[0] * vp[0] + Mg.m[3] * vp[1] + Mg.m[6] * vp[2]) - (Ma.m[0] * gvp[0] + Ma.m[3] * gvp[1] + Ma.m[6] * gvp[2]);
  gfx[1] = sgy - (Mg.m[1] * vp[0] + Mg.m[4] * vp[1] + Mg.m[7] * vp[2]) - (Ma.m[1] * gvp[0] + Ma.m[4] * gvp[1] + Ma.m[7] * gvp[2]);
  gfx[2] = sgz - (Mg.m[2] * vp[0] + Mg.m[5] * vp[1] + Mg.m[8] * vp[2]) - (Ma.m[2] * gvp[0] + Ma.m[5] * gvp[1] + Ma.m[8] * gvp[2]);
}

// Parameter-gradient reduction of k_particle_grad<kMat, true>: the lanes in `live` (the particles of the warp that contribute) add (dmu, dlam,
// dmass) to row `row` of P.pg_mat.  Warps are cell-sorted and scenes have few rows, so a warp nearly always holds one row and all 32 lanes: a
// butterfly and one fp64 atomic per component.  Otherwise each group of lanes sharing a row sums through shuffles restricted to the group and
// its lowest lane issues the atomics (one per (warp, row) either way).
__device__ __forceinline__ void param_grad_reduce(const KParams& P, const unsigned live, const int row, const float dmu, const float dlam, const float dm) {
  const unsigned peers = __match_any_sync(live, row);
  const int lane = threadIdx.x & 31;
  float a = dmu, b = dlam, c = dm;
  if (peers == 0xffffffffu) {   // warp-uniform: every lane sees the same full mask
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); c += __shfl_xor_sync(0xffffffffu, c, o);
    }
  } else {
    a = b = c = 0.f;
    for (unsigned m = peers; m != 0u; m &= m - 1u) {   // the same trip count on every lane of the group
      const int l = __ffs((int)m) - 1;
      a += __shfl_sync(peers, dmu, l); b += __shfl_sync(peers, dlam, l); c += __shfl_sync(peers, dm, l);
    }
  }
  if (lane == __ffs((int)peers) - 1) {
    double* g = P.pg_mat + (size_t)row * 4;
    atomic_add_f64(g + 0, (double)a); atomic_add_f64(g + 1, (double)b); atomic_add_f64(g + 2, (double)c);
  }
}

// kMat == 1: every particle is a mu = 0 liquid (FmpmConfig.scene_flags): no SVD and no SVD adjoint in the instruction stream, the constitutive
// adjoint is gJ * cof(F~) (+ the J^(1/3) term of F[f+1])
// kPG: also the per-row dL/d(mu, lam, mass) (include/fluidmpm.h, FmpmParamGrad).  dL/dmu needs R = U V^T also where the forward takes no SVD
// (mu = 0 rows: the reference's ti.svd runs for every particle, so dL/dmu is defined and in general non-zero there), so this variant takes one
// svd3 per such particle.
template <int kMat, bool kPG>
__global__ void __launch_bounds__(PG_WARPS * 32, kMat == 1 ? PG_MINB_LIQUID : PG_MINB) k_particle_grad(const KParams P, const int f, const int gin, const int gout) {
  __shared__ float4 tiles[PG_WARPS][2][9 * G2P_ZMAX];
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  float4* tg = tiles[threadIdx.x >> 5][0];
  float4* ta = tiles[threadIdx.x >> 5][1];
  PState st; st.meta = 0; st.x[0] = st.x[1] = st.x[2] = 0.f;
  if (s < P.N) {
    load_A(P.pa, P, f, s, st);
    prefetch_planes4(P.pf, P, f, 2, s); prefetch_plane1(P.pf8, P, f, s);   // read after the footprint staging: F[f], then the adjoint of frame f+1
    prefetch_planes4(P.ga, P, gin, 4, s); prefetch_planes4(P.gf, P, gin, 2, s); prefetch_plane1(P.gf8, P, gin, s);
#if PG_AHEAD > 0
    if ((long long)s + (long long)PG_AHEAD * PG_WARPS * 32 < P.N) prefetch_planes4(P.pa, P, f, 4, s + PG_AHEAD * PG_WARPS * 32);   // the first loads of the CTA that takes this one's place
#endif
  }
  int b[3]; float fx[3];
  const bool ok = (s < P.N) && (st.meta & 1) && base_fx(P, st.x, b, fx);
  unsigned live = 0u;   // kPG: the lanes that reach the parameter-gradient reduction (every lane of the warp is still here)
  if constexpr (kPG) live = __ballot_sync(0xffffffffu, ok);
  const Footprint fp = footprint_of(ok, b);
  if (fp.staged) { footprint_load(P.grid_v, P.n, fp, tg); footprint_load(P.ggrid_pm, P.n, fp, ta); }
  if (s >= P.N) return;
  if (!ok) {  // process_unused_particles.grad (MPM:551): the adjoint passes straight through
#pragma unroll
    for (int k = 0; k < 4; k++) P.ga[pa_idx(P, gout, k, s)] = P.ga[pa_idx(P, gin, k, s)];
    P.gf[pf_idx(P, gout, 0, s)] = P.gf[pf_idx(P, gin, 0, s)];
    P.gf[pf_idx(P, gout, 1, s)] = P.gf[pf_idx(P, gin, 1, s)];
    P.gf8[pf8_idx(P, gout, s)] = P.gf8[pf8_idx(P, gin, s)];
    return;
  }
  load_F(P.pf, P.pf8, P, f, s, st.F);
  const float4 mt = __ldg(P.mats + ((st.meta >> 8) & 0xff));
  const float mu = mt.x, lam = mt.y, m = mt.z; const int cls = __float_as_int(mt.w);
  Constit K;
  if (kMat == 1) {   // F~ = (I + dt C) F, J = det F~, affine = k_stress * lam J (J - 1) I + m C   (MPM:254-258, 339-344 with mu = 0)
    Mat3 IdC0;
#pragma unroll
    for (int i = 0; i < 9; i++) IdC0.m[i] = P.dt * st.C.m[i] + ((i % 4 == 0) ? 1.f : 0.f);
    K.Ft = m3_mul(IdC0, st.F); K.need_svd = false; K.J = m3_det(K.Ft);
    const float iso = lam * K.J * (K.J - 1.f);
#pragma unroll
    for (int i = 0; i < 9; i++) K.A.m[i] = P.k_stress * ((i % 4 == 0) ? iso : 0.f) + m * st.C.m[i];
  } else {
    constitutive(P, st, mu, lam, m, cls, K);
  }
  float w[3][3], dw[3][3]; bspline(fx, w); bspline_d(fx, dw);
  float gxin[3], gve[3], mv[3];
  Mat3 Mg, Ma;
  {
    PState g; load_A(P.ga, P, gin, s, g);  // (gx', gv', gC')
    const float c4 = 4.f * P.inv_dx;
#pragma unroll
    for (int k = 0; k < 3; k++) { gxin[k] = g.x[k]; gve[k] = g.v[k] + P.dt * g.x[k]; mv[k] = m * st.v[k]; }  // advect_kernel.grad (MPM:443)
#pragma unroll
    for (int k = 0; k < 9; k++) { Mg.m[k] = c4 * g.C.m[k]; Ma.m[k] = K.A.m[k] * P.dx; }
  }
  float vp[3], gvp[3], gfx[3], s_am; Mat3 S_ao;
  if (fp.staged) {
    const int zo = b[2] - fp.kmin;
    adjoint_gather<kPG>(fx, w, dw, [&](int c) { return tg + c * G2P_ZMAX + zo; }, [&](int c) { return ta + c * G2P_ZMAX + zo; }, gve, Mg, mv, Ma, m, vp, gvp, S_ao, gfx, s_am);
  } else {
    const int cell = (b[0] * P.n + b[1]) * P.n + b[2];
    const float4* gvo = P.grid_v + cell; const float4* gpm = P.ggrid_pm + cell; const int n = P.n;
    adjoint_gather<kPG>(fx, w, dw, [&](int c) { return gvo + ((c / 3) * n + (c % 3)) * n; }, [&](int c) { return gpm + ((c / 3) * n + (c % 3)) * n; }, gve, Mg, mv, Ma, m, vp, gvp,
                        S_ao, gfx, s_am);
  }
  // gA = sum w a (x) d,  d = (o - fx) dx
  Mat3 gA;
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) gA.m[r * 3 + c] = P.dx * (S_ao.m[r * 3 + c] - gvp[r] * fx[c]);
  float ox[3], ov[3];
#pragma unroll
  for (int k = 0; k < 3; k++) { ox[k] = gxin[k] + P.inv_dx * gfx[k]; ov[k] = m * gvp[k]; }
  Mat3 gFn; load_F(P.gf, P.gf8, P, gin, s, gFn);
  Mat3 gFt;
  if (kMat == 1) {   // constitutive_grad with need_svd == false, cls == MAT_LIQUID
    const float trP = P.k_stress * m3_trace(gA);
    float gJ = lam * (2.f * K.J - 1.f) * trP;
    const float cb = cbrtf(K.J);
    gJ += (1.f / 3.f) * (cb / K.J) * m3_trace(gFn);
    const float* a = K.Ft.m;
    gFt.m[0] = gJ * (a[4] * a[8] - a[5] * a[7]); gFt.m[1] = gJ * (a[5] * a[6] - a[3] * a[8]); gFt.m[2] = gJ * (a[3] * a[7] - a[4] * a[6]);
    gFt.m[3] = gJ * (a[2] * a[7] - a[1] * a[8]); gFt.m[4] = gJ * (a[0] * a[8] - a[2] * a[6]); gFt.m[5] = gJ * (a[1] * a[6] - a[0] * a[7]);
    gFt.m[6] = gJ * (a[1] * a[5] - a[2] * a[4]); gFt.m[7] = gJ * (a[2] * a[3] - a[0] * a[5]); gFt.m[8] = gJ * (a[0] * a[4] - a[1] * a[3]);
  } else {
    gFt = constitutive_grad(P, K, mu, lam, cls, gA, gFn);
  }
  // compute_F_tmp.grad (MPM:546): gC += dt * gFt F^T ; gF += (I + dt C)^T gFt ; plus gC += m * gA
  Mat3 oC = m3_add(m3_scale(gA, m), m3_scale(m3_mul_nt(gFt, st.F), P.dt));
  Mat3 IdC;
#pragma unroll
  for (int i = 0; i < 9; i++) IdC.m[i] = P.dt * st.C.m[i] + ((i % 4 == 0) ? 1.f : 0.f);
  Mat3 oF = m3_mul_tn(IdC, gFt);
  store_A(P.ga, P, gout, s, ox, 0, ov, oC);
  store_F(P.gf, P.gf8, P, gout, s, oF);
  if constexpr (kPG) {
    // P = 2 mu M F~^T + lam J (J - 1) I with M = F~ - R, P̄ = k_stress gA:  dmu = 2 P̄ : (M F~^T), dlam = J (J - 1) tr(P̄)
    // A = k_stress P + m C and the scatter's m v and m weights:  dmass = v . gvp + gA : C + sum_i w_i am_i
    Mat3 R;
    if (kMat == 1 || !K.need_svd) { Mat3 U, V; float sg[3]; svd3(K.Ft, U, sg, V); R = m3_mul_nt(U, V); }
    else R = m3_mul_nt(K.U, K.V);
    const Mat3 MFt = m3_mul_nt(m3_sub(K.Ft, R), K.Ft);
    float gm = 0.f, gc = s_am + st.v[0] * gvp[0] + st.v[1] * gvp[1] + st.v[2] * gvp[2];
#pragma unroll
    for (int i = 0; i < 9; i++) { gm = fmaf(gA.m[i], MFt.m[i], gm); gc = fmaf(gA.m[i], st.C.m[i], gc); }
    param_grad_reduce(P, live, (st.meta >> 8) & 0xff, 2.f * P.k_stress * gm, P.k_stress * K.J * (K.J - 1.f) * m3_trace(gA), gc);
  }
}

// injector act adjoint (act_kernel.grad, agents/agent_injector.py:27-28): gpos[f] += gx[f+1, pid]; an Injector (not a BallInjector)
// also rotates inject_p / inject_v by quat[f] (injector.py:93-96), whose adjoint goes to gquat[f] (6-DOF injectors, agent_transporting.yaml)
__global__ void k_inject_grad(const KParams P, const int f, const int gin, const FmpmInjector inj, float* __restrict__ gpos,
                              const float* __restrict__ equat, float* __restrict__ gquat, const int act_id, const int* __restrict__ inv) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= inj.flux) return;
  const int pid = ((const int*)inj.act_range)[act_id + i];
  const int s = inv ? inv[pid] : pid;
  const float4 g0 = P.ga[pa_idx(P, gin, 0, s)];
  atomicAdd(gpos + f * 3 + 0, g0.x); atomicAdd(gpos + f * 3 + 1, g0.y); atomicAdd(gpos + f * 3 + 2, g0.z);
  if (inj.kind == 1 && gquat) {
    const float4 g1 = P.ga[pa_idx(P, gin, 1, s)];
    const float q[4] = {equat[f * 4], equat[f * 4 + 1], equat[f * 4 + 2], equat[f * 4 + 3]};
    const float gx[3] = {g0.x, g0.y, g0.z}, gv[3] = {g1.x, g1.y, g1.z};
    float gq[4] = {0.f, 0.f, 0.f, 0.f};
    q_rot_adj_q(q, inj.inject_p, gx, gq);
    q_rot_adj_q(q, inj.inject_v, gv, gq);
#pragma unroll
    for (int k = 0; k < 4; k++) atomicAdd(gquat + f * 4 + k, gq[k]);
  }
}

// =============================================================================================
// host entry points
// =============================================================================================
static int check_bound_b(FmpmHandle* h, const char* name) {
  if (!h) return 1;
  if (!h->bound) { snprintf(h->err, sizeof(h->err), "%s: fmpm_bind() has not been called", name); return 1; }
  if (!h->buf.ga || !h->buf.gf || !h->buf.gf8 || !h->buf.ggrid_v || !h->buf.ggrid_pm) {
    snprintf(h->err, sizeof(h->err), "%s: gradient buffers were not bound", name); return 1;
  }
  return 0;
}

int fmpm_grid_op_impl(FmpmHandle* h, int f, int clear_pm, int zero_ggv, int ring_slot, void* stream);  // fmpm_forward.cu
int fmpm_p2g_impl(FmpmHandle* h, int f, int write_F, int ring_slot, void* stream);                       // fmpm_forward.cu

static int g2p_grad_scatter_impl(FmpmHandle* h, int f, int gin, int dense_zero, int ring_slot, void* stream) {
  if (check_bound_b(h, "fmpm_g2p_grad_scatter")) return 1;
  KParams P = make_kparams(h, ring_slot);
  if (dense_zero) {
    cudaError_t e = cudaMemsetAsync(P.ggrid_v, 0, (size_t)P.G * sizeof(float4), (cudaStream_t)stream);
    if (e != cudaSuccess) { snprintf(h->err, sizeof(h->err), "fmpm_g2p_grad_scatter: %s", cudaGetErrorString(e)); return 1; }
  }
  if (P.N == 0) return 0;
  const long long warps = ((long long)P.N + 32 * SC_ROUNDS - 1) / (32 * SC_ROUNDS);
  const int blocks = (int)((warps + SC_WARPS - 1) / SC_WARPS);
  if (h->slab.enabled) FMPM_LAUNCH(k_g2p_grad_scatter<true>, blocks, SC_WARPS * 32, 0, stream, P, f, gin);
  else FMPM_LAUNCH(k_g2p_grad_scatter<false>, blocks, SC_WARPS * 32, 0, stream, P, f, gin);
  FMPM_CHECK_LAUNCH(h, "fmpm_g2p_grad_scatter");
  return 0;
}
extern "C" int fmpm_g2p_grad_scatter(FmpmHandle* h, int f, int gin, void* stream) { return g2p_grad_scatter_impl(h, f, gin, 1, -1, stream); }
static int grid_op_grad_impl(FmpmHandle* h, int f, int clear_pm, int ring_slot, void* stream, int zero_ggv_after = 0) {
  if (check_bound_b(h, "fmpm_grid_op_grad")) return 1;
  KParams P = make_kparams(h, ring_slot, f);   // x-slab mode: the accumulator / block flags of substep parity f
  const int nblk = P.nb * P.nb * P.nb;
  const int grid = nblk < h->sm_count * 8 ? nblk : h->sm_count * 8;
  if (P.pg_mat) FMPM_LAUNCH(k_grid_op_grad<true>, grid, 256, 0, stream, P, f, clear_pm, zero_ggv_after);
  else FMPM_LAUNCH(k_grid_op_grad<false>, grid, 256, 0, stream, P, f, clear_pm, zero_ggv_after);
  FMPM_CHECK_LAUNCH(h, "fmpm_grid_op_grad");
  return 0;
}
extern "C" int fmpm_grid_op_grad(FmpmHandle* h, int f, void* stream) { return grid_op_grad_impl(h, f, 0, -1, stream); }
static int particle_grad_impl(FmpmHandle* h, int f, int gin, int gout, int ring_slot, void* stream) {
  if (check_bound_b(h, "fmpm_particle_grad")) return 1;
  KParams P = make_kparams(h, ring_slot);
  if (P.N == 0) return 0;
  const int blocks = (P.N + PG_WARPS * 32 - 1) / (PG_WARPS * 32);
  const bool liquid = h->cfg.scene_flags & FMPM_SCENE_ALL_LIQUID_MU0;
  void (*kern)(const KParams, const int, const int, const int) =
      P.pg_mat ? (liquid ? k_particle_grad<1, true> : k_particle_grad<0, true>) : (liquid ? k_particle_grad<1, false> : k_particle_grad<0, false>);
  FMPM_LAUNCH(kern, blocks, PG_WARPS * 32, 0, stream, P, f, gin, gout);
  FMPM_CHECK_LAUNCH(h, "fmpm_particle_grad");
  return 0;
}
extern "C" int fmpm_particle_grad(FmpmHandle* h, int f, int gin, int gout, void* stream) { return particle_grad_impl(h, f, gin, gout, -1, stream); }

// the particle-level Dynamic.collide pre-pass; the contact-gradient instantiation only while its accumulator is bound
static void collide_particle_grad_launch(const KParams& P, const int f, const int gin, void* stream) {
  if (P.pg_contact) FMPM_LAUNCH(k_collide_particle_grad<true>, (P.N + 127) / 128, 128, 0, stream, P, f, gin);
  else FMPM_LAUNCH(k_collide_particle_grad<false>, (P.N + 127) / 128, 128, 0, stream, P, f, gin);
}

// zero the v_out adjoint on the active blocks of the substep (stored-grid backward: no grid_op recompute to piggy-back on)
__global__ void __launch_bounds__(256) k_zero_ggv_blocks(const KParams P) {
  const int n = P.n, nb = P.nb, nblk = nb * nb * nb;
  for (int blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
    if (P.blk_flags[blk] == 0) continue;
    const int bx = blk / (nb * nb), by = (blk / nb) % nb, bz = blk % nb;
#pragma unroll
    for (int r = 0; r < 2; r++) {
      const int t = threadIdx.x + r * 256;
      const int i = bx * 8 + (t >> 6), j = by * 8 + ((t >> 3) & 7), k = bz * 8 + (t & 7);
      P.ggrid_v[(i * n + j) * n + k] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}
extern "C" int fmpm_substep_grad_stored(FmpmHandle* h, int f, int gin, int gout, void* stream) {
  if (check_bound_b(h, "fmpm_substep_grad_stored")) return 1;
  if (!h->buf.grid_pm_ring) { snprintf(h->err, sizeof(h->err), "fmpm_substep_grad_stored: the per-frame grid ring was not bound"); return 1; }
  if (gin == gout || (gin | gout) & ~1) { snprintf(h->err, sizeof(h->err), "fmpm_substep_grad_stored: gin/gout must be distinct in {0,1}"); return 1; }
  KParams P = make_kparams(h, f);
  const int nblk = P.nb * P.nb * P.nb;
  const int grid = nblk < h->sm_count * 8 ? nblk : h->sm_count * 8;
  FMPM_LAUNCH(k_zero_ggv_blocks, grid, 256, 0, stream, P);
  FMPM_CHECK_LAUNCH(h, "fmpm_substep_grad_stored(zero)");
  if (h->col.has_rigid && h->col.collide_type != 1 && P.N > 0) {
    collide_particle_grad_launch(P, f, gin, stream); FMPM_CHECK_LAUNCH(h, "fmpm_substep_grad_stored(collide)");
  }
  if (g2p_grad_scatter_impl(h, f, gin, 0, f, stream) || grid_op_grad_impl(h, f, 0, f, stream)) return 1;
  return particle_grad_impl(h, f, gin, gout, f, stream);
}

extern "C" int fmpm_substep_grad(FmpmHandle* h, int f, int gin, int gout, void* stream) {
  if (check_bound_b(h, "fmpm_substep_grad")) return 1;
  if (gin == gout || (gin | gout) & ~1) { snprintf(h->err, sizeof(h->err), "fmpm_substep_grad: gin/gout must be distinct in {0,1}"); return 1; }
  // recompute the forward grid of frame f (accumulators are clear on entry), zeroing the v_out adjoint of the active blocks
  if (fmpm_p2g(h, f, 0, stream) || fmpm_grid_op_impl(h, f, 0, 1, -1, stream)) return 1;
  if (h->col.has_rigid && h->col.collide_type != 1) {  // particle-level agent collide: fold its adjoint into the frame-(f+1) adjoint
    KParams P = make_kparams(h);
    if (P.N > 0) { collide_particle_grad_launch(P, f, gin, stream); FMPM_CHECK_LAUNCH(h, "fmpm_substep_grad(collide)"); }
  }
  // adjoint: grid scatter, grid_op.grad (also leaves the accumulators clear for the next substep), per-particle part
  if (g2p_grad_scatter_impl(h, f, gin, 0, -1, stream) || grid_op_grad_impl(h, f, 1, -1, stream)) return 1;
  return fmpm_particle_grad(h, f, gin, gout, stream);
}
// x-slab backward (SURVEY.md 8e): fmpm_substep_grad cut at its two ghost exchanges.  Sequence per rank and substep:
//   fmpm_p2g(f, 0)  ->  [ghost sum of the (momentum, mass) planes]  ->  fmpm_substep_grad_scatter
//                   ->  [ghost sum of the v_out-adjoint planes]     ->  fmpm_substep_grad_finish
extern "C" int fmpm_substep_grad_scatter(FmpmHandle* h, int f, int gin, void* stream) {
  if (check_bound_b(h, "fmpm_substep_grad_scatter")) return 1;
  if (gin & ~1) { snprintf(h->err, sizeof(h->err), "fmpm_substep_grad_scatter: gin must be 0 or 1"); return 1; }
  // fused ghost reduction of the v_out adjoint (peer_ggv_*): the buffer is all-zero here (grid_op.grad zeroes what it consumes), and a
  // neighbour may already be scattering into it, so it must NOT be zeroed now
  const int fused = h->slab.enabled && (h->slab.peer_ggv_left || h->slab.peer_ggv_right);
  if (fmpm_grid_op_impl(h, f, 0, fused ? 0 : 1, -1, stream)) return 1;
  if (h->col.has_rigid && h->col.collide_type != 1) {
    KParams P = make_kparams(h);
    if (P.N > 0) { collide_particle_grad_launch(P, f, gin, stream); FMPM_CHECK_LAUNCH(h, "fmpm_substep_grad_scatter(collide)"); }
  }
  return g2p_grad_scatter_impl(h, f, gin, 0, -1, stream);
}
// the x-slab backward runs grid_op.grad on the ghost planes of both neighbours: parameter gradients would count those nodes twice
static int reject_param_grad(FmpmHandle* h, const char* name) {
  if (!h->pgrad.gmat && !h->cgrad.gcontact) return 0;
  snprintf(h->err, sizeof(h->err), "%s: parameter gradients (fmpm_set_param_grad / fmpm_set_contact_grad) are not supported by the x-slab backward", name);
  return 1;
}
extern "C" int fmpm_substep_grad_finish(FmpmHandle* h, int f, int gin, int gout, void* stream) {
  if (check_bound_b(h, "fmpm_substep_grad_finish") || reject_param_grad(h, "fmpm_substep_grad_finish")) return 1;
  if (gin == gout || (gin | gout) & ~1) { snprintf(h->err, sizeof(h->err), "fmpm_substep_grad_finish: gin/gout must be distinct in {0,1}"); return 1; }
  const int fused = h->slab.enabled && (h->slab.peer_ggv_left || h->slab.peer_ggv_right);
  if (grid_op_grad_impl(h, f, 1, -1, stream, fused)) return 1;
  return fmpm_particle_grad(h, f, gin, gout, stream);
}
int fmpm_slab_sync_impl(FmpmHandle* h, void* stream);   // fmpm_io.cu
// one backward substep of an x-slab rank in ONE call (peer exchange + neighbour handshakes): recompute scatter, handshake, grid_op +
// adjoint scatter (reducing into the neighbours' adjoint grids), handshake, grid_op.grad + particle side
extern "C" int fmpm_substep_grad_slab(FmpmHandle* h, int f, int gin, int gout, void* stream) {
  if (check_bound_b(h, "fmpm_substep_grad_slab") || reject_param_grad(h, "fmpm_substep_grad_slab")) return 1;
  if (!h->slab.enabled || !h->slab.signal || !(h->slab.peer_ggv_left || h->slab.peer_ggv_right)) {
    snprintf(h->err, sizeof(h->err), "fmpm_substep_grad_slab: needs the x-slab peer pointers of the adjoint grid and the handshake arrays"); return 1;
  }
  if (fmpm_p2g(h, f, 0, stream) || fmpm_slab_sync_impl(h, stream) || fmpm_substep_grad_scatter(h, f, gin, stream) || fmpm_slab_sync_impl(h, stream)) return 1;
  return fmpm_substep_grad_finish(h, f, gin, gout, stream);
}
extern "C" int fmpm_inject_grad(FmpmHandle* h, int f, int gin, const FmpmInjector* inj, const FmpmEffector* e, int act_id,
                                const void* inv, void* stream) {
  if (check_bound_b(h, "fmpm_inject_grad")) return 1;
  KParams P = make_kparams(h);
  FMPM_LAUNCH(k_inject_grad, (inj->flux + 31) / 32, 32, 0, stream, P, f, gin, *inj, (float*)e->gpos, (const float*)e->quat, (float*)e->gquat, act_id, (const int*)inv);
  FMPM_CHECK_LAUNCH(h, "fmpm_inject_grad");
  return 0;
}
