// fmpm_common.cuh — shared device helpers of libfluidmpm.so (sm_90a).
// Data layout and material/boundary semantics follow the reference simulator
// fluidlab/fluidengine/simulators/mpm_simulator.py (MPM) — see include/fluidmpm.h and DESIGN.md.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/fluidmpm.h"

#define FMPM_EPS 1e-12f  // configs/macros.py:213
#define FMPM_NOWHERE (-100.0f)  // configs/macros.py:216

struct SdfDev { const float* vox; int res; float T[12]; float Ainv[9]; float friction, softness; };
struct CollidersDev {
  int n_statics; SdfDev statics[4];
  int has_rigid; int collide_type; SdfDev rigid;
  const float* epos; const float* equat; float* egpos; float* egquat;
  float y_min;
};

#ifdef FMPM_HOST_EMU
struct CUtensorMap_st { alignas(64) unsigned long long opaque[16]; };
typedef CUtensorMap_st CUtensorMap;
#define __grid_constant__
#else
#include <cuda.h>   // CUtensorMap (types only: the encoder is fetched from the driver at run time, no link dependency on libcuda)
#endif

struct FmpmHandle {
  CUtensorMap tm_gv8, tm_gv16;   // TMA descriptors of grid_v as a (4, n, n, n) float tensor with boxes (4, 8 | 16, 4, 4): the footprint tile of k_fwd
  int tma_ok;                    // 0: descriptors not available (encoder missing / FMPM_TMA=0): k_fwd stages its tile with LDG + STS
  FmpmConfig cfg;
  FmpmBuffers buf;
  CollidersDev col;
  FmpmSlab slab;
  FmpmBodies bodies;
  bool bound;
  char err[512];
  int sm_count;
  int fwd_mask;   // fmpm_set_fwd_mask
  int fwd_stride; // 1: no CTA -> slot-block permutation in the lazy-grid_op k_fwd (FMPM_FWD_STRIDE=1)
  int use_pdl;    // programmatic dependent launch of the forward chain (FMPM_PDL=0 switches it off)
  int slab_pull_ok;   // x-slab forward steps: grid_op reads the neighbours' ghost planes instead of p2g pushing them (FMPM_SLAB_PULL=0: push form)
  int slab_pull;      // set by fmpm_substeps_slab around its launches: the scatter kernels stay local, grid_op is k_grid_op_pull
  int slab_fsync;     // pull form, opt-in (FMPM_SLAB_FSYNC=1): the neighbour handshake runs INSIDE k_grid_op_pull instead of in a k_slab_sync launch before it
  FmpmParamGrad pgrad;   // fmpm_set_param_grad: both pointers set = the backward kernels also accumulate dL/d(mu, lam, mass) per row and dL/dg
  FmpmContactGrad cgrad; // fmpm_set_contact_grad (needs pgrad): also dL/d(static friction, rigid friction, rigid softness, restitution)
};

int fmpm_advect_rigid_impl(FmpmHandle* h, int f, void* stream);  // fmpm_rigid.cu; no-op without MAT_RIGID bodies

// kernel-side view (passed by value)
struct KParams {
  int N, n, G, T;
  float dt, dx, inv_dx, k_stress;
  float gx, gy, gz;
  int boundary_type;
  float lo[3], hi[3];
  float cyl_cx, cyl_cz, cyl_r, restitution;
  int lock_mask;
  float4* pa; float4* pf; float* pf8;
  float4* ga; float4* gf; float* gf8;
  float4* grid_pm; float4* grid_v; float4* ggrid_v; float4* ggrid_pm;
  const float4* mats;  // (mu, lam, mass, cls-as-int-bits)
  int* blk_flags; int* blk_list; int* blk_count; int nb;  // sparse grid: 8^3-node blocks
  int* epoch;   // launch epoch of the lazy grid_op (k_fwd, kInline): bumped by the p2g that opens a fused step, see fmpm_forward.cu
  CollidersDev col;
  // x-slab mode: neighbours' accumulators (peer memory over NVLink) and the node-plane ranges shared with them
  float4* peer_l; float4* peer_r; int gl_lo, gl_hi, gr_lo, gr_hi;
  int* peer_fl; int* peer_fr;
  float4* peer_gl; float4* peer_gr;   // the neighbours' v_out adjoint (backward ghost reduction fused into g2p.grad's scatter)
  // last, so that the kernels which never read them keep every other parameter offset: the parameter-gradient accumulators (fmpm_set_param_grad)
  double* pg_mat; double* pg_grav;
  double* pg_contact;   // fmpm_set_contact_grad: double[8], see include/fluidmpm.h (FmpmContactGrad)
};

// ring_slot >= 0: the (momentum, mass) / v_out grids and the active-block list live in slot `ring_slot` of the per-frame ring
static inline KParams make_kparams(const FmpmHandle* h, int ring_slot = -1, int parity = 0) {
  KParams P;
  const FmpmConfig& c = h->cfg;
  P.N = c.n_particles; P.n = c.n_grid; P.G = c.n_grid * c.n_grid * c.n_grid; P.T = c.max_substeps_local;
  P.dt = c.dt; P.dx = c.dx; P.inv_dx = c.inv_dx; P.k_stress = c.k_stress;
  P.gx = c.gravity[0]; P.gy = c.gravity[1]; P.gz = c.gravity[2];
  P.boundary_type = c.boundary_type;
  for (int i = 0; i < 3; i++) { P.lo[i] = c.b_lower[i]; P.hi[i] = c.b_upper[i]; }
  P.cyl_cx = c.cyl_center[0]; P.cyl_cz = c.cyl_center[1]; P.cyl_r = c.cyl_radius; P.restitution = c.restitution;
  P.lock_mask = c.lock_mask;
  P.pa = (float4*)h->buf.pa; P.pf = (float4*)h->buf.pf; P.pf8 = (float*)h->buf.pf8;
  P.ga = (float4*)h->buf.ga; P.gf = (float4*)h->buf.gf; P.gf8 = (float*)h->buf.gf8;
  P.grid_pm = (float4*)h->buf.grid_pm; P.grid_v = (float4*)h->buf.grid_v;
  P.ggrid_v = (float4*)h->buf.ggrid_v; P.ggrid_pm = (float4*)h->buf.ggrid_pm;
  P.mats = (const float4*)h->buf.materials;
  P.col = h->col;
  P.blk_flags = (int*)h->buf.blk_flags; P.blk_list = (int*)h->buf.blk_list; P.blk_count = (int*)h->buf.blk_count; P.nb = c.n_grid / 8;
  P.epoch = nullptr;
  P.peer_l = P.peer_r = nullptr; P.gl_lo = P.gl_hi = P.gr_lo = P.gr_hi = 0; P.peer_fl = P.peer_fr = nullptr; P.peer_gl = P.peer_gr = nullptr;
  if (h->slab.enabled) {  // accumulator double-buffered by substep parity; peers use the same parity
    const size_t off = (size_t)(parity & 1) * P.G;
    P.grid_pm += off;
    if (h->slab.peer_pm_left) P.peer_l = (float4*)h->slab.peer_pm_left + off;
    if (h->slab.peer_pm_right) P.peer_r = (float4*)h->slab.peer_pm_right + off;
    const size_t foff = (size_t)(parity & 1) * P.nb * P.nb * P.nb;
    P.blk_flags += foff;
    if (h->slab.peer_flags_left) P.peer_fl = (int*)h->slab.peer_flags_left + foff;
    if (h->slab.peer_flags_right) P.peer_fr = (int*)h->slab.peer_flags_right + foff;
    P.gl_lo = h->slab.left_lo; P.gl_hi = h->slab.left_hi; P.gr_lo = h->slab.right_lo; P.gr_hi = h->slab.right_hi;
    P.peer_gl = (float4*)h->slab.peer_ggv_left; P.peer_gr = (float4*)h->slab.peer_ggv_right;
  }
  P.pg_mat = (double*)h->pgrad.gmat; P.pg_grav = (double*)h->pgrad.ggrav; P.pg_contact = (double*)h->cgrad.gcontact;
  if (ring_slot <= -2 && h->buf.grid_pm3) {   // -2 - k: accumulator k of the triple-buffered forward path (k_fwd, kInline)
    const int k = -2 - ring_slot;
    const size_t nblk = (size_t)P.nb * P.nb * P.nb;
    P.grid_pm = (float4*)h->buf.grid_pm3 + (size_t)k * P.G;
    P.blk_flags = (int*)h->buf.blk_flags3 + (size_t)k * nblk;
    P.epoch = (int*)h->buf.blk_count;   // (a reserved word of FmpmBuffers: int[1], zero-initialised by the caller)
  }
  if (ring_slot >= 0 && h->buf.grid_pm_ring) {
    const size_t nblk = (size_t)P.nb * P.nb * P.nb;
    P.grid_pm = (float4*)h->buf.grid_pm_ring + (size_t)ring_slot * P.G;
    P.grid_v = (float4*)h->buf.grid_v_ring + (size_t)ring_slot * P.G;
    P.blk_flags = (int*)h->buf.blk_list_ring + (size_t)ring_slot * nblk;  // per-frame block flags
  }
  return P;
}

// ---------------------------------------------------------------------------------------------
// small 3x3 algebra (row-major float[9] in registers)
// ---------------------------------------------------------------------------------------------
struct Mat3 { float m[9]; };

__device__ __forceinline__ Mat3 m3_mul(const Mat3& A, const Mat3& B) {
  Mat3 C;
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) C.m[i * 3 + j] = A.m[i * 3] * B.m[j] + A.m[i * 3 + 1] * B.m[3 + j] + A.m[i * 3 + 2] * B.m[6 + j];
  return C;
}
__device__ __forceinline__ Mat3 m3_mul_nt(const Mat3& A, const Mat3& B) {  // A * B^T
  Mat3 C;
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) C.m[i * 3 + j] = A.m[i * 3] * B.m[j * 3] + A.m[i * 3 + 1] * B.m[j * 3 + 1] + A.m[i * 3 + 2] * B.m[j * 3 + 2];
  return C;
}
__device__ __forceinline__ Mat3 m3_mul_tn(const Mat3& A, const Mat3& B) {  // A^T * B
  Mat3 C;
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) C.m[i * 3 + j] = A.m[i] * B.m[j] + A.m[3 + i] * B.m[3 + j] + A.m[6 + i] * B.m[6 + j];
  return C;
}
__device__ __forceinline__ Mat3 m3_tr(const Mat3& A) {
  Mat3 C;
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) C.m[i * 3 + j] = A.m[j * 3 + i];
  return C;
}
__device__ __forceinline__ Mat3 m3_add(const Mat3& A, const Mat3& B) { Mat3 C;
#pragma unroll
  for (int i = 0; i < 9; i++) C.m[i] = A.m[i] + B.m[i]; return C; }
__device__ __forceinline__ Mat3 m3_sub(const Mat3& A, const Mat3& B) { Mat3 C;
#pragma unroll
  for (int i = 0; i < 9; i++) C.m[i] = A.m[i] - B.m[i]; return C; }
__device__ __forceinline__ Mat3 m3_scale(const Mat3& A, float s) { Mat3 C;
#pragma unroll
  for (int i = 0; i < 9; i++) C.m[i] = A.m[i] * s; return C; }
__device__ __forceinline__ Mat3 m3_zero() { Mat3 C;
#pragma unroll
  for (int i = 0; i < 9; i++) C.m[i] = 0.f; return C; }
__device__ __forceinline__ float m3_det(const Mat3& A) {
  return A.m[0] * (A.m[4] * A.m[8] - A.m[5] * A.m[7]) - A.m[1] * (A.m[3] * A.m[8] - A.m[5] * A.m[6]) +
         A.m[2] * (A.m[3] * A.m[7] - A.m[4] * A.m[6]);
}
__device__ __forceinline__ float m3_trace(const Mat3& A) { return A.m[0] + A.m[4] + A.m[8]; }

// ---------------------------------------------------------------------------------------------
// 3x3 SVD, one lane per matrix (the warp batches 32 of them): one-sided Jacobi with a fixed
// number of sweeps (branch-light, no early exit -> no divergence), then sort + sign fix to the
// ti.svd convention used at MPM:264 (det U = det V = +1, sigma descending, sign on the smallest).
// ---------------------------------------------------------------------------------------------
#define FMPM_SVD_SWEEPS 5
__device__ __forceinline__ void svd_rot(float* B, float* V, const int p, const int q) {
  float alpha = B[p] * B[p] + B[3 + p] * B[3 + p] + B[6 + p] * B[6 + p];
  float beta = B[q] * B[q] + B[3 + q] * B[3 + q] + B[6 + q] * B[6 + q];
  float gamma = B[p] * B[q] + B[3 + p] * B[3 + q] + B[6 + p] * B[6 + q];
  float c = 1.f, s = 0.f;
  if (fabsf(gamma) > 1e-20f && fabsf(gamma) > 2e-8f * sqrtf(alpha * beta)) {
    float zeta = (beta - alpha) / (2.f * gamma);
    float t = copysignf(1.f, zeta) / (fabsf(zeta) + sqrtf(1.f + zeta * zeta));
    c = rsqrtf(1.f + t * t);
    s = c * t;
  }
#pragma unroll
  for (int k = 0; k < 3; k++) {
    float bp = B[k * 3 + p], bq = B[k * 3 + q];
    B[k * 3 + p] = c * bp - s * bq; B[k * 3 + q] = s * bp + c * bq;
    float vp = V[k * 3 + p], vq = V[k * 3 + q];
    V[k * 3 + p] = c * vp - s * vq; V[k * 3 + q] = s * vp + c * vq;
  }
}
__device__ __forceinline__ void svd_swap_cols(float* B, float* V, float* n, const int i, const int j) {
  // conditional swap so that n[i] >= n[j]; a swap negates column j to keep det V = +1 and B V^T unchanged
  if (n[i] < n[j]) {
    float t = n[i]; n[i] = n[j]; n[j] = t;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      float b = B[k * 3 + i]; B[k * 3 + i] = B[k * 3 + j]; B[k * 3 + j] = -b;
      float v = V[k * 3 + i]; V[k * 3 + i] = V[k * 3 + j]; V[k * 3 + j] = -v;
    }
  }
}
__device__ __forceinline__ void svd3(const Mat3& A, Mat3& U, float* sig, Mat3& Vm) {
  float B[9], V[9];
#pragma unroll
  for (int i = 0; i < 9; i++) { B[i] = A.m[i]; V[i] = (i % 4 == 0) ? 1.f : 0.f; }
#pragma unroll 1
  for (int sweep = 0; sweep < FMPM_SVD_SWEEPS; sweep++) {
    svd_rot(B, V, 0, 1); svd_rot(B, V, 0, 2); svd_rot(B, V, 1, 2);
  }
  float n[3];
#pragma unroll
  for (int j = 0; j < 3; j++) n[j] = sqrtf(B[j] * B[j] + B[3 + j] * B[3 + j] + B[6 + j] * B[6 + j]);
  svd_swap_cols(B, V, n, 0, 1); svd_swap_cols(B, V, n, 0, 2); svd_swap_cols(B, V, n, 1, 2);
  // U columns = B columns / norm ; degenerate columns completed by cross products
  float u[9];
#pragma unroll
  for (int j = 0; j < 3; j++) {
    float inv = n[j] > 1e-30f ? 1.f / n[j] : 0.f;
#pragma unroll
    for (int k = 0; k < 3; k++) u[k * 3 + j] = B[k * 3 + j] * inv;
  }
  if (!(n[0] > 1e-30f)) {
#pragma unroll
    for (int i = 0; i < 9; i++) u[i] = (i % 4 == 0) ? 1.f : 0.f;
  } else {
    if (!(n[1] > 1e-30f)) {
      // unit vector orthogonal to u0: drop the smallest component direction
      float ax = fabsf(u[0]), ay = fabsf(u[3]), az = fabsf(u[6]);
      float e0 = (ax <= ay && ax <= az) ? 1.f : 0.f, e1 = (e0 == 0.f && ay <= az) ? 1.f : 0.f, e2 = (e0 == 0.f && e1 == 0.f) ? 1.f : 0.f;
      float d = e0 * u[0] + e1 * u[3] + e2 * u[6];
      float w0 = e0 - d * u[0], w1 = e1 - d * u[3], w2 = e2 - d * u[6];
      float inv = rsqrtf(w0 * w0 + w1 * w1 + w2 * w2);
      u[1] = w0 * inv; u[4] = w1 * inv; u[7] = w2 * inv;
    }
    if (!(n[2] > 1e-30f)) {
      u[2] = u[3] * u[7] - u[6] * u[4];
      u[5] = u[6] * u[1] - u[0] * u[7];
      u[8] = u[0] * u[4] - u[3] * u[1];
    }
  }
  float detU = u[0] * (u[4] * u[8] - u[5] * u[7]) - u[1] * (u[3] * u[8] - u[5] * u[6]) + u[2] * (u[3] * u[7] - u[4] * u[6]);
  if (detU < 0.f) { u[2] = -u[2]; u[5] = -u[5]; u[8] = -u[8]; n[2] = -n[2]; }
#pragma unroll
  for (int i = 0; i < 9; i++) { U.m[i] = u[i]; Vm.m[i] = V[i]; }
  sig[0] = n[0]; sig[1] = n[1]; sig[2] = n[2];
}

// ---------------------------------------------------------------------------------------------
// layout accessors
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ size_t pa_idx(const KParams& P, int f, int k, int s) { return ((size_t)f * 4 + k) * (size_t)P.N + s; }
__device__ __forceinline__ size_t pf_idx(const KParams& P, int f, int k, int s) { return ((size_t)f * 2 + k) * (size_t)P.N + s; }
__device__ __forceinline__ size_t pf8_idx(const KParams& P, int f, int s) { return (size_t)f * (size_t)P.N + s; }

__device__ __forceinline__ float4 ldg4(const float4* p) { return __ldg(p); }

struct PState {  // unpacked particle state of one frame
  float x[3], v[3]; Mat3 C, F; int meta;
};
__device__ __forceinline__ void load_A(const float4* __restrict__ base, const KParams& P, int f, int s, PState& st) {
  float4 a0 = base[pa_idx(P, f, 0, s)], a1 = base[pa_idx(P, f, 1, s)], a2 = base[pa_idx(P, f, 2, s)], a3 = base[pa_idx(P, f, 3, s)];
  st.x[0] = a0.x; st.x[1] = a0.y; st.x[2] = a0.z; st.meta = __float_as_int(a0.w);
  st.v[0] = a1.x; st.v[1] = a1.y; st.v[2] = a1.z;
  st.C.m[0] = a1.w; st.C.m[1] = a2.x; st.C.m[2] = a2.y; st.C.m[3] = a2.z; st.C.m[4] = a2.w;
  st.C.m[5] = a3.x; st.C.m[6] = a3.y; st.C.m[7] = a3.z; st.C.m[8] = a3.w;
}
__device__ __forceinline__ void load_F(const float4* __restrict__ pf, const float* __restrict__ pf8, const KParams& P, int f, int s, Mat3& F) {
  float4 f0 = pf[pf_idx(P, f, 0, s)], f1 = pf[pf_idx(P, f, 1, s)];
  F.m[0] = f0.x; F.m[1] = f0.y; F.m[2] = f0.z; F.m[3] = f0.w; F.m[4] = f1.x; F.m[5] = f1.y; F.m[6] = f1.z; F.m[7] = f1.w;
  F.m[8] = pf8[pf8_idx(P, f, s)];
}
__device__ __forceinline__ void store_F(float4* __restrict__ pf, float* __restrict__ pf8, const KParams& P, int f, int s, const Mat3& F) {
  pf[pf_idx(P, f, 0, s)] = make_float4(F.m[0], F.m[1], F.m[2], F.m[3]);
  pf[pf_idx(P, f, 1, s)] = make_float4(F.m[4], F.m[5], F.m[6], F.m[7]);
  pf8[pf8_idx(P, f, s)] = F.m[8];
}
__device__ __forceinline__ void store_A(float4* __restrict__ base, const KParams& P, int f, int s, const float* x, int meta, const float* v, const Mat3& C) {
  base[pa_idx(P, f, 0, s)] = make_float4(x[0], x[1], x[2], __int_as_float(meta));
  base[pa_idx(P, f, 1, s)] = make_float4(v[0], v[1], v[2], C.m[0]);
  base[pa_idx(P, f, 2, s)] = make_float4(C.m[1], C.m[2], C.m[3], C.m[4]);
  base[pa_idx(P, f, 3, s)] = make_float4(C.m[5], C.m[6], C.m[7], C.m[8]);
}

// MPM:335-337: base / fx / quadratic B-spline weights.  `ok` is false when the 3x3x3 stencil would leave
// the grid (the reference has no bounds check there; such particles are frozen here instead of corrupting memory).
__device__ __forceinline__ bool base_fx(const KParams& P, const float* x, int* b, float* fx) {
  bool ok = true;
  const float tmax = (float)(P.n - 2);
#pragma unroll
  for (int d = 0; d < 3; d++) {
    float g = x[d] * P.inv_dx;
    float t = g - 0.5f;
    ok = ok && (t > -1.0f) && (t < tmax);   // then 0 <= (int)t <= n - 3: the whole 3x3x3 stencil is inside the grid (false for NaN)
    int bi = (int)t;  // cast(int): truncation toward zero
    b[d] = bi; fx[d] = g - (float)bi;
  }
  return ok;
}
__device__ __forceinline__ void bspline(const float* fx, float w[3][3]) {
#pragma unroll
  for (int d = 0; d < 3; d++) {
    float a = 1.5f - fx[d], b = fx[d] - 1.0f, c = fx[d] - 0.5f;
    w[0][d] = 0.5f * a * a; w[1][d] = 0.75f - b * b; w[2][d] = 0.5f * c * c;
  }
}
__device__ __forceinline__ void bspline_d(const float* fx, float dw[3][3]) {
#pragma unroll
  for (int d = 0; d < 3; d++) { dw[0][d] = -(1.5f - fx[d]); dw[1][d] = -2.f * (fx[d] - 1.0f); dw[2][d] = fx[d] - 0.5f; }
}

// boundary.impose_x_v velocity part (boundaries.py:39-63 cylinder, :106-120 cube); fac = d v_out / d v_in (diagonal)
// kPG: *hit = the axes that the wall reflects (fac = -restitution, not locked), where d v_out / d restitution = -v_in.  A mask rather than a
// test of fac against -restitution, which would also match a locked axis at restitution 0 and the radial kill at restitution 0.
template <bool kPG = false>
__device__ __forceinline__ void boundary_v(const KParams& P, const float* pos, float* v, float* fac, int* hit = nullptr) {
  fac[0] = fac[1] = fac[2] = 1.f;
  int h = 0;   // kPG only
  if (P.boundary_type == 0) {
#pragma unroll
    for (int i = 0; i < 3; i++) {
      if (pos[i] >= P.hi[i] && v[i] >= 0.f) { fac[i] = -P.restitution; if constexpr (kPG) h |= 1 << i; }
      else if (pos[i] <= P.lo[i] && v[i] <= 0.f) { fac[i] = -P.restitution; if constexpr (kPG) h |= 1 << i; }
    }
  } else {
    if (pos[1] > P.hi[1] && v[1] > 0.f) { fac[1] = -P.restitution; if constexpr (kPG) h = 2; }
    else if (pos[1] < P.lo[1] && v[1] < 0.f) { fac[1] = -P.restitution; if constexpr (kPG) h = 2; }
    float rx = pos[0] - P.cyl_cx, rz = pos[2] - P.cyl_cz;
    float rn = sqrtf(rx * rx + rz * rz + FMPM_EPS);
    if (rn > P.cyl_r) { fac[0] = 0.f; fac[2] = 0.f; }
  }
#pragma unroll
  for (int i = 0; i < 3; i++) {
    if (P.lock_mask & (1 << i)) fac[i] = 0.f;
    v[i] = (fac[i] == 0.f) ? 0.f : v[i] * fac[i];
  }
  if constexpr (kPG) *hit = h & ~P.lock_mask;
}

// ---------------------------------------------------------------------------------------------
// constitutive update of one particle (MPM:254-264 F_tmp + svd, MPM:339-344 stress/affine,
// MPM:356-378 F update).  Fills what the scatter needs.  `want_svd` outputs are only valid when
// need_svd (mu != 0 or a plastic class).
// ---------------------------------------------------------------------------------------------
struct Constit {
  Mat3 Ft, U, V, A, Fn; float sig[3]; float J; bool need_svd;
};
__device__ __forceinline__ void constitutive(const KParams& P, const PState& st, float mu, float lam, float mass, int cls, Constit& K) {
  // F_tmp = (I + dt*C) @ F
  Mat3 IdC;
#pragma unroll
  for (int i = 0; i < 9; i++) IdC.m[i] = P.dt * st.C.m[i] + ((i % 4 == 0) ? 1.f : 0.f);
  K.Ft = m3_mul(IdC, st.F);
  const bool plastic = (cls == FMPM_MAT_PLASTO_ELASTIC) || (cls == FMPM_MAT_PLASTO_ELASTIC_DEMO);
  K.need_svd = (mu != 0.f) || plastic;
  Mat3 stress;
  if (K.need_svd) {
    svd3(K.Ft, K.U, K.sig, K.V);
    K.J = K.sig[0] * K.sig[1] * K.sig[2];
    Mat3 R = m3_mul_nt(K.U, K.V);
    stress = m3_scale(m3_mul_nt(m3_sub(K.Ft, R), K.Ft), 2.f * mu);
  } else {
    K.J = m3_det(K.Ft);  // == product of singular values with the ti.svd sign convention
    stress = m3_zero();
  }
  float iso = lam * K.J * (K.J - 1.f);
  stress.m[0] += iso; stress.m[4] += iso; stress.m[8] += iso;
#pragma unroll
  for (int i = 0; i < 9; i++) K.A.m[i] = P.k_stress * stress.m[i] + mass * st.C.m[i];
  if (cls == FMPM_MAT_LIQUID) {
    float s = (K.J > 0.f) ? cbrtf(K.J) : __int_as_float(0x7fc00000);  // pow(J, 1/3): NaN for J < 0 like the reference
    if (K.J == 0.f) s = 0.f;
    K.Fn = m3_zero(); K.Fn.m[0] = s; K.Fn.m[4] = s; K.Fn.m[8] = s;
  } else if (plastic) {
    Mat3 US = K.U;
#pragma unroll
    for (int d = 0; d < 3; d++) {
      float sn = fminf(fmaxf(K.sig[d], 0.998f), 1.003f);
      US.m[d] *= sn; US.m[3 + d] *= sn; US.m[6 + d] *= sn;
    }
    K.Fn = m3_mul_nt(US, K.V);
  } else {
    K.Fn = K.Ft;  // elastic / rigid
  }
}

// Kernel launch and the few constructs the host compiler cannot take.  FMPM_HOST_EMU is only ever defined by tests/cuda_emu/cuda_runtime.h:
// with that directory first on the include path g++ builds these translation units UNCHANGED, one host thread per CUDA thread, so the
// kernel bodies and the host launch logic run under `pytest -m "not gpu"` (tests/test_cuda_emu_*.py).  nvcc never sees that header.
#ifdef FMPM_HOST_EMU
#define FMPM_LAUNCH(kern, grid, block, smem, stream, ...) cuemu::launch(dim3(grid), dim3(block), smem, [&]() { kern(__VA_ARGS__); })
#define FMPM_LAUNCH_PDL(pdl, kern, grid, block, smem, stream, ...) FMPM_LAUNCH(kern, grid, block, smem, stream, __VA_ARGS__)
#define FMPM_DYN_SMEM(type, name) type* name = (type*)cuemu::dyn_smem()
__device__ __forceinline__ void fmpm_pdl_trigger() {}
__device__ __forceinline__ void fmpm_pdl_wait() {}
#else
#define FMPM_LAUNCH(kern, grid, block, smem, stream, ...) kern<<<grid, block, smem, (cudaStream_t)(stream)>>>(__VA_ARGS__)
#define FMPM_DYN_SMEM(type, name) extern __shared__ type name[]
// Programmatic dependent launch (the forward substep is a chain of short kernels: p2g, [grid_op, k_fwd] x 9, grid_op, g2p).  A kernel of the
// chain lets its successor's CTAs become resident as soon as all of its own CTAs have started (fmpm_pdl_trigger at the top), so the launch
// latency and the tail of the grid are filled with the successor's prologue; the successor touches NO global memory before fmpm_pdl_wait,
// which returns once the predecessor grid has completed and its writes are visible.  Both are no-ops in a launch without the attribute.
// ---- TMA (cp.async.bulk.tensor) + mbarrier: one elected lane arms the warp's mbarrier with the byte count and issues the tile copy, every
// lane then waits on the barrier's phase.  The wait is bounded: a descriptor that never completes traps instead of hanging the GPU.
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, const unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, const unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* tm, unsigned long long* bar, const int c0, const int c1, const int c2, const int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
               ::"r"(smem_u32(dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, const unsigned phase) {
  unsigned done = 0;
  for (int it = 0; it < (1 << 22) && !done; it++)
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(smem_u32(bar)), "r"(phase) : "memory");
  if (!done) __trap();
}
__device__ __forceinline__ void fmpm_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void fmpm_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
template <class... Params, class... Args>
static inline void fmpm_launch_pdl(const bool pdl, void (*kern)(Params...), const int grid, const int block, const size_t smem, void* stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = smem; cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kern, static_cast<Params>(args)...);
}
#define FMPM_LAUNCH_PDL(pdl, kern, grid, block, smem, stream, ...) fmpm_launch_pdl(pdl, kern, grid, block, smem, stream, __VA_ARGS__)
#endif

#ifdef FMPM_HOST_EMU
__device__ __forceinline__ void atomic_add_f64(double* p, const double v) { std::atomic_ref<double>(*p).fetch_add(v, std::memory_order_relaxed); }
#else
__device__ __forceinline__ void atomic_add_f64(double* p, const double v) { atomicAdd(p, v); }   // native fp64 RED on sm_60+
#endif

// One-component sibling of param_grad_reduce (fmpm_backward.cu): the lanes in `live` add v to acc[row * stride], one fp64 atomic per (warp,
// row).  A warp of one row and 32 live lanes reduces with a butterfly; otherwise each group of lanes sharing a row sums through shuffles
// restricted to the group and its lowest lane issues the atomic.
__device__ __forceinline__ void row_sum_reduce(double* acc, const int stride, const unsigned live, const int row, const float v) {
  const unsigned peers = __match_any_sync(live, row);
  float a = v;
  if (peers == 0xffffffffu) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  } else {
    a = 0.f;
    for (unsigned m = peers; m != 0u; m &= m - 1u) a += __shfl_sync(peers, v, __ffs((int)m) - 1);
  }
  if ((int)(threadIdx.x & 31) == __ffs((int)peers) - 1) atomic_add_f64(acc + (size_t)row * stride, (double)a);
}

__device__ __forceinline__ void prefetch_l2(const void* p) {
#ifndef FMPM_HOST_EMU
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
#endif
}
// ---- neighbour handshake of the x-slab steps (k_slab_sync in fmpm_io.cu, and fused into k_grid_op_pull in fmpm_forward.cu)
#ifdef FMPM_HOST_EMU
#include <chrono>
#define FMPM_SYSTEM_FENCE() std::atomic_thread_fence(std::memory_order_seq_cst)
static inline unsigned long long fmpm_now_ns() { return (unsigned long long)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
#else
#define FMPM_SYSTEM_FENCE() __threadfence_system()
__device__ __forceinline__ unsigned long long fmpm_now_ns() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#endif
#ifndef FMPM_SYNC_TIMEOUT_NS
#define FMPM_SYNC_TIMEOUT_NS 10000000000ULL   // 10 s: ranks enter a step together (the migration census is a collective), real skews are microseconds
#endif
__device__ __forceinline__ void slab_wait(volatile int* slot, const int e, int* err) {
  if (*slot >= e) return;
  if (*(volatile int*)err) return;   // a handshake already timed out: fail fast from here on (the host reads the flag, SlabMPMSimulator.sync_error)
  const unsigned long long t0 = fmpm_now_ns();
  while (*slot < e) {
    if (fmpm_now_ns() - t0 > FMPM_SYNC_TIMEOUT_NS) { *err = 1; return; }   // never hang the GPU on a peer that stopped
  }
}

#define FMPM_CHECK_LAUNCH(h, name)                                                        \
  do {                                                                                    \
    cudaError_t e_ = cudaGetLastError();                                                  \
    if (e_ != cudaSuccess) {                                                              \
      snprintf((h)->err, sizeof((h)->err), "%s: %s", name, cudaGetErrorString(e_));       \
      return 1;                                                                           \
    }                                                                                     \
  } while (0)
