// fmpm_io.cu — handle management, frame ring io, cell sort, grad permutation, effector pose chain and the
// index-matched shape loss of libfluidmpm.so.  Reference semantics cited per entry point in include/fluidmpm.h.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <cub/device/device_radix_sort.cuh>
#include "fmpm_common.cuh"
#include "fmpm_scatter.cuh"

#define FMPM_ABI_VERSION 2

extern "C" int fmpm_abi_version(void) { return FMPM_ABI_VERSION; }

extern "C" int fmpm_create(const FmpmConfig* cfg, FmpmHandle** out) {
  if (!cfg || !out) return 1;
  FmpmHandle* h = new (std::nothrow) FmpmHandle();
  if (!h) return 1;
  h->cfg = *cfg; h->bound = false; h->err[0] = 0; h->sm_count = 132; h->fwd_mask = ~4;   // the lazy in-kernel grid_op (bit 2) is opt-in: it was slower than the separate k_grid_op launch
  { const char* e = getenv("FMPM_FWD_STRIDE"); h->fwd_stride = (e && e[0] == '1' && e[1] == 0) ? 1 : 0; }
  { const char* e = getenv("FMPM_PDL"); h->use_pdl = (e && e[0] == '0') ? 0 : 1; }
  h->slab_pull_ok = 0; h->slab_pull = 0;   // fmpm_set_slab_pull
  { const char* e = getenv("FMPM_SLAB_FSYNC"); h->slab_fsync = (e && e[0] == '1') ? 1 : 0; }   // opt-in: it was slower than the separate k_slab_sync launch
  memset(&h->buf, 0, sizeof(h->buf));
  memset(&h->col, 0, sizeof(h->col));
  memset(&h->slab, 0, sizeof(h->slab));
  memset(&h->bodies, 0, sizeof(h->bodies));
  memset(&h->pgrad, 0, sizeof(h->pgrad));
  memset(&h->cgrad, 0, sizeof(h->cgrad));
  memset(&h->mfield, 0, sizeof(h->mfield));
  memset(&h->mmass, 0, sizeof(h->mmass));
  memset(&h->mplastic, 0, sizeof(h->mplastic));
  *out = h;
  if (cfg->n_grid < 4 || cfg->n_particles < 0 || cfg->max_substeps_local < 1 || cfg->n_materials < 1 || cfg->n_materials > 256) {
    snprintf(h->err, sizeof(h->err), "fmpm_create: invalid config (n_grid %d, n_particles %d, T %d, n_materials %d)", cfg->n_grid,
             cfg->n_particles, cfg->max_substeps_local, cfg->n_materials);
    return 1;
  }
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) {
    snprintf(h->err, sizeof(h->err), "fmpm_create: no CUDA device (this library has no CPU fallback)");
    return 1;
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, cfg->device) == cudaSuccess) h->sm_count = prop.multiProcessorCount;
  return 0;
}
extern "C" void fmpm_destroy(FmpmHandle* h) { delete h; }
extern "C" const char* fmpm_last_error(FmpmHandle* h) { return h ? h->err : "null handle"; }

static void fill_sdf(SdfDev& d, const FmpmSdfMesh& m) {
  d.vox = (const float*)m.voxels; d.res = m.res; d.friction = m.friction; d.softness = m.softness;
  for (int i = 0; i < 12; i++) d.T[i] = m.T_mesh_to_voxels[i];
  // R_voxels_to_mesh = T[:3,:3].inverse() evaluated in f32 like the reference kernels do (static.py:59)
  const float* T = m.T_mesh_to_voxels;
  const float a = T[0], b = T[1], c = T[2], d0 = T[4], e = T[5], f = T[6], g = T[8], hh = T[9], i = T[10];
  const float det = a * (e * i - f * hh) - b * (d0 * i - f * g) + c * (d0 * hh - e * g);
  d.Ainv[0] = (e * i - f * hh) / det; d.Ainv[1] = (c * hh - b * i) / det; d.Ainv[2] = (b * f - c * e) / det;
  d.Ainv[3] = (f * g - d0 * i) / det; d.Ainv[4] = (a * i - c * g) / det; d.Ainv[5] = (c * d0 - a * f) / det;
  d.Ainv[6] = (d0 * hh - e * g) / det; d.Ainv[7] = (b * g - a * hh) / det; d.Ainv[8] = (a * e - b * d0) / det;
}
extern "C" int fmpm_set_colliders(FmpmHandle* h, const FmpmColliders* c) {
  if (!h || !c) return 1;
  if (c->n_statics < 0 || c->n_statics > 4) { snprintf(h->err, sizeof(h->err), "fmpm_set_colliders: at most 4 statics (got %d)", c->n_statics); return 1; }
  if (c->has_rigid && (!c->pos || !c->quat || !c->rigid.voxels)) { snprintf(h->err, sizeof(h->err), "fmpm_set_colliders: rigid collider needs voxels, pos and quat"); return 1; }
  memset(&h->col, 0, sizeof(h->col));
  h->col.n_statics = c->n_statics;
  for (int s = 0; s < c->n_statics; s++) {
    if (!c->statics[s].voxels || c->statics[s].res < 2) { snprintf(h->err, sizeof(h->err), "fmpm_set_colliders: static %d has no SDF volume", s); return 1; }
    fill_sdf(h->col.statics[s], c->statics[s]);
  }
  h->col.has_rigid = c->has_rigid; h->col.collide_type = c->collide_type; h->col.y_min = c->collide_y_min;
  if (c->has_rigid) { fill_sdf(h->col.rigid, c->rigid); h->col.epos = (const float*)c->pos; h->col.equat = (const float*)c->quat; h->col.egpos = (float*)c->gpos; h->col.egquat = (float*)c->gquat; }
  return 0;
}

extern "C" int fmpm_set_param_grad(FmpmHandle* h, const FmpmParamGrad* g) {
  if (!h) return 1;
  if (g && ((g->gmat == nullptr) != (g->ggrav == nullptr))) {
    snprintf(h->err, sizeof(h->err), "fmpm_set_param_grad: gmat and ggrav must both be set or both be NULL"); return 1;
  }
  if (g) h->pgrad = *g; else memset(&h->pgrad, 0, sizeof(h->pgrad));
  if (!h->pgrad.gmat) memset(&h->cgrad, 0, sizeof(h->cgrad));   // the contact gradients ride on the parameter-gradient kernels
  return 0;
}
extern "C" int fmpm_set_contact_grad(FmpmHandle* h, const FmpmContactGrad* g) {
  if (!h) return 1;
  if (g && g->gcontact && !h->pgrad.gmat) {
    snprintf(h->err, sizeof(h->err), "fmpm_set_contact_grad: bind the parameter-gradient accumulators (fmpm_set_param_grad) first"); return 1;
  }
  if (g) h->cgrad = *g; else memset(&h->cgrad, 0, sizeof(h->cgrad));
  return 0;
}
extern "C" int fmpm_set_restitution(FmpmHandle* h, float restitution) {
  if (!h) return 1;
  if (!std::isfinite(restitution)) {
    snprintf(h->err, sizeof(h->err), "fmpm_set_restitution: restitution must be finite"); return 1;
  }
  h->cfg.restitution = restitution;
  return 0;
}
extern "C" int fmpm_set_gravity(FmpmHandle* h, const float g[3]) {
  if (!h || !g) return 1;
  for (int i = 0; i < 3; i++) h->cfg.gravity[i] = g[i];
  return 0;
}
extern "C" int fmpm_set_scene_flags(FmpmHandle* h, int scene_flags) {
  if (!h) return 1;
  if (scene_flags & ~FMPM_SCENE_ALL_LIQUID_MU0) { snprintf(h->err, sizeof(h->err), "fmpm_set_scene_flags: unknown bits 0x%x", scene_flags); return 1; }
  if ((scene_flags & FMPM_SCENE_ALL_LIQUID_MU0) && has_material_field(h)) {
    snprintf(h->err, sizeof(h->err), "fmpm_set_scene_flags: FMPM_SCENE_ALL_LIQUID_MU0 while a material field is bound (the all-liquid kernels take mu = 0)"); return 1;
  }
  h->cfg.scene_flags = scene_flags;
  return 0;
}
extern "C" int fmpm_set_material_field(FmpmHandle* h, const FmpmMaterialField* m) {
  if (!h) return 1;
  if (!m || !m->field) {
    if (has_mass_field(h)) { snprintf(h->err, sizeof(h->err), "fmpm_set_material_field: a mass field is bound (it runs with a mu, lam field): unbind it first"); return 1; }
    memset(&h->mfield, 0, sizeof(h->mfield)); return 0;
  }
  if (h->slab.enabled) { snprintf(h->err, sizeof(h->err), "fmpm_set_material_field: not available in x-slab mode"); return 1; }
  if (h->cfg.scene_flags & FMPM_SCENE_ALL_LIQUID_MU0) {
    snprintf(h->err, sizeof(h->err), "fmpm_set_material_field: clear FMPM_SCENE_ALL_LIQUID_MU0 first (the all-liquid kernels take mu = 0)"); return 1;
  }
  h->mfield = *m;
  return 0;
}
extern "C" int fmpm_set_mass_field(FmpmHandle* h, const FmpmMassField* m) {
  if (!h) return 1;
  if (!m || !m->mass) {
    if (has_plastic_field(h)) { snprintf(h->err, sizeof(h->err), "fmpm_set_mass_field: a plastic field is bound (it runs with a mass field): unbind it first"); return 1; }
    memset(&h->mmass, 0, sizeof(h->mmass)); return 0;
  }
  if (h->slab.enabled) { snprintf(h->err, sizeof(h->err), "fmpm_set_mass_field: not available in x-slab mode"); return 1; }
  if (!has_material_field(h)) {
    snprintf(h->err, sizeof(h->err), "fmpm_set_mass_field: bind a material field first (the mass-field kernels take mu, lam and mass per slot)"); return 1;
  }
  h->mmass = *m;
  return 0;
}
extern "C" int fmpm_set_plastic_field(FmpmHandle* h, const FmpmPlasticField* m) {
  if (!h) return 1;
  if (!m || !m->field) { memset(&h->mplastic, 0, sizeof(h->mplastic)); return 0; }
  if (h->slab.enabled) { snprintf(h->err, sizeof(h->err), "fmpm_set_plastic_field: not available in x-slab mode"); return 1; }
  if (!has_mass_field(h)) {
    snprintf(h->err, sizeof(h->err), "fmpm_set_plastic_field: bind a mass field first (the plastic-field kernels take mu, lam, the limits and mass per slot)"); return 1;
  }
  h->mplastic = *m;
  return 0;
}

extern "C" int fmpm_set_slab(FmpmHandle* h, const FmpmSlab* s) {
  if (!h || !s) return 1;
  if (s->enabled && has_plastic_field(h)) { snprintf(h->err, sizeof(h->err), "fmpm_set_slab: not available while a plastic field is bound"); return 1; }
  if (s->enabled && has_mass_field(h)) { snprintf(h->err, sizeof(h->err), "fmpm_set_slab: not available while a mass field is bound"); return 1; }
  if (s->enabled && has_material_field(h)) { snprintf(h->err, sizeof(h->err), "fmpm_set_slab: not available while a material field is bound"); return 1; }
  if (s->enabled && ((s->peer_pm_left && s->left_hi <= s->left_lo) || (s->peer_pm_right && s->right_hi <= s->right_lo))) {
    snprintf(h->err, sizeof(h->err), "fmpm_set_slab: empty ghost plane range"); return 1;
  }
  h->slab = *s;
  return 0;
}

// neighbour handshake of the x-slab mode: epochs in peer-addressable memory.  A rank posts e = ++epoch into its neighbours' slots (after a
// system-scope fence: its peer reductions of the kernels before are visible first) and waits until both neighbours posted >= e.  The spin
// is bounded IN TIME (globaltimer): a rank that never arrives (a crashed peer) raises the error flag instead of hanging the GPU.
// (FMPM_SYSTEM_FENCE, fmpm_now_ns, slab_wait: fmpm_common.cuh — k_grid_op_pull runs the same handshake inside the grid_op launch)
__global__ void k_slab_sync(int* sig, int* peer_l, int* peer_r) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int e = sig[2] + 1;
  sig[2] = e;
  FMPM_SYSTEM_FENCE();
  if (peer_l) ((volatile int*)peer_l)[1] = e;   // I am my left neighbour's RIGHT neighbour
  if (peer_r) ((volatile int*)peer_r)[0] = e;   // and my right neighbour's LEFT neighbour
  FMPM_SYSTEM_FENCE();
  if (peer_l) slab_wait((volatile int*)sig + 0, e, sig + 3);
  if (peer_r) slab_wait((volatile int*)sig + 1, e, sig + 3);
  FMPM_SYSTEM_FENCE();
}
int fmpm_slab_sync_impl(FmpmHandle* h, void* stream);
extern "C" int fmpm_slab_sync(FmpmHandle* h, void* stream) { return fmpm_slab_sync_impl(h, stream); }
int fmpm_slab_sync_impl(FmpmHandle* h, void* stream) {
  if (!h) return 1;
  if (!h->slab.enabled || !h->slab.signal) { snprintf(h->err, sizeof(h->err), "fmpm_slab_sync: the handshake arrays were not set (FmpmSlab.signal)"); return 1; }
  FMPM_LAUNCH(k_slab_sync, 1, 32, 0, stream, (int*)h->slab.signal, (int*)h->slab.peer_signal_left, (int*)h->slab.peer_signal_right);
  FMPM_CHECK_LAUNCH(h, "fmpm_slab_sync");
  return 0;
}
int fmpm_fwd_step_impl(FmpmHandle* h, int f, int full, void* stream);   // fmpm_forward.cu: k_fwd (or k_g2p2g) with everything the scene allows
int fmpm_clear_blocks_launch(FmpmHandle* h, const KParams& P, void* stream);   // fmpm_forward.cu
// pull form of the ghost reduction (k_grid_op_pull, fmpm_forward.cu) when every neighbour's accumulator and flags are peer-addressable and the
// two ghost ranges of this slab do not overlap; otherwise the push form (kSlab scatter kernels)
extern "C" int fmpm_set_slab_pull(FmpmHandle* h, int on) { if (!h) return 1; h->slab_pull_ok = on ? 1 : 0; return 0; }
static bool slab_can_pull(const FmpmHandle* h) {
  const FmpmSlab& s = h->slab;
  if (!h->slab_pull_ok || !s.enabled) return false;
  if (!s.peer_pm_left && !s.peer_pm_right) return false;
  if ((s.peer_pm_left && !s.peer_flags_left) || (s.peer_pm_right && !s.peer_flags_right)) return false;
  if (s.peer_pm_left && s.peer_pm_right && s.left_hi > s.right_lo) return false;
  return true;
}
extern "C" int fmpm_substeps_slab(FmpmHandle* h, int f0, int n, int fuse, void* stream) {
  if (!h) return 1;
  if (n < 1) { snprintf(h->err, sizeof(h->err), "fmpm_substeps_slab: n must be >= 1"); return 1; }
  h->slab_pull = slab_can_pull(h) ? 1 : 0;
  int rc = 0;
  for (int i = 0; i < n && !rc; i++) {
    const int f = f0 + i;
    if (!(fuse && i > 0)) rc = fmpm_p2g(h, f, 1, stream);    // fused: the previous substep's g2p2g scattered frame f already
    if (!rc) rc = ((h->slab_pull && h->slab_fsync) ? 0 : fmpm_slab_sync(h, stream)) || fmpm_grid_op(h, f, 1, stream);   // pull form: the handshake runs inside k_grid_op_pull
    if (rc) break;
    if (fuse && i + 1 < n) rc = fmpm_fwd_step_impl(h, f, i + 2 == n, stream);   // the last fused substep completes F[f+2] (all-liquid scenes)
    else rc = fmpm_g2p(h, f, stream);
  }
  if (!rc && h->slab_pull) {   // the ghost blocks of the last substep: cleared once the neighbours are known to have read them
    rc = fmpm_slab_sync(h, stream) || fmpm_clear_blocks_launch(h, make_kparams(h, -1, f0 + n - 1), stream);
  }
  h->slab_pull = 0;
  return rc ? 1 : 0;
}

static int sort_bits(const FmpmHandle* h) {
  long long G = (long long)h->cfg.n_grid * h->cfg.n_grid * h->cfg.n_grid;  // keys in [0, G]
  int bits = 1;
  while ((1LL << bits) <= G) bits++;
  return bits;
}
extern "C" unsigned long long fmpm_sort_workspace_bytes(FmpmHandle* h) {
  size_t bytes = 0;
  int N = h->cfg.n_particles > 0 ? h->cfg.n_particles : 1;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const int*)nullptr, (int*)nullptr, (const int*)nullptr, (int*)nullptr, N, 0, sort_bits(h));
  return (unsigned long long)bytes + 256;
}
// TMA descriptors of grid_v for k_fwd's footprint tile: the grid as a rank-4 float tensor (component, z, y, x) with boxes of 4 x {8, 16} x 4 x 4
// elements = 4 x 4 node columns of 8 / 16 nodes.  The encoder lives in the driver (cuTensorMapEncodeTiled): fetched through the runtime,
// so the library has no link-time dependency on libcuda.  Any failure leaves tma_ok = 0 and k_fwd stages its tile with plain loads.
static void fmpm_encode_tensor_maps(FmpmHandle* h) {
  h->tma_ok = 0;
#ifndef FMPM_HOST_EMU
  const char* e = getenv("FMPM_TMA");
  if (e && e[0] == '0') return;
  if (!h->buf.grid_v) return;
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                               CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) { cudaGetLastError(); return; }
  const cuuint64_t n = (cuuint64_t)h->cfg.n_grid;
  const cuuint64_t dims[4] = {4, n, n, n};
  const cuuint64_t strides[3] = {16, n * 16, n * n * 16};   // bytes, dimensions 1..3
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  for (int k = 0; k < 2; k++) {
    const cuuint32_t box[4] = {4, k == 0 ? 8u : 16u, 4, 4};
    CUtensorMap* tm = k == 0 ? &h->tm_gv8 : &h->tm_gv16;
    if (((EncodeFn)fn)(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, h->buf.grid_v, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                       CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) return;
  }
  h->tma_ok = 1;
#endif
}
extern "C" int fmpm_bind(FmpmHandle* h, const FmpmBuffers* b) {
  if (!h || !b) return 1;
  if (!b->pa || !b->pf || !b->pf8 || !b->grid_pm || !b->grid_v || !b->materials) {
    snprintf(h->err, sizeof(h->err), "fmpm_bind: state ring / grid / material table pointers must be non-null");
    return 1;
  }
  h->buf = *b; h->bound = true;
  fmpm_encode_tensor_maps(h);
  return 0;
}

#define CHECK_BOUND(h, name)                                                                         \
  do {                                                                                               \
    if (!(h)) return 1;                                                                              \
    if (!(h)->bound) { snprintf((h)->err, sizeof((h)->err), "%s: fmpm_bind() has not been called", name); return 1; } \
  } while (0)
#define CHECK_CUDA(h, name, call)                                                                    \
  do {                                                                                               \
    cudaError_t e_ = (call);                                                                         \
    if (e_ != cudaSuccess) { snprintf((h)->err, sizeof((h)->err), "%s: %s", name, cudaGetErrorString(e_)); return 1; } \
  } while (0)

// ---------------------------------------------------------------------------------------------
// frame io (API layout <-> planar slot layout)
// ---------------------------------------------------------------------------------------------
__global__ void k_write_planar(const KParams P, float4* __restrict__ pa, float4* __restrict__ pf, float* __restrict__ pf8, const int f,
                               const float* __restrict__ x, const float* __restrict__ v, const float* __restrict__ C, const float* __restrict__ F,
                               const int* __restrict__ used, const int* __restrict__ mrow, const int* __restrict__ ids) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= P.N) return;
  const int p = ids ? ids[s] : s;
  int meta = 0;
  if (used) meta = (used[p] ? 1 : 0) | ((mrow ? mrow[p] : 0) << 8);
  const float* xp = x + (size_t)p * 3; const float* vp = v + (size_t)p * 3; const float* Cp = C + (size_t)p * 9; const float* Fp = F + (size_t)p * 9;
  pa[pa_idx(P, f, 0, s)] = make_float4(xp[0], xp[1], xp[2], __int_as_float(meta));
  pa[pa_idx(P, f, 1, s)] = make_float4(vp[0], vp[1], vp[2], Cp[0]);
  pa[pa_idx(P, f, 2, s)] = make_float4(Cp[1], Cp[2], Cp[3], Cp[4]);
  pa[pa_idx(P, f, 3, s)] = make_float4(Cp[5], Cp[6], Cp[7], Cp[8]);
  pf[pf_idx(P, f, 0, s)] = make_float4(Fp[0], Fp[1], Fp[2], Fp[3]);
  pf[pf_idx(P, f, 1, s)] = make_float4(Fp[4], Fp[5], Fp[6], Fp[7]);
  pf8[pf8_idx(P, f, s)] = Fp[8];
}
__global__ void k_read_planar(const KParams P, const float4* __restrict__ pa, const float4* __restrict__ pf, const float* __restrict__ pf8, const int f,
                              float* __restrict__ x, float* __restrict__ v, float* __restrict__ C, float* __restrict__ F, int* __restrict__ used,
                              const int* __restrict__ ids) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= P.N) return;
  const int p = ids ? ids[s] : s;
  const float4 a0 = pa[pa_idx(P, f, 0, s)];
  if (x) { x[(size_t)p * 3] = a0.x; x[(size_t)p * 3 + 1] = a0.y; x[(size_t)p * 3 + 2] = a0.z; }
  if (used) used[p] = __float_as_int(a0.w) & 1;
  if (v || C) {
    const float4 a1 = pa[pa_idx(P, f, 1, s)];
    if (v) { v[(size_t)p * 3] = a1.x; v[(size_t)p * 3 + 1] = a1.y; v[(size_t)p * 3 + 2] = a1.z; }
    if (C) {
      const float4 a2 = pa[pa_idx(P, f, 2, s)], a3 = pa[pa_idx(P, f, 3, s)];
      float* Cp = C + (size_t)p * 9;
      Cp[0] = a1.w; Cp[1] = a2.x; Cp[2] = a2.y; Cp[3] = a2.z; Cp[4] = a2.w; Cp[5] = a3.x; Cp[6] = a3.y; Cp[7] = a3.z; Cp[8] = a3.w;
    }
  }
  if (F) {
    const float4 f0 = pf[pf_idx(P, f, 0, s)], f1 = pf[pf_idx(P, f, 1, s)];
    float* Fp = F + (size_t)p * 9;
    Fp[0] = f0.x; Fp[1] = f0.y; Fp[2] = f0.z; Fp[3] = f0.w; Fp[4] = f1.x; Fp[5] = f1.y; Fp[6] = f1.z; Fp[7] = f1.w;
    Fp[8] = pf8[pf8_idx(P, f, s)];
  }
}

static inline int nblk(int n, int t) { return (n + t - 1) / t; }

extern "C" int fmpm_write_frame(FmpmHandle* h, int f, const void* x, const void* v, const void* C, const void* F, const void* used,
                                const void* mrow, const void* ids, void* stream) {
  CHECK_BOUND(h, "fmpm_write_frame");
  if (f < 0 || f > h->cfg.max_substeps_local) { snprintf(h->err, sizeof(h->err), "fmpm_write_frame: frame %d out of range", f); return 1; }
  if (!x || !v || !C || !F || !used) { snprintf(h->err, sizeof(h->err), "fmpm_write_frame: null input"); return 1; }
  KParams P = make_kparams(h);
  if (P.N == 0) return 0;
  FMPM_LAUNCH(k_write_planar, nblk(P.N, 256), 256, 0, stream, P, P.pa, P.pf, P.pf8, f, (const float*)x, (const float*)v, (const float*)C,
                                                                     (const float*)F, (const int*)used, (const int*)mrow, (const int*)ids);
  FMPM_CHECK_LAUNCH(h, "fmpm_write_frame");
  return 0;
}
extern "C" int fmpm_read_frame(FmpmHandle* h, int f, void* x, void* v, void* C, void* F, void* used, const void* ids, void* stream) {
  CHECK_BOUND(h, "fmpm_read_frame");
  if (f < 0 || f > h->cfg.max_substeps_local) { snprintf(h->err, sizeof(h->err), "fmpm_read_frame: frame %d out of range", f); return 1; }
  KParams P = make_kparams(h);
  if (P.N == 0) return 0;
  FMPM_LAUNCH(k_read_planar, nblk(P.N, 256), 256, 0, stream, P, P.pa, P.pf, P.pf8, f, (float*)x, (float*)v, (float*)C, (float*)F, (int*)used,
                                                                    (const int*)ids);
  FMPM_CHECK_LAUNCH(h, "fmpm_read_frame");
  return 0;
}
extern "C" int fmpm_write_grad(FmpmHandle* h, int g, const void* x, const void* v, const void* C, const void* F, const void* ids, void* stream) {
  CHECK_BOUND(h, "fmpm_write_grad");
  if (!h->buf.ga || (g & ~1)) { snprintf(h->err, sizeof(h->err), "fmpm_write_grad: no grad buffers / bad index"); return 1; }
  KParams P = make_kparams(h);
  if (P.N == 0) return 0;
  FMPM_LAUNCH(k_write_planar, nblk(P.N, 256), 256, 0, stream, P, P.ga, P.gf, P.gf8, g, (const float*)x, (const float*)v, (const float*)C,
                                                                     (const float*)F, nullptr, nullptr, (const int*)ids);
  FMPM_CHECK_LAUNCH(h, "fmpm_write_grad");
  return 0;
}
extern "C" int fmpm_read_grad(FmpmHandle* h, int g, void* x, void* v, void* C, void* F, const void* ids, void* stream) {
  CHECK_BOUND(h, "fmpm_read_grad");
  if (!h->buf.ga || (g & ~1)) { snprintf(h->err, sizeof(h->err), "fmpm_read_grad: no grad buffers / bad index"); return 1; }
  KParams P = make_kparams(h);
  if (P.N == 0) return 0;
  FMPM_LAUNCH(k_read_planar, nblk(P.N, 256), 256, 0, stream, P, P.ga, P.gf, P.gf8, g, (float*)x, (float*)v, (float*)C, (float*)F, nullptr,
                                                                    (const int*)ids);
  FMPM_CHECK_LAUNCH(h, "fmpm_read_grad");
  return 0;
}
extern "C" int fmpm_zero_grad(FmpmHandle* h, int g, void* stream) {
  CHECK_BOUND(h, "fmpm_zero_grad");
  if (!h->buf.ga || (g & ~1)) { snprintf(h->err, sizeof(h->err), "fmpm_zero_grad: no grad buffers / bad index"); return 1; }
  const size_t N = h->cfg.n_particles;
  cudaStream_t st = (cudaStream_t)stream;
  CHECK_CUDA(h, "fmpm_zero_grad", cudaMemsetAsync((float4*)h->buf.ga + (size_t)g * 4 * N, 0, 4 * N * sizeof(float4), st));
  CHECK_CUDA(h, "fmpm_zero_grad", cudaMemsetAsync((float4*)h->buf.gf + (size_t)g * 2 * N, 0, 2 * N * sizeof(float4), st));
  CHECK_CUDA(h, "fmpm_zero_grad", cudaMemsetAsync((float*)h->buf.gf8 + (size_t)g * N, 0, N * sizeof(float), st));
  return 0;
}
extern "C" int fmpm_copy_frame(FmpmHandle* h, int src, int dst, void* stream) {
  CHECK_BOUND(h, "fmpm_copy_frame");
  const int T = h->cfg.max_substeps_local;
  if (src < 0 || src > T || dst < 0 || dst > T) { snprintf(h->err, sizeof(h->err), "fmpm_copy_frame: frame out of range"); return 1; }
  if (src == dst) return 0;
  const size_t N = h->cfg.n_particles;
  cudaStream_t st = (cudaStream_t)stream;
  CHECK_CUDA(h, "fmpm_copy_frame", cudaMemcpyAsync((float4*)h->buf.pa + (size_t)dst * 4 * N, (float4*)h->buf.pa + (size_t)src * 4 * N, 4 * N * sizeof(float4), cudaMemcpyDeviceToDevice, st));
  CHECK_CUDA(h, "fmpm_copy_frame", cudaMemcpyAsync((float4*)h->buf.pf + (size_t)dst * 2 * N, (float4*)h->buf.pf + (size_t)src * 2 * N, 2 * N * sizeof(float4), cudaMemcpyDeviceToDevice, st));
  CHECK_CUDA(h, "fmpm_copy_frame", cudaMemcpyAsync((float*)h->buf.pf8 + (size_t)dst * N, (float*)h->buf.pf8 + (size_t)src * N, N * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

// ---------------------------------------------------------------------------------------------
// grad permutation between slot orders
// ---------------------------------------------------------------------------------------------
__global__ void k_permute_grad(const KParams P, const int gsrc, const int gdst, const int* __restrict__ ids_src, const int* __restrict__ inv_dst) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= P.N) return;
  const int pid = ids_src ? ids_src[s] : s;
  const int d = inv_dst ? inv_dst[pid] : pid;
#pragma unroll
  for (int k = 0; k < 4; k++) P.ga[pa_idx(P, gdst, k, d)] = P.ga[pa_idx(P, gsrc, k, s)];
  P.gf[pf_idx(P, gdst, 0, d)] = P.gf[pf_idx(P, gsrc, 0, s)];
  P.gf[pf_idx(P, gdst, 1, d)] = P.gf[pf_idx(P, gsrc, 1, s)];
  P.gf8[pf8_idx(P, gdst, d)] = P.gf8[pf8_idx(P, gsrc, s)];
}
extern "C" int fmpm_permute_grad(FmpmHandle* h, int gsrc, int gdst, const void* ids_src, const void* inv_dst, void* stream) {
  CHECK_BOUND(h, "fmpm_permute_grad");
  if (!h->buf.ga || gsrc == gdst || ((gsrc | gdst) & ~1)) { snprintf(h->err, sizeof(h->err), "fmpm_permute_grad: bad buffers"); return 1; }
  KParams P = make_kparams(h);
  if (P.N == 0) return 0;
  FMPM_LAUNCH(k_permute_grad, nblk(P.N, 256), 256, 0, stream, P, gsrc, gdst, (const int*)ids_src, (const int*)inv_dst);
  FMPM_CHECK_LAUNCH(h, "fmpm_permute_grad");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// cell sort: key = linear index of the particle's stencil base cell (z fastest), unused/frozen last
// ---------------------------------------------------------------------------------------------
__global__ void k_sort_keys(const KParams P, const int f, int* __restrict__ keys, int* __restrict__ vals) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= P.N) return;
  const float4 a0 = P.pa[pa_idx(P, f, 0, s)];
  const float x[3] = {a0.x, a0.y, a0.z};
  int b[3]; float fx[3];
  int key = P.G;
  if ((__float_as_int(a0.w) & 1) && base_fx(P, x, b, fx)) key = (b[0] * P.n + b[1]) * P.n + b[2];
  keys[s] = key; vals[s] = s;
}
__global__ void k_reorder(const KParams P, const int f, const int* __restrict__ src_of, const int* __restrict__ ids_in, int* __restrict__ ids_out,
                          int* __restrict__ inv_out, float4* __restrict__ sa, float4* __restrict__ sf, float* __restrict__ sf8) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P.N) return;
  const int s = src_of[j];
  const size_t N = P.N;
#pragma unroll
  for (int k = 0; k < 4; k++) sa[k * N + j] = P.pa[pa_idx(P, f, k, s)];
  sf[j] = P.pf[pf_idx(P, f, 0, s)]; sf[N + j] = P.pf[pf_idx(P, f, 1, s)];
  sf8[j] = P.pf8[pf8_idx(P, f, s)];
  const int pid = ids_in ? ids_in[s] : s;
  ids_out[j] = pid; inv_out[pid] = j;
}
extern "C" int fmpm_sort(FmpmHandle* h, int f, const void* ids_in, void* ids_out, void* inv_out, void* stream) {
  CHECK_BOUND(h, "fmpm_sort");
  const FmpmBuffers& b = h->buf;
  if (!b.scratch_a || !b.scratch_f || !b.scratch_f8 || !b.sort_keys_in || !b.sort_keys_out || !b.sort_vals_in || !b.sort_vals_out || !b.sort_tmp) {
    snprintf(h->err, sizeof(h->err), "fmpm_sort: sort workspace was not bound"); return 1;
  }
  if (f < 0 || f > h->cfg.max_substeps_local || !ids_out || !inv_out) { snprintf(h->err, sizeof(h->err), "fmpm_sort: bad arguments"); return 1; }
  KParams P = make_kparams(h);
  if (P.N == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  FMPM_LAUNCH(k_sort_keys, nblk(P.N, 256), 256, 0, st, P, f, (int*)b.sort_keys_in, (int*)b.sort_vals_in);
  FMPM_CHECK_LAUNCH(h, "fmpm_sort(keys)");
  size_t bytes = (size_t)b.sort_tmp_bytes;
  CHECK_CUDA(h, "fmpm_sort(radix)", cub::DeviceRadixSort::SortPairs(b.sort_tmp, bytes, (const int*)b.sort_keys_in, (int*)b.sort_keys_out,
                                                                    (const int*)b.sort_vals_in, (int*)b.sort_vals_out, P.N, 0, sort_bits(h), st));
  FMPM_LAUNCH(k_reorder, nblk(P.N, 256), 256, 0, st, P, f, (const int*)b.sort_vals_out, (const int*)ids_in, (int*)ids_out, (int*)inv_out, (float4*)b.scratch_a,
                                            (float4*)b.scratch_f, (float*)b.scratch_f8);
  FMPM_CHECK_LAUNCH(h, "fmpm_sort(reorder)");
  const size_t N = P.N;
  CHECK_CUDA(h, "fmpm_sort(copy)", cudaMemcpyAsync(P.pa + (size_t)f * 4 * N, b.scratch_a, 4 * N * sizeof(float4), cudaMemcpyDeviceToDevice, st));
  CHECK_CUDA(h, "fmpm_sort(copy)", cudaMemcpyAsync(P.pf + (size_t)f * 2 * N, b.scratch_f, 2 * N * sizeof(float4), cudaMemcpyDeviceToDevice, st));
  CHECK_CUDA(h, "fmpm_sort(copy)", cudaMemcpyAsync(P.pf8 + (size_t)f * N, b.scratch_f8, N * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

// ---------------------------------------------------------------------------------------------
// grid accessors (phase-level parity tests)
// ---------------------------------------------------------------------------------------------
__global__ void k_read_grid(const int G, const float4* __restrict__ a, const float4* __restrict__ b, float* __restrict__ o3a, float* __restrict__ o1a,
                            float* __restrict__ o3b) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  if (a) { const float4 t = a[g]; if (o3a) { o3a[(size_t)g * 3] = t.x; o3a[(size_t)g * 3 + 1] = t.y; o3a[(size_t)g * 3 + 2] = t.z; } if (o1a) o1a[g] = t.w; }
  if (b && o3b) { const float4 t = b[g]; o3b[(size_t)g * 3] = t.x; o3b[(size_t)g * 3 + 1] = t.y; o3b[(size_t)g * 3 + 2] = t.z; }
}
__global__ void k_write_grid(const int G, float4* __restrict__ a, float4* __restrict__ b, const float* __restrict__ i3a, const float* __restrict__ i1a,
                             const float* __restrict__ i3b) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  if (a && i3a) a[g] = make_float4(i3a[(size_t)g * 3], i3a[(size_t)g * 3 + 1], i3a[(size_t)g * 3 + 2], i1a ? i1a[g] : 0.f);
  if (b && i3b) b[g] = make_float4(i3b[(size_t)g * 3], i3b[(size_t)g * 3 + 1], i3b[(size_t)g * 3 + 2], 0.f);
}
extern "C" int fmpm_read_grid(FmpmHandle* h, void* v_in, void* mass, void* v_out, void* stream) {
  CHECK_BOUND(h, "fmpm_read_grid");
  KParams P = make_kparams(h);
  FMPM_LAUNCH(k_read_grid, nblk(P.G, 256), 256, 0, stream, P.G, P.grid_pm, P.grid_v, (float*)v_in, (float*)mass, (float*)v_out);
  FMPM_CHECK_LAUNCH(h, "fmpm_read_grid");
  return 0;
}
extern "C" int fmpm_read_grid_grad(FmpmHandle* h, void* gv_in, void* gmass, void* gv_out, void* stream) {
  CHECK_BOUND(h, "fmpm_read_grid_grad");
  KParams P = make_kparams(h);
  FMPM_LAUNCH(k_read_grid, nblk(P.G, 256), 256, 0, stream, P.G, P.ggrid_pm, P.ggrid_v, (float*)gv_in, (float*)gmass, (float*)gv_out);
  FMPM_CHECK_LAUNCH(h, "fmpm_read_grid_grad");
  return 0;
}
extern "C" int fmpm_write_grid_grad(FmpmHandle* h, const void* gv_in, const void* gmass, const void* gv_out, void* stream) {
  CHECK_BOUND(h, "fmpm_write_grid_grad");
  KParams P = make_kparams(h);
  FMPM_LAUNCH(k_write_grid, nblk(P.G, 256), 256, 0, stream, P.G, P.ggrid_pm, P.ggrid_v, (const float*)gv_in, (const float*)gmass, (const float*)gv_out);
  FMPM_CHECK_LAUNCH(h, "fmpm_write_grid_grad");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// effector pose chain (one thread: O(n_substeps) scalars)
// ---------------------------------------------------------------------------------------------
__device__ void effector_impose_x(const FmpmEffector& e, const float* in, float* out, float* jac) {
#pragma unroll
  for (int k = 0; k < 9; k++) jac[k] = 0.f;
  float lo[3], hi[3];
  if (e.boundary_type == 0) { for (int i = 0; i < 3; i++) { lo[i] = e.b_lower[i]; hi[i] = e.b_upper[i]; } }
  else { lo[0] = 0.f; hi[0] = 1.f; lo[2] = 0.f; hi[2] = 1.f; lo[1] = e.b_lower[1]; hi[1] = e.b_upper[1]; }
  for (int i = 0; i < 3; i++) {
    const float m = fminf(in[i], hi[i]); bool pass = in[i] < hi[i];   // min(a,b): adjoint to a iff a < b
    const float mm = fmaxf(m, lo[i]); pass = pass && (lo[i] < m);      // max(a,b): adjoint to a iff b < a
    out[i] = mm; jac[i * 4] = pass ? 1.f : 0.f;
  }
  if (e.boundary_type == 1) {
    const float rx = in[0] - e.cyl_center[0], rz = in[2] - e.cyl_center[1];
    const float rn = sqrtf(rx * rx + rz * rz + FMPM_EPS);
    if (rn > e.cyl_radius) {
      const float R = e.cyl_radius;
      out[0] = rx / rn * R + e.cyl_center[0];
      out[2] = rz / rn * R + e.cyl_center[1];
      const float i3 = 1.f / (rn * rn * rn);
      jac[0] = R * (1.f / rn - rx * rx * i3); jac[2] = R * (-rx * rz * i3);
      jac[6] = R * (-rz * rx * i3);           jac[8] = R * (1.f / rn - rz * rz * i3);
    }
  }
}
__global__ void k_effector_step(const FmpmEffector e, const int s, const int s_global, const int ns, const float* __restrict__ action) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float* pos = (float*)e.pos; float* quat = (float*)e.quat; float* v = (float*)e.v; float* w = (float*)e.w; float* act = (float*)e.act;
  const int ad = e.action_dim;
  for (int j = 0; j < ad; j++) act[(size_t)s_global * ad + j] = action[j];              // set_action_kernel, effector.py:218-221
  for (int f = s * ns; f < (s + 1) * ns; f++) {
    if (ad > 0) {                                                                        // set_velocity, effector.py:252-260
      for (int k = 0; k < 3; k++) v[f * 3 + k] = act[(size_t)s_global * ad + k] * e.scale_v[k] / (float)ns;
      if (ad > 3) for (int k = 0; k < 3; k++) w[f * 3 + k] = act[(size_t)s_global * ad + k + 3] * e.scale_v[k + 3] / (float)ns;
    }
    float in[3], out[3], jac[9];                                                         // move_kernel, effector.py:157-161
    for (int k = 0; k < 3; k++) in[k] = pos[f * 3 + k] + v[f * 3 + k];
    effector_impose_x(e, in, out, jac);
    for (int k = 0; k < 3; k++) pos[(f + 1) * 3 + k] = out[k];
    const float wv[3] = {w[f * 3], w[f * 3 + 1], w[f * 3 + 2]};
    const float wn = sqrtf(wv[0] * wv[0] + wv[1] * wv[1] + wv[2] * wv[2] + FMPM_EPS);     // w2quat, utils/geom.py:18-28
    const float sh = sinf(wn * 0.5f);
    const float q[4] = {cosf(wn * 0.5f), wv[0] / wn * sh, wv[1] / wn * sh, wv[2] / wn * sh};
    const float* r = quat + f * 4;                                                       // qmul(q, r), utils/geom.py:7-16
    float o[4] = {r[0] * q[0] - r[1] * q[1] - r[2] * q[2] - r[3] * q[3], r[0] * q[1] + r[1] * q[0] - r[2] * q[3] + r[3] * q[2],
                  r[0] * q[2] + r[1] * q[3] + r[2] * q[0] - r[3] * q[1], r[0] * q[3] - r[1] * q[2] + r[2] * q[1] + r[3] * q[0]};
    const float on = sqrtf(o[0] * o[0] + o[1] * o[1] + o[2] * o[2] + o[3] * o[3]);
    for (int k = 0; k < 4; k++) quat[(f + 1) * 4 + k] = o[k] / on;
  }
}
__global__ void k_effector_step_grad(const FmpmEffector e, const int s, const int s_global, const int ns) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const float* pos = (const float*)e.pos; const float* v = (const float*)e.v; const float* quat = (const float*)e.quat; const float* w = (const float*)e.w;
  float* gpos = (float*)e.gpos; float* gv = (float*)e.gv; float* gw = (float*)e.gw; float* gquat = (float*)e.gquat; float* gact = (float*)e.gact;
  const int ad = e.action_dim;
  for (int f = (s + 1) * ns - 1; f >= s * ns; f--) {                                     // move_kernel.grad, effector.py:155
    float in[3], out[3], jac[9];
    for (int k = 0; k < 3; k++) in[k] = pos[f * 3 + k] + v[f * 3 + k];
    effector_impose_x(e, in, out, jac);
    for (int a = 0; a < 3; a++) {
      float g = 0.f;
      for (int b = 0; b < 3; b++) g += jac[b * 3 + a] * gpos[(f + 1) * 3 + b];
      gpos[f * 3 + a] += g; gv[f * 3 + a] += g;
    }
    if (gquat) {
      // quat[f+1] = normalize(qmul_raw(w2quat(w[f]), quat[f]))  (utils/geom.py:7-28): adjoints of quat[f] and w[f]
      const float* wv = w + f * 3; const float* r = quat + f * 4; const float* g1 = gquat + (f + 1) * 4;
      const float wn = sqrtf(wv[0] * wv[0] + wv[1] * wv[1] + wv[2] * wv[2] + FMPM_EPS);
      const float sh = sinf(wn * 0.5f), ch = cosf(wn * 0.5f);
      const float q[4] = {ch, wv[0] / wn * sh, wv[1] / wn * sh, wv[2] / wn * sh};
      const float o[4] = {r[0] * q[0] - r[1] * q[1] - r[2] * q[2] - r[3] * q[3], r[0] * q[1] + r[1] * q[0] - r[2] * q[3] + r[3] * q[2],
                          r[0] * q[2] + r[1] * q[3] + r[2] * q[0] - r[3] * q[1], r[0] * q[3] - r[1] * q[2] + r[2] * q[1] + r[3] * q[0]};
      const float on = sqrtf(o[0] * o[0] + o[1] * o[1] + o[2] * o[2] + o[3] * o[3]);
      float dd = 0.f;
      for (int k = 0; k < 4; k++) dd += o[k] / on * g1[k];
      float go[4];
      for (int k = 0; k < 4; k++) go[k] = (g1[k] - o[k] / on * dd) / on;
      const float gr[4] = {go[0] * q[0] + go[1] * q[1] + go[2] * q[2] + go[3] * q[3], -go[0] * q[1] + go[1] * q[0] + go[2] * q[3] - go[3] * q[2],
                           -go[0] * q[2] - go[1] * q[3] + go[2] * q[0] + go[3] * q[1], -go[0] * q[3] + go[1] * q[2] - go[2] * q[1] + go[3] * q[0]};
      const float gq[4] = {go[0] * r[0] + go[1] * r[1] + go[2] * r[2] + go[3] * r[3], -go[0] * r[1] + go[1] * r[0] - go[2] * r[3] + go[3] * r[2],
                           -go[0] * r[2] + go[1] * r[3] + go[2] * r[0] - go[3] * r[1], -go[0] * r[3] - go[1] * r[2] + go[2] * r[1] + go[3] * r[0]};
      for (int k = 0; k < 4; k++) gquat[f * 4 + k] += gr[k];
      float gwn = -sh * 0.5f * gq[0];
      for (int k = 0; k < 3; k++) gwn += gq[k + 1] * wv[k] * (ch * 0.5f * wn - sh) / (wn * wn);
      for (int k = 0; k < 3; k++) gw[f * 3 + k] += gq[k + 1] * sh / wn + gwn * wv[k] / wn;
    }
  }
  if (ad > 0) {                                                                          // set_velocity.grad, effector.py:270-274
    for (int f = s * ns; f < (s + 1) * ns; f++) {
      for (int k = 0; k < 3; k++) gact[(size_t)s_global * ad + k] += gv[f * 3 + k] * e.scale_v[k] / (float)ns;
      if (ad > 3) for (int k = 0; k < 3; k++) gact[(size_t)s_global * ad + k + 3] += gw[f * 3 + k] * e.scale_v[k + 3] / (float)ns;
    }
  }
}
__global__ void k_effector_apply_p(const FmpmEffector e, const int grad) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const float* act_p = (const float*)e.act_p;
  float in[3], out[3], jac[9];
  for (int k = 0; k < 3; k++) in[k] = act_p[k] * e.scale_p[k];
  effector_impose_x(e, in, out, jac);
  if (!grad) { float* pos = (float*)e.pos; for (int k = 0; k < 3; k++) pos[k] = out[k]; }
  else {
    const float* gpos = (const float*)e.gpos; float* gact_p = (float*)e.gact_p;
    for (int a = 0; a < 3; a++) { float g = 0.f; for (int b = 0; b < 3; b++) g += jac[b * 3 + a] * gpos[b]; gact_p[a] += g * e.scale_p[a]; }
  }
}
extern "C" int fmpm_effector_step(FmpmHandle* h, const FmpmEffector* e, int s, int s_global, const void* action, void* stream) {
  if (!h || !e) return 1;
  if ((s + 1) * h->cfg.n_substeps > h->cfg.max_substeps_local) { snprintf(h->err, sizeof(h->err), "fmpm_effector_step: step %d exceeds the local ring", s); return 1; }
  FMPM_LAUNCH(k_effector_step, 1, 32, 0, stream, *e, s, s_global, h->cfg.n_substeps, (const float*)action);
  FMPM_CHECK_LAUNCH(h, "fmpm_effector_step");
  return 0;
}
extern "C" int fmpm_effector_step_grad(FmpmHandle* h, const FmpmEffector* e, int s, int s_global, void* stream) {
  if (!h || !e) return 1;
  FMPM_LAUNCH(k_effector_step_grad, 1, 32, 0, stream, *e, s, s_global, h->cfg.n_substeps);
  FMPM_CHECK_LAUNCH(h, "fmpm_effector_step_grad");
  return 0;
}
extern "C" int fmpm_effector_apply_action_p(FmpmHandle* h, const FmpmEffector* e, void* stream) {
  if (!h || !e) return 1;
  FMPM_LAUNCH(k_effector_apply_p, 1, 32, 0, stream, *e, 0);
  FMPM_CHECK_LAUNCH(h, "fmpm_effector_apply_action_p");
  return 0;
}
extern "C" int fmpm_effector_apply_action_p_grad(FmpmHandle* h, const FmpmEffector* e, void* stream) {
  if (!h || !e) return 1;
  FMPM_LAUNCH(k_effector_apply_p, 1, 32, 0, stream, *e, 1);
  FMPM_CHECK_LAUNCH(h, "fmpm_effector_apply_action_p_grad");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// index-matched shape loss (losses/shapematching_loss.py:80-93)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_loss_chamfer(const KParams P, const int f, const int* __restrict__ ids, const float* __restrict__ tgt,
                                                      const unsigned mask, const float weight, float* __restrict__ out) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  float acc = 0.f;
  if (s < P.N) {
    const float4 a0 = P.pa[pa_idx(P, f, 0, s)];
    const int meta = __float_as_int(a0.w);
    const int row = (meta >> 8) & 0xff;
    if ((meta & 1) && row < 32 && ((mask >> row) & 1u)) {
      const int p = ids ? ids[s] : s;
      const float d0 = a0.x - tgt[(size_t)p * 3], d1 = a0.y - tgt[(size_t)p * 3 + 1], d2 = a0.z - tgt[(size_t)p * 3 + 2];
      acc = d0 * d0 + d1 * d1 + d2 * d2;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ float ws[8];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; i++) t += ws[i];
    if (t != 0.f) atomicAdd(out, t * weight);
  }
}
__global__ void k_loss_chamfer_grad(const KParams P, const int f, const int g, const int* __restrict__ ids, const float* __restrict__ tgt,
                                    const unsigned mask, const float weight) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= P.N) return;
  const float4 a0 = P.pa[pa_idx(P, f, 0, s)];
  const int meta = __float_as_int(a0.w);
  const int row = (meta >> 8) & 0xff;
  if ((meta & 1) && row < 32 && ((mask >> row) & 1u)) {
    const int p = ids ? ids[s] : s;
    float4 gx = P.ga[pa_idx(P, g, 0, s)];
    gx.x += 2.f * weight * (a0.x - tgt[(size_t)p * 3]);
    gx.y += 2.f * weight * (a0.y - tgt[(size_t)p * 3 + 1]);
    gx.z += 2.f * weight * (a0.z - tgt[(size_t)p * 3 + 2]);
    P.ga[pa_idx(P, g, 0, s)] = gx;
  }
}
extern "C" int fmpm_loss_chamfer(FmpmHandle* h, int f, const void* ids, const void* tgt, unsigned int mask, float weight, void* loss_out, void* stream) {
  CHECK_BOUND(h, "fmpm_loss_chamfer");
  KParams P = make_kparams(h);
  if (P.N == 0) return 0;
  FMPM_LAUNCH(k_loss_chamfer, nblk(P.N, 256), 256, 0, stream, P, f, (const int*)ids, (const float*)tgt, mask, weight, (float*)loss_out);
  FMPM_CHECK_LAUNCH(h, "fmpm_loss_chamfer");
  return 0;
}
extern "C" int fmpm_loss_chamfer_grad(FmpmHandle* h, int f, int g, const void* ids, const void* tgt, unsigned int mask, float weight, void* stream) {
  CHECK_BOUND(h, "fmpm_loss_chamfer_grad");
  if (!h->buf.ga || (g & ~1)) { snprintf(h->err, sizeof(h->err), "fmpm_loss_chamfer_grad: no grad buffers / bad index"); return 1; }
  KParams P = make_kparams(h);
  if (P.N == 0) return 0;
  FMPM_LAUNCH(k_loss_chamfer_grad, nblk(P.N, 256), 256, 0, stream, P, f, g, (const int*)ids, (const float*)tgt, mask, weight);
  FMPM_CHECK_LAUNCH(h, "fmpm_loss_chamfer_grad");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// correspondence-free density loss on the simulation grid (DESIGN.md §4):
//   m_i = sum_p m_p w_ip over the used, in-grid particles of the masked rows,  L = w_d sum_i (m_i - m*_i)^2 + w_s sum_i m_i phi*_i
// ---------------------------------------------------------------------------------------------
#define DL_THREADS 256
// the particle's deposit stencil: false when it deposits nothing (unused, row not in the mask, frozen at the grid edge, beyond N)
__device__ __forceinline__ bool density_particle(const KParams& P, const int f, const int s, const unsigned mask, int* b, float* fx, int& row) {
  if (s >= P.N) return false;
  const float4 a0 = P.pa[pa_idx(P, f, 0, s)];
  const int meta = __float_as_int(a0.w);
  row = (meta >> 8) & 0xff;
  const float x[3] = {a0.x, a0.y, a0.z};
  return (meta & 1) && row < 32 && ((mask >> row) & 1u) && base_fx(P, x, b, fx);
}
// One lane per slot.  The lanes of a warp that share a stencil base (MATCH.ANY on the cell key) sum their 27 weighted masses first: a
// segmented reduction along the group's lanes by pointer jumping (log2 of the largest group in the warp, full-warp shuffles, no divergence).
// The group's lowest lane then holds the 27 sums; it parks them in shared memory and the group's lanes issue the 27 float reductions
// round-robin, so a group of g lanes issues ceil(27 / g) RED instructions per lane instead of 27 per particle.  Slots need not be sorted:
// an aged or missing cell sort only makes the groups smaller.
// kMass: the particle's mass from the per-slot mass field (fmpm_set_mass_field) instead of its row; the k_loss_mfield_* entry points
template <bool kMass>
__device__ __forceinline__ void density_deposit_body(const KParams& P, const int f, const unsigned mask, float* __restrict__ mass) {
  __shared__ float park[DL_THREADS / 32][27][32];
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int b[3], row = 0; float fx[3];
  const bool ok = density_particle(P, f, s, mask, b, fx, row);
  const int key = ok ? (b[0] * P.n + b[1]) * P.n + b[2] : -1;
  const unsigned grp = __match_any_sync(0xffffffffu, key);
  float v[27];
  {
    float w[3][3];
    bspline(fx, w);
    const float m = ok ? (kMass ? __ldg(P.mmass + s) : P.mats[row].z) : 0.f;
#pragma unroll
    for (int t = 0; t < 27; t++) v[t] = m * w[t / 9][0] * w[(t / 3) % 3][1] * w[t % 3][2];
  }
  const unsigned above = grp & ~((2u << lane) - 1u);   // the group's lanes after mine (2u << 31 wraps to 0: none)
  int nxt = above ? __ffs((int)above) - 1 : -1;
  while (__any_sync(0xffffffffu, nxt >= 0)) {   // v = the sum over my lane and the next 2^k - 1 of my group, nxt = my 2^k-th successor
    const int src = nxt >= 0 ? nxt : lane;
#pragma unroll
    for (int t = 0; t < 27; t++) {
      const float o = __shfl_sync(0xffffffffu, v[t], src);
      if (nxt >= 0) v[t] += o;
    }
    const int n2 = __shfl_sync(0xffffffffu, nxt, src);
    nxt = nxt >= 0 ? n2 : -1;
  }
  const int leader = __ffs((int)grp) - 1;
  if (ok && lane == leader) {
#pragma unroll
    for (int t = 0; t < 27; t++) park[warp][t][lane] = v[t];
  }
  __syncwarp();
  if (!ok) return;
  const int rank = __popc(grp & ((1u << lane) - 1u)), gsz = __popc(grp);
  for (int t = rank; t < 27; t += gsz) {
    const int node = ((b[0] + t / 9) * P.n + b[1] + (t / 3) % 3) * P.n + b[2] + t % 3;
    atomicAdd(mass + node, park[warp][t][leader]);
  }
}
__global__ void __launch_bounds__(DL_THREADS) k_loss_density_deposit(const KParams P, const int f, const unsigned mask, float* __restrict__ mass) {
  density_deposit_body<false>(P, f, mask, mass);
}
__global__ void __launch_bounds__(DL_THREADS) k_loss_mfield_density_deposit(const KParams P, const int f, const unsigned mask, float* __restrict__ mass) {
  density_deposit_body<true>(P, f, mask, mass);
}
// dense over the nodes.  kGrad = false: loss_out[0] += L (fp32 partial sums per CTA, one atomic per CTA).  kGrad = true: m is overwritten
// with its adjoint gbar = 2 w_d (m - m*) + w_s phi*.  A NULL target / sdf reads as 0.
template <bool kGrad>
__global__ void __launch_bounds__(DL_THREADS) k_loss_density_node(const int G, float* __restrict__ mass, const float* __restrict__ target,
                                                                  const float* __restrict__ sdf, const float wd, const float ws, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float acc = 0.f;
  if (i < G) {
    const float m = mass[i], t = target ? target[i] : 0.f, phi = sdf ? sdf[i] : 0.f;
    if constexpr (kGrad) mass[i] = 2.f * wd * (m - t) + ws * phi;
    else acc = wd * (m - t) * (m - t) + ws * m * phi;
  }
  if constexpr (!kGrad) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __shared__ float ws_[DL_THREADS / 32];
    if ((threadIdx.x & 31) == 0) ws_[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int k = 0; k < DL_THREADS / 32; k++) t += ws_[k];
      if (t != 0.f) atomicAdd(out, t);
    }
  }
}
// One lane per slot: gathers gbar at the 27 nodes; x-plane of adjoint buffer g += m_p sum_i gbar_i grad w_ip (the base held fixed).
// kPG: also dL/dm of the particle's row, sum_i gbar_i w_ip, reduced per (warp, row) into P.pg_mat[row][2] (row_sum_reduce).
// kMass: m_p from the mass field, and with kPG dL/dm added to P.gmass[s] (one lane per slot: no atomics) instead of the row.
template <bool kPG, bool kMass>
__device__ __forceinline__ void density_grad_body(const KParams& P, const int f, const int g, const unsigned mask, const float* __restrict__ gbar) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  int b[3], row = 0; float fx[3];
  const bool ok = density_particle(P, f, s, mask, b, fx, row);
  float dm = 0.f;
  if (ok) {
    float w[3][3], dw[3][3];
    bspline(fx, w); bspline_d(fx, dw);
    float gx = 0.f, gy = 0.f, gz = 0.f;
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
      for (int j = 0; j < 3; j++)
#pragma unroll
        for (int k = 0; k < 3; k++) {
          const float gb = gbar[((b[0] + i) * P.n + b[1] + j) * P.n + b[2] + k];
          gx += gb * dw[i][0] * w[j][1] * w[k][2];
          gy += gb * w[i][0] * dw[j][1] * w[k][2];
          gz += gb * w[i][0] * w[j][1] * dw[k][2];
          dm += gb * w[i][0] * w[j][1] * w[k][2];
        }
    const float c = (kMass ? __ldg(P.mmass + s) : P.mats[row].z) * P.inv_dx;
    float4 a = P.ga[pa_idx(P, g, 0, s)];
    a.x += c * gx; a.y += c * gy; a.z += c * gz;
    P.ga[pa_idx(P, g, 0, s)] = a;
  }
  if constexpr (kPG && kMass) {
    if (ok) P.gmass[s] += dm;
  } else if constexpr (kPG) {
    const unsigned live = __ballot_sync(0xffffffffu, ok);
    if (ok) row_sum_reduce(P.pg_mat + 2, 4, live, row, dm);
  }
}
template <bool kPG>
__global__ void __launch_bounds__(DL_THREADS) k_loss_density_grad(const KParams P, const int f, const int g, const unsigned mask, const float* __restrict__ gbar) {
  density_grad_body<kPG, false>(P, f, g, mask, gbar);
}
template <bool kPG>
__global__ void __launch_bounds__(DL_THREADS) k_loss_mfield_density_grad(const KParams P, const int f, const int g, const unsigned mask, const float* __restrict__ gbar) {
  density_grad_body<kPG, true>(P, f, g, mask, gbar);
}
static int density_loss_args(FmpmHandle* h, const int f, const FmpmDensityLoss* l, const char* name) {
  if (f < 0 || f > h->cfg.max_substeps_local) { snprintf(h->err, sizeof(h->err), "%s: frame %d out of range", name, f); return 1; }
  if (!l || !l->mass) { snprintf(h->err, sizeof(h->err), "%s: no mass scratch (FmpmDensityLoss.mass)", name); return 1; }
  return 0;
}
// the loss gradients with parameter gradients and a mass field add dL/dm per slot
static int loss_gmass_check(FmpmHandle* h, const char* name) {
  if (has_mass_field(h) && h->pgrad.gmat && !h->mmass.gmass) {
    snprintf(h->err, sizeof(h->err), "%s: parameter gradients with a mass field need FmpmMassField.gmass", name); return 1;
  }
  return 0;
}
// zero the scratch and deposit frame f into it
static int density_deposit(FmpmHandle* h, const KParams& P, const int f, const FmpmDensityLoss* l, void* stream, const char* name) {
  CHECK_CUDA(h, name, cudaMemsetAsync(l->mass, 0, (size_t)P.G * sizeof(float), (cudaStream_t)stream));
  if (P.N > 0 && l->mrow_mask_lo) {
    if (P.mmass) FMPM_LAUNCH(k_loss_mfield_density_deposit, nblk(P.N, DL_THREADS), DL_THREADS, 0, stream, P, f, l->mrow_mask_lo, (float*)l->mass);
    else FMPM_LAUNCH(k_loss_density_deposit, nblk(P.N, DL_THREADS), DL_THREADS, 0, stream, P, f, l->mrow_mask_lo, (float*)l->mass);
    FMPM_CHECK_LAUNCH(h, name);
  }
  return 0;
}
extern "C" int fmpm_loss_density(FmpmHandle* h, int f, const FmpmDensityLoss* l, void* loss_out, void* stream) {
  CHECK_BOUND(h, "fmpm_loss_density");
  if (density_loss_args(h, f, l, "fmpm_loss_density")) return 1;
  if (!loss_out) { snprintf(h->err, sizeof(h->err), "fmpm_loss_density: loss_out is NULL"); return 1; }
  KParams P = make_kparams(h);
  if (density_deposit(h, P, f, l, stream, "fmpm_loss_density")) return 1;
  FMPM_LAUNCH(k_loss_density_node<false>, nblk(P.G, DL_THREADS), DL_THREADS, 0, stream, P.G, (float*)l->mass, (const float*)l->target, (const float*)l->sdf,
              l->w_density, l->w_sdf, (float*)loss_out);
  FMPM_CHECK_LAUNCH(h, "fmpm_loss_density");
  return 0;
}
extern "C" int fmpm_loss_density_grad(FmpmHandle* h, int f, int g, const FmpmDensityLoss* l, void* stream) {
  CHECK_BOUND(h, "fmpm_loss_density_grad");
  if (!h->buf.ga || (g & ~1)) { snprintf(h->err, sizeof(h->err), "fmpm_loss_density_grad: no grad buffers / bad index"); return 1; }
  if (density_loss_args(h, f, l, "fmpm_loss_density_grad") || loss_gmass_check(h, "fmpm_loss_density_grad")) return 1;
  KParams P = make_kparams(h);
  if (P.N == 0 || !l->mrow_mask_lo) return 0;   // no particle carries an adjoint
  if (density_deposit(h, P, f, l, stream, "fmpm_loss_density_grad")) return 1;
  FMPM_LAUNCH(k_loss_density_node<true>, nblk(P.G, DL_THREADS), DL_THREADS, 0, stream, P.G, (float*)l->mass, (const float*)l->target, (const float*)l->sdf,
              l->w_density, l->w_sdf, (float*)nullptr);
  FMPM_CHECK_LAUNCH(h, "fmpm_loss_density_grad");
  if (P.mmass) {
    if (P.pg_mat) FMPM_LAUNCH(k_loss_mfield_density_grad<true>, nblk(P.N, DL_THREADS), DL_THREADS, 0, stream, P, f, g, l->mrow_mask_lo, (const float*)l->mass);
    else FMPM_LAUNCH(k_loss_mfield_density_grad<false>, nblk(P.N, DL_THREADS), DL_THREADS, 0, stream, P, f, g, l->mrow_mask_lo, (const float*)l->mass);
  } else if (P.pg_mat) FMPM_LAUNCH(k_loss_density_grad<true>, nblk(P.N, DL_THREADS), DL_THREADS, 0, stream, P, f, g, l->mrow_mask_lo, (const float*)l->mass);
  else FMPM_LAUNCH(k_loss_density_grad<false>, nblk(P.N, DL_THREADS), DL_THREADS, 0, stream, P, f, g, l->mrow_mask_lo, (const float*)l->mass);
  FMPM_CHECK_LAUNCH(h, "fmpm_loss_density_grad");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// correspondence-free momentum loss on the simulation grid (DESIGN.md §4): the density loss's particles also deposit p2g's APIC momentum,
//   P_i = sum_p m_p w_ip u_ip, u_ip = v_p + C_p d_ip, d_ip = (o_i - fx_p) dx,
//   L = w_d sum_i (m_i - m*_i)^2 + w_s sum_i m_i phi*_i + w_m sum_i |P_i - P*_i|^2
// ---------------------------------------------------------------------------------------------
#define ML_REC 16   // floats parked per particle: m, fx[3], v[3], C[9] (plane 1 .. 3 order)
__device__ __forceinline__ float bspline_at(const float fx, const int o) {
  const float a = 1.5f - fx, b = fx - 1.0f, c = fx - 0.5f;
  return o == 0 ? 0.5f * a * a : (o == 1 ? 0.75f - b * b : 0.5f * c * c);
}
// Node-major.  Every selected lane parks its particle's record in shared memory, component-major with the lane fastest: the lanes of a group
// read one particle's component as a broadcast and the groups of a warp read distinct banks.  The lanes that share a stencil base (MATCH.ANY
// on the cell key) take the group's 27 nodes round-robin; a lane sums (P, m) at its node over the group's particles in lane order and issues
// one vector reduction.  Reducing the 108 values per particle through the density kernel's segmented shuffles would cost four times its
// shuffles; here a group of g lanes issues ceil(27 / g) RED.v4 per lane, and an unsorted frame (groups of one) 27 per particle.
template <bool kMass>   // kMass: m_p from the mass field
__device__ __forceinline__ void momentum_deposit_body(const KParams& P, const int f, const unsigned mask, float4* __restrict__ field) {
  __shared__ float park[DL_THREADS / 32][ML_REC][32];
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int b[3], row = 0; float fx[3];
  const bool ok = density_particle(P, f, s, mask, b, fx, row);
  const int key = ok ? (b[0] * P.n + b[1]) * P.n + b[2] : -1;
  const unsigned grp = __match_any_sync(0xffffffffu, key);
  if (ok) {
    const float4 a1 = P.pa[pa_idx(P, f, 1, s)], a2 = P.pa[pa_idx(P, f, 2, s)], a3 = P.pa[pa_idx(P, f, 3, s)];
    const float r[ML_REC] = {kMass ? __ldg(P.mmass + s) : P.mats[row].z, fx[0], fx[1], fx[2], a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w, a3.x, a3.y, a3.z, a3.w};
#pragma unroll
    for (int c = 0; c < ML_REC; c++) park[warp][c][lane] = r[c];
  }
  __syncwarp();
  if (!ok) return;
  const int rank = __popc(grp & ((1u << lane) - 1u)), gsz = __popc(grp);
  for (int t = rank; t < 27; t += gsz) {
    const int o[3] = {t / 9, (t / 3) % 3, t % 3};
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (unsigned m = grp; m != 0u; m &= m - 1u) {
      const int q = __ffs((int)m) - 1;
      float r[ML_REC];
#pragma unroll
      for (int c = 0; c < ML_REC; c++) r[c] = park[warp][c][q];
      float w = r[0], d[3];
#pragma unroll
      for (int a = 0; a < 3; a++) { w *= bspline_at(r[1 + a], o[a]); d[a] = ((float)o[a] - r[1 + a]) * P.dx; }
      acc.x += w * (r[4] + r[7] * d[0] + r[8] * d[1] + r[9] * d[2]);
      acc.y += w * (r[5] + r[10] * d[0] + r[11] * d[1] + r[12] * d[2]);
      acc.z += w * (r[6] + r[13] * d[0] + r[14] * d[1] + r[15] * d[2]);
      acc.w += w;
    }
    red_add_v4(field + ((b[0] + o[0]) * P.n + b[1] + o[1]) * P.n + b[2] + o[2], acc);
  }
}
__global__ void __launch_bounds__(DL_THREADS) k_loss_momentum_deposit(const KParams P, const int f, const unsigned mask, float4* __restrict__ field) {
  momentum_deposit_body<false>(P, f, mask, field);
}
__global__ void __launch_bounds__(DL_THREADS) k_loss_mfield_momentum_deposit(const KParams P, const int f, const unsigned mask, float4* __restrict__ field) {
  momentum_deposit_body<true>(P, f, mask, field);
}
// dense over the nodes.  kGrad = false: loss_out[0] += L (fp32 partial sums per CTA, one atomic per CTA).  kGrad = true: (P, m) is overwritten
// with its adjoint (b, a), b = 2 w_m (P - P*), a = 2 w_d (m - m*) + w_s phi*.  A NULL target / sdf reads as 0.
template <bool kGrad>
__global__ void __launch_bounds__(DL_THREADS) k_loss_momentum_node(const int G, float4* __restrict__ field, const float4* __restrict__ target,
                                                                   const float* __restrict__ sdf, const float wd, const float ws, const float wm,
                                                                   float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float acc = 0.f;
  if (i < G) {
    const float4 v = field[i], t = target ? target[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    const float phi = sdf ? sdf[i] : 0.f;
    const float ex = v.x - t.x, ey = v.y - t.y, ez = v.z - t.z, em = v.w - t.w;
    if constexpr (kGrad) field[i] = make_float4(2.f * wm * ex, 2.f * wm * ey, 2.f * wm * ez, 2.f * wd * em + ws * phi);
    else acc = wd * em * em + ws * v.w * phi + wm * (ex * ex + ey * ey + ez * ez);
  }
  if constexpr (!kGrad) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __shared__ float ws_[DL_THREADS / 32];
    if ((threadIdx.x & 31) == 0) ws_[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int k = 0; k < DL_THREADS / 32; k++) t += ws_[k];
      if (t != 0.f) atomicAdd(out, t);
    }
  }
}
// One lane per slot: gathers (b, a) at the 27 nodes and adds, with s_i = a_i + b_i . u_ip and the stencil base held fixed,
//   v += m_p sum_i w_ip b_i,  C += m_p sum_i w_ip b_i d_ip^T,  x += m_p sum_i [grad w_ip s_i - w_ip C_p^T b_i]   (d u_ip / d x = -C_p)
// into planes 0 .. 3 of adjoint buffer g.  kPG: also dL/dm of the particle's row, sum_i w_ip s_i, reduced per (warp, row) into
// P.pg_mat[row][2] (row_sum_reduce).  kMass: m_p from the mass field, and with kPG dL/dm added to P.gmass[s] instead of the row.
template <bool kPG, bool kMass>
__device__ __forceinline__ void momentum_grad_body(const KParams& P, const int f, const int g, const unsigned mask, const float4* __restrict__ adj) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  int b[3], row = 0; float fx[3];
  const bool ok = density_particle(P, f, s, mask, b, fx, row);
  float dm = 0.f;
  if (ok) {
    const float4 a1 = P.pa[pa_idx(P, f, 1, s)], a2 = P.pa[pa_idx(P, f, 2, s)], a3 = P.pa[pa_idx(P, f, 3, s)];
    const float v[3] = {a1.x, a1.y, a1.z};
    const float C[3][3] = {{a1.w, a2.x, a2.y}, {a2.z, a2.w, a3.x}, {a3.y, a3.z, a3.w}};
    float w[3][3], dw[3][3];
    bspline(fx, w); bspline_d(fx, dw);
    float gx[3] = {0.f, 0.f, 0.f}, gv[3] = {0.f, 0.f, 0.f}, gC[3][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
      for (int j = 0; j < 3; j++)
#pragma unroll
        for (int k = 0; k < 3; k++) {
          const float4 q = adj[((b[0] + i) * P.n + b[1] + j) * P.n + b[2] + k];
          const float d[3] = {((float)i - fx[0]) * P.dx, ((float)j - fx[1]) * P.dx, ((float)k - fx[2]) * P.dx};
          const float wt = w[i][0] * w[j][1] * w[k][2];
          const float bq[3] = {q.x, q.y, q.z}, bw[3] = {wt * q.x, wt * q.y, wt * q.z};
          float sc = q.w;
#pragma unroll
          for (int a = 0; a < 3; a++) {
            sc += bq[a] * (v[a] + C[a][0] * d[0] + C[a][1] * d[1] + C[a][2] * d[2]);
            gv[a] += bw[a];
#pragma unroll
            for (int e = 0; e < 3; e++) gC[a][e] += bw[a] * d[e];
          }
          gx[0] += sc * dw[i][0] * w[j][1] * w[k][2];
          gx[1] += sc * w[i][0] * dw[j][1] * w[k][2];
          gx[2] += sc * w[i][0] * w[j][1] * dw[k][2];
          dm += sc * wt;
        }
    const float m = kMass ? __ldg(P.mmass + s) : P.mats[row].z, c = m * P.inv_dx;
    float4 a0 = P.ga[pa_idx(P, g, 0, s)], g1 = P.ga[pa_idx(P, g, 1, s)], g2 = P.ga[pa_idx(P, g, 2, s)], g3 = P.ga[pa_idx(P, g, 3, s)];
    a0.x += c * gx[0] - m * (C[0][0] * gv[0] + C[1][0] * gv[1] + C[2][0] * gv[2]);
    a0.y += c * gx[1] - m * (C[0][1] * gv[0] + C[1][1] * gv[1] + C[2][1] * gv[2]);
    a0.z += c * gx[2] - m * (C[0][2] * gv[0] + C[1][2] * gv[1] + C[2][2] * gv[2]);
    g1.x += m * gv[0]; g1.y += m * gv[1]; g1.z += m * gv[2]; g1.w += m * gC[0][0];
    g2.x += m * gC[0][1]; g2.y += m * gC[0][2]; g2.z += m * gC[1][0]; g2.w += m * gC[1][1];
    g3.x += m * gC[1][2]; g3.y += m * gC[2][0]; g3.z += m * gC[2][1]; g3.w += m * gC[2][2];
    P.ga[pa_idx(P, g, 0, s)] = a0; P.ga[pa_idx(P, g, 1, s)] = g1; P.ga[pa_idx(P, g, 2, s)] = g2; P.ga[pa_idx(P, g, 3, s)] = g3;
  }
  if constexpr (kPG && kMass) {
    if (ok) P.gmass[s] += dm;
  } else if constexpr (kPG) {
    const unsigned live = __ballot_sync(0xffffffffu, ok);
    if (ok) row_sum_reduce(P.pg_mat + 2, 4, live, row, dm);
  }
}
template <bool kPG>
__global__ void __launch_bounds__(DL_THREADS) k_loss_momentum_grad(const KParams P, const int f, const int g, const unsigned mask, const float4* __restrict__ adj) {
  momentum_grad_body<kPG, false>(P, f, g, mask, adj);
}
template <bool kPG>
__global__ void __launch_bounds__(DL_THREADS) k_loss_mfield_momentum_grad(const KParams P, const int f, const int g, const unsigned mask, const float4* __restrict__ adj) {
  momentum_grad_body<kPG, true>(P, f, g, mask, adj);
}
static int momentum_loss_args(FmpmHandle* h, const int f, const FmpmMomentumLoss* l, const char* name) {
  if (f < 0 || f > h->cfg.max_substeps_local) { snprintf(h->err, sizeof(h->err), "%s: frame %d out of range", name, f); return 1; }
  if (!l || !l->field) { snprintf(h->err, sizeof(h->err), "%s: no field scratch (FmpmMomentumLoss.field)", name); return 1; }
  return 0;
}
// zero the scratch and deposit (P, m) of frame f into it
static int momentum_deposit(FmpmHandle* h, const KParams& P, const int f, const FmpmMomentumLoss* l, void* stream, const char* name) {
  CHECK_CUDA(h, name, cudaMemsetAsync(l->field, 0, (size_t)P.G * sizeof(float4), (cudaStream_t)stream));
  if (P.N > 0 && l->mrow_mask_lo) {
    if (P.mmass) FMPM_LAUNCH(k_loss_mfield_momentum_deposit, nblk(P.N, DL_THREADS), DL_THREADS, 0, stream, P, f, l->mrow_mask_lo, (float4*)l->field);
    else FMPM_LAUNCH(k_loss_momentum_deposit, nblk(P.N, DL_THREADS), DL_THREADS, 0, stream, P, f, l->mrow_mask_lo, (float4*)l->field);
    FMPM_CHECK_LAUNCH(h, name);
  }
  return 0;
}
extern "C" int fmpm_loss_momentum(FmpmHandle* h, int f, const FmpmMomentumLoss* l, void* loss_out, void* stream) {
  CHECK_BOUND(h, "fmpm_loss_momentum");
  if (momentum_loss_args(h, f, l, "fmpm_loss_momentum")) return 1;
  if (!loss_out) { snprintf(h->err, sizeof(h->err), "fmpm_loss_momentum: loss_out is NULL"); return 1; }
  KParams P = make_kparams(h);
  if (momentum_deposit(h, P, f, l, stream, "fmpm_loss_momentum")) return 1;
  FMPM_LAUNCH(k_loss_momentum_node<false>, nblk(P.G, DL_THREADS), DL_THREADS, 0, stream, P.G, (float4*)l->field, (const float4*)l->target,
              (const float*)l->sdf, l->w_density, l->w_sdf, l->w_momentum, (float*)loss_out);
  FMPM_CHECK_LAUNCH(h, "fmpm_loss_momentum");
  return 0;
}
extern "C" int fmpm_loss_momentum_grad(FmpmHandle* h, int f, int g, const FmpmMomentumLoss* l, void* stream) {
  CHECK_BOUND(h, "fmpm_loss_momentum_grad");
  if (!h->buf.ga || (g & ~1)) { snprintf(h->err, sizeof(h->err), "fmpm_loss_momentum_grad: no grad buffers / bad index"); return 1; }
  if (momentum_loss_args(h, f, l, "fmpm_loss_momentum_grad") || loss_gmass_check(h, "fmpm_loss_momentum_grad")) return 1;
  KParams P = make_kparams(h);
  if (P.N == 0 || !l->mrow_mask_lo) return 0;   // no particle carries an adjoint
  if (momentum_deposit(h, P, f, l, stream, "fmpm_loss_momentum_grad")) return 1;
  FMPM_LAUNCH(k_loss_momentum_node<true>, nblk(P.G, DL_THREADS), DL_THREADS, 0, stream, P.G, (float4*)l->field, (const float4*)l->target,
              (const float*)l->sdf, l->w_density, l->w_sdf, l->w_momentum, (float*)nullptr);
  FMPM_CHECK_LAUNCH(h, "fmpm_loss_momentum_grad");
  if (P.mmass) {
    if (P.pg_mat) FMPM_LAUNCH(k_loss_mfield_momentum_grad<true>, nblk(P.N, DL_THREADS), DL_THREADS, 0, stream, P, f, g, l->mrow_mask_lo, (const float4*)l->field);
    else FMPM_LAUNCH(k_loss_mfield_momentum_grad<false>, nblk(P.N, DL_THREADS), DL_THREADS, 0, stream, P, f, g, l->mrow_mask_lo, (const float4*)l->field);
  } else if (P.pg_mat) FMPM_LAUNCH(k_loss_momentum_grad<true>, nblk(P.N, DL_THREADS), DL_THREADS, 0, stream, P, f, g, l->mrow_mask_lo, (const float4*)l->field);
  else FMPM_LAUNCH(k_loss_momentum_grad<false>, nblk(P.N, DL_THREADS), DL_THREADS, 0, stream, P, f, g, l->mrow_mask_lo, (const float4*)l->field);
  FMPM_CHECK_LAUNCH(h, "fmpm_loss_momentum_grad");
  return 0;
}

// =============================================================================================
// Adam on the composite action table (optimizer/optim.py:22-41, TrainablePolicy.optimize policies.py:152-164)
// =============================================================================================
// NumPy's evaluation order and dtypes: `(1 - beta) * grads` and `grads * grads` are float32 products (grads is float32, the Python scalar is
// weak), everything that touches the float64 moment buffers is float64; each operation rounds once (the _rn intrinsics keep ptxas from
// contracting a*b+c), so the table stays bit-identical to the reference's across iterations.
#ifdef FMPM_HOST_EMU
static inline double adam_dmul(double a, double b) { volatile double r = a * b; return r; }
static inline double adam_dadd(double a, double b) { volatile double r = a + b; return r; }
static inline float adam_fmul(float a, float b) { volatile float r = a * b; return r; }
static inline double adam_ddiv(double a, double b) { return a / b; }
static inline double adam_dsqrt(double a) { return sqrt(a); }
#else
__device__ __forceinline__ double adam_dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double adam_dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float adam_fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double adam_ddiv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double adam_dsqrt(double a) { return __dsqrt_rn(a); }
#endif
__global__ void k_adam_step(const FmpmAdamCfg c, double* __restrict__ params, double* __restrict__ m, double* __restrict__ v, const float* __restrict__ grads,
                            const unsigned char* __restrict__ trainable) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.rows * c.cols) return;
  const int row = i / c.cols, col = i % c.cols;
  float g = grads[i];
  if ((trainable && !trainable[row]) || (col < 32 && ((c.fix_dim_mask >> col) & 1u))) g = 0.f;
  const double m_t = adam_dadd(adam_dmul(c.beta_1, m[i]), (double)adam_fmul((float)(1.0 - c.beta_1), g));
  const double v_t = adam_dadd(adam_dmul(c.beta_2, v[i]), (double)adam_fmul((float)(1.0 - c.beta_2), adam_fmul(g, g)));
  m[i] = m_t; v[i] = v_t;
  const double m_cap = adam_ddiv(m_t, c.bias_1), v_cap = adam_ddiv(v_t, c.bias_2);
  double p = adam_dadd(params[i], -adam_ddiv(adam_dmul(c.lr, m_cap), adam_dadd(adam_dsqrt(v_cap), c.epsilon)));
  if (row < c.rows - 1) p = p < c.clip_lo ? c.clip_lo : (p > c.clip_hi ? c.clip_hi : p);   // ndarray.clip: min(max(p, lo), hi)
  params[i] = p;
}
extern "C" int fmpm_adam_step(FmpmHandle* h, const FmpmAdamCfg* c, void* params, void* m, void* v, const void* grads, const void* trainable, void* stream) {
  if (!h) return 1;
  if (!c || !params || !m || !v || !grads || c->rows < 1 || c->cols < 1 || c->cols > 32) {
    snprintf(h->err, sizeof(h->err), "fmpm_adam_step: null buffer or bad shape (rows >= 1, 1 <= cols <= 32)"); return 1;
  }
  const int n = c->rows * c->cols;
  FMPM_LAUNCH(k_adam_step, (n + 127) / 128, 128, 0, stream, *c, (double*)params, (double*)m, (double*)v, (const float*)grads, (const unsigned char*)trainable);
  FMPM_CHECK_LAUNCH(h, "fmpm_adam_step");
  return 0;
}
