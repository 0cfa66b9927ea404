// oracle/smoke_oracle_capi.cpp — TEST INFRASTRUCTURE ONLY.  C interface (ctypes) of oracle/smoke_oracle.hpp; doubles at the boundary,
// the arithmetic runs in the precision chosen at creation (32: the reference's f32; 64: ground truth for finite differences).
#include "smoke_oracle.hpp"

using namespace orc;

namespace {
struct SHandle { int precision; Smoke<float>* f32; Smoke<double>* f64; };
#define SDISPATCH(h, expr) do { if ((h)->precision == 32) { auto& S = *(h)->f32; expr; } else { auto& S = *(h)->f64; expr; } } while (0)

template <class R> void set_frame_t(Smoke<R>& S, int s, const double* v, const double* vt, const double* dv, const double* p, const double* q) {
  const size_t o = (size_t)s * S.G;
  for (size_t i = 0; i < S.G * 3; i++) { S.v[o * 3 + i] = (R)v[i]; S.v_tmp[o * 3 + i] = (R)vt[i]; }
  for (size_t i = 0; i < S.G; i++) { S.dv[o + i] = (R)dv[i]; S.p[o + i] = (R)p[i]; }
  for (size_t i = 0; i < S.G * S.c.q_dim; i++) S.q[o * S.c.q_dim + i] = (R)q[i];
}
template <class R> void get_frame_t(Smoke<R>& S, int s, double* v, double* vt, double* dv, double* p, double* q, bool grad) {
  const size_t o = (size_t)s * S.G;
  auto &av = grad ? S.gv : S.v, &avt = grad ? S.gv_tmp : S.v_tmp, &adv = grad ? S.gdv : S.dv, &ap = grad ? S.gp : S.p, &aq = grad ? S.gq : S.q;
  for (size_t i = 0; i < S.G * 3; i++) { v[i] = av[o * 3 + i]; vt[i] = avt[o * 3 + i]; }
  for (size_t i = 0; i < S.G; i++) { dv[i] = adv[o + i]; p[i] = ap[o + i]; }
  for (size_t i = 0; i < S.G * S.c.q_dim; i++) q[i] = aq[o * S.c.q_dim + i];
}
template <class R> void set_grad_frame_t(Smoke<R>& S, int s, const double* v, const double* vt, const double* dv, const double* p, const double* q) {
  const size_t o = (size_t)s * S.G;
  for (size_t i = 0; i < S.G * 3; i++) { S.gv[o * 3 + i] = (R)v[i]; S.gv_tmp[o * 3 + i] = (R)vt[i]; }
  for (size_t i = 0; i < S.G; i++) { S.gdv[o + i] = (R)dv[i]; S.gp[o + i] = (R)p[i]; }
  for (size_t i = 0; i < S.G * S.c.q_dim; i++) S.gq[o * S.c.q_dim + i] = (R)q[i];
}
template <class R> void add_static_t(Smoke<R>& S, int res, const double* vox, const double* T) {
  SdfMesh<R> M; M.res = res; M.vox.resize((size_t)res * res * res);
  for (size_t i = 0; i < M.vox.size(); i++) M.vox[i] = (R)vox[i];
  for (int i = 0; i < 16; i++) M.T[i] = (R)T[i];
  for (int i = 0; i < 9; i++) M.Ainv[i] = 0;   // unused here (no normals)
  M.has_dynamics = 1;
  S.statics.push_back(M);
}
template <class R> void set_aircon_t(Smoke<R>& S, int f, const double* st) {
  for (int d = 0; d < 3; d++) S.a_pos[(size_t)f * 3 + d] = (R)st[d];
  for (int d = 0; d < 4; d++) S.a_quat[(size_t)f * 4 + d] = (R)st[3 + d];
  S.a_s[f] = (R)st[7]; S.a_r[f] = (R)st[8];
}
template <class R> void get_aircon_grad_t(Smoke<R>& S, int f, double* out) {
  for (int d = 0; d < 3; d++) out[d] = S.ga_pos[(size_t)f * 3 + d];
  for (int d = 0; d < 4; d++) out[3 + d] = S.ga_quat[(size_t)f * 4 + d];
  out[7] = S.ga_s[f]; out[8] = S.ga_r[f];
}
template <class R> void get_free_t(Smoke<R>& S, int s, int* out) { for (size_t i = 0; i < S.G; i++) out[i] = S.is_free[(size_t)s * S.G + i]; }
template <class R> void set_free_t(Smoke<R>& S, int s, const int* m) { for (size_t i = 0; i < S.G; i++) S.is_free[(size_t)s * S.G + i] = m[i] ? 1 : 0; }
}  // namespace

extern "C" {
void* orc_smoke_create(const SmokeConfig* cfg, int precision) {
  SHandle* h = new SHandle{precision, nullptr, nullptr};
  if (precision == 32) h->f32 = new Smoke<float>(*cfg); else h->f64 = new Smoke<double>(*cfg);
  return h;
}
void orc_smoke_destroy(void* hp) { SHandle* h = (SHandle*)hp; delete h->f32; delete h->f64; delete h; }
void orc_smoke_add_static(void* hp, int res, const double* vox, const double* T) { SHandle* h = (SHandle*)hp; SDISPATCH(h, add_static_t(S, res, vox, T)); }
void orc_smoke_set_aircon(void* hp, int f, const double* st) { SHandle* h = (SHandle*)hp; SDISPATCH(h, set_aircon_t(S, f, st)); }
void orc_smoke_get_aircon_grad(void* hp, int f, double* out) { SHandle* h = (SHandle*)hp; SDISPATCH(h, get_aircon_grad_t(S, f, out)); }
void orc_smoke_set_frame(void* hp, int s, const double* v, const double* vt, const double* dv, const double* p, const double* q) {
  SHandle* h = (SHandle*)hp; SDISPATCH(h, set_frame_t(S, s, v, vt, dv, p, q)); }
void orc_smoke_get_frame(void* hp, int s, double* v, double* vt, double* dv, double* p, double* q) {
  SHandle* h = (SHandle*)hp; SDISPATCH(h, get_frame_t(S, s, v, vt, dv, p, q, false)); }
void orc_smoke_set_grad_frame(void* hp, int s, const double* v, const double* vt, const double* dv, const double* p, const double* q) {
  SHandle* h = (SHandle*)hp; SDISPATCH(h, set_grad_frame_t(S, s, v, vt, dv, p, q)); }
void orc_smoke_get_grad_frame(void* hp, int s, double* v, double* vt, double* dv, double* p, double* q) {
  SHandle* h = (SHandle*)hp; SDISPATCH(h, get_frame_t(S, s, v, vt, dv, p, q, true)); }
void orc_smoke_get_free(void* hp, int s, int* out) { SHandle* h = (SHandle*)hp; SDISPATCH(h, get_free_t(S, s, out)); }
void orc_smoke_set_free(void* hp, int s, const int* mask) { SHandle* h = (SHandle*)hp; SDISPATCH(h, set_free_t(S, s, mask)); }
// one phase of Smoke<R> at a time (tests that compare the kernels launch by launch, each started from the kernel's own inputs)
void orc_smoke_free_space(void* hp, int s) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.compute_free_space(s)); }
void orc_smoke_advect(void* hp, int s, int f) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.advect_and_impulse(s, f)); }
void orc_smoke_divergence(void* hp, int s) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.divergence(s)); }
void orc_smoke_pressure(void* hp, int s) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.pressure_solve(s)); }
void orc_smoke_project(void* hp, int s) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.subtract_gradient(s)); }
void orc_smoke_project_grad(void* hp, int s) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.subtract_gradient_grad(s)); }
void orc_smoke_pressure_grad(void* hp, int s) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.pressure_solve_grad(s)); }
void orc_smoke_divergence_grad(void* hp, int s) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.divergence_grad(s)); }
void orc_smoke_advect_grad(void* hp, int s, int f) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.advect_and_impulse_grad(s, f)); }
void orc_smoke_step(void* hp, int s, int f) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.step(s, f)); }
void orc_smoke_step_grad(void* hp, int s, int f) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.step_grad(s, f)); }
void orc_smoke_reset_grad(void* hp) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.reset_grad()); }
void orc_smoke_copy_frame(void* hp, int a, int b) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.copy_frame(a, b)); }
void orc_smoke_copy_grad(void* hp, int a, int b) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.copy_grad(a, b)); }
void orc_smoke_reset_grad_till_frame(void* hp, int s) { SHandle* h = (SHandle*)hp; SDISPATCH(h, S.reset_grad_till_frame(s)); }
}
