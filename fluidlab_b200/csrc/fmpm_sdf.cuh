// fmpm_sdf.cuh — SDF mesh colliders on the device: Static.collide (meshes/static.py:26-104, called in grid_op MPM:388-390)
// and Dynamic.collide of a Rigid effector (meshes/dynamic.py:29-121 via effectors/rigid.py:36-38 and
// agents/agent_rigid.py:21-23; called in g2p MPM:419-422 and/or grid_op MPM:393-395), forward and adjoint.
// The baked volume format is the reference's pickle: voxels[res^3] + T_mesh_to_voxels (utils/mesh.py:63-87,
// meshes/mesh.py:121-127); 128^3 fp32 = 8 MB per mesh, L2 resident on H100 (50 MB L2).
#pragma once
#include "fmpm_common.cuh"

__device__ __forceinline__ void q_rot(const float* q, const float* v, float* o) {  // utils/geom.py:92-97
  const float uv0 = q[2] * v[2] - q[3] * v[1], uv1 = q[3] * v[0] - q[1] * v[2], uv2 = q[1] * v[1] - q[2] * v[0];
  const float uu0 = q[2] * uv2 - q[3] * uv1, uu1 = q[3] * uv0 - q[1] * uv2, uu2 = q[1] * uv1 - q[2] * uv0;
  o[0] = v[0] + 2.f * (q[0] * uv0 + uu0); o[1] = v[1] + 2.f * (q[0] * uv1 + uu1); o[2] = v[2] + 2.f * (q[0] * uv2 + uu2);
}
__device__ __forceinline__ void q_inv(const float* q, float* qi) {  // utils/geom.py:30-32
  const float n = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  qi[0] = q[0] / n; qi[1] = -q[1] / n; qi[2] = -q[2] / n; qi[3] = -q[3] / n;
}
// adjoint of o = q_rot(q, v) with respect to q (the polynomial of utils/geom.py:92-97 differentiated as written): gq += ...
__device__ __forceinline__ void q_rot_adj_q(const float* q, const float* v, const float* go, float* gq) {
  const float uv0 = q[2] * v[2] - q[3] * v[1], uv1 = q[3] * v[0] - q[1] * v[2], uv2 = q[1] * v[1] - q[2] * v[0];
  const float gu0 = 2.f * (q[0] * go[0] + go[1] * q[3] - go[2] * q[2]), gu1 = 2.f * (q[0] * go[1] + go[2] * q[1] - go[0] * q[3]),
              gu2 = 2.f * (q[0] * go[2] + go[0] * q[2] - go[1] * q[1]);   // adjoint of uv = 2 q0 go + 2 go x qv
  gq[0] += 2.f * (go[0] * uv0 + go[1] * uv1 + go[2] * uv2);
  gq[1] += 2.f * (uv1 * go[2] - uv2 * go[1]) + (v[1] * gu2 - v[2] * gu1);
  gq[2] += 2.f * (uv2 * go[0] - uv0 * go[2]) + (v[2] * gu0 - v[0] * gu2);
  gq[3] += 2.f * (uv0 * go[1] - uv1 * go[0]) + (v[0] * gu1 - v[1] * gu0);
}
// adjoint of qi = q_inv(q): gq += ...
__device__ __forceinline__ void q_inv_adj(const float* q, const float* qi, const float* gqi, float* gq) {
  const float n = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const float d = qi[0] * gqi[0] + qi[1] * gqi[1] + qi[2] * gqi[2] + qi[3] * gqi[3];
  gq[0] += (gqi[0] - qi[0] * d) / n; gq[1] -= (gqi[1] - qi[1] * d) / n; gq[2] -= (gqi[2] - qi[2] * d) / n; gq[3] -= (gqi[3] - qi[3] * d) / n;
}

// trilinear lookup, 1.0 outside (static.py:35-48); grad = d sdf / d pos_voxels when kGrad
template <bool kGrad>
__device__ __forceinline__ float sdf_lookup(const SdfDev& M, const float* pv, float* grad) {
  const float f0 = floorf(pv[0]), f1 = floorf(pv[1]), f2 = floorf(pv[2]);
  const int b0 = (int)f0, b1 = (int)f1, b2 = (int)f2;
  if (kGrad) { grad[0] = grad[1] = grad[2] = 0.f; }
  if (b0 >= M.res - 1 || b1 >= M.res - 1 || b2 >= M.res - 1 || b0 < 0 || b1 < 0 || b2 < 0) return 1.f;
  float sd = 0.f;
#pragma unroll
  for (int i = 0; i < 2; i++)
#pragma unroll
    for (int j = 0; j < 2; j++)
#pragma unroll
      for (int k = 0; k < 2; k++) {
        const float t0 = pv[0] - (float)(b0 + i), t1 = pv[1] - (float)(b1 + j), t2 = pv[2] - (float)(b2 + k);
        const float w0 = 1.f - fabsf(t0), w1 = 1.f - fabsf(t1), w2 = 1.f - fabsf(t2);
        const float val = __ldg(M.vox + ((size_t)(b0 + i) * M.res + (b1 + j)) * M.res + (b2 + k));
        sd += w0 * w1 * w2 * val;
        if (kGrad) {
          const float d0 = t0 > 0.f ? -1.f : (t0 < 0.f ? 1.f : 0.f), d1 = t1 > 0.f ? -1.f : (t1 < 0.f ? 1.f : 0.f), d2 = t2 > 0.f ? -1.f : (t2 < 0.f ? 1.f : 0.f);
          grad[0] += d0 * w1 * w2 * val; grad[1] += w0 * d1 * w2 * val; grad[2] += w0 * w1 * d2 * val;
        }
      }
  return sd;
}

// One collide evaluation.  Static: dynamic = false (pos/quat ignored).  kGrad: adjoints of (v, p) are ACCUMULATED into gv, gp and,
// for dynamic colliders, those of the poses of frames f / f+1 into gpose0[7] / gpose1[7] = (pos[3], quat[4]) (6-DOF Rigid
// effectors, agent_pouring.yaml; the quaternion part stays zero-gradient downstream when action_dim = 3).
// kPG (with kGrad): also ACCUMULATES the adjoints of the contact parameters into gparam[0] (friction) and gparam[1] (softness, dynamic only):
//   d friction += vn sbar / rtn   (flag set and rtn + vn friction > 0; sbar = sum_k rt_k infl gout_k; 0 on the sticky branch)
//   d softness += ginfl (-sd) infl   (ex < 1; the hit test carries no gradient)
template <bool kGrad, bool kPG = false>
__device__ __forceinline__ void sdf_collide(const SdfDev& M, const bool dynamic, const float* pos0, const float* q0, const float* pos1, const float* q1,
                                            const float dt, const float* p, const float* v, float* out, const float* gout, float* gv, float* gp,
                                            float* gpose0, float* gpose1, float* gparam = nullptr) {
  out[0] = v[0]; out[1] = v[1]; out[2] = v[2];
  float qi[4] = {1.f, 0.f, 0.f, 0.f}, pm[3] = {p[0], p[1], p[2]}, d0[3] = {0.f, 0.f, 0.f};
  if (dynamic) {
    q_inv(q0, qi);
#pragma unroll
    for (int k = 0; k < 3; k++) d0[k] = p[k] - pos0[k];
    q_rot(qi, d0, pm);
  }
  float pv[3];
#pragma unroll
  for (int r = 0; r < 3; r++) pv[r] = M.T[r * 4] * pm[0] + M.T[r * 4 + 1] * pm[1] + M.T[r * 4 + 2] * pm[2] + M.T[r * 4 + 3];
  float gsd[3];
  const float sd = sdf_lookup<kGrad>(M, pv, gsd);
  const float ex = dynamic ? expf(-sd * M.softness) : 1.f;
  const float infl = dynamic ? fminf(ex, 1.f) : 1.f;
  const bool hit = dynamic ? (sd <= 0.f || (M.softness > 0.f && infl > 0.1f)) : (sd <= 0.f);
  if (!hit) { if (kGrad) { gv[0] += gout[0]; gv[1] += gout[1]; gv[2] += gout[2]; } return; }
  float cv[3] = {0.f, 0.f, 0.f};
  if (dynamic) {
    float pw1[3]; q_rot(q1, pm, pw1);
#pragma unroll
    for (int k = 0; k < 3; k++) cv[k] = (pw1[k] + pos1[k] - p[k]) / dt;  // collider_v, dynamic.py:86-91
  }
  const bool sticky = dynamic && (M.friction > 10.f);
  float rel[3] = {0.f, 0.f, 0.f}, nvx[3] = {0.f, 0.f, 0.f}, gnorm = 1.f, un = 1.f, n[3] = {0.f, 0.f, 0.f}, vn = 0.f, m = 0.f, rt[3] = {0.f, 0.f, 0.f},
        rtn = 0.f, g = 0.f, rt2[3] = {0.f, 0.f, 0.f}, nm[3] = {0.f, 0.f, 0.f};
  bool flag = false;
  if (sticky) { out[0] = cv[0]; out[1] = cv[1]; out[2] = cv[2]; }
  else {
#pragma unroll
    for (int k = 0; k < 3; k++) rel[k] = v[k] - cv[k];
    // normal_: central differences of the trilinear SDF with delta = 1e-2 voxel (static.py:66-79)
    const float delta = 1e-2f;
    float graw[3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
      float inc[3] = {pv[0], pv[1], pv[2]}, dec[3] = {pv[0], pv[1], pv[2]};
      inc[i] += delta; dec[i] -= delta;
      graw[i] = (sdf_lookup<false>(M, inc, nullptr) - sdf_lookup<false>(M, dec, nullptr)) / (2.f * delta);
    }
    gnorm = sqrtf(graw[0] * graw[0] + graw[1] * graw[1] + graw[2] * graw[2] + FMPM_EPS);
#pragma unroll
    for (int i = 0; i < 3; i++) nvx[i] = graw[i] / gnorm;
    float u[3];
#pragma unroll
    for (int r = 0; r < 3; r++) nm[r] = M.Ainv[r * 3] * nvx[0] + M.Ainv[r * 3 + 1] * nvx[1] + M.Ainv[r * 3 + 2] * nvx[2];
    if (dynamic) q_rot(q0, nm, u); else { u[0] = nm[0]; u[1] = nm[1]; u[2] = nm[2]; }
    un = sqrtf(u[0] * u[0] + u[1] * u[1] + u[2] * u[2] + FMPM_EPS);
#pragma unroll
    for (int k = 0; k < 3; k++) n[k] = u[k] / un;
    vn = rel[0] * n[0] + rel[1] * n[1] + rel[2] * n[2];
    m = fminf(vn, 0.f);
#pragma unroll
    for (int k = 0; k < 3; k++) rt[k] = rel[k] - m * n[k];
    rtn = sqrtf(rt[0] * rt[0] + rt[1] * rt[1] + rt[2] * rt[2]);
    g = fmaxf(0.f, rtn + vn * M.friction);
    flag = (vn < 0.f) && (rtn > FMPM_EPS);
#pragma unroll
    for (int k = 0; k < 3; k++) { rt2[k] = flag ? rt[k] / rtn * g : rt[k]; out[k] = cv[k] + rt2[k] * infl + rel[k] * (1.f - infl); }
  }
  if (!kGrad) return;
  float gcv[3] = {gout[0], gout[1], gout[2]}, gpv[3] = {0.f, 0.f, 0.f}, gsdv = 0.f;
  if (!sticky) {
    float grt2[3], grel[3], ginfl = 0.f;
#pragma unroll
    for (int k = 0; k < 3; k++) { grt2[k] = infl * gout[k]; ginfl += gout[k] * (rt2[k] - rel[k]); grel[k] = (1.f - infl) * gout[k]; }
    float grt[3] = {0.f, 0.f, 0.f}, gvn = 0.f, gn[3] = {0.f, 0.f, 0.f};
    if (flag) {
      const float sc = g / rtn;
      float sbar = 0.f;
#pragma unroll
      for (int k = 0; k < 3; k++) { grt[k] += sc * grt2[k]; sbar += rt[k] * grt2[k]; }
      float grtn = -sbar * g / (rtn * rtn);
      if (rtn + vn * M.friction > 0.f) {
        grtn += sbar / rtn; gvn += sbar / rtn * M.friction;
        if constexpr (kPG) gparam[0] += vn * sbar / rtn;
      }
#pragma unroll
      for (int k = 0; k < 3; k++) grt[k] += grtn * rt[k] / rtn;
    } else {
#pragma unroll
      for (int k = 0; k < 3; k++) grt[k] += grt2[k];
    }
    float gm = 0.f;
#pragma unroll
    for (int k = 0; k < 3; k++) { grel[k] += grt[k]; gm -= grt[k] * n[k]; gn[k] -= m * grt[k]; }
    if (vn < 0.f) gvn += gm;
#pragma unroll
    for (int k = 0; k < 3; k++) { grel[k] += gvn * n[k]; gn[k] += gvn * rel[k]; }
#pragma unroll
    for (int k = 0; k < 3; k++) { gv[k] += grel[k]; gcv[k] -= grel[k]; }
    if (dynamic) {
      const float nd = n[0] * gn[0] + n[1] * gn[1] + n[2] * gn[2];
      float gu[3], gnm[3], gnvx[3], ggraw[3];
#pragma unroll
      for (int k = 0; k < 3; k++) gu[k] = (gn[k] - n[k] * nd) / un;
      q_rot(qi, gu, gnm);
      q_rot_adj_q(q0, nm, gu, gpose0 + 3);                                     // u = R(q0) nm
#pragma unroll
      for (int c = 0; c < 3; c++) gnvx[c] = M.Ainv[c] * gnm[0] + M.Ainv[3 + c] * gnm[1] + M.Ainv[6 + c] * gnm[2];
      const float nd2 = nvx[0] * gnvx[0] + nvx[1] * gnvx[1] + nvx[2] * gnvx[2];
#pragma unroll
      for (int k = 0; k < 3; k++) ggraw[k] = (gnvx[k] - nvx[k] * nd2) / gnorm;
      const float delta = 1e-2f;
#pragma unroll
      for (int i = 0; i < 3; i++) {
        float inc[3] = {pv[0], pv[1], pv[2]}, dec[3] = {pv[0], pv[1], pv[2]}, gi[3], gd[3];
        inc[i] += delta; dec[i] -= delta;
        sdf_lookup<true>(M, inc, gi); sdf_lookup<true>(M, dec, gd);
#pragma unroll
        for (int k = 0; k < 3; k++) gpv[k] += ggraw[i] * (gi[k] - gd[k]) / (2.f * delta);
      }
      if (ex < 1.f) {
        gsdv += ginfl * (-M.softness) * infl;
        if constexpr (kPG) gparam[1] += ginfl * (-sd) * infl;
      }
    }
  }
  if (dynamic) {
#pragma unroll
    for (int k = 0; k < 3; k++) gpv[k] += gsdv * gsd[k];
    float q1i[4]; q_inv(q1, q1i);
    const float t1[3] = {gcv[0] / dt, gcv[1] / dt, gcv[2] / dt};
    float gpm[3]; q_rot(q1i, t1, gpm);
    q_rot_adj_q(q1, pm, t1, gpose1 + 3);                                       // pw1 = R(q1) pm
#pragma unroll
    for (int k = 0; k < 3; k++) { gpose1[k] += t1[k]; gp[k] -= t1[k]; }
#pragma unroll
    for (int c = 0; c < 3; c++) gpm[c] += M.T[c] * gpv[0] + M.T[4 + c] * gpv[1] + M.T[8 + c] * gpv[2];
    float gd0[3]; q_rot(q0, gpm, gd0);
#pragma unroll
    for (int k = 0; k < 3; k++) { gp[k] += gd0[k]; gpose0[k] -= gd0[k]; }
    float gqi[4] = {0.f, 0.f, 0.f, 0.f};
    q_rot_adj_q(qi, d0, gpm, gqi);                                             // pm = R(inv(q0)) (p - pos0)
    q_inv_adj(q0, qi, gqi, gpose0 + 3);
  }
}

// agent.collide for AgentRigid (identity for other agents): reads the effector pose of frames f and f+1; kPG: gparam as in sdf_collide
template <bool kGrad, bool kPG = false>
__device__ __forceinline__ void agent_collide(const KParams& P, const int f, const float* p, const float* v, float* out, const float* gout, float* gv,
                                              float* gp, float* g0, float* g1, float* gparam = nullptr) {
  if (!(p[1] > P.col.y_min)) {  // AgentIceCreamDynamic.collide: identity below y_min
    out[0] = v[0]; out[1] = v[1]; out[2] = v[2];
    if (kGrad) { gv[0] += gout[0]; gv[1] += gout[1]; gv[2] += gout[2]; }
    return;
  }
  const float* pos0 = P.col.epos + f * 3; const float* pos1 = P.col.epos + (f + 1) * 3;
  const float* q0 = P.col.equat + f * 4; const float* q1 = P.col.equat + (f + 1) * 4;
  const float a0[3] = {pos0[0], pos0[1], pos0[2]}, a1[3] = {pos1[0], pos1[1], pos1[2]};
  const float b0[4] = {q0[0], q0[1], q0[2], q0[3]}, b1[4] = {q1[0], q1[1], q1[2], q1[3]};
  sdf_collide<kGrad, kPG>(P.col.rigid, true, a0, b0, a1, b1, P.dt, p, v, out, gout, gv, gp, g0, g1, gparam);
}

// warp-reduced accumulation of the effector pose adjoints of frames f / f+1 (g0[7], g1[7] = pos[3] + quat[4]) — one atomic per
// warp and component; gquat may be null (pose quaternion adjoint not requested)
__device__ __forceinline__ void reduce_pose_grad(float* gpos, float* gquat, const int f, const float* g0, const float* g1) {
#pragma unroll
  for (int i = 0; i < 14; i++) {
    float x = i < 7 ? g0[i] : g1[i - 7];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0 && x != 0.f) {
      const int ff = i < 7 ? f : f + 1, c = i < 7 ? i : i - 7;
      if (c < 3) atomicAdd(gpos + ff * 3 + c, x);
      else if (gquat) atomicAdd(gquat + ff * 4 + (c - 3), x);
    }
  }
}
