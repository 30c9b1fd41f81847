// Warp-per-environment rigid-body pipeline: kinematics, bias forces, mass matrix, collision.
// Everything is fp64 (the path's arithmetic type, like MuJoCo's mjtNum).  `ws` is this warp's shared-memory
// workspace (doubles), `wi` its int area; offsets come from the Layout in constant memory.
//
// Replaces the `mj_step` internals behind `self.sim.step()` (reference: MujocoController.py:379); the stage
// order and formulas follow SURVEY.md Appendix A.5.  Parallelisation pattern: a "lane loop"
//   for (i = lane; i < n; i += 32) ...
// over independent items (bodies, dofs, geoms, pairs, contacts), separated by __syncwarp().
#pragma once
#include "ge_math.cuh"
#include "ge_model.cuh"

namespace ge {

__constant__ DevModel c_m;
__constant__ Layout c_L;
__shared__ double* g_hovf;    // CTA-per-env build: HBM overflow row for the Hessian blocks of the env this CTA holds (may be null)
__constant__ int c_nancheck;  // GE_NANCHECK=1: record in status bits 8.. the first pipeline stage that produced a non-finite value

#define LANE_LOOP(i, n) for (int i = lane; i < (n); i += GE_LANES)

// ------------------------------------------------------------------------------------------------ kinematics
// Three lane-parallel phases, no level synchronisation: (1) every body's transform relative to its parent,
// (2) every body composes its own ancestor chain, (3) motion axes / spatial inertias / geom frames.
__device__ __noinline__ void stage_fk(double* ws, int lane) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double* qpos = ws + L.qpos;
  double *lpos = ws + L.lpos, *lquat = ws + L.lquat, *janchor = ws + L.janchor, *jaxis = ws + L.jaxis;
  LANE_LOOP(b, m.nbody) {
    double pos[3], quat[4], R[9], t[3];
    v3copy(pos, m.body_pos + 3 * b);
    for (int k = 0; k < 4; k++) quat[k] = m.body_quat[4 * b + k];
    int jn = m.body_jntnum[b], ja = m.body_jntadr[b];
    for (int k = 0; k < jn; k++) {
      int j = ja + k, qa = m.jnt_qposadr[j], type = m.jnt_type[j];
      if (type == J_FREE) {
        v3copy(pos, qpos + qa);
        for (int c = 0; c < 4; c++) quat[c] = qpos[qa + 3 + c];
        qnormalize(quat);
        v3copy(janchor + 3 * j, pos); v3set(jaxis + 3 * j, 0, 0, 1);
        continue;
      }
      q2mat(R, quat);
      m3mulv(t, R, m.jnt_pos + 3 * j); v3add(janchor + 3 * j, pos, t);
      m3mulv(jaxis + 3 * j, R, m.jnt_axis + 3 * j);
      if (type == J_SLIDE) {
        v3addscl(pos, pos, jaxis + 3 * j, qpos[qa] - m.qpos0[qa]);
      } else {
        double dq[4], nq[4];
        if (type == J_HINGE) qaxisangle(dq, m.jnt_axis + 3 * j, qpos[qa] - m.qpos0[qa]);
        else { for (int c = 0; c < 4; c++) dq[c] = qpos[qa + c]; qnormalize(dq); }
        qmul(nq, quat, dq);
        for (int c = 0; c < 4; c++) quat[c] = nq[c];
        q2mat(R, quat);
        m3mulv(t, R, m.jnt_pos + 3 * j); v3sub(pos, janchor + 3 * j, t);
      }
    }
    qnormalize(quat);
    v3copy(lpos + 3 * b, pos);
    for (int c = 0; c < 4; c++) lquat[4 * b + c] = quat[c];
  }
  gsync();
  double *xpos = ws + L.xpos, *xmat = ws + L.xmat;
  LANE_LOOP(b, m.nbody) {
    double pos[3], quat[4], t[3], nq[4];
    v3copy(pos, lpos + 3 * b);
    for (int c = 0; c < 4; c++) quat[c] = lquat[4 * b + c];
    for (int a = (b > 0 ? m.body_parentid[b] : 0); a > 0; a = m.body_parentid[a]) {
      qrot(t, lquat + 4 * a, pos); v3add(pos, lpos + 3 * a, t);
      qmul(nq, lquat + 4 * a, quat);
      for (int c = 0; c < 4; c++) quat[c] = nq[c];
    }
    qnormalize(quat);
    v3copy(xpos + 3 * b, pos);
    double R[9];
    q2mat(R, quat);
    for (int c = 0; c < 9; c++) xmat[9 * b + c] = R[c];
  }
  gsync();
  double* cdof = ws + L.cdof;
  LANE_LOOP(d, m.nv) {
    int j = m.dof_jntid[d], b = m.dof_bodyid[d], k = d - m.jnt_dofadr[j], type = m.jnt_type[j], p = m.body_parentid[b];
    double* c = cdof + 6 * d;
    double ax[3], an[3], t[3];
    if (type == J_FREE) {
      if (k < 3) { v3set(c, 0, 0, 0); v3set(c + 3, 0, 0, 0); c[3 + k] = 1; }
      else { m3col(ax, xmat + 9 * b, k - 3); v3copy(c, ax); v3cross(c + 3, xpos + 3 * b, ax); }
      continue;
    }
    m3mulv(t, xmat + 9 * p, janchor + 3 * j); v3add(an, xpos + 3 * p, t);
    if (type == J_BALL) m3col(ax, xmat + 9 * b, k); else m3mulv(ax, xmat + 9 * p, jaxis + 3 * j);
    if (type == J_SLIDE) { v3set(c, 0, 0, 0); v3copy(c + 3, ax); }
    else { v3copy(c, ax); v3cross(c + 3, an, ax); }
  }
  gsync();  // the local joint frames (janchor, jaxis) are dead from here on: cinert overwrites them
  double* cinert = ws + L.cinert;
  LANE_LOOP(b, m.nbody) {
    double* I = cinert + 10 * b;
    double mass = m.body_mass[b];
    double c[3];
    m3mulv(c, xmat + 9 * b, m.body_ipos + 3 * b); v3add(c, c, xpos + 3 * b);
    const double* R = xmat + 9 * b;
    const double* Ib = m.body_inertia + 6 * b;
    double Il[9] = {Ib[0], Ib[3], Ib[4], Ib[3], Ib[1], Ib[5], Ib[4], Ib[5], Ib[2]}, RI[9], Rt[9], Iw[9];
    for (int i = 0; i < 3; i++) for (int jj = 0; jj < 3; jj++) Rt[3 * i + jj] = R[3 * jj + i];
    m3mul(RI, R, Il); m3mul(Iw, RI, Rt);
    double cc = v3dot(c, c);
    I[0] = mass; I[1] = mass * c[0]; I[2] = mass * c[1]; I[3] = mass * c[2];
    I[4] = Iw[0] + mass * (cc - c[0] * c[0]); I[5] = Iw[4] + mass * (cc - c[1] * c[1]); I[6] = Iw[8] + mass * (cc - c[2] * c[2]);
    I[7] = Iw[1] - mass * c[0] * c[1]; I[8] = Iw[2] - mass * c[0] * c[2]; I[9] = Iw[5] - mass * c[1] * c[2];
  }
  double *gpos = ws + L.gpos, *gmat = ws + L.gmat;
  LANE_LOOP(g, m.ngeom) {
    int b = m.geom_bodyid[g];
    double t[3];
    m3mulv(t, xmat + 9 * b, m.geom_pos + 3 * g); v3add(gpos + 3 * g, xpos + 3 * b, t);
    m3mul(gmat + 9 * g, xmat + 9 * b, m.geom_lmat + 9 * g);
    m3mulv(t, gmat + 9 * g, m.geom_obbcenter + 3 * g); v3add(ws + L.gcen + 3 * g, gpos + 3 * g, t);  // bounding-sphere / OBB centre
  }
  gsync();
}

// ------------------------------------------------------------------------------------------------ bias forces (RNE) -> ws[qfrc_smooth] := qfrc_bias
__device__ __noinline__ void stage_rne(double* ws, int lane) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *qvel = ws + L.qvel, *cdof = ws + L.cdof, *cinert = ws + L.cinert;
  double *cdofdot = ws + L.cdofdot, *cvel = ws + L.cvel, *cacc = ws + L.cacc, *cfrc = ws + L.cfrc;
  LANE_LOOP(d, m.nv) {
    int j = m.dof_jntid[d], type = m.jnt_type[j], k = d - m.jnt_dofadr[j];
    double* out = cdofdot + 6 * d;
    if (type == J_FREE && k < 3) { for (int c = 0; c < 6; c++) out[c] = 0; continue; }
    int grp0 = m.jnt_dofadr[j] + (type == J_FREE ? 3 : 0);  // first dof of the rotational group of this joint
    double v[6] = {0, 0, 0, 0, 0, 0};
    for (int a = m.dof_parentid[d]; a >= 0; a = m.dof_parentid[a]) {
      if ((type == J_BALL || type == J_FREE) && a >= grp0) continue;  // axes of one joint share the velocity before the joint
      double qd = qvel[a];
      for (int c = 0; c < 6; c++) v[c] += cdof[6 * a + c] * qd;
    }
    cross_motion(out, v, cdof + 6 * d);
  }
  gsync();
  LANE_LOOP(b, m.nbody) {
    double v[6] = {0, 0, 0, 0, 0, 0}, a[6] = {0, 0, 0, -m.gravity[0], -m.gravity[1], -m.gravity[2]};
    for (int d = m.body_lastdof[b]; d >= 0; d = m.dof_parentid[d]) {
      double qd = qvel[d];
      for (int c = 0; c < 6; c++) { v[c] += cdof[6 * d + c] * qd; a[c] += cdofdot[6 * d + c] * qd; }
    }
    double Ia[6], Iv[6], x[6];
    inert_mul(Ia, cinert + 10 * b, a); inert_mul(Iv, cinert + 10 * b, v); cross_force(x, v, Iv);
    for (int c = 0; c < 6; c++) { cvel[6 * b + c] = v[c]; cfrc[6 * b + c] = Ia[c] + x[c]; }
  }
  gsync();
  LANE_LOOP(b, m.nbody) {  // subtree sums: depth-first numbering makes a subtree a contiguous range
    double s[6] = {0, 0, 0, 0, 0, 0};
    int n = m.body_subtreenum[b];
    for (int c2 = b; c2 < b + n; c2++) for (int c = 0; c < 6; c++) s[c] += cfrc[6 * c2 + c];
    for (int c = 0; c < 6; c++) cacc[6 * b + c] = s[c];
  }
  gsync();
  double* bias = ws + L.qfrc_smooth;
  LANE_LOOP(d, m.nv) bias[d] = dot6(cdof + 6 * d, cacc + 6 * m.dof_bodyid[d]);
  gsync();
}

// ------------------------------------------------------------------------------------------------ CRBA -> qM (tree-sparse rows: self, parent, grandparent, ...)
__device__ __noinline__ void stage_crb(double* ws, int lane) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *cdof = ws + L.cdof, *cinert = ws + L.cinert;
  double *crb = ws + L.cvel, *qM = ws + L.qM;  // composite inertias reuse the (dead) cvel/cacc area
  LANE_LOOP(b, m.nbody) {
    double s[10];
    for (int c = 0; c < 10; c++) s[c] = 0;
    int n = m.body_subtreenum[b];
    for (int c2 = b; c2 < b + n; c2++) for (int c = 0; c < 10; c++) s[c] += cinert[10 * c2 + c];
    for (int c = 0; c < 10; c++) crb[10 * b + c] = s[c];
  }
  gsync();
  LANE_LOOP(i, m.nv) {
    double f[6];
    inert_mul(f, crb + 10 * m.dof_bodyid[i], cdof + 6 * i);
    int adr = m.dof_Madr[i], k = 1;
    qM[adr] = dot6(cdof + 6 * i, f) + m.dof_armature[i];
    for (int j = m.dof_parentid[i]; j >= 0; j = m.dof_parentid[j], k++) qM[adr + k] = dot6(cdof + 6 * j, f);
  }
  gsync();
}

// L^T D L factorisation / solve of the tree-sparse mass matrix; one lane per kinematic tree (trees are independent)
__device__ __noinline__ void factor_trees(double* LD, int lane) {
  const DevModel& m = c_m;
  LANE_LOOP(t, m.ntree) {
    int lo = m.tree_dofadr[t], hi = lo + m.tree_dofnum[t];
    for (int k = hi - 1; k >= lo; k--) {
      int ak = m.dof_Madr[k], ki = 1;
      double inv = 1.0 / LD[ak];
      for (int i = m.dof_parentid[k]; i >= 0; i = m.dof_parentid[i], ki++) {
        double a = LD[ak + ki] * inv;
        int ai = m.dof_Madr[i], kj = ki, ij = 0;
        for (int j = i; j >= 0; j = m.dof_parentid[j], kj++, ij++) LD[ai + ij] -= a * LD[ak + kj];
        LD[ak + ki] = a;
      }
    }
  }
  gsync();
}
__device__ __noinline__ void solve_trees(const double* LD, double* x, int lane) {
  const DevModel& m = c_m;
  LANE_LOOP(t, m.ntree) {
    int lo = m.tree_dofadr[t], hi = lo + m.tree_dofnum[t];
    for (int k = hi - 1; k >= lo; k--) {
      int ak = m.dof_Madr[k], ki = 1;
      double xk = x[k];
      for (int i = m.dof_parentid[k]; i >= 0; i = m.dof_parentid[i], ki++) x[i] -= LD[ak + ki] * xk;
    }
    for (int k = lo; k < hi; k++) x[k] /= LD[m.dof_Madr[k]];
    for (int k = lo; k < hi; k++) {
      int ak = m.dof_Madr[k], ki = 1;
      double xk = x[k];
      for (int i = m.dof_parentid[k]; i >= 0; i = m.dof_parentid[i], ki++) xk -= LD[ak + ki] * x[i];
      x[k] = xk;
    }
  }
  gsync();
}
// r = M v, one lane per dof (ancestors from the dof's own row, descendants from theirs)
__device__ __noinline__ void mul_M(const double* qM, double* r, const double* v, int lane) {
  const DevModel& m = c_m;
  LANE_LOOP(i, m.nv) {
    int a = m.dof_Madr[i], k = 1;
    double s = qM[a] * v[i];
    for (int j = m.dof_parentid[i]; j >= 0; j = m.dof_parentid[j], k++) s += qM[a + k] * v[j];
    int n = m.dof_subtreenum[i], di = m.dof_depth[i];
    for (int c = i + 1; c < i + n; c++) s += qM[m.dof_Madr[c] + m.dof_depth[c] - di] * v[c];
    r[i] = s;
  }
  gsync();
}

// ------------------------------------------------------------------------------------------------ collision
struct PairContacts { int n; double normal[3]; double pos[8][3]; double dist[8]; };

__device__ __forceinline__ bool obb_separated(const double* c1, const double* R1, const double* h1, const double* c2, const double* R2, const double* h2, double margin) {
  double d[3], C[3][3], AC[3][3], da[3], db[3];
  v3sub(d, c2, c1);
#pragma unroll
  for (int i = 0; i < 3; i++) {
    da[i] = d[0] * R1[i] + d[1] * R1[3 + i] + d[2] * R1[6 + i];
    db[i] = d[0] * R2[i] + d[1] * R2[3 + i] + d[2] * R2[6 + i];
#pragma unroll
    for (int j = 0; j < 3; j++) { C[i][j] = R1[i] * R2[j] + R1[3 + i] * R2[3 + j] + R1[6 + i] * R2[6 + j]; AC[i][j] = fabs(C[i][j]) + 1e-9; }
  }
#pragma unroll
  for (int i = 0; i < 3; i++) if (fabs(da[i]) > h1[i] + h2[0] * AC[i][0] + h2[1] * AC[i][1] + h2[2] * AC[i][2] + margin) return true;
#pragma unroll
  for (int j = 0; j < 3; j++) if (fabs(db[j]) > h2[j] + h1[0] * AC[0][j] + h1[1] * AC[1][j] + h1[2] * AC[2][j] + margin) return true;
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) {
      const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
      double ra = h1[i1] * AC[i2][j] + h1[i2] * AC[i1][j], rb = h2[j1] * AC[i][j2] + h2[j2] * AC[i][j1];
      double len2 = 1.0 - C[i][j] * C[i][j];
      if (len2 < 1e-8) continue;
      if (fabs(da[i2] * C[i1][j] - da[i1] * C[i2][j]) > ra + rb + margin * sqrt(len2)) return true;
    }
  return false;
}

__device__ __forceinline__ void col_plane_sphere(const double* ws, int g1, int g2, double margin, PairContacts& out) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *gpos = ws + L.gpos, *gmat = ws + L.gmat;
  double n[3], d[3];
  m3col(n, gmat + 9 * g1, 2); v3sub(d, gpos + 3 * g2, gpos + 3 * g1);
  double r = m.geom_size[3 * g2], dist = v3dot(d, n) - r;
  if (dist >= margin) return;
  v3copy(out.normal, n);
  v3addscl(out.pos[0], gpos + 3 * g2, n, -(r + 0.5 * dist));
  out.dist[0] = dist; out.n = 1;
}
// sphere vs capsule, capsule vs capsule, sphere vs cylinder: closed forms (mirror the oracle's functions of the same names)
__device__ __noinline__ void col_sphere_capsule(const double* ws, int g1, int g2, double margin, PairContacts& out) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *c = ws + L.gpos + 3 * g1, *p = ws + L.gpos + 3 * g2;
  double ax[3], d[3], q[3], n[3];
  m3col(ax, ws + L.gmat + 9 * g2, 2);
  double r1 = m.geom_size[3 * g1], r2 = m.geom_size[3 * g2], h = m.geom_size[3 * g2 + 1];
  v3sub(d, c, p);
  double t = v3dot(d, ax);
  if (t > h) t = h; else if (t < -h) t = -h;
  v3addscl(q, p, ax, t); v3sub(d, q, c);
  double len = v3norm(d);
  if (len < 1e-12) { m3col(n, ws + L.gmat + 9 * g2, 0); len = 0; } else v3scl(n, d, 1.0 / len);
  double dist = len - r1 - r2;
  if (dist >= margin) return;
  v3copy(out.normal, n);
  v3addscl(out.pos[0], c, n, r1 + 0.5 * dist);
  out.dist[0] = dist; out.n = 1;
}
__device__ __noinline__ void col_capsule_capsule(const double* ws, int g1, int g2, double margin, PairContacts& out) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *p1 = ws + L.gpos + 3 * g1, *p2 = ws + L.gpos + 3 * g2;
  double a1[3], a2[3], w[3], q1[3], q2[3], d[3], n[3];
  m3col(a1, ws + L.gmat + 9 * g1, 2); m3col(a2, ws + L.gmat + 9 * g2, 2);
  double r1 = m.geom_size[3 * g1], h1 = m.geom_size[3 * g1 + 1], r2 = m.geom_size[3 * g2], h2 = m.geom_size[3 * g2 + 1];
  v3sub(w, p1, p2);
  double b = v3dot(a1, a2), dd = v3dot(a1, w), ee = v3dot(a2, w), den = 1.0 - b * b, s, t;
  if (den < 1e-10) {
    double c2 = -dd, lo = c2 - h2, hi = c2 + h2;
    if (lo < -h1) lo = -h1;
    if (hi > h1) hi = h1;
    s = lo <= hi ? 0.5 * (lo + hi) : (c2 > 0 ? h1 : -h1);
  } else {
    s = (b * ee - dd) / den;
    if (s > h1) s = h1; else if (s < -h1) s = -h1;
  }
  t = b * s + ee;
  if (t > h2) t = h2; else if (t < -h2) t = -h2;
  s = b * t - dd;
  if (s > h1) s = h1; else if (s < -h1) s = -h1;
  v3addscl(q1, p1, a1, s); v3addscl(q2, p2, a2, t); v3sub(d, q2, q1);
  double len = v3norm(d);
  if (len < 1e-12) { v3cross(n, a1, a2); if (v3norm(n) < 1e-12) m3col(n, ws + L.gmat + 9 * g1, 0); v3normalize(n); len = 0; } else v3scl(n, d, 1.0 / len);
  double dist = len - r1 - r2;
  if (dist >= margin) return;
  v3copy(out.normal, n);
  v3addscl(out.pos[0], q1, n, r1 + 0.5 * dist);
  out.dist[0] = dist; out.n = 1;
}
__device__ __noinline__ void col_sphere_cylinder(const double* ws, int g1, int g2, double margin, PairContacts& out) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *c = ws + L.gpos + 3 * g1, *R = ws + L.gmat + 9 * g2;
  double t[3], l[3], o[3], n[3];
  v3sub(t, c, ws + L.gpos + 3 * g2); m3Tmulv(l, R, t);
  double r1 = m.geom_size[3 * g1], r = m.geom_size[3 * g2], h = m.geom_size[3 * g2 + 1];
  double rho = sqrt(l[0] * l[0] + l[1] * l[1]), sz = l[2] >= 0 ? 1.0 : -1.0, dz = fabs(l[2]) - h, dr = rho - r, sd;
  double ux = rho > 1e-12 ? l[0] / rho : 1.0, uy = rho > 1e-12 ? l[1] / rho : 0.0;
  if (dz <= 0 && dr <= 0) {
    if (dr > dz) { v3set(o, ux, uy, 0); sd = dr; } else { v3set(o, 0, 0, sz); sd = dz; }
  } else if (dz <= 0) { v3set(o, ux, uy, 0); sd = dr; }
  else if (dr <= 0) { v3set(o, 0, 0, sz); sd = dz; }
  else { sd = sqrt(dr * dr + dz * dz); v3set(o, dr * ux / sd, dr * uy / sd, sz * dz / sd); }
  double dist = sd - r1;
  if (dist >= margin) return;
  m3mulv(n, R, o); v3scl(n, n, -1.0);
  v3copy(out.normal, n);
  v3addscl(out.pos[0], c, n, r1 + 0.5 * dist);
  out.dist[0] = dist; out.n = 1;
}
// plane vs capsule: the two end spheres (+axis end first); plane vs cylinder: deepest rim point of each cap (+axis cap first),
// a cap parallel to the plane contributes its centre (mirrors the oracle's col_plane_capsule / col_plane_cylinder)
__device__ __noinline__ void col_plane_capsule(const double* ws, int g1, int g2, double margin, PairContacts& out) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *gpos = ws + L.gpos, *gmat = ws + L.gmat;
  double n[3], ax[3];
  m3col(n, gmat + 9 * g1, 2); m3col(ax, gmat + 9 * g2, 2);
  double r = m.geom_size[3 * g2], h = m.geom_size[3 * g2 + 1];
  v3copy(out.normal, n);
  for (int s = 0; s < 2; s++) {
    double c[3], d[3];
    v3addscl(c, gpos + 3 * g2, ax, s ? -h : h);
    v3sub(d, c, gpos + 3 * g1);
    double dist = v3dot(d, n) - r;
    if (dist >= margin) continue;
    v3addscl(out.pos[out.n], c, n, -(r + 0.5 * dist));
    out.dist[out.n] = dist; out.n++;
  }
}
__device__ __noinline__ void col_plane_cylinder(const double* ws, int g1, int g2, double margin, PairContacts& out) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *gpos = ws + L.gpos, *gmat = ws + L.gmat;
  double n[3], ax[3], rim[3];
  m3col(n, gmat + 9 * g1, 2); m3col(ax, gmat + 9 * g2, 2);
  double r = m.geom_size[3 * g2], h = m.geom_size[3 * g2 + 1];
  v3addscl(rim, n, ax, -v3dot(n, ax));
  double len = v3norm(rim);
  if (len > 1e-6) v3scl(rim, rim, -r / len); else v3set(rim, 0, 0, 0);
  v3copy(out.normal, n);
  for (int s = 0; s < 2; s++) {
    double c[3], d[3];
    v3addscl(c, gpos + 3 * g2, ax, s ? -h : h);
    v3add(c, c, rim);
    v3sub(d, c, gpos + 3 * g1);
    double dist = v3dot(d, n);
    if (dist >= margin) continue;
    v3addscl(out.pos[out.n], c, n, -0.5 * dist);
    out.dist[out.n] = dist; out.n++;
  }
}
__device__ __noinline__ void col_plane_box(const double* ws, int g1, int g2, double margin, PairContacts& out) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *gpos = ws + L.gpos, *gmat = ws + L.gmat;
  double n[3];
  m3col(n, gmat + 9 * g1, 2);
  const double* h = m.geom_size + 3 * g2;
  v3copy(out.normal, n);
  for (int k = 0; k < 8 && out.n < 4; k++) {
    double loc[3] = {(k & 1 ? h[0] : -h[0]), (k & 2 ? h[1] : -h[1]), (k & 4 ? h[2] : -h[2])}, w[3], d[3];
    m3mulv(w, gmat + 9 * g2, loc); v3add(w, w, gpos + 3 * g2);
    v3sub(d, w, gpos + 3 * g1);
    double dist = v3dot(d, n);
    if (dist >= margin) continue;
    v3addscl(out.pos[out.n], w, n, -0.5 * dist);
    out.dist[out.n] = dist; out.n++;
  }
}
__device__ __noinline__ void col_plane_mesh(const double* ws, int g1, int g2, double margin, PairContacts& out) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *gpos = ws + L.gpos, *gmat = ws + L.gmat;
  double n[3], nl[3];
  m3col(n, gmat + 9 * g1, 2);
  m3Tmulv(nl, gmat + 9 * g2, n);
  int k = m.geom_meshid[g2], best = 0;
  const double* v = m.mesh_vert + 3 * m.mesh_vertadr[k];
  double bv = 1e300;
  for (int i = 0; i < m.mesh_vertnum[k]; i++) { double s = v3dot(v + 3 * i, nl); if (s < bv) { bv = s; best = i; } }
  double w[3], d[3];
  m3mulv(w, gmat + 9 * g2, v + 3 * best); v3add(w, w, gpos + 3 * g2);
  v3sub(d, w, gpos + 3 * g1);
  double dist = v3dot(d, n);
  if (dist >= margin) return;
  v3copy(out.normal, n);
  v3addscl(out.pos[0], w, n, -0.5 * dist);
  out.dist[0] = dist; out.n = 1;
}
__device__ __forceinline__ void col_sphere_sphere(const double* ws, int g1, int g2, double margin, PairContacts& out) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double* gpos = ws + L.gpos;
  double d[3];
  v3sub(d, gpos + 3 * g2, gpos + 3 * g1);
  double len = v3norm(d), r1 = m.geom_size[3 * g1], r2 = m.geom_size[3 * g2], dist = len - r1 - r2;
  if (dist >= margin) return;
  if (len < GE_MINVAL) v3set(d, 0, 0, 1); else v3scl(d, d, 1.0 / len);
  v3copy(out.normal, d);
  v3addscl(out.pos[0], gpos + 3 * g1, d, r1 + 0.5 * dist);
  out.dist[0] = dist; out.n = 1;
}
__device__ __noinline__ void col_sphere_box(const double* ws, int g1, int g2, double margin, PairContacts& out) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *gpos = ws + L.gpos, *gmat = ws + L.gmat;
  const double* h = m.geom_size + 3 * g2;
  double r = m.geom_size[3 * g1], d[3], p[3], q[3];
  v3sub(d, gpos + 3 * g1, gpos + 3 * g2);
  m3Tmulv(p, gmat + 9 * g2, d);
  bool inside = true;
  for (int k = 0; k < 3; k++) { q[k] = p[k] < -h[k] ? -h[k] : (p[k] > h[k] ? h[k] : p[k]); if (q[k] != p[k]) inside = false; }
  double nl[3] = {0, 0, 0}, dist;
  if (inside) {
    int best = 0; double bd = 1e300;
    for (int k = 0; k < 3; k++) { double s = h[k] - fabs(p[k]); if (s < bd) { bd = s; best = k; } }
    for (int k = 0; k < 3; k++) if (k == best) { nl[k] = p[k] >= 0 ? 1 : -1; q[k] = nl[k] * h[k]; }
    dist = -bd - r;
  } else {
    v3sub(nl, p, q);
    double len = v3normalize(nl);
    dist = len - r;
  }
  if (dist >= margin) return;
  double nw[3], qw[3];
  m3mulv(nw, gmat + 9 * g2, nl); m3mulv(qw, gmat + 9 * g2, q); v3add(qw, qw, gpos + 3 * g2);
  v3addscl(out.pos[0], qw, nw, 0.5 * dist);
  v3scl(out.normal, nw, -1.0);
  out.dist[0] = dist; out.n = 1;
}

__device__ __forceinline__ int clip_poly(const double (*p)[2], int n, int axis, double lim, double (*out)[2]) {
  int k = 0;
  for (int i = 0; i < n; i++) {
    const double *a = p[i], *b = p[(i + 1 == n) ? 0 : i + 1];
    double da = a[axis] - lim, db = b[axis] - lim;
    if (da <= 0) { out[k][0] = a[0]; out[k][1] = a[1]; k++; }
    if ((da < 0 && db > 0) || (da > 0 && db < 0)) { double t = da / (da - db); out[k][0] = a[0] + t * (b[0] - a[0]); out[k][1] = a[1] + t * (b[1] - a[1]); k++; }
  }
  return k;
}
// box-box manifold: 15-axis SAT, then reference-face clipping or edge-edge closest points (same contract as the oracle's col_box_box)
__device__ __noinline__ void col_box_box(const double* ws, int g1, int g2, double margin, PairContacts& out) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *c1 = ws + L.gpos + 3 * g1, *c2 = ws + L.gpos + 3 * g2, *R1 = ws + L.gmat + 9 * g1, *R2 = ws + L.gmat + 9 * g2;
  const double *h1 = m.geom_size + 3 * g1, *h2 = m.geom_size + 3 * g2;
  double d[3], a[3][3], b[3][3], C[3][3], AC[3][3];
  v3sub(d, c2, c1);
  for (int i = 0; i < 3; i++) { m3col(a[i], R1, i); m3col(b[i], R2, i); }
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { C[i][j] = v3dot(a[i], b[j]); AC[i][j] = fabs(C[i][j]); }
  double best_s = -1e300; int best_axis = -1;
  for (int i = 0; i < 3; i++) {
    double s = fabs(v3dot(d, a[i])) - (h1[i] + h2[0] * AC[i][0] + h2[1] * AC[i][1] + h2[2] * AC[i][2]);
    if (s >= margin) return;
    if (s > best_s) { best_s = s; best_axis = i; }
  }
  for (int j = 0; j < 3; j++) {
    double s = fabs(v3dot(d, b[j])) - (h2[j] + h1[0] * AC[0][j] + h1[1] * AC[1][j] + h1[2] * AC[2][j]);
    if (s >= margin) return;
    if (s > best_s) { best_s = s; best_axis = 3 + j; }
  }
  double edge_s = -1e300; int ei = -1, ej = -1; double en[3] = {0, 0, 0};
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    double Lx[3];
    v3cross(Lx, a[i], b[j]);
    double len = v3norm(Lx);
    if (len < 1e-6) continue;
    v3scl(Lx, Lx, 1.0 / len);
    double ra = 0, rb = 0;
    for (int k = 0; k < 3; k++) { ra += h1[k] * fabs(v3dot(Lx, a[k])); rb += h2[k] * fabs(v3dot(Lx, b[k])); }
    double s = fabs(v3dot(d, Lx)) - ra - rb;
    if (s >= margin) return;
    if (s > edge_s) { edge_s = s; ei = i; ej = j; v3copy(en, Lx); }
  }
  if (ei >= 0 && edge_s > best_s + 1e-6) {
    double n[3], p1[3], p2[3];
    v3copy(n, en);
    if (v3dot(d, n) < 0) v3scl(n, n, -1.0);
    v3copy(p1, c1); v3copy(p2, c2);
    for (int k = 0; k < 3; k++) {
      if (k != ei) v3addscl(p1, p1, a[k], (v3dot(n, a[k]) >= 0 ? 1.0 : -1.0) * h1[k]);
      if (k != ej) v3addscl(p2, p2, b[k], (v3dot(n, b[k]) >= 0 ? -1.0 : 1.0) * h2[k]);
    }
    double w[3];
    v3sub(w, p1, p2);
    double ab = C[ei][ej], aw = v3dot(a[ei], w), bw = v3dot(b[ej], w), den = 1.0 - ab * ab;
    double t = (ab * bw - aw) / den, u = (bw - ab * aw) / den;
    double q1[3], q2[3], dd[3];
    v3addscl(q1, p1, a[ei], t); v3addscl(q2, p2, b[ej], u);
    v3sub(dd, q2, q1);
    double dist = v3dot(dd, n);
    if (dist >= margin) return;
    v3add(out.pos[0], q1, q2); v3scl(out.pos[0], out.pos[0], 0.5);
    v3copy(out.normal, n); out.dist[0] = dist; out.n = 1;
    return;
  }
  bool ref1 = best_axis < 3;
  int ax = ref1 ? best_axis : best_axis - 3;
  const double *cr = ref1 ? c1 : c2, *ci = ref1 ? c2 : c1, *hr = ref1 ? h1 : h2, *hi = ref1 ? h2 : h1;
  double (*ar)[3] = ref1 ? a : b;
  double (*ai)[3] = ref1 ? b : a;
  double dr[3], nref[3];
  v3sub(dr, ci, cr);
  v3scl(nref, ar[ax], v3dot(dr, ar[ax]) >= 0 ? 1.0 : -1.0);
  int inc = 0; double bestd = -1;
  for (int k = 0; k < 3; k++) { double s = fabs(v3dot(ai[k], nref)); if (s > bestd) { bestd = s; inc = k; } }
  double sgn = v3dot(ai[inc], nref) > 0 ? -1.0 : 1.0;
  double fc[3];
  v3addscl(fc, ci, ai[inc], sgn * hi[inc]);
  int u1 = (inc + 1) % 3, u2 = (inc + 2) % 3, r1 = (ax + 1) % 3, r2 = (ax + 2) % 3;
  double poly[16][2], tmp[16][2], height[4];
  const double sg[4][2] = {{1, 1}, {-1, 1}, {-1, -1}, {1, -1}};
  for (int k = 0; k < 4; k++) {
    double corner[3], rel[3];
    v3addscl(corner, fc, ai[u1], sg[k][0] * hi[u1]); v3addscl(corner, corner, ai[u2], sg[k][1] * hi[u2]);
    v3sub(rel, corner, cr);
    poly[k][0] = v3dot(rel, ar[r1]); poly[k][1] = v3dot(rel, ar[r2]);
    height[k] = v3dot(rel, nref) - hr[ax];
  }
  double ex[2] = {poly[1][0] - poly[0][0], poly[1][1] - poly[0][1]}, ey[2] = {poly[3][0] - poly[0][0], poly[3][1] - poly[0][1]};
  double det = ex[0] * ey[1] - ex[1] * ey[0], gx = 0, gy = 0;
  if (fabs(det) > 1e-14) {
    double dh1 = height[1] - height[0], dh3 = height[3] - height[0];
    gx = (dh1 * ey[1] - dh3 * ex[1]) / det; gy = (dh3 * ex[0] - dh1 * ey[0]) / det;
  }
  double g0 = height[0] - gx * poly[0][0] - gy * poly[0][1];
  int n = 4;
  n = clip_poly(poly, n, 0, hr[r1], tmp); if (!n) return;
  for (int k = 0; k < n; k++) tmp[k][0] = -tmp[k][0];
  n = clip_poly(tmp, n, 0, hr[r1], poly); if (!n) return;
  for (int k = 0; k < n; k++) poly[k][0] = -poly[k][0];
  n = clip_poly(poly, n, 1, hr[r2], tmp); if (!n) return;
  for (int k = 0; k < n; k++) tmp[k][1] = -tmp[k][1];
  n = clip_poly(tmp, n, 1, hr[r2], poly); if (!n) return;
  for (int k = 0; k < n; k++) poly[k][1] = -poly[k][1];
  v3scl(out.normal, nref, ref1 ? 1.0 : -1.0);
  for (int k = 0; k < n && out.n < 8; k++) {
    double dist = g0 + gx * poly[k][0] + gy * poly[k][1];
    if (dist >= margin) continue;
    double* pos = out.pos[out.n];
    v3addscl(pos, cr, ar[r1], poly[k][0]); v3addscl(pos, pos, ar[r2], poly[k][1]);
    v3addscl(pos, pos, nref, hr[ax] + 0.5 * dist);
    out.dist[out.n] = dist; out.n++;
  }
}

// ---- warp-cooperative Minkowski Portal Refinement: every lane carries the same portal, the hull support function is a
// 32-lane strided arg-max over the vertices followed by a butterfly reduction (lowest index wins ties, like the oracle's scan)
struct SP { double v[3], a[3], b[3]; };
__device__ __noinline__ void support_w(const double* ws, int g, double inflate, const double* dir, double* out, int lane) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *R = ws + L.gmat + 9 * g, *size = m.geom_size + 3 * g;
  double dl[3], pl[3] = {0, 0, 0};
  m3Tmulv(dl, R, dir);
  int type = m.geom_type[g];
  if (type == G_SPHERE) v3scl(pl, dl, size[0]);
  else if (type == G_BOX) { for (int k = 0; k < 3; k++) pl[k] = dl[k] >= 0 ? size[k] : -size[k]; }
  else if (type == G_CAPSULE) { v3scl(pl, dl, size[0]); pl[2] += dl[2] >= 0 ? size[1] : -size[1]; }
  else if (type == G_CYLINDER) {
    double n = sqrt(dl[0] * dl[0] + dl[1] * dl[1]);
    if (n > GE_MINVAL) { pl[0] = dl[0] / n * size[0]; pl[1] = dl[1] / n * size[0]; }
    pl[2] = dl[2] >= 0 ? size[1] : -size[1];
  } else {
    int k = m.geom_meshid[g], nvert = m.mesh_vertnum[k], best = 0x7fffffff;
    const double* v = m.mesh_vert + 3 * m.mesh_vertadr[k];
    double bv = -1e300;
    // four vertices per lane and trip: 12 independent loads in flight before the (ordered) comparisons
    for (int i0 = lane; i0 < nvert; i0 += 128) {
      double c[4][3];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        int i = i0 + 32 * u;
        bool ok = i < nvert;
        c[u][0] = ok ? __ldg(v + 3 * i) : 0.0; c[u][1] = ok ? __ldg(v + 3 * i + 1) : 0.0; c[u][2] = ok ? __ldg(v + 3 * i + 2) : 0.0;
      }
#pragma unroll
      for (int u = 0; u < 4; u++) {
        int i = i0 + 32 * u;
        double t = c[u][0] * dl[0] + c[u][1] * dl[1] + c[u][2] * dl[2];
        if (i < nvert && t > bv) { bv = t; best = i; }
      }
    }
    warp_argmax(bv, best);
    if (best >= nvert) best = 0;  // a non-finite direction matches no vertex: stay inside the table (the step is flagged as non-finite later)
    v3copy(pl, v + 3 * best);
  }
  m3mulv(out, R, pl); v3add(out, out, ws + L.gpos + 3 * g); v3addscl(out, out, dir, inflate);
}
__device__ __forceinline__ void mink_w(const double* ws, int g1, int g2, double inflate, const double* dir, SP& s, int lane) {
  double u[3], nd[3];
  v3copy(u, dir); v3normalize(u); v3scl(nd, u, -1.0);
  support_w(ws, g1, inflate, u, s.a, lane); support_w(ws, g2, inflate, nd, s.b, lane); v3sub(s.v, s.a, s.b);
}
__device__ __forceinline__ void tri_closest_origin(const double* p, const double* q, const double* r, double* w) {
  double ab[3], ac[3], ap[3];
  v3sub(ab, q, p); v3sub(ac, r, p); v3scl(ap, p, -1.0);
  double d1 = v3dot(ab, ap), d2 = v3dot(ac, ap);
  if (d1 <= 0 && d2 <= 0) { w[0] = 1; w[1] = 0; w[2] = 0; return; }
  double bp[3]; v3scl(bp, q, -1.0);
  double d3 = v3dot(ab, bp), d4 = v3dot(ac, bp);
  if (d3 >= 0 && d4 <= d3) { w[0] = 0; w[1] = 1; w[2] = 0; return; }
  double vc = d1 * d4 - d3 * d2;
  if (vc <= 0 && d1 >= 0 && d3 <= 0) { double v = d1 / (d1 - d3); w[0] = 1 - v; w[1] = v; w[2] = 0; return; }
  double cp[3]; v3scl(cp, r, -1.0);
  double d5 = v3dot(ab, cp), d6 = v3dot(ac, cp);
  if (d6 >= 0 && d5 <= d6) { w[0] = 0; w[1] = 0; w[2] = 1; return; }
  double vb = d5 * d2 - d1 * d6;
  if (vb <= 0 && d2 >= 0 && d6 <= 0) { double v = d2 / (d2 - d6); w[0] = 1 - v; w[1] = 0; w[2] = v; return; }
  double va = d3 * d6 - d5 * d4;
  if (va <= 0 && (d4 - d3) >= 0 && (d5 - d6) >= 0) { double v = (d4 - d3) / ((d4 - d3) + (d5 - d6)); w[0] = 0; w[1] = 1 - v; w[2] = v; return; }
  double den = 1.0 / (va + vb + vc);
  w[1] = vb * den; w[2] = vc * den; w[0] = 1 - w[1] - w[2];
}
// returns true and (depth, dir, pos) if the inflated shapes intersect.  Control flow is warp-uniform.
__device__ __noinline__ bool mpr_w(const double* ws, int g1, int g2, double inflate, double* depth, double* pdir, double* ppos, int lane) {
  const DevModel& m = c_m; const Layout& L = c_L;
  SP v0, v1, v2, v3, v4;
  double dir[3], t1[3], t2[3], cr[3];
  for (int s = 0; s < 2; s++) {
    int g = s ? g2 : g1;
    double* out = s ? v0.b : v0.a;
    if (m.geom_type[g] == G_MESH) { m3mulv(out, ws + L.gmat + 9 * g, m.mesh_center + 3 * m.geom_meshid[g]); v3add(out, out, ws + L.gpos + 3 * g); }
    else v3copy(out, ws + L.gpos + 3 * g);
  }
  v3sub(v0.v, v0.a, v0.b);
  if (v3dot(v0.v, v0.v) < 1e-20) v3set(v0.v, 1e-5, 0, 0);
  v3scl(dir, v0.v, -1.0);
  mink_w(ws, g1, g2, inflate, dir, v1, lane);
  v3normalize(dir);
  if (v3dot(v1.v, dir) <= 0) return false;
  v3cross(cr, v1.v, v0.v);
  if (v3dot(cr, cr) < 1e-20 * v3dot(v1.v, v1.v) * v3dot(v0.v, v0.v) + 1e-300) {
    *depth = v3dot(v1.v, dir); v3copy(pdir, dir);
    v3add(ppos, v1.a, v1.b); v3scl(ppos, ppos, 0.5);
    return true;
  }
  mink_w(ws, g1, g2, inflate, cr, v2, lane);
  if (v3dot(v2.v, cr) <= 0) return false;
  v3sub(t1, v1.v, v0.v); v3sub(t2, v2.v, v0.v); v3cross(dir, t1, t2);
  if (v3dot(dir, v0.v) > 0) { SP t = v1; v1 = v2; v2 = t; v3scl(dir, dir, -1.0); }
  for (int it = 0;; it++) {
    if (it > 100) return false;
    mink_w(ws, g1, g2, inflate, dir, v3, lane);
    if (v3dot(v3.v, dir) <= 0) return false;
    v3cross(cr, v1.v, v3.v);
    if (v3dot(cr, v0.v) < 0) { v2 = v3; v3sub(t1, v1.v, v0.v); v3sub(t2, v3.v, v0.v); v3cross(dir, t1, t2); continue; }
    v3cross(cr, v3.v, v2.v);
    if (v3dot(cr, v0.v) < 0) { v1 = v3; v3sub(t1, v3.v, v0.v); v3sub(t2, v2.v, v0.v); v3cross(dir, t1, t2); continue; }
    break;
  }
  bool hit = false;
  for (int it = 0;; it++) {
    v3sub(t1, v2.v, v1.v); v3sub(t2, v3.v, v1.v); v3cross(dir, t1, t2); v3normalize(dir);
    if (!hit && v3dot(v1.v, dir) >= 0) hit = true;
    mink_w(ws, g1, g2, inflate, dir, v4, lane);
    double dv4 = v3dot(v4.v, dir);
    if (!hit && dv4 < 0) return false;
    double dmin = fmin(v3dot(v1.v, dir), fmin(v3dot(v2.v, dir), v3dot(v3.v, dir)));
    if (dv4 - dmin <= m.mpr_tol || it >= m.mpr_iter) { if (!hit) return false; break; }
    v3cross(cr, v4.v, v0.v);
    if (v3dot(v1.v, cr) > 0) { if (v3dot(v2.v, cr) > 0) v1 = v4; else v3 = v4; }
    else { if (v3dot(v3.v, cr) > 0) v2 = v4; else v1 = v4; }
  }
  double w[3], cp[3];
  tri_closest_origin(v1.v, v2.v, v3.v, w);
  for (int k = 0; k < 3; k++) cp[k] = w[0] * v1.v[k] + w[1] * v2.v[k] + w[2] * v3.v[k];
  double dep = v3norm(cp);
  if (dep > 1e-12) v3scl(pdir, cp, 1.0 / dep); else v3copy(pdir, dir);
  *depth = dep;
  for (int k = 0; k < 3; k++) ppos[k] = 0.5 * (w[0] * (v1.a[k] + v1.b[k]) + w[1] * (v2.a[k] + v2.b[k]) + w[2] * (v3.a[k] + v3.b[k]));
  return true;
}

// contact record: [dist, pos3, frame9, D, B, Kr, mu(maxdim-1), vel(maxdim), ja(maxdim), jv(maxdim)]
#define C_DIST 0
#define C_POS 1
#define C_FRAME 4
#define C_D 13
#define C_B 14
#define C_KR 15
#define C_MU 16
__device__ __forceinline__ int c_vel() { return C_MU + c_m.maxdim - 1; }
__device__ __forceinline__ int c_ja() { return C_MU + 2 * c_m.maxdim - 1; }
__device__ __forceinline__ int c_jv() { return C_MU + 3 * c_m.maxdim - 1; }

__device__ __forceinline__ void make_frame(double* fr) {
  double t[3] = {0, 0, 0};
  if (fabs(fr[1]) < 0.5) t[1] = 1; else t[2] = 1;
  double d = v3dot(fr, t);
  v3addscl(fr + 3, t, fr, -d); v3normalize(fr + 3);
  v3cross(fr + 6, fr, fr + 3);
}

// Broad phase over the static candidate pair list (bounding spheres, then oriented boxes), analytic narrow phase one lane
// per surviving pair, then the MPR pairs, each with one whole warp (the warps of a CTA-per-env build take them round-robin).
// Returns the number of contacts; sets bit 0 of *status on overflow.  (The oracle emits contacts in the same order: analytic
// pairs first, then MPR pairs, both in candidate order.)  A list that overflows keeps the first maxcon contacts of that order.
__device__ __forceinline__ bool pair_is_analytic(int t1, int t2) {
  return (t1 == G_PLANE) || (t1 == G_SPHERE && (t2 == G_SPHERE || t2 == G_BOX || t2 == G_CAPSULE || t2 == G_CYLINDER)) ||
         (t1 == G_BOX && t2 == G_BOX) || (t1 == G_CAPSULE && t2 == G_CAPSULE);
}
// what one collision stage found: contacts kept, broad-phase survivors (before the maxcand cut), MPR pairs among the kept candidates
struct CollisionCounts { int ncon, ncand, nmpr; };
__device__ __noinline__ CollisionCounts stage_collision(double* ws, int* wi, int lane, int* status) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *gpos = ws + L.gpos, *gmat = ws + L.gmat, *gcen = ws + L.gcen;
  const int wl = lane & 31, wid = lane >> 5;
  int* cand = wi + L.i_cand;
  int ncand = 0;
  for (int base = 0; base < m.npair; base += GE_LANES) {
    int p = base + lane;
    bool pass = false;
    if (p < m.npair) {
      // one 16-byte record per pair (geom ids + types) and the precomputed sum of bounding radii + margin; the world-space
      // bounding-sphere centres of all geoms were computed once in stage_fk (gcen)
      const int4 pr = __ldg((const int4*)m.pair_rec + p);
      const int g1 = pr.x, g2 = pr.y, t1 = pr.z, t2 = pr.w;
      const double rs = __ldg(m.pair_rsum + p);
      const double* c2 = gcen + 3 * g2;
      if (t1 == G_PLANE) {
        double n[3], d[3];
        m3col(n, gmat + 9 * g1, 2); v3sub(d, c2, gpos + 3 * g1);
        pass = !(v3dot(d, n) > rs);
      } else {
        const double* c1 = gcen + 3 * g1;
        double d[3];
        v3sub(d, c2, c1);
        pass = !(v3dot(d, d) > rs * rs);
        if (pass && !(t1 == G_SPHERE && t2 == G_SPHERE))
          pass = !obb_separated(c1, gmat + 9 * g1, m.geom_obbhalf + 3 * g1, c2, gmat + 9 * g2, m.geom_obbhalf + 3 * g2, m.pair_margin[p]);
      }
    }
    int total;
    int pos = ncand + group_exscan(pass ? 1 : 0, lane, total);
    if (pass && pos < L.maxcand) cand[pos] = p;
    ncand += total;
  }
  const int nsurv = ncand;
  if (ncand > L.maxcand) { ncand = L.maxcand; *status |= 1; }
  gsync();
  double* con = ws + L.con;
  int *cb1 = wi + L.i_cb1, *cb2 = wi + L.i_cb2, *cdim = wi + L.i_cdim, *cpair = wi + L.i_cpair;
  int ncon = 0;
#ifdef GE_DIAG
  int dg_na = 0, dg_k = 0, dg_nhit = 0, dg_nslots = 0, dg_maxn = 0;
#endif
  // ---- analytic pairs
  for (int base = 0; base < ncand; base += GE_LANES) {
    int ci = base + lane;
    PairContacts pc;
    pc.n = 0;
    int p = -1;
    if (ci < ncand) {
      p = cand[ci];
      int g1 = m.pair_geom[2 * p], g2 = m.pair_geom[2 * p + 1], t1 = m.geom_type[g1], t2 = m.geom_type[g2];
      double margin = m.pair_margin[p];
      if (t1 == G_PLANE) {
        if (t2 == G_SPHERE) col_plane_sphere(ws, g1, g2, margin, pc);
        else if (t2 == G_BOX) col_plane_box(ws, g1, g2, margin, pc);
        else if (t2 == G_MESH) col_plane_mesh(ws, g1, g2, margin, pc);
        else if (t2 == G_CAPSULE) col_plane_capsule(ws, g1, g2, margin, pc);
        else if (t2 == G_CYLINDER) col_plane_cylinder(ws, g1, g2, margin, pc);
      } else if (t1 == G_SPHERE && t2 == G_SPHERE) col_sphere_sphere(ws, g1, g2, margin, pc);
      else if (t1 == G_SPHERE && t2 == G_BOX) col_sphere_box(ws, g1, g2, margin, pc);
      else if (t1 == G_BOX && t2 == G_BOX) col_box_box(ws, g1, g2, margin, pc);
      else if (t1 == G_SPHERE && t2 == G_CAPSULE) col_sphere_capsule(ws, g1, g2, margin, pc);
      else if (t1 == G_SPHERE && t2 == G_CYLINDER) col_sphere_cylinder(ws, g1, g2, margin, pc);
      else if (t1 == G_CAPSULE && t2 == G_CAPSULE) col_capsule_capsule(ws, g1, g2, margin, pc);
    }
    // ordered compaction of the per-lane contact lists
#ifdef GE_DIAG
    if (pc.n > dg_maxn) dg_maxn = pc.n;
    if (pc.n < 0 || pc.n > 8) printf("DIAG pc.n %d lane %d block %d pair %d\n", pc.n, lane, (int)blockIdx.x, p);
#endif
    int total;
    int off = ncon + group_exscan(pc.n, lane, total);
    for (int k = 0; k < pc.n; k++) {
      int idx = off + k;
      if (idx >= L.maxcon) break;
      double* c = con + idx * L.cstride;
      c[C_DIST] = pc.dist[k]; v3copy(c + C_POS, pc.pos[k]); v3copy(c + C_FRAME, pc.normal);
      cpair[idx] = p;
    }
    ncon += total;
  }
#ifdef GE_DIAG
  dg_na = ncon;
#endif
  if (ncon > L.maxcon) { ncon = L.maxcon; *status |= 1; }
  gsync();
  // ---- convex pairs through MPR
  int nmpr = 0;
#if GE_NW == 1
  bool full = false;  // a hit found no room: the rest of the MPR pairs are only counted
  for (int ci = 0; ci < ncand; ci++) {
    int p = cand[ci];
    int g1 = m.pair_geom[2 * p], g2 = m.pair_geom[2 * p + 1], t1 = m.geom_type[g1], t2 = m.geom_type[g2];
    if (pair_is_analytic(t1, t2)) continue;
    nmpr++;
    if (full) continue;
    double margin = m.pair_margin[p], depth, dir[3], pos[3];
    if (!mpr_w(ws, g1, g2, 0.5 * margin, &depth, dir, pos, lane)) continue;
    double dist = margin - depth;
    if (dist >= margin) continue;
    if (ncon >= L.maxcon) { *status |= 1; full = true; continue; }
    if (lane == 0) {
      double* c = con + ncon * L.cstride;
      c[C_DIST] = dist; v3copy(c + C_POS, pos); v3copy(c + C_FRAME, dir);
      cpair[ncon] = p;
    }
    ncon++;
  }
  gsync();
#else
  {
    // Rounds: with `room` = maxcon - ncon free slots, the next (at most room) MPR pairs are dealt out, pair number k of the stage to
    // warp k % GE_NW; the j-th pair of the round writes its result into contact slot ncon + j (cpair = -1: no contact), then the slots
    // are compacted in order.  A round whose pairs missed leaves room for the next one, so the list ends as the first maxcon contacts
    // of the emission order.  Normally every MPR pair fits the first round (one round, three barriers).  Once the list is full, the
    // remaining pairs are only tested for a hit, which is an overflow.
    int k = 0, ci = 0;
    bool overflow = false;
    for (;;) {
      const int room = L.maxcon - ncon, k0 = k;
      if (room <= 0) {
        bool hit_any = false;
        for (; ci < ncand; ci++) {
          int p = cand[ci];
          int g1 = m.pair_geom[2 * p], g2 = m.pair_geom[2 * p + 1], t1 = m.geom_type[g1], t2 = m.geom_type[g2];
          if (pair_is_analytic(t1, t2)) continue;
          const bool mine = (k % GE_NW) == wid;
          k++;
          if (!mine || hit_any) continue;
          double margin = m.pair_margin[p], depth = 0, dir[3], pos[3];
          const bool hit = mpr_w(ws, g1, g2, 0.5 * margin, &depth, dir, pos, wl) && margin - depth < margin;
          hit_any = __any_sync(FULL, hit) != 0;  // (warp-uniform: the warp's later pairs are skipped together)
        }
        overflow |= group_any(hit_any);
        break;
      }
      for (; ci < ncand; ci++) {
        int p = cand[ci];
        int g1 = m.pair_geom[2 * p], g2 = m.pair_geom[2 * p + 1], t1 = m.geom_type[g1], t2 = m.geom_type[g2];
        if (pair_is_analytic(t1, t2)) continue;
        if (k - k0 >= room) break;  // this pair opens the next round
        const int slot = ncon + k - k0;
        const bool mine = (k % GE_NW) == wid;
        k++;
        if (!mine) continue;
        double margin = m.pair_margin[p], depth = 0, dir[3], pos[3];
        bool hit = mpr_w(ws, g1, g2, 0.5 * margin, &depth, dir, pos, wl);
        double dist = margin - depth;
        if (hit && dist >= margin) hit = false;
        if (wl == 0) {
          double* c = con + slot * L.cstride;
          if (hit) { c[C_DIST] = dist; v3copy(c + C_POS, pos); v3copy(c + C_FRAME, dir); }
          cpair[slot] = hit ? p : -1;
        }
      }
      gsync();
      const int nslots = ncon + k - k0;
      // every thread counts the hits first (read-only), THEN warp 0 alone compacts in place: record j moves down to the next free slot
      // (never overtakes an unread record).  (r02d: a version in which all threads walked the flags while warp 0 was already moving
      // records let a slow thread read a flag that had just been overwritten - its contact count then differed from the others';
      // found by racecheck once the workspace was in shared memory.)
      int nhit = 0;
      for (int j = ncon; j < nslots; j++) nhit += cpair[j] >= 0;
      gsync();
      if (wid == 0) {
        int o2 = ncon;
        for (int j = ncon; j < nslots; j++) {
          const int p = cpair[j];
          __syncwarp();  // every lane has read flag j before lane 0 may overwrite a lower slot
          if (p < 0) continue;
          if (o2 != j) {
            for (int q = wl; q < C_FRAME + 3; q += 32) con[o2 * L.cstride + q] = con[j * L.cstride + q];
            if (wl == 0) cpair[o2] = p;
          }
          o2++;
        }
      }
#ifdef GE_DIAG
      dg_k = k; dg_nhit = nhit; dg_nslots = nslots;
#endif
      ncon += nhit;
      gsync();
      if (ci >= ncand) break;
    }
    if (overflow) *status |= 1;
    nmpr = k;
  }
#endif
  // ---- per-contact frame and solver parameters
  bool bad_pair = false;
  LANE_LOOP(i, ncon) {
    double* c = con + i * L.cstride;
    int p = cpair[i];
#ifdef GE_DIAG
    if ((unsigned)p >= (unsigned)m.npair)
      printf("DIAG bad pair index: block %d lane %d i %d p %d ncon %d (analytic total %d, max per lane %d) ncand %d mpr k %d nhit %d nslots %d maxcon %d\n", (int)blockIdx.x,
             lane, i, p, ncon, dg_na, dg_maxn, ncand, dg_k, dg_nhit, dg_nslots, L.maxcon);
#endif
    // Safety net (r02m): a contact record whose pair index is not a pair of the model must never be dereferenced - the record is
    // neutralised (pair 0, far outside its margin: no force) and the environment flagged (status bit 6 = 64, below).  See DESIGN.md
    // section 4 for the open issue this guards.
    if ((unsigned)p >= (unsigned)m.npair) { bad_pair = true; p = 0; cpair[i] = 0; c[C_DIST] = 1e3; }
    make_frame(c + C_FRAME);
    int g1 = m.pair_geom[2 * p], g2 = m.pair_geom[2 * p + 1], b1 = m.geom_bodyid[g1], b2 = m.geom_bodyid[g2], dim = m.pair_condim[p];
    cb1[i] = b1; cb2[i] = b2; cdim[i] = dim;
    { int d1 = m.body_lastdof[b1], d2 = m.body_lastdof[b2]; wi[L.i_ct1 + i] = d1 < 0 ? -1 : m.dof_treeindex[d1]; wi[L.i_ct2 + i] = d2 < 0 ? -1 : m.dof_treeindex[d2]; }
    const double* f = m.pair_friction + 3 * p;
    double mu[5] = {f[0], f[0], f[1], f[2], f[2]};
    for (int k = 0; k < dim - 1; k++) c[C_MU + k] = mu[k];
    double margin = m.pair_margin[p], dist = c[C_DIST];
    const double *solref = m.pair_solref + 2 * p, *solimp = m.pair_solimp + 5 * p;
    // impedance (SURVEY A.5): d(r) between solimp[0] and solimp[1] over `width`; K, B from (timeconst, dampratio)
    double d0 = solimp[0], dw = solimp[1], width = solimp[2], mid = solimp[3], power = solimp[4];
    double x = fabs(dist - margin) / (width > GE_MINVAL ? width : GE_MINVAL), y;
    if (x >= 1) y = 1; else if (x <= 0) y = 0; else if (power == 1) y = x;
    else if (x <= mid) y = pow(x / mid, power) * mid; else y = 1 - pow((1 - x) / (1 - mid), power) * (1 - mid);
    double imp = d0 + y * (dw - d0);
    double tc = solref[0], dr = solref[1];
    if (tc < 2 * m.timestep) tc = 2 * m.timestep;
    double kk = dw * dw * tc * tc * dr * dr, bb = dw * tc;
    double K = 1.0 / (kk > GE_MINVAL ? kk : GE_MINVAL), B = 2.0 / (bb > GE_MINVAL ? bb : GE_MINVAL);
    double tran = m.body_invweight0[2 * b1] + m.body_invweight0[2 * b2];
    double diag0 = dim == 1 ? tran : tran + mu[0] * mu[0] * tran;
    double R = (1 - imp) / imp * diag0;
    if (R < GE_MINVAL) R = GE_MINVAL;
    if (dim > 1) { R = 2 * mu[0] * mu[0] / m.impratio * R; if (R < GE_MINVAL) R = GE_MINVAL; }
    c[C_D] = 1.0 / R; c[C_B] = B; c[C_KR] = K * imp * (dist - margin);
  }
  if (group_any(bad_pair)) *status |= 64;  // (every thread keeps its own copy of the status word: the flag has to be set by all of them)
  gsync();
  return CollisionCounts{ncon, nsurv, nmpr};
}

}  // namespace ge
