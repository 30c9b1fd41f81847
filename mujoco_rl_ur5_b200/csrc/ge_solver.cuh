// Constraint construction and the Newton solver, one warp per environment, matrix-free Jacobians.
//
// The constraint Jacobian is never stored.  Products with it go through per-body spatial vectors:
//   J x   : V_b = sum_{d in chain(b)} cdof_d x_d  (one lane per body), then one lane per contact projects
//           (V_b2 - V_b1) at the contact point onto the contact frame;
//   J^T f : one lane per body gathers the wrenches of its contacts, subtree sums over contiguous body ranges,
//           then one lane per dof takes cdof_d . W_subtree(body_d).
// Only the Newton Hessian  H = M + J^T D_active J  is formed explicitly (packed lower triangle, skyline Cholesky);
// the per-contact Jacobian block it needs is rebuilt in registers, one lane per dof of the two kinematic chains.
//
// Stands in for mj_makeConstraint + mj_solNewton behind `sim.step()` (reference: MujocoController.py:379; the
// scenes set no <option solver=...>, so MuJoCo's default Newton solver and pyramidal cones are in force —
// UR5gripper_2_finger.xml:19-22).  Mirrors oracle/grasp_oracle.c solve_newton().
#pragma once
#include "ge_physics.cuh"

namespace ge {

#define SR_CA 0
#define SR_CB 1
#define SR_D 2
#define SR_AREF 3
#define SR_JA 4
#define SR_JV 5
__device__ __forceinline__ double& srv(double* ws, int field, int i) { return ws[c_L.sr + field * GE_MAXSR + i]; }

__device__ __forceinline__ void impedance(const double* solref, const double* solimp, double pos, double margin, double& imp, double& K, double& B) {
  double d0 = solimp[0], dw = solimp[1], width = solimp[2], mid = solimp[3], power = solimp[4];
  double x = fabs(pos - margin) / (width > GE_MINVAL ? width : GE_MINVAL), y;
  if (x >= 1) y = 1; else if (x <= 0) y = 0; else if (power == 1) y = x;
  else if (x <= mid) y = pow(x / mid, power) * mid; else y = 1 - pow((1 - x) / (1 - mid), power) * (1 - mid);
  imp = d0 + y * (dw - d0);
  double tc = solref[0], dr = solref[1];
  if (tc < 2 * c_m.timestep) tc = 2 * c_m.timestep;
  double kk = dw * dw * tc * tc * dr * dr, bb = dw * tc;
  K = 1.0 / (kk > GE_MINVAL ? kk : GE_MINVAL); B = 2.0 / (bb > GE_MINVAL ? bb : GE_MINVAL);
}

// V_b = sum over the dofs on the path world -> b of cdof_d x_d
__device__ __noinline__ void body_vel(double* ws, const double* x, int lane) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double* cdof = ws + L.cdof;
  double* Vb = ws + L.Vb;
  LANE_LOOP(b, m.nbody) {
    double v[6] = {0, 0, 0, 0, 0, 0};
    for (int d = m.body_lastdof[b]; d >= 0; d = m.dof_parentid[d]) {
      double xd = x[d];
      for (int c = 0; c < 6; c++) v[c] += cdof[6 * d + c] * xd;
    }
    for (int c = 0; c < 6; c++) Vb[6 * b + c] = v[c];
  }
  gsync();
}
// base rows of every contact applied to the current V_b: out slot `slot` (offset inside the contact record)
__device__ __noinline__ void contact_base(double* ws, const int* wi, int ncon, int slot, int lane) {
  const Layout& L = c_L;
  const double* Vb = ws + L.Vb;
  LANE_LOOP(i, ncon) {
    double* c = ws + L.con + i * L.cstride;
    int b1 = wi[L.i_cb1 + i], b2 = wi[L.i_cb2 + i], dim = wi[L.i_cdim + i];
    double rel[6], pv[3], t[3];
    for (int k = 0; k < 6; k++) rel[k] = Vb[6 * b2 + k] - Vb[6 * b1 + k];
    v3cross(t, rel, c + C_POS); v3add(pv, rel + 3, t);
    for (int k = 0; k < dim; k++) c[slot + k] = k < 3 ? v3dot(c + C_FRAME + 3 * k, pv) : v3dot(c + C_FRAME + 3 * (k - 3), rel);
  }
}
__device__ __noinline__ void simple_base(double* ws, const int* wi, int nsr, const double* x, int field, int lane) {
  const Layout& L = c_L;
  LANE_LOOP(i, nsr) {
    int A = wi[L.i_srA + i], B = wi[L.i_srB + i];
    srv(ws, field, i) = srv(ws, SR_CA, i) * x[A] + (B >= 0 ? srv(ws, SR_CB, i) * x[B] : 0.0);
  }
}

// equality + limit rows and the velocity-dependent part of every row's reference acceleration.  Returns #simple rows.
__device__ __noinline__ int stage_constraints(double* ws, int* wi, int lane, int ncon, int* status) {
  const DevModel& m = c_m; const Layout& L = c_L;
  const double *qpos = ws + L.qpos, *qvel = ws + L.qvel;
  int nsr = 0;
  LANE_LOOP(i, m.neq) {  // joint coupling q1 - q1_0 = poly(q2 - q2_0)
    int j1 = m.eq_jnt1[i], j2 = m.eq_jnt2[i];
    const double* c = m.eq_polycoef + 5 * i;
    int a1 = m.jnt_qposadr[j1], d1 = m.jnt_dofadr[j1], d2 = -1;
    double x1 = qpos[a1] - m.qpos0[a1], pos, deriv = 0, diag = m.dof_invweight0[d1];
    if (j2 >= 0) {
      int a2 = m.jnt_qposadr[j2];
      d2 = m.jnt_dofadr[j2];
      double x2 = qpos[a2] - m.qpos0[a2];
      pos = x1 - (c[0] + x2 * (c[1] + x2 * (c[2] + x2 * (c[3] + x2 * c[4]))));
      deriv = c[1] + x2 * (2 * c[2] + x2 * (3 * c[3] + x2 * 4 * c[4]));
      diag += m.dof_invweight0[d2];
    } else pos = x1 - c[0];
    double imp, K, B;
    impedance(m.eq_solref + 2 * i, m.eq_solimp + 5 * i, pos, 0, imp, K, B);
    double vel = qvel[d1] - (d2 >= 0 ? deriv * qvel[d2] : 0.0);
    double R = (1 - imp) / imp * diag;
    if (R < GE_MINVAL) R = GE_MINVAL;
    wi[L.i_srA + i] = d1; wi[L.i_srB + i] = d2; wi[L.i_srtype + i] = 0;
    srv(ws, SR_CA, i) = 1; srv(ws, SR_CB, i) = -deriv; srv(ws, SR_D, i) = 1.0 / R; srv(ws, SR_AREF, i) = -B * vel - K * imp * pos;
  }
  nsr = m.neq;
  for (int base = 0; base < m.njnt; base += GE_LANES) {  // joint limits, ordered compaction (joint order, lower side first)
    int j = base + lane, cnt = 0;
    double dist[2];
    if (j < m.njnt && m.jnt_limited[j]) {
      double q = qpos[m.jnt_qposadr[j]], mg = m.jnt_margin[j];
      dist[0] = q - m.jnt_range[2 * j]; dist[1] = m.jnt_range[2 * j + 1] - q;
      cnt = (dist[0] < mg) + (dist[1] < mg);
    }
    int total;
    int off = nsr + group_exscan(cnt, lane, total);
    if (cnt) {
      double mg = m.jnt_margin[j];
      int d = m.jnt_dofadr[j];
      for (int side = 0; side < 2; side++) {
        if (!(dist[side] < mg)) continue;
        if (off >= GE_MAXSR) break;
        double imp, K, B, sgn = side == 0 ? 1.0 : -1.0;
        impedance(m.jnt_solref + 2 * j, m.jnt_solimp + 5 * j, dist[side], mg, imp, K, B);
        double R = (1 - imp) / imp * m.dof_invweight0[d];
        if (R < GE_MINVAL) R = GE_MINVAL;
        wi[L.i_srA + off] = d; wi[L.i_srB + off] = -1; wi[L.i_srtype + off] = 1;
        srv(ws, SR_CA, off) = sgn; srv(ws, SR_CB, off) = 0; srv(ws, SR_D, off) = 1.0 / R;
        srv(ws, SR_AREF, off) = -B * sgn * qvel[d] - K * imp * (dist[side] - mg);
        off++;
      }
    }
    nsr += total;
  }
  if (nsr > GE_MAXSR) { nsr = GE_MAXSR; *status |= 8; }  // GE_STATUS_ROW_OVERFLOW
  body_vel(ws, qvel, lane);
  contact_base(ws, wi, ncon, c_vel(), lane);
  gsync();
  return nsr;
}

// value and alpha-derivative of pyramid row r of a contact given base values a[] (+ alpha * v[]); rows: r=2(k-1)+s
struct RowIter {
  const double* c; int dim, nrow;
  __device__ __forceinline__ RowIter(const double* c_, int dim_) : c(c_), dim(dim_), nrow(dim_ == 1 ? 1 : 2 * (dim_ - 1)) {}
  // x = J_r a - aref_r for base values `a`
  __device__ __forceinline__ double value(const double* a, int r, double& smu, int& k) const {
    const double* vel = c + c_vel();
    if (dim == 1) { smu = 0; k = 0; return a[0] + c[C_B] * vel[0] + c[C_KR]; }
    k = 1 + (r >> 1);
    smu = (r & 1) ? -c[C_MU + k - 1] : c[C_MU + k - 1];
    return (a[0] + smu * a[k]) + c[C_B] * (vel[0] + smu * vel[k]) + c[C_KR];
  }
};

// forces / active sets / constraint cost at the current ja; writes base forces into the jv slots and qfrc_constraint
__device__ __noinline__ double nt_update(double* ws, int* wi, int ncon, int nsr, int lane) {
  const DevModel& m = c_m; const Layout& L = c_L;
  double cost = 0;
  const int ja = c_ja(), jv = c_jv();
  LANE_LOOP(i, ncon) {
    double* c = ws + L.con + i * L.cstride;
    int dim = wi[L.i_cdim + i], mask = 0;
    RowIter it(c, dim);
    double F[6] = {0, 0, 0, 0, 0, 0}, D = c[C_D];
    for (int r = 0; r < it.nrow; r++) {
      double smu; int k;
      double x = it.value(c + ja, r, smu, k);
      if (x < 0) { double f = -D * x; cost += 0.5 * D * x * x; F[0] += f; if (k) F[k] += smu * f; mask |= 1 << r; }
    }
    for (int k = 0; k < dim; k++) c[jv + k] = F[k];
    wi[L.i_cact + i] = mask;
  }
  LANE_LOOP(i, nsr) {
    double x = srv(ws, SR_JA, i) - srv(ws, SR_AREF, i), D = srv(ws, SR_D, i);
    int act = wi[L.i_srtype + i] == 0 || x < 0;
    wi[L.i_sract + i] = act;
    srv(ws, SR_JV, i) = act ? -D * x : 0.0;
    if (act) cost += 0.5 * D * x * x;
  }
  cost = group_sum(cost);
  gsync();
  // J^T f: one lane per contact forms the contact wrench about the world origin once (scratch: the Hessian storage, free
  // between two Newton directions), one lane per body then adds the wrenches of its contacts in contact order
  double *Wb = ws + L.Wb, *Wsub = ws + L.Vb, *Wc = ws + L.H;
  LANE_LOOP(i, ncon) {
    const double* c = ws + L.con + i * L.cstride;
    int dim = wi[L.i_cdim + i];
    double f[3] = {0, 0, 0}, tq[3], tr[3] = {0, 0, 0};
    for (int k = 0; k < dim && k < 3; k++) v3addscl(f, f, c + C_FRAME + 3 * k, c[jv + k]);
    for (int k = 3; k < dim; k++) v3addscl(tr, tr, c + C_FRAME + 3 * (k - 3), c[jv + k]);
    v3cross(tq, c + C_POS, f); v3add(tq, tq, tr);
    for (int k = 0; k < 3; k++) { Wc[6 * i + k] = tq[k]; Wc[6 * i + 3 + k] = f[k]; }
  }
  gsync();
  LANE_LOOP(b, m.nbody) {
    double w[6] = {0, 0, 0, 0, 0, 0};
    if (m.body_lastdof[b] >= 0)
      NO_UNROLL for (int i = 0; i < ncon; i++) {
        int b1 = wi[L.i_cb1 + i], b2 = wi[L.i_cb2 + i];
        if (b2 == b) for (int k = 0; k < 6; k++) w[k] += Wc[6 * i + k];
        if (b1 == b) for (int k = 0; k < 6; k++) w[k] -= Wc[6 * i + k];
      }
    for (int k = 0; k < 6; k++) Wb[6 * b + k] = w[k];
  }
  gsync();
  LANE_LOOP(b, m.nbody) {
    double s[6] = {0, 0, 0, 0, 0, 0};
    int n = m.body_subtreenum[b];
    NO_UNROLL for (int c2 = b; c2 < b + n; c2++) for (int k = 0; k < 6; k++) s[k] += Wb[6 * c2 + k];
    for (int k = 0; k < 6; k++) Wsub[6 * b + k] = s[k];
  }
  gsync();
  double* qfc = ws + L.qfrc_constraint;
  const double* cdof = ws + L.cdof;
  LANE_LOOP(d, m.nv) {
    double s = dot6(cdof + 6 * d, Wsub + 6 * m.dof_bodyid[d]);
    NO_UNROLL for (int i = 0; i < nsr; i++) {
      double f = srv(ws, SR_JV, i);
      if (wi[L.i_srA + i] == d) s += srv(ws, SR_CA, i) * f;
      if (wi[L.i_srB + i] == d) s += srv(ws, SR_CB, i) * f;
    }
    qfc[d] = s;
  }
  gsync();
  return cost;
}

// constraint cost only (used for the warm-start choice); base values taken from slot `slot` / simple-row field `field`
__device__ __noinline__ double rows_cost(double* ws, const int* wi, int ncon, int nsr, int slot, int field, int lane) {
  const Layout& L = c_L;
  double cost = 0;
  LANE_LOOP(i, ncon) {
    const double* c = ws + L.con + i * L.cstride;
    RowIter it(c, wi[L.i_cdim + i]);
    for (int r = 0; r < it.nrow; r++) { double smu; int k; double x = it.value(c + slot, r, smu, k); if (x < 0) cost += 0.5 * c[C_D] * x * x; }
  }
  LANE_LOOP(i, nsr) {
    double x = srv(ws, field, i) - srv(ws, SR_AREF, i);
    if (wi[L.i_srtype + i] == 0 || x < 0) cost += 0.5 * srv(ws, SR_D, i) * x * x;
  }
  return group_sum(cost);
}

}  // namespace ge
#include "ge_hessian.cuh"
namespace ge {

// Newton solver; returns the number of iterations. Output: ws[qacc], ws[qfrc_constraint].
// CTA barriers inside the FIRST Newton iteration (which every stepping warp executes): keeps the warps of a CTA on the same
// code so that they share instruction-cache lines; later iterations run unsynchronised.
#define GE_NEWTON_BARRIERS 4
__device__ __forceinline__ void newton_barrier(bool sync) { if (sync) asm volatile("barrier.sync 1, %0;" ::"r"((int)(blockDim.x * blockDim.y)) : "memory"); }

__device__ __noinline__ int solve_newton(double* ws, int* wi, int lane, int ncon, int nsr, bool sync = false) {
  const DevModel& m = c_m; const Layout& L = c_L;
  int nv = m.nv;
  double *qacc = ws + L.qacc, *qacc_smooth = ws + L.qacc_smooth, *qfrc_smooth = ws + L.qfrc_smooth, *qaccws = ws + L.qaccws;
  double *Ma = ws + L.Ma, *Mv = ws + L.Mv, *grad = ws + L.grad, *search = ws + L.search, *qfc = ws + L.qfrc_constraint;
  const double* qM = ws + L.qM;
  const int ja = c_ja(), jv = c_jv();
  LANE_LOOP(d, nv) { qacc[d] = qacc_smooth[d]; qfc[d] = 0; }
  gsync();
  if (ncon + nsr == 0) { for (int k = 0; k < GE_NEWTON_BARRIERS; k++) newton_barrier(sync); return 0; }
  // warm start choice
  LANE_LOOP(d, nv) grad[d] = qaccws[d] - qacc_smooth[d];
  gsync();
  mul_M(qM, Mv, grad, lane);
  double gws = 0;
  LANE_LOOP(d, nv) gws += 0.5 * grad[d] * Mv[d];
  gws = group_sum(gws);
  body_vel(ws, qaccws, lane); contact_base(ws, wi, ncon, jv, lane); simple_base(ws, wi, nsr, qaccws, SR_JV, lane);
  gsync();
  body_vel(ws, qacc_smooth, lane); contact_base(ws, wi, ncon, ja, lane); simple_base(ws, wi, nsr, qacc_smooth, SR_JA, lane);
  gsync();
  double cost_ws = gws + rows_cost(ws, wi, ncon, nsr, jv, SR_JV, lane), cost_0 = rows_cost(ws, wi, ncon, nsr, ja, SR_JA, lane);
  if (cost_ws < cost_0) {
    LANE_LOOP(d, nv) qacc[d] = qaccws[d];
    LANE_LOOP(i, ncon) { double* c = ws + L.con + i * L.cstride; for (int k = 0; k < wi[L.i_cdim + i]; k++) c[ja + k] = c[jv + k]; }
    LANE_LOOP(i, nsr) srv(ws, SR_JA, i) = srv(ws, SR_JV, i);
  }
  gsync();
  GE_CLK(SC_NEWTON);
  mul_M(qM, Ma, qacc, lane);
  GE_CLK(SC_MULM_COLD);
  GE_WARM(SC_MULM_COLD, SC_WARM_MULM, mul_M(qM, Ma, qacc, lane));
  double cost_c = nt_update(ws, wi, ncon, nsr, lane), gauss = 0;
  GE_CLK(SC_NT_UPDATE);
  LANE_LOOP(d, nv) gauss += 0.5 * (Ma[d] - qfrc_smooth[d]) * (qacc[d] - qacc_smooth[d]);
  double cost = group_sum(gauss) + cost_c;
  double scale = 1.0 / (m.meaninertia * (nv > 1 ? nv : 1));
  int niter = 0;
  NO_UNROLL for (int it = 0; it < m.iterations; it++) {
    double gn = 0;
    LANE_LOOP(d, nv) { double g = Ma[d] - qfrc_smooth[d] - qfc[d]; grad[d] = g; gn += g * g; }
    gn = group_sum(gn);
    gsync();
    if (it > 0 && scale * sqrt(gn) < m.tolerance) break;
    GE_CLK(SC_NEWTON);
    if (it == 0) newton_barrier(sync);
    GE_CLK(SC_BARRIER);
    build_hessian(ws, wi, ncon, nsr, lane);
    GE_CLK(SC_HESSIAN);
    if (it == 0) newton_barrier(sync);
    GE_CLK(SC_BARRIER);
    cholesky_solve(ws, wi, search, grad, lane);
    GE_CLK(SC_CHOL);
    mul_M(qM, Mv, search, lane);
    double g1 = 0, g2 = 0, sn = 0;
    LANE_LOOP(d, nv) { g1 += search[d] * (Ma[d] - qfrc_smooth[d]); g2 += 0.5 * search[d] * Mv[d]; sn += search[d] * search[d]; }
    g1 = group_sum(g1); g2 = group_sum(g2); sn = sqrt(group_sum(sn));
    body_vel(ws, search, lane); contact_base(ws, wi, ncon, jv, lane); simple_base(ws, wi, nsr, search, SR_JV, lane);
    gsync();
    GE_CLK(SC_NEWTON);
    if (it == 0) newton_barrier(sync);
    GE_CLK(SC_BARRIER);
    // exact line search: safeguarded 1-D Newton on the convex piecewise-quadratic cost along `search`
    double gtol = m.tolerance * 0.01 * sn * m.meaninertia * (nv > 1 ? nv : 1);
    if (gtol < GE_MINVAL) gtol = GE_MINVAL;
    double alpha = 0, lo = 0, hi = -1;
    NO_UNROLL for (int ls = 0; ls < 50; ls++) {
      double d1 = 0, d2 = 0;
      LANE_LOOP(i, ncon) {
        const double* c = ws + L.con + i * L.cstride;
        RowIter ri(c, wi[L.i_cdim + i]);
        double a[6];
        for (int k = 0; k < ri.dim; k++) a[k] = c[ja + k] + alpha * c[jv + k];
        for (int r = 0; r < ri.nrow; r++) {
          double smu; int k;
          double x = ri.value(a, r, smu, k);
          if (x < 0) { double v = c[jv] + (k ? smu * c[jv + k] : 0.0); d1 += c[C_D] * x * v; d2 += c[C_D] * v * v; }
        }
      }
      LANE_LOOP(i, nsr) {
        double v = srv(ws, SR_JV, i), x = srv(ws, SR_JA, i) + alpha * v - srv(ws, SR_AREF, i);
        if (wi[L.i_srtype + i] == 0 || x < 0) { double D = srv(ws, SR_D, i); d1 += D * x * v; d2 += D * v * v; }
      }
      d1 = group_sum(d1) + g1 + 2 * g2 * alpha; d2 = group_sum(d2) + 2 * g2;
      if (fabs(d1) < gtol) break;
      if (d1 < 0) lo = alpha; else hi = alpha;
      double next = alpha - d1 / d2;
      if (hi >= 0 && (next <= lo || next >= hi)) next = 0.5 * (lo + hi);
      alpha = next;
    }
    GE_CLK(SC_LINESEARCH);
    if (it == 0) newton_barrier(sync);
    GE_CLK(SC_BARRIER);
    niter = it + 1;
    if (alpha == 0) break;
    LANE_LOOP(d, nv) { qacc[d] += alpha * search[d]; Ma[d] += alpha * Mv[d]; }
    LANE_LOOP(i, ncon) { double* c = ws + L.con + i * L.cstride; for (int k = 0; k < wi[L.i_cdim + i]; k++) c[ja + k] += alpha * c[jv + k]; }
    LANE_LOOP(i, nsr) srv(ws, SR_JA, i) += alpha * srv(ws, SR_JV, i);
    gsync();
    double oldcost = cost;
    GE_CLK(SC_NEWTON);
    cost_c = nt_update(ws, wi, ncon, nsr, lane);
    GE_CLK(SC_NT_UPDATE);
    gauss = 0;
    LANE_LOOP(d, nv) gauss += 0.5 * (Ma[d] - qfrc_smooth[d]) * (qacc[d] - qacc_smooth[d]);
    cost = group_sum(gauss) + cost_c;
    if (scale * (oldcost - cost) < m.tolerance) break;
  }
  return niter;
}

}  // namespace ge
