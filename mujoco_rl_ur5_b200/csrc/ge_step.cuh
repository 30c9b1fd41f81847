// One simulation sub-step, the PID movement loop and the grasp program, all inside one warp.
//
// Reference call sites: MJ_Controller.move_group_to_joint_target (MujocoController.py:269-393, loop :318-382),
// MJ_Controller.stay (:621-637), move_ee / ik (:446-517), GraspEnv.move_and_grasp (GraspingEnv.py:205-386).
#pragma once
#include "ge_solver.cuh"

namespace ge {

#define CTL_TARGET 0
#define CTL_LAST 8
#define CTL_KP 16
#define CTL_CTRL 24

struct StepInfo { int ncon, nsr, niter, ncand, nmpr; };  // ncand, nmpr: see CollisionCounts

// Stage barriers (warp-per-env build): all warps of the CTA (one env each) enter collision, the constraint solver and the
// integrator together, so that the SM's instruction cache serves the (large) stage code once per CTA instead of once per warp.
// Warps that do not step in an iteration must call stage_barriers_idle() to keep the barrier counts equal.
#define GE_NUM_STAGE_BARRIERS (3 + GE_NEWTON_BARRIERS)
// The warps of a CTA reach these barriers from DIFFERENT code locations (a stepping warp inside forward() / solve_newton(), a warp
// whose environment does not step this iteration in stage_barriers_idle()).  That is legal for the unaligned PTX barrier
// (`barrier.sync id, count`: any convergent warp may arrive from anywhere, the hardware counts arrivals) but not for __syncthreads()
// (`barrier.sync.aligned` semantics in CUDA C++; compute-sanitizer synccheck reported "divergent thread(s) in block", r02b), so the
// stage barriers use named barrier 1 with the CTA's thread count.
__device__ __forceinline__ void cta_barrier_unaligned() {
  asm volatile("barrier.sync 1, %0;" ::"r"((int)(blockDim.x * blockDim.y)) : "memory");
}
__device__ __forceinline__ void stage_barrier(bool sync) { if (sync) cta_barrier_unaligned(); }
__device__ __forceinline__ void stage_barriers_idle(bool on) { if (on) for (int k = 0; k < GE_NUM_STAGE_BARRIERS; k++) cta_barrier_unaligned(); }

// debugging aid (GE_NANCHECK=1): first stage whose output holds a non-finite value -> one of status bits 8..15 (only the first is kept)
__device__ __noinline__ void nan_probe(const double* a, int n, int lane, int* status, int bit) {
  bool bad = false;
  LANE_LOOP(i, n) if (!isfinite(a[i])) bad = true;
  bad = group_any(bad);
  if (bad && !(*status & 0xff00)) *status |= 1 << bit;
}
// mj_forward: kinematics -> bias -> mass matrix -> collision -> constraints -> smooth acceleration -> Newton
__device__ __noinline__ StepInfo forward(double* ws, int* wi, int lane, int* status, bool sync = false) {
  const DevModel& m = c_m; const Layout& L = c_L;
  StepInfo si;
  const bool dbg = c_nancheck != 0;
  if (dbg) { nan_probe(ws + L.qpos, m.nq, lane, status, 8); nan_probe(ws + L.qvel, m.nv, lane, status, 8); nan_probe(ws + L.ctl, 32, lane, status, 8); }
  stage_fk(ws, lane);
  GE_CLK(SC_FK);
  GE_WARM(SC_FK, SC_WARM_FK, stage_fk(ws, lane));
  if (dbg) { nan_probe(ws + L.gmat, 9 * m.ngeom, lane, status, 9); nan_probe(ws + L.cdof, 6 * m.nv, lane, status, 9); }
  stage_barrier(sync);
  GE_CLK(SC_BARRIER);
  {
    const CollisionCounts cc = stage_collision(ws, wi, lane, status);  // needs the geom frames only; bias forces / mass matrix reuse their storage
    si.ncon = cc.ncon; si.ncand = cc.ncand; si.nmpr = cc.nmpr;
  }
  GE_CLK(SC_COLLISION);
  stage_rne(ws, lane);  // qfrc_smooth := bias
  stage_crb(ws, lane);
  GE_CLK(SC_RNE_CRB);
  GE_WARM(SC_RNE_CRB, SC_WARM_RNE_CRB, stage_rne(ws, lane); stage_crb(ws, lane));
  if (dbg) { nan_probe(ws + L.qM, m.nM, lane, status, 11); nan_probe(ws + L.qfrc_smooth, m.nv, lane, status, 11); }
  // smooth forces: passive (joint damping) - bias + actuation (torque motors, gear * clamp(ctrl))
  const double *qvel = ws + L.qvel, *ctrl = ws + L.ctl + CTL_CTRL;
  double *qfs = ws + L.qfrc_smooth, *qas = ws + L.qacc_smooth;
  LANE_LOOP(d, m.nv) qfs[d] = -m.dof_damping[d] * qvel[d] - qfs[d];
  gsync();
  if (lane < m.nu) {
    double c = ctrl[lane], lo = m.actuator_ctrlrange[2 * lane], hi = m.actuator_ctrlrange[2 * lane + 1];
    c = c < lo ? lo : (c > hi ? hi : c);
    qfs[m.jnt_dofadr[m.actuator_jntid[lane]]] += m.actuator_gear[lane] * c;  // one actuator per joint in these scenes
  }
  gsync();
  LANE_LOOP(d, m.nv) qas[d] = qfs[d];
  gsync();
  // qacc_smooth = M^-1 qfrc_smooth: dense per-tree Cholesky in 8-lane groups (Hessian storage is free here)
  mass_block_solve(ws, qas, 0.0, lane);
  if (dbg) nan_probe(qas, m.nv, lane, status, 12);
  GE_CLK(SC_MASS);
  stage_barrier(sync);
  GE_CLK(SC_BARRIER);
  si.nsr = stage_constraints(ws, wi, lane, si.ncon, status);
  GE_CLK(SC_CONSTRAINTS);
  si.niter = solve_newton(ws, wi, lane, si.ncon, si.nsr, sync);
  if (dbg) nan_probe(ws + L.qacc, m.nv, lane, status, 14);
  if (si.niter >= m.iterations) *status |= 4;
  LANE_LOOP(d, m.nv) ws[L.qaccws + d] = ws[L.qacc + d];
  gsync();
  GE_CLK(SC_NEWTON);
  return si;
}

// mj_step = mj_forward + semi-implicit Euler with implicit joint damping
__device__ __noinline__ StepInfo sim_step(double* ws, int* wi, int lane, int* status, bool sync = false) {
  const DevModel& m = c_m; const Layout& L = c_L;
  StepInfo si = forward(ws, wi, lane, status, sync);
  stage_barrier(sync);
  GE_CLK(SC_BARRIER);
  double h = m.timestep;
  double *acc = ws + L.grad, *qvel = ws + L.qvel, *qpos = ws + L.qpos;
  LANE_LOOP(d, m.nv) acc[d] = ws[L.qfrc_smooth + d] + ws[L.qfrc_constraint + d];
  gsync();
  mass_block_solve(ws, acc, m.any_damping ? h : 0.0, lane);
  LANE_LOOP(d, m.nv) qvel[d] += h * acc[d];
  gsync();
  bool bad = false;
  LANE_LOOP(j, m.njnt) {
    int qa = m.jnt_qposadr[j], d = m.jnt_dofadr[j], type = m.jnt_type[j];
    if (type == J_HINGE || type == J_SLIDE) { qpos[qa] += h * qvel[d]; if (!isfinite(qpos[qa])) bad = true; continue; }
    if (type == J_FREE) { for (int k = 0; k < 3; k++) qpos[qa + k] += h * qvel[d + k]; qa += 3; d += 3; }
    double w[3] = {qvel[d], qvel[d + 1], qvel[d + 2]}, dq[4], nq[4];
    double ang = v3normalize(w) * h;
    qaxisangle(dq, w, ang);
    qmul(nq, qpos + qa, dq); qnormalize(nq);
    for (int k = 0; k < 4; k++) qpos[qa + k] = nq[k];
    if (!isfinite(nq[0])) bad = true;
  }
  if (group_any(bad)) *status |= 2;
  gsync();
  GE_CLK(SC_EULER);
  GE_CLK_COUNT(SC_SUBSTEPS);
  return si;
}

// 7 PID controllers (Ki = 0), derivative on measurement with the fixed controller period dt_pid (SURVEY A.2)
__device__ __noinline__ double pid_and_delta(double* ws, int lane, int group_mask, double dt_pid) {
  const DevModel& m = c_m; const Layout& L = c_L;
  double* ctl = ws + L.ctl;
  double delta = 0;
  if (lane < GE_NU) {
    double x = ws[L.qpos + m.jnt_qposadr[m.actuator_jntid[lane]]];
    double lim = m.pid_lim[lane];
    double u = ctl[CTL_KP + lane] * (ctl[CTL_TARGET + lane] - x) - m.pid_kd[lane] * (x - ctl[CTL_LAST + lane]) / dt_pid;
    u = u < -lim ? -lim : (u > lim ? lim : u);
    ctl[CTL_LAST + lane] = x; ctl[CTL_CTRL + lane] = u;
    if (group_mask >> lane & 1) delta = fabs(ctl[CTL_TARGET + lane] - x);
  }
  delta = group_max(delta);
  gsync();
  return delta;
}

// analytic tool-down IK of the ur5_gripper.urdf chain (SURVEY A.4); base = world position of base_link
__device__ __noinline__ bool ik_solve(const double* ee_pos, const double* base, double* q5) {
  const DevModel& m = c_m;
  const double* ch = m.ik_chain;
  double d1 = ch[0], d4 = ch[1], a1 = ch[2], a2 = ch[3], d5 = ch[4], d6 = ch[5], p[3];
  const double PI = 3.14159265358979323846;
  for (int k = 0; k < 3; k++) p[k] = ee_pos[k] - base[k] + m.ik_offset[k];
  double r2 = p[0] * p[0] + p[1] * p[1];
  if (r2 < d4 * d4 + 1e-12) return false;
  double r = sqrt(r2), phi = atan2(p[1], p[0]);
  double pan = phi - asin(d4 / r);
  if (pan < -PI) pan += 2 * PI;
  if (pan > PI) pan -= 2 * PI;
  double rho = sqrt(r2 - d4 * d4), Wx = rho - d5, Wz = p[2] + d6 - d1;
  double L2 = Wx * Wx + Wz * Wz, c = (L2 - a1 * a1 - a2 * a2) / (2 * a1 * a2);
  if (c > 1) c = 1;
  if (c < -1) c = -1;
  double elbow = acos(c);
  double alpha = atan2(Wz, Wx) + atan2(a2 * sin(elbow), a1 + a2 * cos(elbow));
  double lift = -alpha, w1 = -0.5 * PI - lift - elbow, w2 = -0.5 * PI;
  if (w1 < -PI) w1 += 2 * PI;
  if (w1 > PI) w1 -= 2 * PI;
  double fx = a1 * cos(alpha) + a2 * cos(alpha - elbow), fz = a1 * sin(alpha) + a2 * sin(alpha - elbow);
  double err = sqrt((fx - Wx) * (fx - Wx) + (fz - Wz) * (fz - Wz));
  q5[0] = pan; q5[1] = lift; q5[2] = elbow; q5[3] = w1; q5[4] = w2;
  for (int k = 0; k < 5; k++) if (q5[k] < m.ik_lower[k] - 1e-9 || q5[k] > m.ik_upper[k] + 1e-9) return false;
  return err <= 0.02;
}

// ---- movement command + grasp program state, kept in registers while the kernel runs (all lanes hold the same values)
struct Cmd {
  int active, mask, maxsteps, steps, result, reached;
  double tol;
};
struct Prog {
  int phase, rot, grasp, aux, r1, rfinal;
  double coords[3], table;
};
enum { PH_NONE = 0, PH_PRE = 1, PH_PRE_CENTRE = 2, PH_ROTATE = 3, PH_OPEN_HALF = 4, PH_DESCEND = 5, PH_STAY1 = 6, PH_CLOSE = 7,
       PH_CENTRE = 8, PH_DROP = 9, PH_CHECK = 10, PH_OPEN = 11, PH_STAY2 = 12, PH_ROTATE_BACK = 13, PH_STAY_ONLY = 20 };

__device__ __noinline__ void start_group(Cmd& c, double* ws, int lane, int mask, const double* target, double tol, int maxsteps) {
  const Layout& L = c_L;
  if (target && lane == 0) { int k = 0; for (int i = 0; i < GE_NU; i++) if (mask >> i & 1) ws[L.ctl + CTL_TARGET + i] = target[k++]; }
  gsync();
  c.active = 1; c.mask = mask; c.tol = tol; c.maxsteps = maxsteps; c.steps = 1; c.result = 0; c.reached = 0;
}
__device__ __noinline__ void start_ee(Cmd& c, double* ws, int lane, const double* xyz, const double* base, double tol, int maxsteps) {
  double q5[5];
  if (!ik_solve(xyz, base, q5)) { c.active = 0; c.result = 3; c.steps = 0; return; }
  start_group(c, ws, lane, 0x1f, q5, tol, maxsteps);
}

// Called when the current movement has ended; starts the next movement of the grasp program (if any).
// info[12] mirrors the oracle's per-phase record.  Returns false when the program is finished.
__device__ __noinline__ bool prog_advance(Prog& p, Cmd& c, double* ws, int lane, const double* base, int* info, unsigned char* reward) {
  const Layout& L = c_L;
  const double centre[3] = {0.0, -0.6, 1.1}, drop[3] = {0.6, 0.0, 1.15};
  const double ROT_DEG[6] = {0, 30, 60, 90, -30, -60};
  const double PI = 3.14159265358979323846;
  while (true) {
    switch (p.phase) {
      case PH_PRE:
        if (c.result == 3) {  // IK failed: try the table centre as pre-grasp position (GraspingEnv.py:227-239)
          p.phase = PH_PRE_CENTRE;
          start_ee(c, ws, lane, centre, base, 0.05, 1000);
          if (c.active) return true;
          continue;
        }
        info[0] = c.result == 3 ? 0 : c.result; info[1] = c.steps; p.r1 = info[0];
        goto after_pre;
      case PH_PRE_CENTRE:
        p.r1 = c.result == 3 ? 0 : c.result; info[0] = 10 + p.r1; info[1] = c.steps;
      after_pre:
        if (p.r1 != 2) {
          if (lane == 0) ws[L.ctl + CTL_TARGET + 5] = ROT_DEG[p.rot] * PI / 180.0;
          p.phase = PH_ROTATE;
          start_group(c, ws, lane, 0x7f, nullptr, 0.05, 500);
          return true;
        }
        p.grasp = 0;
        goto to_centre;
      case PH_ROTATE: {
        info[2] = c.steps;
        const double half[1] = {0.0};
        p.phase = PH_OPEN_HALF;
        start_group(c, ws, lane, 0x40, half, 0.05, 1000);
        return true;
      }
      case PH_OPEN_HALF: {
        double z = p.coords[2] - 0.01;
        double c2[3] = {p.coords[0], p.coords[1], z > p.table ? z : p.table};
        p.phase = PH_DESCEND;
        start_ee(c, ws, lane, c2, base, 0.01, 300);
        if (c.active) return true;
        continue;
      }
      case PH_DESCEND:
        info[3] = c.result == 3 ? 0 : c.result; info[4] = c.steps;
        if (c.result == 2) { p.grasp = 0; goto to_centre; }
        p.phase = PH_STAY1; p.aux = 5;  // stay(100 ms) = 5 chunks of 10 sub-steps
        start_group(c, ws, lane, 0x7f, nullptr, 1e-7, 10);
        return true;
      case PH_STAY1:
        if (--p.aux > 0) { start_group(c, ws, lane, 0x7f, nullptr, 1e-7, 10); return true; }
        {
          const double cl[1] = {-0.4};
          p.phase = PH_CLOSE;
          start_group(c, ws, lane, 0x40, cl, 0.01, 300);
          return true;
        }
      case PH_CLOSE:
        p.grasp = c.result != 1; info[5] = c.steps;
      to_centre:
        if (lane == 0) ws[L.ctl + CTL_KP + 0] = 10.0;  // GraspingEnv.py:282
        gsync();
        p.phase = PH_CENTRE;
        start_ee(c, ws, lane, centre, base, 0.05, 1000);
        if (c.active) return true;
        continue;
      case PH_CENTRE:
        info[6] = c.steps;
        p.phase = PH_DROP;
        start_ee(c, ws, lane, drop, base, 0.01, 1200);
        if (c.active) return true;
        continue;
      case PH_DROP:
        info[7] = c.steps;
        p.rfinal = -1;
        if (p.grasp) {
          const double cl[1] = {-0.4};
          p.phase = PH_CHECK;
          start_group(c, ws, lane, 0x40, cl, 0.01, 1000);
          return true;
        }
        goto do_open;
      case PH_CHECK:
        p.rfinal = c.result; info[8] = c.steps;
      do_open: {
        const double op[1] = {0.4};
        p.phase = PH_OPEN;
        start_group(c, ws, lane, 0x40, op, 0.05, 1000);
        return true;
      }
      case PH_OPEN:
        info[9] = c.steps;
        if (p.rfinal == 2 && p.grasp) {
          *reward = 1;
          p.phase = PH_STAY2; p.aux = 10;  // stay(200 ms)
          start_group(c, ws, lane, 0x7f, nullptr, 1e-7, 10);
          return true;
        }
        *reward = 0;
        goto rotate_back;
      case PH_STAY2:
        if (--p.aux > 0) { start_group(c, ws, lane, 0x7f, nullptr, 1e-7, 10); return true; }
      rotate_back:
        if (lane == 0) ws[L.ctl + CTL_TARGET + 5] = 0.0;
        p.phase = PH_ROTATE_BACK;
        start_group(c, ws, lane, 0x7f, nullptr, 0.05, 500);
        return true;
      case PH_ROTATE_BACK:
        info[10] = c.steps; info[11] = p.grasp;
        if (lane == 0) ws[L.ctl + CTL_KP + 0] = 20.0;  // GraspingEnv.py:347
        gsync();
        p.phase = PH_NONE;
        return false;
      case PH_STAY_ONLY:
        if (--p.aux > 0) { start_group(c, ws, lane, 0x7f, nullptr, 1e-7, 10); return true; }
        p.phase = PH_NONE;
        return false;
      default:
        return false;
    }
  }
}

}  // namespace ge
