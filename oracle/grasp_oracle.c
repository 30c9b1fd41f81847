/* ===========================================================================================
 * TEST INFRASTRUCTURE — CPU ORACLE.  NOT PART OF THE SHIPPED PRODUCT.
 *
 * Single-environment, single-thread, fp64 restatement of the reference's hot path:
 *   PID actuation -> mj_step sub-step loop   (gym_grasper/controller/MujocoController.py:269-393)
 *   grasp state machine                      (gym_grasper/envs/GraspingEnv.py:205-386)
 *   top-down IK                              (MujocoController.py:467-517, ikpy [EXT])
 *   RGB-D observation                        (MujocoController.py:708-740)
 *
 * PARITY UNPINNED: the arithmetic of `sim.step()` lives in MuJoCo / mujoco_py, `PID` in simple_pid and the
 * IK in ikpy; none of them is vendored in /root/reference, none is pinned (requirements.txt:1-9) and none
 * can be installed here.  This file restates the algorithms from the MuJoCo documentation ("Computation"
 * chapter) as summarised in SURVEY.md Appendix A.  It is pinned only by the weak known-answer vectors of
 * SURVEY.md section 8(c) (tests/test_oracle_kat.py) and by physics invariants.  Every place where a MuJoCo
 * internal had to be re-derived is marked DECISION.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may load this.
 * =========================================================================================== */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include "orc_math.h"

#define G_PLANE 0
#define G_SPHERE 2
#define G_CAPSULE 3
#define G_CYLINDER 5
#define G_BOX 6
#define G_MESH 7
#define J_FREE 0
#define J_BALL 1
#define J_SLIDE 2
#define J_HINGE 3

#define MAXCON 256
#define NU 7

/* ------------------------------------------------------------------ blob access */
typedef struct { char name[32]; int32_t dtype, ndim; int64_t shape[4]; int64_t offset, nbytes; } BlobEntry;
static const void* blob_get(const void* blob, const char* name, int64_t* count) {
  const char* b = (const char*)blob;
  if (memcmp(b, "GEBLOB01", 8) != 0) return NULL;
  int64_t n = *(const int64_t*)(b + 8);
  const BlobEntry* e = (const BlobEntry*)(b + 24);
  for (int64_t i = 0; i < n; i++)
    if (strncmp(e[i].name, name, 32) == 0) {
      int64_t c = 1;
      for (int k = 0; k < e[i].ndim; k++) c *= e[i].shape[k];
      if (count) *count = c;
      return b + e[i].offset;
    }
  fprintf(stderr, "oracle: blob entry '%s' missing\n", name);
  return NULL;
}
#define BD(name) ((const double*)blob_get(blob, name, NULL))
#define BI(name) ((const int32_t*)blob_get(blob, name, NULL))

typedef struct {
  void* blob;
  int nbody, njnt, nq, nv, nu, ngeom, neq, npair, nmesh, nM;
  double timestep, gravity[3], tolerance, impratio, mpr_tol, meaninertia, extent, znear, zfar;
  int iterations, mpr_iter;
  const double *qpos0, *body_pos, *body_quat, *body_mass, *body_ipos, *body_inertia, *body_invweight0;
  const int32_t *body_parentid, *body_jntadr, *body_jntnum, *body_dofadr, *body_dofnum, *body_lastdof;
  const int32_t *jnt_type, *jnt_bodyid, *jnt_qposadr, *jnt_dofadr, *jnt_limited;
  const double *jnt_pos, *jnt_axis, *jnt_range, *jnt_margin, *jnt_solref, *jnt_solimp;
  const int32_t *dof_bodyid, *dof_jntid, *dof_parentid, *dof_Madr;
  const double *dof_armature, *dof_damping, *dof_invweight0;
  const int32_t *geom_type, *geom_bodyid, *geom_meshid;
  const double *geom_pos, *geom_quat, *geom_size, *geom_rbound, *geom_obbcenter, *geom_obbhalf, *geom_rgba;
  const int32_t *mesh_vertadr, *mesh_vertnum, *mesh_faceadr, *mesh_facenum, *mesh_face;
  const double *mesh_vert, *mesh_center;
  const int32_t *pair_geom, *pair_condim;
  const double *pair_friction, *pair_margin, *pair_solref, *pair_solimp;
  const int32_t* actuator_jntid;
  const double *actuator_gear, *actuator_ctrlrange;
  const int32_t *eq_jnt1, *eq_jnt2;
  const double *eq_polycoef, *eq_solref, *eq_solimp;
  const double *cam_pos0, *cam_mat0, *cam_fovy;
  const double *pid_kp, *pid_kd, *pid_lim, *ik_chain, *ik_lower, *ik_upper, *ik_offset;
  int ik_base_body, ee_body;
  double* geom_lmat; /* geom rotation in body frame, 9 per geom */
  double* face_plane; /* per hull face: outward normal + offset (geom-local), 4 per face */
  int any_damping;
} Model;

typedef struct {
  double dist, pos[3], frame[9], margin, friction[5], solref[2], solimp[5];
  int dim, geom1, geom2;
} Contact;

/* "boxbox" diagnostics, one record of BBX_W doubles per col_box_box call of the last collision stage: geom1, geom2, outcome
 * (0 separated, 1 face contact, 2 edge-edge), the reference box (1, 2; 0 unless a face contact), the best face axis (0-5),
 * face axes whose SAT separation equals the best one bit for bit (1: no tie), edge axes with 0 < |a_i x b_j| < 1e-6 (skipped by
 * the guard), incident-face vertices that lie exactly on a clip line (kept by `da <= 0`), contacts the pair emitted */
#define BBX_MAX 64
#define BBX_W 9
typedef struct {
  Model* m;
  /* state */
  double *qpos, *qvel, *qacc_ws, ctrl[NU];
  /* controller (MujocoController.py:157-254) */
  double kp[NU], kd[NU], lim[NU], target[NU], last_input[NU], dt_pid;
  long substeps;
  /* kinematics */
  double *xpos, *xquat, *xmat, *xipos, *xanchor, *xaxis, *cdof, *cdof_dot, *cvel, *cacc, *cfrc, *cinert, *crb;
  double *gpos, *gmat;
  /* dynamics */
  double *qM, *qLD, *qH, *qfrc_bias, *qfrc_passive, *qfrc_actuator, *qfrc_smooth, *qacc_smooth, *qfrc_constraint, *qacc;
  /* contacts + constraints */
  int ncon, nefc, ne, nl, nefc_max, maxcon; /* maxcon: contacts kept (<= MAXCON, orc_set_maxcon), later ones set con_overflow */
  int maxsr, sr_overflow;                    /* maxsr: equality + limit rows kept (orc_set_maxsr; default: all), later ones set sr_overflow */
  Contact con[MAXCON];
  double *efc_J, *efc_B, *efc_pos, *efc_margin, *efc_diag, *efc_R, *efc_aref, *efc_force, *efc_AR;
  int* efc_type;
  int solver_iter, con_overflow, solver; /* solver: 0 = Newton (MuJoCo default, what the MJCF implies), 1 = PGS */
  int ncand;                             /* pairs that passed the broad phase in the last collision stage */
  int nfound, ncon_peak;                 /* contacts the last collision stage found (uncapped); the most since orc_ncon_peak reset it */
  int nbbx;                              /* box-box pairs the last collision stage ran col_box_box on (orc_field "boxbox") */
  double bbx[BBX_MAX * BBX_W];
  double *tmp1, *tmp2, *nt_H, *nt_grad, *nt_search, *nt_Ma, *nt_Mv, *nt_jar, *nt_jv;
  int* nt_active;
} Env;

/* ------------------------------------------------------------------ model */
Model* orc_model_load(const void* blob_in, int64_t nbytes) {
  Model* m = (Model*)calloc(1, sizeof(Model));
  m->blob = malloc(nbytes);
  memcpy(m->blob, blob_in, nbytes);
  const void* blob = m->blob;
  if (!blob_get(blob, "nbody", NULL)) { free(m->blob); free(m); return NULL; }
  m->nbody = BI("nbody")[0]; m->njnt = BI("njnt")[0]; m->nq = BI("nq")[0]; m->nv = BI("nv")[0]; m->nu = BI("nu")[0];
  m->ngeom = BI("ngeom")[0]; m->neq = BI("neq")[0]; m->npair = BI("npair")[0]; m->nmesh = BI("nmesh")[0]; m->nM = BI("nM")[0];
  m->timestep = BD("opt_timestep")[0]; memcpy(m->gravity, BD("opt_gravity"), 24);
  m->tolerance = BD("opt_tolerance")[0]; m->impratio = BD("opt_impratio")[0]; m->iterations = BI("opt_iterations")[0];
  m->mpr_tol = BD("opt_mpr_tolerance")[0]; m->mpr_iter = BI("opt_mpr_iterations")[0];
  m->meaninertia = BD("stat_meaninertia")[0]; m->extent = BD("stat_extent")[0];
  m->znear = BD("vis_znear")[0]; m->zfar = BD("vis_zfar")[0];
  m->qpos0 = BD("qpos0");
  m->body_pos = BD("body_pos"); m->body_quat = BD("body_quat"); m->body_mass = BD("body_mass"); m->body_ipos = BD("body_ipos");
  m->body_inertia = BD("body_inertia"); m->body_invweight0 = BD("body_invweight0");
  m->body_parentid = BI("body_parentid"); m->body_jntadr = BI("body_jntadr"); m->body_jntnum = BI("body_jntnum");
  m->body_dofadr = BI("body_dofadr"); m->body_dofnum = BI("body_dofnum"); m->body_lastdof = BI("body_lastdof");
  m->jnt_type = BI("jnt_type"); m->jnt_bodyid = BI("jnt_bodyid"); m->jnt_qposadr = BI("jnt_qposadr"); m->jnt_dofadr = BI("jnt_dofadr");
  m->jnt_limited = BI("jnt_limited"); m->jnt_pos = BD("jnt_pos"); m->jnt_axis = BD("jnt_axis"); m->jnt_range = BD("jnt_range");
  m->jnt_margin = BD("jnt_margin"); m->jnt_solref = BD("jnt_solref"); m->jnt_solimp = BD("jnt_solimp");
  m->dof_bodyid = BI("dof_bodyid"); m->dof_jntid = BI("dof_jntid"); m->dof_parentid = BI("dof_parentid"); m->dof_Madr = BI("dof_Madr");
  m->dof_armature = BD("dof_armature"); m->dof_damping = BD("dof_damping"); m->dof_invweight0 = BD("dof_invweight0");
  m->geom_type = BI("geom_type"); m->geom_bodyid = BI("geom_bodyid"); m->geom_meshid = BI("geom_meshid");
  m->geom_pos = BD("geom_pos"); m->geom_quat = BD("geom_quat"); m->geom_size = BD("geom_size"); m->geom_rbound = BD("geom_rbound");
  m->geom_obbcenter = BD("geom_obbcenter"); m->geom_obbhalf = BD("geom_obbhalf"); m->geom_rgba = BD("geom_rgba");
  m->mesh_vertadr = BI("mesh_vertadr"); m->mesh_vertnum = BI("mesh_vertnum"); m->mesh_faceadr = BI("mesh_faceadr");
  m->mesh_facenum = BI("mesh_facenum"); m->mesh_face = BI("mesh_face"); m->mesh_vert = BD("mesh_vert"); m->mesh_center = BD("mesh_center");
  m->pair_geom = BI("pair_geom"); m->pair_condim = BI("pair_condim"); m->pair_friction = BD("pair_friction");
  m->pair_margin = BD("pair_margin"); m->pair_solref = BD("pair_solref"); m->pair_solimp = BD("pair_solimp");
  m->actuator_jntid = BI("actuator_jntid"); m->actuator_gear = BD("actuator_gear"); m->actuator_ctrlrange = BD("actuator_ctrlrange");
  m->eq_jnt1 = BI("eq_jnt1"); m->eq_jnt2 = BI("eq_jnt2"); m->eq_polycoef = BD("eq_polycoef"); m->eq_solref = BD("eq_solref"); m->eq_solimp = BD("eq_solimp");
  m->cam_pos0 = BD("cam_pos0"); m->cam_mat0 = BD("cam_mat0"); m->cam_fovy = BD("cam_fovy");
  m->pid_kp = BD("pid_kp"); m->pid_kd = BD("pid_kd"); m->pid_lim = BD("pid_lim");
  m->ik_chain = BD("ik_chain"); m->ik_lower = BD("ik_lower"); m->ik_upper = BD("ik_upper"); m->ik_offset = BD("ik_offset");
  m->ik_base_body = BI("ik_base_body")[0]; m->ee_body = BI("ee_body")[0];
  if (m->nu != NU) { fprintf(stderr, "oracle: expects %d actuators\n", NU); return NULL; }
  m->geom_lmat = (double*)malloc(sizeof(double) * 9 * m->ngeom);
  for (int g = 0; g < m->ngeom; g++) q2mat(m->geom_lmat + 9 * g, m->geom_quat + 4 * g);
  int64_t nface = 0;
  blob_get(blob, "mesh_face", &nface);
  nface /= 3;
  m->face_plane = (double*)malloc(sizeof(double) * 4 * (nface + 1));
  for (int k = 0; k < m->nmesh; k++)
    for (int f = 0; f < m->mesh_facenum[k]; f++) {
      const int32_t* idx = m->mesh_face + 3 * (m->mesh_faceadr[k] + f);
      const double* v = m->mesh_vert + 3 * m->mesh_vertadr[k];
      double e1[3], e2[3], n[3];
      v3sub(e1, v + 3 * idx[1], v + 3 * idx[0]); v3sub(e2, v + 3 * idx[2], v + 3 * idx[0]);
      v3cross(n, e1, e2); v3normalize(n);
      double* pl = m->face_plane + 4 * (m->mesh_faceadr[k] + f);
      v3copy(pl, n); pl[3] = v3dot(n, v + 3 * idx[0]);
    }
  m->any_damping = 0;
  for (int d = 0; d < m->nv; d++) if (m->dof_damping[d] != 0) m->any_damping = 1;
  return m;
}
void orc_model_free(Model* m) { if (m) { free(m->blob); free(m->geom_lmat); free(m->face_plane); free(m); } }
int orc_model_size(const Model* m, int what) {
  switch (what) { case 0: return m->nq; case 1: return m->nv; case 2: return m->nbody; case 3: return m->ngeom; case 4: return m->nM; case 5: return m->njnt; }
  return -1;
}

#define DALLOC(n) ((double*)calloc((size_t)(n) + 1, sizeof(double)))
Env* orc_env_create(Model* m) {
  Env* e = (Env*)calloc(1, sizeof(Env));
  e->m = m;
  int nv = m->nv, nb = m->nbody;
  e->qpos = DALLOC(m->nq); e->qvel = DALLOC(nv); e->qacc_ws = DALLOC(nv);
  e->xpos = DALLOC(3 * nb); e->xquat = DALLOC(4 * nb); e->xmat = DALLOC(9 * nb); e->xipos = DALLOC(3 * nb);
  e->xanchor = DALLOC(3 * m->njnt); e->xaxis = DALLOC(3 * m->njnt);
  e->cdof = DALLOC(6 * nv); e->cdof_dot = DALLOC(6 * nv); e->cvel = DALLOC(6 * nb); e->cacc = DALLOC(6 * nb); e->cfrc = DALLOC(6 * nb);
  e->cinert = DALLOC(10 * nb); e->crb = DALLOC(10 * nb);
  e->gpos = DALLOC(3 * m->ngeom); e->gmat = DALLOC(9 * m->ngeom);
  e->qM = DALLOC(m->nM); e->qLD = DALLOC(m->nM); e->qH = DALLOC(m->nM);
  e->qfrc_bias = DALLOC(nv); e->qfrc_passive = DALLOC(nv); e->qfrc_actuator = DALLOC(nv); e->qfrc_smooth = DALLOC(nv);
  e->qacc_smooth = DALLOC(nv); e->qfrc_constraint = DALLOC(nv); e->qacc = DALLOC(nv);
  e->nefc_max = m->neq + m->njnt + 10 * MAXCON;
  e->maxcon = MAXCON;
  e->maxsr = e->nefc_max;
  e->efc_J = DALLOC((size_t)e->nefc_max * nv); e->efc_B = DALLOC((size_t)e->nefc_max * nv);
  e->efc_pos = DALLOC(e->nefc_max); e->efc_margin = DALLOC(e->nefc_max); e->efc_diag = DALLOC(e->nefc_max);
  e->efc_R = DALLOC(e->nefc_max); e->efc_aref = DALLOC(e->nefc_max); e->efc_force = DALLOC(e->nefc_max); e->efc_AR = DALLOC(e->nefc_max);
  e->efc_type = (int*)calloc(e->nefc_max + 1, sizeof(int));
  e->tmp1 = DALLOC(nv); e->tmp2 = DALLOC(nv);
  e->nt_H = DALLOC((size_t)nv * nv); e->nt_grad = DALLOC(nv); e->nt_search = DALLOC(nv); e->nt_Ma = DALLOC(nv); e->nt_Mv = DALLOC(nv);
  e->nt_jar = DALLOC(e->nefc_max); e->nt_jv = DALLOC(e->nefc_max); e->nt_active = (int*)calloc(e->nefc_max + 1, sizeof(int));
  memcpy(e->qpos, m->qpos0, sizeof(double) * m->nq);
  e->dt_pid = m->timestep;
  for (int i = 0; i < NU; i++) {
    e->kp[i] = m->pid_kp[i]; e->kd[i] = m->pid_kd[i]; e->lim[i] = m->pid_lim[i];
    e->target[i] = e->qpos[m->jnt_qposadr[m->actuator_jntid[i]]];
    e->last_input[i] = e->target[i];
  }
  return e;
}
void orc_env_free(Env* e) {
  if (!e) return;
  double** p[] = {&e->qpos, &e->qvel, &e->qacc_ws, &e->xpos, &e->xquat, &e->xmat, &e->xipos, &e->xanchor, &e->xaxis, &e->cdof, &e->cdof_dot,
                  &e->cvel, &e->cacc, &e->cfrc, &e->cinert, &e->crb, &e->gpos, &e->gmat, &e->qM, &e->qLD, &e->qH, &e->qfrc_bias, &e->qfrc_passive,
                  &e->qfrc_actuator, &e->qfrc_smooth, &e->qacc_smooth, &e->qfrc_constraint, &e->qacc, &e->efc_J, &e->efc_B, &e->efc_pos,
                  &e->efc_margin, &e->efc_diag, &e->efc_R, &e->efc_aref, &e->efc_force, &e->efc_AR, &e->tmp1, &e->tmp2, &e->nt_H, &e->nt_grad, &e->nt_search, &e->nt_Ma, &e->nt_Mv, &e->nt_jar, &e->nt_jv};
  for (size_t i = 0; i < sizeof(p) / sizeof(p[0]); i++) free(*p[i]);
  free(e->efc_type); free(e->nt_active);
  free(e);
}

/* ------------------------------------------------------------------ stage 1: kinematics (mj_kinematics + mj_comPos restated)
 * Spatial quantities are expressed in world axes about the WORLD ORIGIN (DECISION: MuJoCo uses the subtree COM;
 * the choice only changes rounding). Motion vectors are [angular; linear-at-origin], forces [torque-about-origin; force]. */
static void fk(Env* e) {
  const Model* m = e->m;
  v3set(e->xpos, 0, 0, 0); e->xquat[0] = 1; e->xquat[1] = e->xquat[2] = e->xquat[3] = 0;
  q2mat(e->xmat, e->xquat);
  for (int b = 1; b < m->nbody; b++) {
    int p = m->body_parentid[b];
    double pos[3], quat[4], R[9], t[3];
    m3mulv(t, e->xmat + 9 * p, m->body_pos + 3 * b); v3add(pos, e->xpos + 3 * p, t);
    qmul(quat, e->xquat + 4 * p, m->body_quat + 4 * b);
    for (int k = 0; k < m->body_jntnum[b]; k++) {
      int j = m->body_jntadr[b] + k, qa = m->jnt_qposadr[j], type = m->jnt_type[j];
      if (type == J_FREE) {
        v3copy(pos, e->qpos + qa);
        memcpy(quat, e->qpos + qa + 3, 32); qnormalize(quat);
        v3copy(e->xanchor + 3 * j, pos); v3set(e->xaxis + 3 * j, 0, 0, 1);
        continue;
      }
      q2mat(R, quat);
      m3mulv(t, R, m->jnt_pos + 3 * j); v3add(e->xanchor + 3 * j, pos, t);
      m3mulv(e->xaxis + 3 * j, R, m->jnt_axis + 3 * j);
      if (type == J_SLIDE) {
        v3addscl(pos, pos, e->xaxis + 3 * j, e->qpos[qa] - m->qpos0[qa]);
      } else {
        double dq[4], nq_[4];
        if (type == J_HINGE) qaxisangle(dq, m->jnt_axis + 3 * j, e->qpos[qa] - m->qpos0[qa]);
        else { memcpy(dq, e->qpos + qa, 32); qnormalize(dq); }
        qmul(nq_, quat, dq); memcpy(quat, nq_, 32);
        q2mat(R, quat);
        m3mulv(t, R, m->jnt_pos + 3 * j); v3sub(pos, e->xanchor + 3 * j, t);
      }
    }
    qnormalize(quat);
    v3copy(e->xpos + 3 * b, pos); memcpy(e->xquat + 4 * b, quat, 32); q2mat(e->xmat + 9 * b, quat);
    m3mulv(t, e->xmat + 9 * b, m->body_ipos + 3 * b); v3add(e->xipos + 3 * b, pos, t);
  }
  /* motion axes per dof */
  for (int d = 0; d < m->nv; d++) {
    int j = m->dof_jntid[d], b = m->dof_bodyid[d], k = d - m->jnt_dofadr[j], type = m->jnt_type[j];
    double* c = e->cdof + 6 * d;
    double ax[3];
    if (type == J_SLIDE) { v3set(c, 0, 0, 0); v3copy(c + 3, e->xaxis + 3 * j); }
    else if (type == J_HINGE) { v3copy(c, e->xaxis + 3 * j); v3cross(c + 3, e->xanchor + 3 * j, c); }
    else if (type == J_BALL) { m3col(ax, e->xmat + 9 * b, k); v3copy(c, ax); v3cross(c + 3, e->xanchor + 3 * j, ax); }
    else { /* free: 3 world translations, then 3 body-frame rotations about the body origin */
      if (k < 3) { v3set(c, 0, 0, 0); v3set(c + 3, 0, 0, 0); c[3 + k] = 1; }
      else { m3col(ax, e->xmat + 9 * b, k - 3); v3copy(c, ax); v3cross(c + 3, e->xpos + 3 * b, ax); }
    }
  }
  /* geoms */
  for (int g = 0; g < m->ngeom; g++) {
    int b = m->geom_bodyid[g];
    double t[3];
    m3mulv(t, e->xmat + 9 * b, m->geom_pos + 3 * g); v3add(e->gpos + 3 * g, e->xpos + 3 * b, t);
    m3mul(e->gmat + 9 * g, e->xmat + 9 * b, m->geom_lmat + 9 * g);
  }
  /* spatial inertia about the world origin: [m, h(3)=m*c, I_o(6: xx yy zz xy xz yz)] */
  for (int b = 0; b < m->nbody; b++) {
    double* I = e->cinert + 10 * b;
    double mass = m->body_mass[b];
    const double* c = e->xipos + 3 * b;
    const double* R = e->xmat + 9 * b;
    const double* Ib = m->body_inertia + 6 * b;
    double Il[9] = {Ib[0], Ib[3], Ib[4], Ib[3], Ib[1], Ib[5], Ib[4], Ib[5], Ib[2]}, RI[9], Rt[9], Iw[9];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Rt[3 * i + j] = R[3 * j + i];
    m3mul(RI, R, Il); m3mul(Iw, RI, Rt);
    double cc = v3dot(c, c);
    I[0] = mass; I[1] = mass * c[0]; I[2] = mass * c[1]; I[3] = mass * c[2];
    I[4] = Iw[0] + mass * (cc - c[0] * c[0]); I[5] = Iw[4] + mass * (cc - c[1] * c[1]); I[6] = Iw[8] + mass * (cc - c[2] * c[2]);
    I[7] = Iw[1] - mass * c[0] * c[1]; I[8] = Iw[2] - mass * c[0] * c[2]; I[9] = Iw[5] - mass * c[1] * c[2];
  }
}

/* f(6) = I(10) * v(6) : f = [I_o w + h x v ; m v + w x h] */
static void inert_mul(double* f, const double* I, const double* v) {
  const double *w = v, *l = v + 3, *h = I + 1;
  double hv[3], wh[3];
  v3cross(hv, h, l); v3cross(wh, w, h);
  f[0] = I[4] * w[0] + I[7] * w[1] + I[8] * w[2] + hv[0];
  f[1] = I[7] * w[0] + I[5] * w[1] + I[9] * w[2] + hv[1];
  f[2] = I[8] * w[0] + I[9] * w[1] + I[6] * w[2] + hv[2];
  f[3] = I[0] * l[0] + wh[0]; f[4] = I[0] * l[1] + wh[1]; f[5] = I[0] * l[2] + wh[2];
}
static double dot6(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3] + a[4] * b[4] + a[5] * b[5]; }
/* motion cross: r = v x s */
static void cross_motion(double* r, const double* v, const double* s) {
  double a[3], b[3], c[3];
  v3cross(a, v, s); v3cross(b, v, s + 3); v3cross(c, v + 3, s);
  v3copy(r, a); v3add(r + 3, b, c);
}
/* force cross: r = v x* f = [w x L + l x p ; w x p] */
static void cross_force(double* r, const double* v, const double* f) {
  double a[3], b[3], c[3];
  v3cross(a, v, f); v3cross(b, v + 3, f + 3); v3cross(c, v, f + 3);
  v3add(r, a, b); v3copy(r + 3, c);
}

/* ------------------------------------------------------------------ stage 2: CRBA (mj_crb) + L^T D L (mj_factorM) */
static void crb(Env* e) {
  const Model* m = e->m;
  memcpy(e->crb, e->cinert, sizeof(double) * 10 * m->nbody);
  for (int b = m->nbody - 1; b > 0; b--) {
    int p = m->body_parentid[b];
    for (int k = 0; k < 10; k++) e->crb[10 * p + k] += e->crb[10 * b + k];
  }
  for (int i = 0; i < m->nv; i++) {
    double f[6];
    inert_mul(f, e->crb + 10 * m->dof_bodyid[i], e->cdof + 6 * i);
    int adr = m->dof_Madr[i];
    e->qM[adr] = dot6(e->cdof + 6 * i, f) + m->dof_armature[i];
    int k = 1;
    for (int j = m->dof_parentid[i]; j >= 0; j = m->dof_parentid[j], k++) e->qM[adr + k] = dot6(e->cdof + 6 * j, f);
  }
}
static void factor(const Model* m, double* LD) {
  for (int k = m->nv - 1; k >= 0; k--) {
    int ak = m->dof_Madr[k];
    double Mkk = LD[ak];
    int ki = 1;
    for (int i = m->dof_parentid[k]; i >= 0; i = m->dof_parentid[i], ki++) {
      double a = LD[ak + ki] / Mkk;
      int ai = m->dof_Madr[i], kj = ki, ij = 0;
      for (int j = i; j >= 0; j = m->dof_parentid[j], kj++, ij++) LD[ai + ij] -= a * LD[ak + kj];
      LD[ak + ki] = a;
    }
  }
}
static void solve_ld(const Model* m, const double* LD, double* x) {
  for (int k = m->nv - 1; k >= 0; k--) {
    int ak = m->dof_Madr[k], ki = 1;
    for (int i = m->dof_parentid[k]; i >= 0; i = m->dof_parentid[i], ki++) x[i] -= LD[ak + ki] * x[k];
  }
  for (int k = 0; k < m->nv; k++) x[k] /= LD[m->dof_Madr[k]];
  for (int k = 0; k < m->nv; k++) {
    int ak = m->dof_Madr[k], ki = 1;
    for (int i = m->dof_parentid[k]; i >= 0; i = m->dof_parentid[i], ki++) x[k] -= LD[ak + ki] * x[i];
  }
}
static void mul_m(const Model* m, const double* M, double* r, const double* v) {
  for (int i = 0; i < m->nv; i++) r[i] = 0;
  for (int i = 0; i < m->nv; i++) {
    int a = m->dof_Madr[i], k = 1;
    r[i] += M[a] * v[i];
    for (int j = m->dof_parentid[i]; j >= 0; j = m->dof_parentid[j], k++) { r[i] += M[a + k] * v[j]; r[j] += M[a + k] * v[i]; }
  }
}

/* ------------------------------------------------------------------ stage 3: velocity + bias forces (mj_comVel + mj_rne) */
static void rne(Env* e) {
  const Model* m = e->m;
  for (int k = 0; k < 6; k++) { e->cvel[k] = 0; e->cacc[k] = 0; }
  e->cacc[3] = -m->gravity[0]; e->cacc[4] = -m->gravity[1]; e->cacc[5] = -m->gravity[2];
  for (int b = 1; b < m->nbody; b++) {
    int p = m->body_parentid[b];
    double* v = e->cvel + 6 * b;
    double* a = e->cacc + 6 * b;
    memcpy(v, e->cvel + 6 * p, 48); memcpy(a, e->cacc + 6 * p, 48);
    for (int k = 0; k < m->body_jntnum[b]; k++) {
      int j = m->body_jntadr[b] + k, d = m->jnt_dofadr[j], type = m->jnt_type[j];
      int nd = type == J_FREE ? 6 : (type == J_BALL ? 3 : 1);
      int d0 = 0;
      if (type == J_FREE) { /* translations first: constant axes */
        for (int i = 0; i < 3; i++) { for (int c = 0; c < 6; c++) e->cdof_dot[6 * (d + i) + c] = 0; for (int c = 0; c < 6; c++) v[c] += e->cdof[6 * (d + i) + c] * e->qvel[d + i]; }
        d0 = 3;
      }
      /* all axes of one joint are differentiated with the velocity accumulated before that joint (SURVEY A.5) */
      for (int i = d0; i < nd; i++) cross_motion(e->cdof_dot + 6 * (d + i), v, e->cdof + 6 * (d + i));
      for (int i = d0; i < nd; i++)
        for (int c = 0; c < 6; c++) { v[c] += e->cdof[6 * (d + i) + c] * e->qvel[d + i]; a[c] += e->cdof_dot[6 * (d + i) + c] * e->qvel[d + i]; }
    }
  }
  for (int b = 0; b < m->nbody; b++) {
    double Ia[6], Iv[6], x[6];
    inert_mul(Ia, e->cinert + 10 * b, e->cacc + 6 * b);
    inert_mul(Iv, e->cinert + 10 * b, e->cvel + 6 * b);
    cross_force(x, e->cvel + 6 * b, Iv);
    for (int c = 0; c < 6; c++) e->cfrc[6 * b + c] = Ia[c] + x[c];
  }
  for (int b = m->nbody - 1; b > 0; b--) {
    int p = m->body_parentid[b];
    for (int c = 0; c < 6; c++) e->cfrc[6 * p + c] += e->cfrc[6 * b + c];
  }
  for (int d = 0; d < m->nv; d++) e->qfrc_bias[d] = dot6(e->cdof + 6 * d, e->cfrc + 6 * m->dof_bodyid[d]);
}

/* ------------------------------------------------------------------ stage 4: collision */
static void make_frame(double* fr) { /* fr[0..2] = unit normal given; fill two tangents */
  double t[3] = {0, 0, 0};
  if (fabs(fr[1]) < 0.5) t[1] = 1; else t[2] = 1;
  double d = v3dot(fr, t);
  v3addscl(fr + 3, t, fr, -d); v3normalize(fr + 3);
  v3cross(fr + 6, fr, fr + 3);
}
static void add_contact(Env* e, int pair, double dist, const double* pos, const double* normal) {
  const Model* m = e->m;
  if (++e->nfound > e->ncon_peak) e->ncon_peak = e->nfound;
  if (e->ncon >= e->maxcon) { e->con_overflow = 1; return; }
  Contact* c = &e->con[e->ncon++];
  c->dist = dist; v3copy(c->pos, pos); v3copy(c->frame, normal); make_frame(c->frame);
  c->margin = m->pair_margin[pair]; c->dim = m->pair_condim[pair];
  const double* f = m->pair_friction + 3 * pair;
  c->friction[0] = c->friction[1] = f[0]; c->friction[2] = f[1]; c->friction[3] = c->friction[4] = f[2];
  memcpy(c->solref, m->pair_solref + 2 * pair, 16); memcpy(c->solimp, m->pair_solimp + 5 * pair, 40);
  c->geom1 = m->pair_geom[2 * pair]; c->geom2 = m->pair_geom[2 * pair + 1];
}

/* conservative oriented-box overlap test (15-axis SAT) with margin */
static int obb_separated(const double* c1, const double* R1, const double* h1, const double* c2, const double* R2, const double* h2, double margin) {
  double d[3], a[3][3], b[3][3];
  v3sub(d, c2, c1);
  for (int i = 0; i < 3; i++) { m3col(a[i], R1, i); m3col(b[i], R2, i); }
  double C[3][3], AC[3][3];
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { C[i][j] = v3dot(a[i], b[j]); AC[i][j] = fabs(C[i][j]) + 1e-9; }
  double da[3] = {v3dot(d, a[0]), v3dot(d, a[1]), v3dot(d, a[2])};
  double db[3] = {v3dot(d, b[0]), v3dot(d, b[1]), v3dot(d, b[2])};
  for (int i = 0; i < 3; i++) if (fabs(da[i]) > h1[i] + h2[0] * AC[i][0] + h2[1] * AC[i][1] + h2[2] * AC[i][2] + margin) return 1;
  for (int j = 0; j < 3; j++) if (fabs(db[j]) > h2[j] + h1[0] * AC[0][j] + h1[1] * AC[1][j] + h1[2] * AC[2][j] + margin) return 1;
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
    double ra = h1[i1] * AC[i2][j] + h1[i2] * AC[i1][j], rb = h2[j1] * AC[i][j2] + h2[j2] * AC[i][j1];
    double len2 = 1.0 - C[i][j] * C[i][j];
    if (len2 < 1e-8) continue;
    if (fabs(da[i2] * C[i1][j] - da[i1] * C[i2][j]) > ra + rb + margin * sqrt(len2)) return 1;
  }
  return 0;
}

static void col_plane_sphere(Env* e, int pair, int g1, int g2) {
  const Model* m = e->m;
  double n[3], d[3];
  m3col(n, e->gmat + 9 * g1, 2); v3sub(d, e->gpos + 3 * g2, e->gpos + 3 * g1);
  double r = m->geom_size[3 * g2], dist = v3dot(d, n) - r;
  if (dist >= m->pair_margin[pair]) return;
  double pos[3];
  v3addscl(pos, e->gpos + 3 * g2, n, -(r + 0.5 * dist));
  add_contact(e, pair, dist, pos, n);
}
static void col_plane_box(Env* e, int pair, int g1, int g2) {
  const Model* m = e->m;
  double n[3];
  m3col(n, e->gmat + 9 * g1, 2);
  const double* h = m->geom_size + 3 * g2;
  int cnt = 0;
  for (int k = 0; k < 8 && cnt < 4; k++) {
    double loc[3] = {(k & 1 ? h[0] : -h[0]), (k & 2 ? h[1] : -h[1]), (k & 4 ? h[2] : -h[2])}, w[3], d[3];
    m3mulv(w, e->gmat + 9 * g2, loc); v3add(w, w, e->gpos + 3 * g2);
    v3sub(d, w, e->gpos + 3 * g1);
    double dist = v3dot(d, n);
    if (dist >= m->pair_margin[pair]) continue;
    double pos[3];
    v3addscl(pos, w, n, -0.5 * dist);
    add_contact(e, pair, dist, pos, n);
    cnt++;
  }
}
static void col_plane_mesh(Env* e, int pair, int g1, int g2) { /* DECISION: deepest hull vertex only */
  const Model* m = e->m;
  double n[3], nl[3];
  m3col(n, e->gmat + 9 * g1, 2);
  m3Tmulv(nl, e->gmat + 9 * g2, n);
  int k = m->geom_meshid[g2], best = 0;
  const double* v = m->mesh_vert + 3 * m->mesh_vertadr[k];
  double bv = 1e300;
  for (int i = 0; i < m->mesh_vertnum[k]; i++) { double s = v3dot(v + 3 * i, nl); if (s < bv) { bv = s; best = i; } }
  double w[3], d[3];
  m3mulv(w, e->gmat + 9 * g2, v + 3 * best); v3add(w, w, e->gpos + 3 * g2);
  v3sub(d, w, e->gpos + 3 * g1);
  double dist = v3dot(d, n);
  if (dist >= m->pair_margin[pair]) return;
  double pos[3];
  v3addscl(pos, w, n, -0.5 * dist);
  add_contact(e, pair, dist, pos, n);
}
/* plane vs capsule: the two end spheres (+axis end first).  plane vs cylinder (DECISION: MuJoCo's mjc_PlaneCylinder is not
 * documented): the deepest rim point of each cap (+axis cap first); a cap parallel to the plane contributes its centre. */
static void col_plane_capsule(Env* e, int pair, int g1, int g2) {
  const Model* m = e->m;
  double n[3], ax[3];
  m3col(n, e->gmat + 9 * g1, 2); m3col(ax, e->gmat + 9 * g2, 2);
  double r = m->geom_size[3 * g2], h = m->geom_size[3 * g2 + 1];
  for (int s = 0; s < 2; s++) {
    double c[3], d[3], pos[3];
    v3addscl(c, e->gpos + 3 * g2, ax, s ? -h : h);
    v3sub(d, c, e->gpos + 3 * g1);
    double dist = v3dot(d, n) - r;
    if (dist >= m->pair_margin[pair]) continue;
    v3addscl(pos, c, n, -(r + 0.5 * dist));
    add_contact(e, pair, dist, pos, n);
  }
}
static void col_plane_cylinder(Env* e, int pair, int g1, int g2) {
  const Model* m = e->m;
  double n[3], ax[3], rim[3];
  m3col(n, e->gmat + 9 * g1, 2); m3col(ax, e->gmat + 9 * g2, 2);
  double r = m->geom_size[3 * g2], h = m->geom_size[3 * g2 + 1];
  v3addscl(rim, n, ax, -v3dot(n, ax)); /* component of the plane normal perpendicular to the axis */
  double len = v3norm(rim);
  if (len > 1e-6) v3scl(rim, rim, -r / len); else v3set(rim, 0, 0, 0);
  for (int s = 0; s < 2; s++) {
    double c[3], d[3], pos[3];
    v3addscl(c, e->gpos + 3 * g2, ax, s ? -h : h);
    v3add(c, c, rim);
    v3sub(d, c, e->gpos + 3 * g1);
    double dist = v3dot(d, n);
    if (dist >= m->pair_margin[pair]) continue;
    v3addscl(pos, c, n, -0.5 * dist);
    add_contact(e, pair, dist, pos, n);
  }
}
static void col_sphere_sphere(Env* e, int pair, int g1, int g2) {
  const Model* m = e->m;
  double d[3];
  v3sub(d, e->gpos + 3 * g2, e->gpos + 3 * g1);
  double len = v3norm(d), r1 = m->geom_size[3 * g1], r2 = m->geom_size[3 * g2], dist = len - r1 - r2;
  if (dist >= m->pair_margin[pair]) return;
  if (len < ORC_MINVAL) v3set(d, 0, 0, 1); else v3scl(d, d, 1.0 / len);
  double pos[3];
  v3addscl(pos, e->gpos + 3 * g1, d, r1 + 0.5 * dist);
  add_contact(e, pair, dist, pos, d);
}
/* sphere vs capsule, capsule vs capsule, sphere vs cylinder: closed forms (MuJoCo also treats these pairs analytically; MPR on two
 * smooth surfaces converges slowly and its portal choice is ill-conditioned).  Normal points from geom1 to geom2. */
static void col_sphere_capsule(Env* e, int pair, int g1, int g2) {
  const Model* m = e->m;
  const double *c = e->gpos + 3 * g1, *p = e->gpos + 3 * g2;
  double ax[3], d[3], q[3], n[3], pos[3];
  m3col(ax, e->gmat + 9 * g2, 2);
  double r1 = m->geom_size[3 * g1], r2 = m->geom_size[3 * g2], h = m->geom_size[3 * g2 + 1];
  v3sub(d, c, p);
  double t = v3dot(d, ax);
  if (t > h) t = h; else if (t < -h) t = -h;
  v3addscl(q, p, ax, t); v3sub(d, q, c);
  double len = v3norm(d);
  if (len < 1e-12) { m3col(n, e->gmat + 9 * g2, 0); len = 0; } else v3scl(n, d, 1.0 / len);
  double dist = len - r1 - r2;
  if (dist >= m->pair_margin[pair]) return;
  v3addscl(pos, c, n, r1 + 0.5 * dist);
  add_contact(e, pair, dist, pos, n);
}
static void col_capsule_capsule(Env* e, int pair, int g1, int g2) {
  const Model* m = e->m;
  const double *p1 = e->gpos + 3 * g1, *p2 = e->gpos + 3 * g2;
  double a1[3], a2[3], w[3], q1[3], q2[3], d[3], n[3], pos[3];
  m3col(a1, e->gmat + 9 * g1, 2); m3col(a2, e->gmat + 9 * g2, 2);
  double r1 = m->geom_size[3 * g1], h1 = m->geom_size[3 * g1 + 1], r2 = m->geom_size[3 * g2], h2 = m->geom_size[3 * g2 + 1];
  v3sub(w, p1, p2);
  double b = v3dot(a1, a2), dd = v3dot(a1, w), ee = v3dot(a2, w), den = 1.0 - b * b, s, t;
  if (den < 1e-10) { /* parallel axes: middle of the overlap of the two segments (measured along axis 1) */
    double c2 = -dd, lo = c2 - h2, hi = c2 + h2; /* segment 2 projected on axis 1: centre -dd, half length h2 */
    if (lo < -h1) lo = -h1;
    if (hi > h1) hi = h1;
    s = lo <= hi ? 0.5 * (lo + hi) : (c2 > 0 ? h1 : -h1);
  } else {
    s = (b * ee - dd) / den;
    if (s > h1) s = h1; else if (s < -h1) s = -h1;
  }
  t = b * s + ee;
  if (t > h2) t = h2; else if (t < -h2) t = -h2;
  s = b * t - dd; /* re-project onto segment 1 with t fixed */
  if (s > h1) s = h1; else if (s < -h1) s = -h1;
  v3addscl(q1, p1, a1, s); v3addscl(q2, p2, a2, t); v3sub(d, q2, q1);
  double len = v3norm(d);
  if (len < 1e-12) { v3cross(n, a1, a2); if (v3norm(n) < 1e-12) m3col(n, e->gmat + 9 * g1, 0); v3normalize(n); len = 0; } else v3scl(n, d, 1.0 / len);
  double dist = len - r1 - r2;
  if (dist >= m->pair_margin[pair]) return;
  v3addscl(pos, q1, n, r1 + 0.5 * dist);
  add_contact(e, pair, dist, pos, n);
}
static void col_sphere_cylinder(Env* e, int pair, int g1, int g2) {
  const Model* m = e->m;
  const double *c = e->gpos + 3 * g1, *R = e->gmat + 9 * g2;
  double t[3], l[3], out[3], n[3], pos[3];
  v3sub(t, c, e->gpos + 3 * g2); m3Tmulv(l, R, t);
  double r1 = m->geom_size[3 * g1], r = m->geom_size[3 * g2], h = m->geom_size[3 * g2 + 1];
  double rho = sqrt(l[0] * l[0] + l[1] * l[1]), sz = l[2] >= 0 ? 1.0 : -1.0, dz = fabs(l[2]) - h, dr = rho - r, sd;
  double ux = rho > 1e-12 ? l[0] / rho : 1.0, uy = rho > 1e-12 ? l[1] / rho : 0.0;
  if (dz <= 0 && dr <= 0) {
    if (dr > dz) { v3set(out, ux, uy, 0); sd = dr; } else { v3set(out, 0, 0, sz); sd = dz; }
  } else if (dz <= 0) { v3set(out, ux, uy, 0); sd = dr; }
  else if (dr <= 0) { v3set(out, 0, 0, sz); sd = dz; }
  else { sd = sqrt(dr * dr + dz * dz); v3set(out, dr * ux / sd, dr * uy / sd, sz * dz / sd); }
  double dist = sd - r1;
  if (dist >= m->pair_margin[pair]) return;
  m3mulv(n, R, out); v3scl(n, n, -1.0);
  v3addscl(pos, c, n, r1 + 0.5 * dist);
  add_contact(e, pair, dist, pos, n);
}
static void col_sphere_box(Env* e, int pair, int g1, int g2) {
  const Model* m = e->m;
  const double* h = m->geom_size + 3 * g2;
  double r = m->geom_size[3 * g1], d[3], p[3], q[3];
  v3sub(d, e->gpos + 3 * g1, e->gpos + 3 * g2);
  m3Tmulv(p, e->gmat + 9 * g2, d);
  int inside = 1;
  for (int k = 0; k < 3; k++) { q[k] = p[k] < -h[k] ? -h[k] : (p[k] > h[k] ? h[k] : p[k]); if (q[k] != p[k]) inside = 0; }
  double nl[3] = {0, 0, 0}, dist;
  if (inside) {
    int best = 0; double bd = 1e300;
    for (int k = 0; k < 3; k++) { double s = h[k] - fabs(p[k]); if (s < bd) { bd = s; best = k; } }
    nl[best] = p[best] >= 0 ? 1 : -1;
    q[best] = nl[best] * h[best];
    dist = -bd - r;
  } else {
    v3sub(nl, p, q);
    double len = v3normalize(nl);
    dist = len - r;
  }
  if (dist >= m->pair_margin[pair]) return;
  double nw[3], qw[3], pos[3], nrm[3];
  m3mulv(nw, e->gmat + 9 * g2, nl); m3mulv(qw, e->gmat + 9 * g2, q); v3add(qw, qw, e->gpos + 3 * g2);
  v3addscl(pos, qw, nw, 0.5 * dist);
  v3scl(nrm, nw, -1.0); /* geom1 = sphere -> geom2 = box */
  add_contact(e, pair, dist, pos, nrm);
}

/* box-box: 15-axis SAT, then reference-face clipping (Sutherland-Hodgman) or edge-edge closest points.
 * DECISION: MuJoCo's mjc_BoxBox is not restated (undocumented); this is an independent manifold generator
 * with the same contract (<= 8 points, normal from geom1 to geom2, dist < margin). */
static int clip_poly(double (*p)[2], int n, int axis, double lim, double (*out)[2], double* on_line) {
  /* keep the part with sign*coord[axis] <= lim; called for +/- */
  int k = 0;
  for (int i = 0; i < n; i++) {
    const double *a = p[i], *b = p[(i + 1) % n];
    double da = a[axis] - lim, db = b[axis] - lim;
    if (da == 0) *on_line += 1;
    if (da <= 0) { out[k][0] = a[0]; out[k][1] = a[1]; k++; }
    if ((da < 0 && db > 0) || (da > 0 && db < 0)) { double t = da / (da - db); out[k][0] = a[0] + t * (b[0] - a[0]); out[k][1] = a[1] + t * (b[1] - a[1]); k++; }
  }
  return k;
}
static void col_box_box(Env* e, int pair, int g1, int g2) {
  const Model* m = e->m;
  const double *c1 = e->gpos + 3 * g1, *c2 = e->gpos + 3 * g2, *R1 = e->gmat + 9 * g1, *R2 = e->gmat + 9 * g2;
  const double *h1 = m->geom_size + 3 * g1, *h2 = m->geom_size + 3 * g2;
  double margin = m->pair_margin[pair];
  double d[3], a[3][3], b[3][3], C[3][3], AC[3][3];
  double dummy[BBX_W], *rec = e->nbbx < BBX_MAX ? e->bbx + BBX_W * e->nbbx++ : dummy;
  memset(rec, 0, sizeof(dummy));
  rec[0] = g1; rec[1] = g2;
  int ncon0 = e->ncon;
  v3sub(d, c2, c1);
  for (int i = 0; i < 3; i++) { m3col(a[i], R1, i); m3col(b[i], R2, i); }
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { C[i][j] = v3dot(a[i], b[j]); AC[i][j] = fabs(C[i][j]); }
  double best_s = -1e300, face_s[6]; int best_axis = -1;
  for (int i = 0; i < 3; i++) { /* face axes of box 1 */
    double s = fabs(v3dot(d, a[i])) - (h1[i] + h2[0] * AC[i][0] + h2[1] * AC[i][1] + h2[2] * AC[i][2]);
    if (s >= margin) return;
    if (s > best_s) { best_s = s; best_axis = i; }
    face_s[i] = s;
  }
  for (int j = 0; j < 3; j++) { /* face axes of box 2 */
    double s = fabs(v3dot(d, b[j])) - (h2[j] + h1[0] * AC[0][j] + h1[1] * AC[1][j] + h1[2] * AC[2][j]);
    if (s >= margin) return;
    if (s > best_s) { best_s = s; best_axis = 3 + j; }
    face_s[3 + j] = s;
  }
  for (int k = 0; k < 6; k++) rec[5] += face_s[k] == best_s;
  double edge_s = -1e300; int ei = -1, ej = -1; double en[3] = {0, 0, 0};
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    double L[3];
    v3cross(L, a[i], b[j]);
    double len = v3norm(L);
    if (len < 1e-6) { rec[6] += len > 0; continue; }
    v3scl(L, L, 1.0 / len);
    double ra = 0, rb = 0;
    for (int k = 0; k < 3; k++) { ra += h1[k] * fabs(v3dot(L, a[k])); rb += h2[k] * fabs(v3dot(L, b[k])); }
    double s = fabs(v3dot(d, L)) - ra - rb;
    if (s >= margin) return;
    if (s > edge_s) { edge_s = s; ei = i; ej = j; v3copy(en, L); }
  }
  if (ei >= 0 && edge_s > best_s + 1e-6) { /* edge-edge */
    double n[3], p1[3], p2[3];
    v3copy(n, en);
    if (v3dot(d, n) < 0) v3scl(n, n, -1.0);
    v3copy(p1, c1); v3copy(p2, c2);
    for (int k = 0; k < 3; k++) {
      if (k != ei) v3addscl(p1, p1, a[k], (v3dot(n, a[k]) >= 0 ? 1.0 : -1.0) * h1[k]);
      if (k != ej) v3addscl(p2, p2, b[k], (v3dot(n, b[k]) >= 0 ? -1.0 : 1.0) * h2[k]);
    }
    /* closest points between lines p1 + t a[ei], p2 + u b[ej] */
    double w[3];
    v3sub(w, p1, p2);
    double ab = C[ei][ej], aw = v3dot(a[ei], w), bw = v3dot(b[ej], w), den = 1.0 - ab * ab;
    double t = (ab * bw - aw) / den, u = (bw - ab * aw) / den;
    double q1[3], q2[3], pos[3], dd[3];
    v3addscl(q1, p1, a[ei], t); v3addscl(q2, p2, b[ej], u);
    v3sub(dd, q2, q1);
    double dist = v3dot(dd, n);
    if (dist >= margin) return;
    v3add(pos, q1, q2); v3scl(pos, pos, 0.5);
    add_contact(e, pair, dist, pos, n);
    rec[2] = 2; rec[8] = e->ncon - ncon0;
    return;
  }
  /* face contact: reference box owns the axis */
  int ref1 = best_axis < 3, ax = ref1 ? best_axis : best_axis - 3;
  rec[2] = 1; rec[3] = ref1 ? 1 : 2; rec[4] = best_axis;
  const double *cr = ref1 ? c1 : c2, *ci = ref1 ? c2 : c1, *hr = ref1 ? h1 : h2, *hi = ref1 ? h2 : h1;
  double (*ar)[3] = ref1 ? a : b;
  double (*ai)[3] = ref1 ? b : a;
  double dr[3], nref[3];
  v3sub(dr, ci, cr);
  v3scl(nref, ar[ax], v3dot(dr, ar[ax]) >= 0 ? 1.0 : -1.0); /* from reference box towards incident box */
  /* incident face: most anti-parallel to nref */
  int inc = 0; double bestd = -1;
  for (int k = 0; k < 3; k++) { double s = fabs(v3dot(ai[k], nref)); if (s > bestd) { bestd = s; inc = k; } }
  double sgn = v3dot(ai[inc], nref) > 0 ? -1.0 : 1.0; /* face normal = sgn*ai[inc], pointing against nref */
  double fc[3];
  v3addscl(fc, ci, ai[inc], sgn * hi[inc]);
  int u1 = (inc + 1) % 3, u2 = (inc + 2) % 3, r1 = (ax + 1) % 3, r2 = (ax + 2) % 3;
  double poly[16][2], tmp[16][2], height[4];
  double corner[4][3];
  static const double sg[4][2] = {{1, 1}, {-1, 1}, {-1, -1}, {1, -1}};
  for (int k = 0; k < 4; k++) {
    v3addscl(corner[k], fc, ai[u1], sg[k][0] * hi[u1]); v3addscl(corner[k], corner[k], ai[u2], sg[k][1] * hi[u2]);
    double rel[3];
    v3sub(rel, corner[k], cr);
    poly[k][0] = v3dot(rel, ar[r1]); poly[k][1] = v3dot(rel, ar[r2]);
    height[k] = v3dot(rel, nref) - hr[ax];
  }
  /* plane through the incident face in reference 2-D coordinates: height = g0 + gx*x + gy*y (exact for a planar quad) */
  double ex[2] = {poly[1][0] - poly[0][0], poly[1][1] - poly[0][1]}, ey[2] = {poly[3][0] - poly[0][0], poly[3][1] - poly[0][1]};
  double det = ex[0] * ey[1] - ex[1] * ey[0];
  double gx = 0, gy = 0;
  if (fabs(det) > 1e-14) {
    double dh1 = height[1] - height[0], dh3 = height[3] - height[0];
    gx = (dh1 * ey[1] - dh3 * ex[1]) / det; gy = (dh3 * ex[0] - dh1 * ey[0]) / det;
  }
  double g0 = height[0] - gx * poly[0][0] - gy * poly[0][1];
  int n = 4;
  /* clip against the four side planes of the reference face */
  n = clip_poly(poly, n, 0, hr[r1], tmp, rec + 7); if (!n) return;
  for (int k = 0; k < n; k++) { tmp[k][0] = -tmp[k][0]; }
  n = clip_poly(tmp, n, 0, hr[r1], poly, rec + 7); if (!n) return;
  for (int k = 0; k < n; k++) { poly[k][0] = -poly[k][0]; }
  n = clip_poly(poly, n, 1, hr[r2], tmp, rec + 7); if (!n) return;
  for (int k = 0; k < n; k++) { tmp[k][1] = -tmp[k][1]; }
  n = clip_poly(tmp, n, 1, hr[r2], poly, rec + 7); if (!n) return;
  for (int k = 0; k < n; k++) { poly[k][1] = -poly[k][1]; }
  double n12[3];
  v3scl(n12, nref, ref1 ? 1.0 : -1.0);
  int cnt = 0;
  for (int k = 0; k < n && cnt < 8; k++) {
    double dist = g0 + gx * poly[k][0] + gy * poly[k][1];
    if (dist >= margin) continue;
    double pos[3];
    v3addscl(pos, cr, ar[r1], poly[k][0]); v3addscl(pos, pos, ar[r2], poly[k][1]);
    v3addscl(pos, pos, nref, hr[ax] + 0.5 * dist);
    add_contact(e, pair, dist, pos, n12);
    cnt++;
  }
  rec[8] = e->ncon - ncon0;
}

/* ---- generic convex pair: Minkowski Portal Refinement (restates the published XenoCollide/MPR algorithm that MuJoCo
 * reaches through libccd [EXT]); both shapes inflated by margin/2 so that dist = margin - depth (SURVEY A.5) */
typedef struct { const Env* e; int g; double inflate; } Shape;
static void support(const Shape* s, const double* dir, double* out) { /* dir: unit, world */
  const Env* e = s->e; const Model* m = e->m; int g = s->g;
  const double *R = e->gmat + 9 * g, *size = m->geom_size + 3 * g;
  double dl[3], pl[3] = {0, 0, 0};
  m3Tmulv(dl, R, dir);
  switch (m->geom_type[g]) {
    case G_SPHERE: v3scl(pl, dl, size[0]); break;
    case G_BOX: for (int k = 0; k < 3; k++) pl[k] = dl[k] >= 0 ? size[k] : -size[k]; break;
    case G_CAPSULE: v3scl(pl, dl, size[0]); pl[2] += dl[2] >= 0 ? size[1] : -size[1]; break;
    case G_CYLINDER: { double n = sqrt(dl[0] * dl[0] + dl[1] * dl[1]); if (n > ORC_MINVAL) { pl[0] = dl[0] / n * size[0]; pl[1] = dl[1] / n * size[0]; } pl[2] = dl[2] >= 0 ? size[1] : -size[1]; break; }
    case G_MESH: {
      int k = m->geom_meshid[g], best = 0; const double* v = m->mesh_vert + 3 * m->mesh_vertadr[k]; double bv = -1e300;
      for (int i = 0; i < m->mesh_vertnum[k]; i++) { double t = v3dot(v + 3 * i, dl); if (t > bv) { bv = t; best = i; } }
      v3copy(pl, v + 3 * best); break;
    }
  }
  m3mulv(out, R, pl); v3add(out, out, e->gpos + 3 * g); v3addscl(out, out, dir, s->inflate);
}
static void shape_center(const Shape* s, double* out) {
  const Env* e = s->e; const Model* m = e->m; int g = s->g;
  if (m->geom_type[g] == G_MESH) { m3mulv(out, e->gmat + 9 * g, m->mesh_center + 3 * m->geom_meshid[g]); v3add(out, out, e->gpos + 3 * g); }
  else v3copy(out, e->gpos + 3 * g);
}
typedef struct { double v[3], a[3], b[3]; } SP;
static void mink(const Shape* A, const Shape* B, const double* dir, SP* s) {
  double nd[3], u[3];
  v3copy(u, dir); v3normalize(u); v3scl(nd, u, -1.0);
  support(A, u, s->a); support(B, nd, s->b); v3sub(s->v, s->a, s->b);
}
/* closest point to the origin on triangle (p,q,r): barycentric weights */
static void tri_closest_origin(const double* p, const double* q, const double* r, double* w) {
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
static int mpr_penetration(const Env* e, const Shape* A, const Shape* B, double* depth, double* pdir, double* ppos) {
  const Model* m = e->m;
  SP v0, v1, v2, v3, v4;
  double dir[3], t1[3], t2[3];
  shape_center(A, v0.a); shape_center(B, v0.b); v3sub(v0.v, v0.a, v0.b);
  if (v3dot(v0.v, v0.v) < 1e-20) v3set(v0.v, 1e-5, 0, 0);
  v3scl(dir, v0.v, -1.0);
  mink(A, B, dir, &v1);
  v3normalize(dir);
  if (v3dot(v1.v, dir) <= 0) return 0;
  double cr[3];
  v3cross(cr, v1.v, v0.v);
  if (v3dot(cr, cr) < 1e-20 * v3dot(v1.v, v1.v) * v3dot(v0.v, v0.v) + 1e-300) {
    /* origin lies on the ray centre -> v1: the boundary point in that direction is v1 itself */
    *depth = v3dot(v1.v, dir); v3copy(pdir, dir);
    v3add(ppos, v1.a, v1.b); v3scl(ppos, ppos, 0.5);
    return 1;
  }
  mink(A, B, cr, &v2);
  if (v3dot(v2.v, cr) <= 0) return 0;
  v3sub(t1, v1.v, v0.v); v3sub(t2, v2.v, v0.v); v3cross(dir, t1, t2);
  if (v3dot(dir, v0.v) > 0) { SP t = v1; v1 = v2; v2 = t; v3scl(dir, dir, -1.0); }
  for (int it = 0;; it++) { /* portal discovery */
    if (it > 100) return 0;
    mink(A, B, dir, &v3);
    if (v3dot(v3.v, dir) <= 0) return 0;
    v3cross(cr, v1.v, v3.v);
    if (v3dot(cr, v0.v) < 0) { v2 = v3; v3sub(t1, v1.v, v0.v); v3sub(t2, v3.v, v0.v); v3cross(dir, t1, t2); continue; }
    v3cross(cr, v3.v, v2.v);
    if (v3dot(cr, v0.v) < 0) { v1 = v3; v3sub(t1, v3.v, v0.v); v3sub(t2, v2.v, v0.v); v3cross(dir, t1, t2); continue; }
    break;
  }
  int hit = 0;
  for (int it = 0;; it++) { /* portal refinement; `hit` = the portal has been seen beyond the origin (shapes intersect) */
    v3sub(t1, v2.v, v1.v); v3sub(t2, v3.v, v1.v); v3cross(dir, t1, t2); v3normalize(dir);
    if (!hit && v3dot(v1.v, dir) >= 0) hit = 1;
    mink(A, B, dir, &v4);
    double dv4 = v3dot(v4.v, dir);
    if (!hit && dv4 < 0) return 0;
    double dmin = v3dot(v1.v, dir), dd = v3dot(v2.v, dir);
    if (dd < dmin) dmin = dd;
    dd = v3dot(v3.v, dir);
    if (dd < dmin) dmin = dd;
    if (dv4 - dmin <= m->mpr_tol || it >= m->mpr_iter) { if (!hit) return 0; break; }
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
  return 1;
}
long g_mpr_calls = 0, g_mpr_pairmask[64];
static void col_convex(Env* e, int pair, int g1, int g2) {
  const Model* m = e->m;
  g_mpr_calls++; g_mpr_pairmask[(g1 * 7 + g2) & 63]++;
  double margin = m->pair_margin[pair];
  Shape A = {e, g1, 0.5 * margin}, B = {e, g2, 0.5 * margin};
  double depth, dir[3], pos[3];
  if (!mpr_penetration(e, &A, &B, &depth, dir, pos)) return;
  double dist = margin - depth;
  if (dist >= margin) return;
  /* `dir` is the direction in which translating geom2 separates the pair = normal from geom1 to geom2 */
  add_contact(e, pair, dist, pos, dir);
}

static int pair_is_analytic(int t1, int t2) {
  return t1 == G_PLANE || (t1 == G_SPHERE && (t2 == G_SPHERE || t2 == G_BOX || t2 == G_CAPSULE || t2 == G_CYLINDER)) || (t1 == G_BOX && t2 == G_BOX) ||
         (t1 == G_CAPSULE && t2 == G_CAPSULE);
}
/* Two passes over the static candidate list: analytic pair functions first, then the generic convex (MPR) pairs.
 * (Contact order only affects floating-point summation order in the solver; the CUDA engine emits the same order.) */
static void collision(Env* e) {
  const Model* m = e->m;
  e->ncon = 0; e->con_overflow = 0; e->ncand = 0; e->nbbx = 0; e->nfound = 0;
  for (int pass = 0; pass < 2; pass++)
  for (int p = 0; p < m->npair; p++) {
    int g1 = m->pair_geom[2 * p], g2 = m->pair_geom[2 * p + 1], t1 = m->geom_type[g1], t2 = m->geom_type[g2];
    if (pair_is_analytic(t1, t2) != (pass == 0)) continue;
    double margin = m->pair_margin[p], c1[3], c2[3], t[3];
    m3mulv(t, e->gmat + 9 * g2, m->geom_obbcenter + 3 * g2); v3add(c2, e->gpos + 3 * g2, t);
    if (t1 == G_PLANE) {
      double n[3], d[3];
      m3col(n, e->gmat + 9 * g1, 2); v3sub(d, c2, e->gpos + 3 * g1);
      if (v3dot(d, n) > m->geom_rbound[g2] + margin) continue;
      e->ncand++;
      if (t2 == G_SPHERE) col_plane_sphere(e, p, g1, g2);
      else if (t2 == G_BOX) col_plane_box(e, p, g1, g2);
      else if (t2 == G_MESH) col_plane_mesh(e, p, g1, g2);
      else if (t2 == G_CAPSULE) col_plane_capsule(e, p, g1, g2);
      else if (t2 == G_CYLINDER) col_plane_cylinder(e, p, g1, g2);
      continue;
    }
    m3mulv(t, e->gmat + 9 * g1, m->geom_obbcenter + 3 * g1); v3add(c1, e->gpos + 3 * g1, t);
    double d[3];
    v3sub(d, c2, c1);
    double rs = m->geom_rbound[g1] + m->geom_rbound[g2] + margin;
    if (v3dot(d, d) > rs * rs) continue;
    if (!(t1 == G_SPHERE && t2 == G_SPHERE) &&
        obb_separated(c1, e->gmat + 9 * g1, m->geom_obbhalf + 3 * g1, c2, e->gmat + 9 * g2, m->geom_obbhalf + 3 * g2, margin)) continue;
    e->ncand++;
    if (t1 == G_SPHERE && t2 == G_SPHERE) col_sphere_sphere(e, p, g1, g2);
    else if (t1 == G_SPHERE && t2 == G_BOX) col_sphere_box(e, p, g1, g2);
    else if (t1 == G_BOX && t2 == G_BOX) col_box_box(e, p, g1, g2);
    else if (t1 == G_SPHERE && t2 == G_CAPSULE) col_sphere_capsule(e, p, g1, g2);
    else if (t1 == G_SPHERE && t2 == G_CYLINDER) col_sphere_cylinder(e, p, g1, g2);
    else if (t1 == G_CAPSULE && t2 == G_CAPSULE) col_capsule_capsule(e, p, g1, g2);
    else col_convex(e, p, g1, g2);
  }
}

/* ------------------------------------------------------------------ stage 5: constraints (mj_makeConstraint restated) */
static double* add_row(Env* e, int type, double pos, double margin, double diag) {
  int i = e->nefc++;
  e->efc_type[i] = type; e->efc_pos[i] = pos; e->efc_margin[i] = margin; e->efc_diag[i] = diag;
  double* J = e->efc_J + (size_t)i * e->m->nv;
  memset(J, 0, sizeof(double) * e->m->nv);
  return J;
}
/* J row of  u . (velocity of world point p on body b)  and  w . (angular velocity of body b), scaled */
static void jac_point(const Env* e, double* J, int b, const double* p, const double* u, const double* w, double scale) {
  const Model* m = e->m;
  double pu[3];
  if (u) v3cross(pu, p, u);
  for (int d = m->body_lastdof[b]; d >= 0; d = m->dof_parentid[d]) {
    const double* c = e->cdof + 6 * d;
    double s = 0;
    if (u) s += v3dot(u, c + 3) + v3dot(pu, c);
    if (w) s += v3dot(w, c);
    J[d] += scale * s;
  }
}
static void impedance(const double* solref, const double* solimp, double pos, double margin, double* imp, double* K, double* B, double timestep) {
  double d0 = solimp[0], dw = solimp[1], width = solimp[2], mid = solimp[3], power = solimp[4];
  double x = fabs(pos - margin) / (width > ORC_MINVAL ? width : ORC_MINVAL), y;
  if (x >= 1) y = 1;
  else if (x <= 0) y = 0;
  else if (power == 1) y = x;
  else if (x <= mid) y = pow(x / mid, power) * mid; /* a*x^p with a = 1/mid^(p-1) */
  else y = 1 - pow((1 - x) / (1 - mid), power) * (1 - mid);
  *imp = d0 + y * (dw - d0);
  double tc = solref[0], dr = solref[1];
  if (tc < 2 * timestep) tc = 2 * timestep; /* "refsafe" */
  double dmax = dw;
  double k = dmax * dmax * tc * tc * dr * dr, bb = dmax * tc;
  *K = 1.0 / (k > ORC_MINVAL ? k : ORC_MINVAL); *B = 2.0 / (bb > ORC_MINVAL ? bb : ORC_MINVAL);
}
static void make_constraint(Env* e) {
  const Model* m = e->m;
  int nv = m->nv;
  e->nefc = 0;
  /* equality: joint coupling q1 - q1_0 = poly(q2 - q2_0) */
  for (int i = 0; i < m->neq; i++) {
    int j1 = m->eq_jnt1[i], j2 = m->eq_jnt2[i];
    const double* c = m->eq_polycoef + 5 * i;
    int a1 = m->jnt_qposadr[j1], d1 = m->jnt_dofadr[j1];
    double x1 = e->qpos[a1] - m->qpos0[a1], pos, deriv = 0, diag = m->dof_invweight0[d1];
    if (j2 >= 0) {
      int a2 = m->jnt_qposadr[j2], d2 = m->jnt_dofadr[j2];
      double x2 = e->qpos[a2] - m->qpos0[a2];
      pos = x1 - (c[0] + x2 * (c[1] + x2 * (c[2] + x2 * (c[3] + x2 * c[4]))));
      deriv = c[1] + x2 * (2 * c[2] + x2 * (3 * c[3] + x2 * 4 * c[4]));
      diag += m->dof_invweight0[d2];
      double* J = add_row(e, 0, pos, 0, diag);
      J[d1] = 1; J[d2] = -deriv;
    } else {
      pos = x1 - c[0];
      double* J = add_row(e, 0, pos, 0, diag);
      J[d1] = 1;
    }
  }
  e->ne = e->nefc;
  e->sr_overflow = 0;
  /* joint limits (hinge / slide), in joint order with the lower side first; rows past maxsr are dropped */
  for (int j = 0; j < m->njnt; j++) {
    if (!m->jnt_limited[j]) continue;
    int qa = m->jnt_qposadr[j], d = m->jnt_dofadr[j];
    double q = e->qpos[qa], mg = m->jnt_margin[j];
    for (int side = 0; side < 2; side++) {
      double dist = side == 0 ? q - m->jnt_range[2 * j] : m->jnt_range[2 * j + 1] - q;
      if (!(dist < mg)) continue;
      if (e->nefc >= e->maxsr) { e->sr_overflow = 1; continue; }
      double* J = add_row(e, 1, dist, mg, m->dof_invweight0[d]);
      J[d] = side == 0 ? 1 : -1;
    }
  }
  e->nl = e->nefc - e->ne;
  /* contacts: pyramidal cone, 2*(dim-1) rows J_n +/- mu_k J_k */
  for (int ci = 0; ci < e->ncon; ci++) {
    Contact* c = &e->con[ci];
    int b1 = m->geom_bodyid[c->geom1], b2 = m->geom_bodyid[c->geom2];
    double tran = m->body_invweight0[2 * b1] + m->body_invweight0[2 * b2], rot = m->body_invweight0[2 * b1 + 1] + m->body_invweight0[2 * b2 + 1];
    double Jb[6][64 * 8];
    if (nv > 64 * 8) { fprintf(stderr, "oracle: nv too large\n"); return; }
    for (int k = 0; k < c->dim; k++) {
      memset(Jb[k], 0, sizeof(double) * nv);
      if (k < 3) { jac_point(e, Jb[k], b2, c->pos, c->frame + 3 * k, NULL, 1.0); jac_point(e, Jb[k], b1, c->pos, c->frame + 3 * k, NULL, -1.0); }
      else { const double* ax = c->frame + 3 * (k - 3); jac_point(e, Jb[k], b2, c->pos, NULL, ax, 1.0); jac_point(e, Jb[k], b1, c->pos, NULL, ax, -1.0); }
    }
    if (c->dim == 1) {
      double* J = add_row(e, 2, c->dist, c->margin, tran);
      memcpy(J, Jb[0], sizeof(double) * nv);
      continue;
    }
    for (int k = 1; k < c->dim; k++) {
      double mu = c->friction[k - 1];
      double diag = tran + mu * mu * (k < 3 ? tran : rot);
      for (int s = 0; s < 2; s++) {
        double* J = add_row(e, 3, c->dist, c->margin, diag);
        for (int d = 0; d < nv; d++) J[d] = Jb[0][d] + (s == 0 ? mu : -mu) * Jb[k][d];
      }
    }
  }
  /* reference acceleration, regularisation */
  {
    int i = 0;
    for (int q = 0; q < m->neq; q++, i++) {
      double imp, K, B, vel = 0;
      impedance(m->eq_solref + 2 * q, m->eq_solimp + 5 * q, e->efc_pos[i], 0, &imp, &K, &B, m->timestep);
      for (int d = 0; d < nv; d++) vel += e->efc_J[(size_t)i * nv + d] * e->qvel[d];
      e->efc_aref[i] = -B * vel - K * imp * e->efc_pos[i];
      double R = (1 - imp) / imp * e->efc_diag[i];
      e->efc_R[i] = R > ORC_MINVAL ? R : ORC_MINVAL;
    }
    for (int j = 0; j < m->njnt; j++) {
      if (!m->jnt_limited[j]) continue;
      int qa = m->jnt_qposadr[j];
      double q = e->qpos[qa], mg = m->jnt_margin[j];
      for (int side = 0; side < 2; side++) {
        double dist = side == 0 ? q - m->jnt_range[2 * j] : m->jnt_range[2 * j + 1] - q;
        if (!(dist < mg)) continue;
        if (i >= e->ne + e->nl) break;
        double imp, K, B, vel = 0;
        impedance(m->jnt_solref + 2 * j, m->jnt_solimp + 5 * j, e->efc_pos[i], mg, &imp, &K, &B, m->timestep);
        for (int d = 0; d < nv; d++) vel += e->efc_J[(size_t)i * nv + d] * e->qvel[d];
        e->efc_aref[i] = -B * vel - K * imp * (e->efc_pos[i] - mg);
        double R = (1 - imp) / imp * e->efc_diag[i];
        e->efc_R[i] = R > ORC_MINVAL ? R : ORC_MINVAL;
        i++;
      }
    }
    for (int ci = 0; ci < e->ncon; ci++) {
      Contact* c = &e->con[ci];
      int nrow = c->dim == 1 ? 1 : 2 * (c->dim - 1), first = i;
      for (int r = 0; r < nrow; r++, i++) {
        double imp, K, B, vel = 0;
        impedance(c->solref, c->solimp, c->dist, c->margin, &imp, &K, &B, m->timestep);
        for (int d = 0; d < nv; d++) vel += e->efc_J[(size_t)i * nv + d] * e->qvel[d];
        e->efc_aref[i] = -B * vel - K * imp * (c->dist - c->margin);
        double R = (1 - imp) / imp * e->efc_diag[i];
        e->efc_R[i] = R > ORC_MINVAL ? R : ORC_MINVAL;
      }
      if (c->dim > 1) { /* DECISION (SURVEY A.5): all pyramid edges share Rpy = 2 mu^2 R_first, mu = friction[0]/sqrt(impratio) */
        double mu2 = c->friction[0] * c->friction[0] / m->impratio;
        double Rpy = 2 * mu2 * e->efc_R[first];
        if (Rpy < ORC_MINVAL) Rpy = ORC_MINVAL;
        for (int r = 0; r < nrow; r++) e->efc_R[first + r] = Rpy;
      }
    }
  }
}

/* ------------------------------------------------------------------ stage 6: PGS in the dual (mj_solPGS restated; pyramidal rows are plain f >= 0) */
static void solve_pgs(Env* e) {
  const Model* m = e->m;
  int nv = m->nv, n = e->nefc;
  memcpy(e->qacc, e->qacc_smooth, sizeof(double) * nv);
  memset(e->qfrc_constraint, 0, sizeof(double) * nv);
  e->solver_iter = 0;
  if (n == 0) return;
  /* B_i = M^-1 J_i^T ; AR_ii */
  for (int i = 0; i < n; i++) {
    double* B = e->efc_B + (size_t)i * nv;
    const double* J = e->efc_J + (size_t)i * nv;
    memcpy(B, J, sizeof(double) * nv);
    solve_ld(m, e->qLD, B);
    double a = 0;
    for (int d = 0; d < nv; d++) a += J[d] * B[d];
    e->efc_AR[i] = a + e->efc_R[i];
  }
  /* warm start from qacc_warmstart (mj_constraintUpdate semantics), accepted only if it beats the unconstrained start */
  double cost_ws = 0, cost_0 = 0;
  for (int d = 0; d < nv; d++) e->tmp1[d] = e->qacc_ws[d] - e->qacc_smooth[d];
  mul_m(m, e->qM, e->tmp2, e->tmp1);
  for (int d = 0; d < nv; d++) cost_ws += 0.5 * e->tmp1[d] * e->tmp2[d];
  for (int i = 0; i < n; i++) {
    const double* J = e->efc_J + (size_t)i * nv;
    double jw = 0, j0 = 0;
    for (int d = 0; d < nv; d++) { jw += J[d] * e->qacc_ws[d]; j0 += J[d] * e->qacc_smooth[d]; }
    jw -= e->efc_aref[i]; j0 -= e->efc_aref[i];
    double D = 1.0 / e->efc_R[i];
    int eq = e->efc_type[i] == 0;
    e->efc_force[i] = (eq || jw < 0) ? -D * jw : 0;
    if (eq || jw < 0) cost_ws += 0.5 * D * jw * jw;
    if (eq || j0 < 0) cost_0 += 0.5 * D * j0 * j0;
  }
  if (!(cost_ws < cost_0)) for (int i = 0; i < n; i++) e->efc_force[i] = 0;
  for (int i = 0; i < n; i++) {
    const double* B = e->efc_B + (size_t)i * nv;
    double f = e->efc_force[i];
    if (f != 0) for (int d = 0; d < nv; d++) e->qacc[d] += B[d] * f;
  }
  double scale = 1.0 / (m->meaninertia * (nv > 1 ? nv : 1));
  for (int it = 0; it < m->iterations; it++) {
    double improvement = 0;
    for (int i = 0; i < n; i++) {
      const double* J = e->efc_J + (size_t)i * nv;
      const double* B = e->efc_B + (size_t)i * nv;
      double res = 0;
      for (int d = 0; d < nv; d++) res += J[d] * e->qacc[d];
      res += e->efc_R[i] * e->efc_force[i] - e->efc_aref[i];
      double fo = e->efc_force[i], fn = fo - res / e->efc_AR[i];
      if (e->efc_type[i] != 0 && fn < 0) fn = 0;
      double delta = fn - fo;
      if (delta != 0) {
        e->efc_force[i] = fn;
        for (int d = 0; d < nv; d++) e->qacc[d] += B[d] * delta;
        improvement -= delta * (0.5 * delta * e->efc_AR[i] + res);
      }
    }
    e->solver_iter = it + 1;
    if (improvement * scale < m->tolerance) break;
  }
  for (int i = 0; i < n; i++) {
    const double* J = e->efc_J + (size_t)i * nv;
    double f = e->efc_force[i];
    if (f != 0) for (int d = 0; d < nv; d++) e->qfrc_constraint[d] += J[d] * f;
  }
}


/* ------------------------------------------------------------------ stage 6': Newton solver on the primal problem (mj_solNewton restated).
 *   minimise over a:  1/2 (a - a_smooth)^T M (a - a_smooth) + sum_i s_i(J_i a - aref_i),
 *   s_i(x) = 1/2 D_i x^2 when the row is an equality or x < 0 (limits, pyramidal contact edges), else 0.
 * Exact Newton direction from H = M + J^T D_active J (dense Cholesky), exact line search by safeguarded 1-D Newton
 * on the piecewise-quadratic cost.  DECISION: MuJoCo's incremental Cholesky updates and its three-point bracketing
 * line search are replaced by a full refactorisation and a bracketed Newton iteration (same minimiser). */
static double nt_update(Env* e, const double* jar) { /* forces, active flags, constraint cost, qfrc_constraint */
  const Model* m = e->m;
  int nv = m->nv, n = e->nefc;
  double cost = 0;
  memset(e->qfrc_constraint, 0, sizeof(double) * nv);
  for (int i = 0; i < n; i++) {
    double D = 1.0 / e->efc_R[i];
    int act = e->efc_type[i] == 0 || jar[i] < 0;
    e->nt_active[i] = act;
    e->efc_force[i] = act ? -D * jar[i] : 0;
    if (act) {
      cost += 0.5 * D * jar[i] * jar[i];
      const double* J = e->efc_J + (size_t)i * nv;
      double f = e->efc_force[i];
      for (int d = 0; d < nv; d++) e->qfrc_constraint[d] += J[d] * f;
    }
  }
  return cost;
}
/* solver statistics (profiling aid for the GPU kernel work, read with orc_newton_stats):
 * [0] solves with constraints, [1] Hessian builds (= Newton iterations that factorise), [2] builds whose active set equals the one of the
 * previous build of the same solve (H unchanged: the factor could be reused), [3] line-search iterations, [4] constraint rows summed over
 * solves, [5] solves that ended after one build, [6] after two, [7] after three or more */
static long g_nt_stats[8];
void orc_newton_stats(long* out, int reset) { memcpy(out, g_nt_stats, sizeof g_nt_stats); if (reset) memset(g_nt_stats, 0, sizeof g_nt_stats); }
static void solve_newton(Env* e) {
  const Model* m = e->m;
  int nv = m->nv, n = e->nefc;
  unsigned char prev_active[4096]; int have_prev = 0, builds = 0;
  memcpy(e->qacc, e->qacc_smooth, sizeof(double) * nv);
  memset(e->qfrc_constraint, 0, sizeof(double) * nv);
  e->solver_iter = 0;
  if (n == 0) return;
  double *jar = e->nt_jar, *jv = e->nt_jv, *Ma = e->nt_Ma, *Mv = e->nt_Mv, *grad = e->nt_grad, *search = e->nt_search, *H = e->nt_H;
  /* warm start: qacc_warmstart if it has the lower cost, else qacc_smooth */
  double cost_ws = 0, cost_0 = 0;
  for (int d = 0; d < nv; d++) e->tmp1[d] = e->qacc_ws[d] - e->qacc_smooth[d];
  mul_m(m, e->qM, e->tmp2, e->tmp1);
  for (int d = 0; d < nv; d++) cost_ws += 0.5 * e->tmp1[d] * e->tmp2[d];
  for (int i = 0; i < n; i++) {
    const double* J = e->efc_J + (size_t)i * nv;
    double jw = 0, j0 = 0;
    for (int d = 0; d < nv; d++) { jw += J[d] * e->qacc_ws[d]; j0 += J[d] * e->qacc_smooth[d]; }
    jw -= e->efc_aref[i]; j0 -= e->efc_aref[i];
    double D = 1.0 / e->efc_R[i];
    int eq = e->efc_type[i] == 0;
    if (eq || jw < 0) cost_ws += 0.5 * D * jw * jw;
    if (eq || j0 < 0) cost_0 += 0.5 * D * j0 * j0;
  }
  if (cost_ws < cost_0) memcpy(e->qacc, e->qacc_ws, sizeof(double) * nv);
  mul_m(m, e->qM, Ma, e->qacc);
  for (int i = 0; i < n; i++) {
    const double* J = e->efc_J + (size_t)i * nv;
    double s = 0;
    for (int d = 0; d < nv; d++) s += J[d] * e->qacc[d];
    jar[i] = s - e->efc_aref[i];
  }
  double cost_c = nt_update(e, jar), gauss = 0;
  for (int d = 0; d < nv; d++) gauss += 0.5 * (Ma[d] - e->qfrc_smooth[d]) * (e->qacc[d] - e->qacc_smooth[d]);
  double cost = gauss + cost_c;
  double scale = 1.0 / (m->meaninertia * (nv > 1 ? nv : 1));
  for (int it = 0; it < m->iterations; it++) {
    double gn = 0;
    for (int d = 0; d < nv; d++) { grad[d] = Ma[d] - e->qfrc_smooth[d] - e->qfrc_constraint[d]; gn += grad[d] * grad[d]; }
    if (it > 0 && scale * sqrt(gn) < m->tolerance) break;
    if (n <= 4096) {
      if (have_prev) { int same = 1; for (int r = 0; r < n; r++) if (prev_active[r] != (unsigned char)e->nt_active[r]) { same = 0; break; } g_nt_stats[2] += same; }
      for (int r = 0; r < n; r++) prev_active[r] = (unsigned char)e->nt_active[r];
      have_prev = 1;
    }
    g_nt_stats[1]++; builds++;
    /* H = M + J^T D_active J */
    memset(H, 0, sizeof(double) * nv * nv);
    for (int i = 0; i < nv; i++) {
      int a = m->dof_Madr[i], k = 0;
      for (int j = i; j >= 0; j = m->dof_parentid[j], k++) { H[i * nv + j] = e->qM[a + k]; H[j * nv + i] = e->qM[a + k]; }
    }
    for (int r = 0; r < n; r++) {
      if (!e->nt_active[r]) continue;
      const double* J = e->efc_J + (size_t)r * nv;
      double D = 1.0 / e->efc_R[r];
      for (int i = 0; i < nv; i++) {
        if (J[i] == 0) continue;
        double s = D * J[i];
        for (int j = 0; j <= i; j++) H[i * nv + j] += s * J[j];
      }
    }
    /* Cholesky H = L L^T (lower, in place), then search = -H^-1 grad */
    for (int j = 0; j < nv; j++) {
      double s = H[j * nv + j];
      for (int k = 0; k < j; k++) s -= H[j * nv + k] * H[j * nv + k];
      if (s < ORC_MINVAL) s = ORC_MINVAL;
      double ljj = sqrt(s);
      H[j * nv + j] = ljj;
      for (int i = j + 1; i < nv; i++) {
        double t = H[i * nv + j];
        for (int k = 0; k < j; k++) t -= H[i * nv + k] * H[j * nv + k];
        H[i * nv + j] = t / ljj;
      }
    }
    for (int i = 0; i < nv; i++) { double t = grad[i]; for (int k = 0; k < i; k++) t -= H[i * nv + k] * search[k]; search[i] = t / H[i * nv + i]; }
    for (int i = nv - 1; i >= 0; i--) { double t = search[i]; for (int k = i + 1; k < nv; k++) t -= H[k * nv + i] * search[k]; search[i] = t / H[i * nv + i]; }
    double snorm = 0;
    for (int d = 0; d < nv; d++) { search[d] = -search[d]; snorm += search[d] * search[d]; }
    snorm = sqrt(snorm);
    /* exact line search */
    mul_m(m, e->qM, Mv, search);
    double g1 = 0, g2 = 0;
    for (int d = 0; d < nv; d++) { g1 += search[d] * (Ma[d] - e->qfrc_smooth[d]); g2 += 0.5 * search[d] * Mv[d]; }
    for (int i = 0; i < n; i++) {
      const double* J = e->efc_J + (size_t)i * nv;
      double s = 0;
      for (int d = 0; d < nv; d++) s += J[d] * search[d];
      jv[i] = s;
    }
    double gtol = m->tolerance * 0.01 * snorm * m->meaninertia * (nv > 1 ? nv : 1);
    if (gtol < ORC_MINVAL) gtol = ORC_MINVAL;
    double alpha = 0, lo = 0, hi = -1;
    for (int ls = 0; ls < 50; ls++) {
      g_nt_stats[3]++;
      double d1 = g1 + 2 * g2 * alpha, d2 = 2 * g2;
      for (int i = 0; i < n; i++) {
        double x = jar[i] + alpha * jv[i];
        if (e->efc_type[i] == 0 || x < 0) { double D = 1.0 / e->efc_R[i]; d1 += D * x * jv[i]; d2 += D * jv[i] * jv[i]; }
      }
      if (fabs(d1) < gtol) break;
      if (d1 < 0) lo = alpha; else hi = alpha;
      double next = alpha - d1 / d2;
      if (hi >= 0 && (next <= lo || next >= hi)) next = 0.5 * (lo + hi);
      alpha = next;
    }
    e->solver_iter = it + 1;
    if (alpha == 0) break;
    for (int d = 0; d < nv; d++) { e->qacc[d] += alpha * search[d]; Ma[d] += alpha * Mv[d]; }
    for (int i = 0; i < n; i++) jar[i] += alpha * jv[i];
    double oldcost = cost;
    cost_c = nt_update(e, jar);
    gauss = 0;
    for (int d = 0; d < nv; d++) gauss += 0.5 * (Ma[d] - e->qfrc_smooth[d]) * (e->qacc[d] - e->qacc_smooth[d]);
    cost = gauss + cost_c;
    if (scale * (oldcost - cost) < m->tolerance) break;
  }
  g_nt_stats[0]++; g_nt_stats[4] += n; g_nt_stats[builds <= 1 ? 5 : (builds == 2 ? 6 : 7)]++;
}
static void solve_constraints(Env* e) { if (e->solver == 1) solve_pgs(e); else solve_newton(e); }

/* ------------------------------------------------------------------ mj_forward + mj_Euler */
void orc_forward(Env* e) {
  const Model* m = e->m;
  int nv = m->nv;
  fk(e);
  crb(e);
  memcpy(e->qLD, e->qM, sizeof(double) * m->nM);
  factor(m, e->qLD);
  collision(e);
  make_constraint(e);
  rne(e);
  for (int d = 0; d < nv; d++) { e->qfrc_passive[d] = -m->dof_damping[d] * e->qvel[d]; e->qfrc_actuator[d] = 0; }
  for (int i = 0; i < m->nu; i++) {
    double c = e->ctrl[i], lo = m->actuator_ctrlrange[2 * i], hi = m->actuator_ctrlrange[2 * i + 1];
    c = c < lo ? lo : (c > hi ? hi : c);
    e->qfrc_actuator[m->jnt_dofadr[m->actuator_jntid[i]]] += m->actuator_gear[i] * c;
  }
  for (int d = 0; d < nv; d++) { e->qfrc_smooth[d] = e->qfrc_passive[d] - e->qfrc_bias[d] + e->qfrc_actuator[d]; e->qacc_smooth[d] = e->qfrc_smooth[d]; }
  solve_ld(m, e->qLD, e->qacc_smooth);
  solve_constraints(e);
  memcpy(e->qacc_ws, e->qacc, sizeof(double) * nv);
}
static void integrate_pos(Env* e) {
  const Model* m = e->m;
  double h = m->timestep;
  for (int j = 0; j < m->njnt; j++) {
    int qa = m->jnt_qposadr[j], d = m->jnt_dofadr[j], type = m->jnt_type[j];
    if (type == J_HINGE || type == J_SLIDE) { e->qpos[qa] += h * e->qvel[d]; continue; }
    if (type == J_FREE) { for (int k = 0; k < 3; k++) e->qpos[qa + k] += h * e->qvel[d + k]; qa += 3; d += 3; }
    double w[3] = {e->qvel[d], e->qvel[d + 1], e->qvel[d + 2]}, dq[4], nq_[4];
    double ang = v3normalize(w) * h;
    qaxisangle(dq, w, ang);
    qmul(nq_, e->qpos + qa, dq); qnormalize(nq_);
    memcpy(e->qpos + qa, nq_, 32);
  }
}
void orc_step(Env* e) {
  const Model* m = e->m;
  int nv = m->nv;
  double h = m->timestep;
  orc_forward(e);
  /* semi-implicit Euler with implicit joint damping: (M + h D) a = qfrc_smooth + qfrc_constraint */
  for (int d = 0; d < nv; d++) e->tmp1[d] = e->qfrc_smooth[d] + e->qfrc_constraint[d];
  if (m->any_damping) {
    memcpy(e->qH, e->qM, sizeof(double) * m->nM);
    for (int d = 0; d < nv; d++) e->qH[m->dof_Madr[d]] += h * m->dof_damping[d];
    factor(m, e->qH);
    solve_ld(m, e->qH, e->tmp1);
  } else solve_ld(m, e->qLD, e->tmp1);
  for (int d = 0; d < nv; d++) e->qvel[d] += h * e->tmp1[d];
  integrate_pos(e);
  e->substeps++;
}

/* ------------------------------------------------------------------ controller (MujocoController.py:269-393; PID = simple_pid [EXT], Ki = 0) */
static void pid_all(Env* e) {
  const Model* m = e->m;
  for (int i = 0; i < NU; i++) {
    double x = e->qpos[m->jnt_qposadr[m->actuator_jntid[i]]];
    double u = e->kp[i] * (e->target[i] - x) - e->kd[i] * (x - e->last_input[i]) / e->dt_pid;
    u = u < -e->lim[i] ? -e->lim[i] : (u > e->lim[i] ? e->lim[i] : u);
    e->last_input[i] = x;
    e->ctrl[i] = u;
  }
}
/* returns 1 = "success", 2 = "max. steps reached"; *steps = last_movement_steps.  group_mask bit i = actuator i in group.
 * target[i] is applied for group members when has_target (MujocoController.py:308-311). */
int orc_move_group(Env* e, int group_mask, const double* target, int has_target, double tol, int max_steps, int* steps_out) {
  const Model* m = e->m;
  int steps = 1, result = 0, reached = 0;
  if (has_target) { int k = 0; for (int i = 0; i < NU; i++) if (group_mask >> i & 1) e->target[i] = target[k++]; }
  while (!reached) {
    pid_all(e);
    double mx = 0;
    for (int i = 0; i < NU; i++) if (group_mask >> i & 1) { double dl = fabs(e->target[i] - e->qpos[m->jnt_qposadr[m->actuator_jntid[i]]]); if (dl > mx) mx = dl; }
    if (mx < tol) { result = 1; reached = 1; }
    if (steps > max_steps) { result = 2; break; }
    orc_step(e);
    steps++;
  }
  if (steps_out) *steps_out = steps;
  return result;
}
/* stay(ms): the reference loops 10-sub-step chunks for `ms` of WALL-CLOCK time (MujocoController.py:621-637).
 * DECISION (SURVEY A.1): deterministic mapping ms -> ceil(ms/2/10) chunks, i.e. ms/2 sub-steps. */
void orc_stay(Env* e, int ms) {
  int chunks = (ms / 2 + 9) / 10;
  for (int c = 0; c < chunks; c++) orc_move_group(e, 0x7f, NULL, 0, 1e-7, 10, NULL);
}

/* analytic tool-down IK for the ur5_gripper.urdf chain (SURVEY A.4). ee_pos in world; out 5 joint angles. returns 1 ok */
int orc_ik(Env* e, const double* ee_pos, double* q5) {
  const Model* m = e->m;
  fk(e);
  const double* ch = m->ik_chain; /* d1, d4, a1, a2, d5, d6 */
  double d1 = ch[0], d4 = ch[1], a1 = ch[2], a2 = ch[3], d5 = ch[4], d6 = ch[5];
  double p[3];
  for (int k = 0; k < 3; k++) p[k] = ee_pos[k] - e->xpos[3 * m->ik_base_body + k] + m->ik_offset[k];
  double r2 = p[0] * p[0] + p[1] * p[1];
  if (r2 < d4 * d4 + 1e-12) return 0;
  double r = sqrt(r2), phi = atan2(p[1], p[0]);
  double pan = phi - asin(d4 / r);
  if (pan < -M_PI) pan += 2 * M_PI;
  if (pan > M_PI) pan -= 2 * M_PI;
  double rho = sqrt(r2 - d4 * d4), Wx = rho - d5, Wz = p[2] + d6 - d1;
  double L2 = Wx * Wx + Wz * Wz, c = (L2 - a1 * a1 - a2 * a2) / (2 * a1 * a2);
  if (c > 1) c = 1;
  if (c < -1) c = -1;
  double elbow = acos(c);
  double alpha = atan2(Wz, Wx) + atan2(a2 * sin(elbow), a1 + a2 * cos(elbow));
  double lift = -alpha, w1 = -0.5 * M_PI - lift - elbow, w2 = -0.5 * M_PI;
  if (w1 < -M_PI) w1 += 2 * M_PI;
  if (w1 > M_PI) w1 -= 2 * M_PI;
  /* forward check of the planar wrist point (error is zero unless the reach was clamped) */
  double fx = a1 * cos(alpha) + a2 * cos(alpha - elbow), fz = a1 * sin(alpha) + a2 * sin(alpha - elbow);
  double err = sqrt((fx - Wx) * (fx - Wx) + (fz - Wz) * (fz - Wz));
  q5[0] = pan; q5[1] = lift; q5[2] = elbow; q5[3] = w1; q5[4] = w2;
  for (int k = 0; k < 5; k++) if (q5[k] < m->ik_lower[k] - 1e-9 || q5[k] > m->ik_upper[k] + 1e-9) return 0;
  return err <= 0.02;
}
/* move_ee (MujocoController.py:446-465): 0 = "No valid joint angles", 1 success, 2 max steps */
int orc_move_ee(Env* e, const double* ee_pos, double tol, int max_steps, int* steps_out) {
  double q5[5];
  if (!orc_ik(e, ee_pos, q5)) { if (steps_out) *steps_out = 0; return 0; }
  return orc_move_group(e, 0x1f, q5, 1, tol, max_steps, steps_out);
}

/* move_and_grasp (GraspingEnv.py:205-386). coords = world target from pixel_2_world, rot index 0..5.
 * info[0..9] receives per-phase step counts / codes. returns reward 0/1 */
static const double ROT_DEG[6] = {0, 30, 60, 90, -30, -60};
int orc_move_and_grasp(Env* e, const double* coords, int rot, double table_height, int* info) {
  int steps = 0, r1, r2 = -1, grasp = 0, rfinal = -1;
  double c1[3] = {coords[0], coords[1], 1.1}, centre[3] = {0.0, -0.6, 1.1}, drop[3] = {0.6, 0.0, 1.15};
  int inf[12] = {0};
  r1 = orc_move_ee(e, c1, 0.05, 1000, &steps); inf[0] = r1; inf[1] = steps;
  if (r1 == 0) { r1 = orc_move_ee(e, centre, 0.05, 1000, &steps); inf[0] = 10 + r1; inf[1] = steps; }
  if (r1 != 2) {
    /* NB: if the fallback IK also failed the reference would still proceed (result string "No..." is neither "max"). */
    double tgt = ROT_DEG[rot] * M_PI / 180.0;
    e->target[5] = tgt;
    orc_move_group(e, 0x7f, NULL, 0, 0.05, 500, &steps); inf[2] = steps;
    double half[1] = {0.0};
    orc_move_group(e, 0x40, half, 1, 0.05, 1000, &steps);
    double c2[3] = {coords[0], coords[1], coords[2] - 0.01 > table_height ? coords[2] - 0.01 : table_height};
    r2 = orc_move_ee(e, c2, 0.01, 300, &steps); inf[3] = r2; inf[4] = steps;
    if (r2 == 2) grasp = 0;
    else {
      orc_stay(e, 100);
      double cl[1] = {-0.4};
      int rg = orc_move_group(e, 0x40, cl, 1, 0.01, 300, &steps);
      grasp = rg != 1; inf[5] = steps;
    }
  }
  e->kp[0] = 10.0;
  int r3 = orc_move_ee(e, centre, 0.05, 1000, &steps); inf[6] = steps; (void)r3;
  int r4 = orc_move_ee(e, drop, 0.01, 1200, &steps); inf[7] = steps; (void)r4;
  if (grasp) { double cl[1] = {-0.4}; rfinal = orc_move_group(e, 0x40, cl, 1, 0.01, 1000, &steps); inf[8] = steps; }
  int grasped = (rfinal == 2) && grasp;
  double op[1] = {0.4};
  orc_move_group(e, 0x40, op, 1, 0.05, 1000, &steps); inf[9] = steps;
  if (grasped) orc_stay(e, 200);
  e->target[5] = 0.0;
  orc_move_group(e, 0x7f, NULL, 0, 0.05, 500, &steps); inf[10] = steps;
  e->kp[0] = 20.0;
  inf[11] = grasp;
  if (info) memcpy(info, inf, sizeof inf);
  return grasped;
}

/* ------------------------------------------------------------------ observation (MujocoController.py:708-740): ray-cast RGB-D.
 * depth is linear eye-space z in metres (= depth_2_meters of a GL depth buffer, SURVEY A.3); image already flipped U/D + L/R. */
static double ray_geom(const Env* e, int g, const double* o, const double* dir, double* nrm) {
  const Model* m = e->m;
  const double *R = e->gmat + 9 * g, *size = m->geom_size + 3 * g;
  double ol[3], dl[3], t[3];
  v3sub(t, o, e->gpos + 3 * g); m3Tmulv(ol, R, t); m3Tmulv(dl, R, dir);
  int type = m->geom_type[g];
  double tn = -1e300, tf = 1e300, nl[3] = {0, 0, 1};
  if (type == G_PLANE) {
    if (dl[2] >= -1e-12) return -1;
    double tt = -ol[2] / dl[2];
    if (tt <= 0) return -1;
    m3col(nrm, R, 2);
    return tt;
  } else if (type == G_SPHERE) {
    double b = v3dot(ol, dl), c = v3dot(ol, ol) - size[0] * size[0], a = v3dot(dl, dl);
    double disc = b * b - a * c;
    if (disc < 0) return -1;
    double tt = (-b - sqrt(disc)) / a;
    if (tt <= 0) return -1;
    v3addscl(nl, ol, dl, tt); v3normalize(nl);
    m3mulv(nrm, R, nl);
    return tt;
  } else if (type == G_BOX) {
    for (int k = 0; k < 3; k++) {
      if (fabs(dl[k]) < 1e-14) { if (fabs(ol[k]) > size[k]) return -1; continue; }
      double t1 = (-size[k] - ol[k]) / dl[k], t2 = (size[k] - ol[k]) / dl[k], s = -1;
      if (t1 > t2) { double x = t1; t1 = t2; t2 = x; s = 1; }
      if (t1 > tn) { tn = t1; v3set(nl, 0, 0, 0); nl[k] = s; }
      if (t2 < tf) tf = t2;
    }
    if (tn > tf || tn <= 0) return -1;
    m3mulv(nrm, R, nl);
    return tn;
  } else if (type == G_MESH) {
    int k = m->geom_meshid[g];
    /* bounding sphere reject */
    double oc[3]; v3sub(oc, ol, m->geom_obbcenter + 3 * g);
    double b = v3dot(oc, dl), c = v3dot(oc, oc) - m->geom_rbound[g] * m->geom_rbound[g], a = v3dot(dl, dl);
    if (b * b - a * c < 0) return -1;
    const double* pl = m->face_plane + 4 * m->mesh_faceadr[k];
    for (int f = 0; f < m->mesh_facenum[k]; f++, pl += 4) {
      double dn = v3dot(pl, dl), on = v3dot(pl, ol) - pl[3];
      if (fabs(dn) < 1e-14) { if (on > 0) return -1; continue; }
      double tt = -on / dn;
      if (dn < 0) { if (tt > tn) { tn = tt; v3copy(nl, pl); } }
      else if (tt < tf) tf = tt;
      if (tn > tf) return -1;
    }
    if (tn <= 0) return -1;
    m3mulv(nrm, R, nl);
    return tn;
  }
  if (type == G_CYLINDER) { /* infinite cylinder and the slab |z| <= h, intersected like the box slabs */
    double r = size[0], h = size[1];
    double a = dl[0] * dl[0] + dl[1] * dl[1], b = ol[0] * dl[0] + ol[1] * dl[1], c = ol[0] * ol[0] + ol[1] * ol[1] - r * r;
    if (a < 1e-14) { if (c > 0) return -1; }
    else {
      double disc = b * b - a * c;
      if (disc < 0) return -1;
      double sq = sqrt(disc);
      tn = (-b - sq) / a; tf = (-b + sq) / a;
      v3set(nl, (ol[0] + tn * dl[0]) / r, (ol[1] + tn * dl[1]) / r, 0);
    }
    if (fabs(dl[2]) < 1e-14) { if (fabs(ol[2]) > h) return -1; }
    else {
      double t1 = (-h - ol[2]) / dl[2], t2 = (h - ol[2]) / dl[2], s = -1;
      if (t1 > t2) { double x = t1; t1 = t2; t2 = x; s = 1; }
      if (t1 > tn) { tn = t1; v3set(nl, 0, 0, s); }
      if (t2 < tf) tf = t2;
    }
    if (tn > tf || tn <= 0) return -1;
    m3mulv(nrm, R, nl);
    return tn;
  }
  if (type == G_CAPSULE) { /* side wall where |z| <= h, otherwise the outward half of either end sphere */
    double r = size[0], h = size[1], best = -1;
    double a = dl[0] * dl[0] + dl[1] * dl[1], b = ol[0] * dl[0] + ol[1] * dl[1], c = ol[0] * ol[0] + ol[1] * ol[1] - r * r;
    if (a >= 1e-14) {
      double disc = b * b - a * c;
      if (disc >= 0) {
        double t1 = (-b - sqrt(disc)) / a, z = ol[2] + t1 * dl[2];
        if (t1 > 0 && fabs(z) <= h) { best = t1; v3set(nl, (ol[0] + t1 * dl[0]) / r, (ol[1] + t1 * dl[1]) / r, 0); }
      }
    }
    for (int s = 0; s < 2; s++) {
      double sg = s ? -1.0 : 1.0, oc[3] = {ol[0], ol[1], ol[2] - sg * h};
      double bb = v3dot(oc, dl), cc = v3dot(oc, oc) - r * r, aa = v3dot(dl, dl), disc = bb * bb - aa * cc;
      if (disc < 0) continue;
      double t1 = (-bb - sqrt(disc)) / aa;
      if (t1 <= 0 || sg * (oc[2] + t1 * dl[2]) < 0) continue;
      if (best < 0 || t1 < best) { best = t1; v3addscl(nl, oc, dl, t1); v3scl(nl, nl, 1.0 / r); }
    }
    if (best <= 0) return -1;
    m3mulv(nrm, R, nl);
    return best;
  }
  return -1;
}
void orc_render(Env* e, int cam, int W, int H, uint8_t* rgb, float* depth) {
  const Model* m = e->m;
  fk(e);
  const double *cp = m->cam_pos0 + 3 * cam, *cm = m->cam_mat0 + 9 * cam;
  double f = 0.5 * H / tan(m->cam_fovy[cam] * M_PI / 360.0);
  double light[3] = {-1, 1, -2.565}; /* directional light at (1,-1,3) aimed at box_link (0,0,0.435): UR5gripper_2_finger.xml:107 */
  v3normalize(light);
  for (int r = 0; r < H; r++) for (int c = 0; c < W; c++) {
    double dc[3] = {(0.5 * W - c - 0.5) / f, (0.5 * H - r - 0.5) / f, -1.0}, dir[3];
    m3mulv(dir, cm, dc);
    double best = 1e300, bn[3] = {0, 0, 1}; int bg = -1;
    for (int g = 0; g < m->ngeom; g++) {
      double n[3];
      double t = ray_geom(e, g, cp, dir, n);
      if (t > 0 && t < best) { best = t; bg = g; v3copy(bn, n); }
    }
    size_t px = (size_t)r * W + c;
    if (bg < 0) { depth[px] = (float)(m->zfar * m->extent); rgb[3 * px] = rgb[3 * px + 1] = rgb[3 * px + 2] = 0; continue; }
    depth[px] = (float)best; /* dir has eye-z = -1, so t is eye-space depth */
    double lam = -v3dot(bn, light);
    if (lam < 0) lam = 0;
    double shade = 0.4 + 0.6 * lam;
    const double* col = m->geom_rgba + 4 * bg;
    double base[3] = {col[0], col[1], col[2]};
    if (m->geom_type[bg] == G_PLANE) { /* builtin checker floor: texrepeat 10 over the 5 m plane */
      double hit[3]; v3addscl(hit, cp, dir, best);
      int cx = (int)floor(hit[0] / 0.25), cy = (int)floor(hit[1] / 0.25);
      if ((cx + cy) & 1) { base[0] = 0.1; base[1] = 0.2; base[2] = 0.3; } else { base[0] = 0.2; base[1] = 0.3; base[2] = 0.4; }
    }
    for (int k = 0; k < 3; k++) { double v = base[k] * shade * 255.0 + 0.5; rgb[3 * px + k] = (uint8_t)(v > 255 ? 255 : v); }
  }
}

/* ------------------------------------------------------------------ render probe: where rounding may decide a pixel.
 * The CUDA renderer evaluates the same fp64 expressions as orc_render, but with FMA contraction and on geom frames from its own
 * kinematics (which agree with fk's to rounding), so its f32 depth and u8 rgb can legitimately differ only where a rounding-sized
 * change of the ray or of the frames changes the answer.  For each listed pixel (index r * W + c) this returns the geom orc_render
 * picks (-1: background) and a bit set of such reasons:
 *   1  the winner, its normal (by more than 1e-6), its f32 depth or its rgb changes when the ray direction moves by +-eps_px pixels
 *      in x or y, or the camera origin by +-eps_m along a world axis (silhouettes, hull edges, frame differences);
 *   2  the nearest hit of another geom is within a relative PROBE_REL_TIE of the winner's (coplanar faces);
 *   4  a shaded channel base * shade * 255 + 0.5 lies within a relative 1e-9 of an integer (u8 truncation boundary);
 *   8  the fp64 depth lies within a relative PROBE_REL_F32 of a rounding midpoint of f32;
 *   16 a floor hit lies within 1e-9 m of a checker line (floor(hit / 0.25)). */
#define PROBE_REL_TIE 1e-9
#define PROBE_REL_F32 1e-12
typedef struct { int g; double t, second, n[3]; float depth; uint8_t rgb[3]; double v[3]; double hit[3]; } ProbeHit;
static void probe_trace(const Env* e, const double* o, const double* dir, ProbeHit* h) {
  const Model* m = e->m;
  h->g = -1; h->t = 1e300; h->second = 1e300; v3set(h->n, 0, 0, 1);
  for (int g = 0; g < m->ngeom; g++) {
    double n[3], t = ray_geom(e, g, o, dir, n);
    if (!(t > 0)) continue;
    if (t < h->t) { h->second = h->t; h->t = t; h->g = g; v3copy(h->n, n); }
    else if (t < h->second) h->second = t;
  }
  if (h->g < 0) { h->depth = (float)(m->zfar * m->extent); h->rgb[0] = h->rgb[1] = h->rgb[2] = 0; return; }
  h->depth = (float)h->t;
  double light[3] = {-1, 1, -2.565};
  v3normalize(light);
  double lam = -v3dot(h->n, light);
  if (lam < 0) lam = 0;
  double shade = 0.4 + 0.6 * lam;
  const double* col = m->geom_rgba + 4 * h->g;
  double base[3] = {col[0], col[1], col[2]};
  v3addscl(h->hit, o, dir, h->t);
  if (m->geom_type[h->g] == G_PLANE) {
    int cx = (int)floor(h->hit[0] / 0.25), cy = (int)floor(h->hit[1] / 0.25);
    if ((cx + cy) & 1) { base[0] = 0.1; base[1] = 0.2; base[2] = 0.3; } else { base[0] = 0.2; base[1] = 0.3; base[2] = 0.4; }
  }
  for (int k = 0; k < 3; k++) { h->v[k] = base[k] * shade * 255.0 + 0.5; h->rgb[k] = (uint8_t)(h->v[k] > 255 ? 255 : h->v[k]); }
}
void orc_render_probe(Env* e, int cam, int W, int H, int n, const int64_t* pix, double eps_px, double eps_m, int* gid, int* flags) {
  const Model* m = e->m;
  fk(e);
  const double *cp = m->cam_pos0 + 3 * cam, *cm = m->cam_mat0 + 9 * cam;
  double f = 0.5 * H / tan(m->cam_fovy[cam] * M_PI / 360.0);
  for (int i = 0; i < n; i++) {
    int r = (int)(pix[i] / W), c = (int)(pix[i] % W), fl = 0;
    double dc[3] = {(0.5 * W - c - 0.5) / f, (0.5 * H - r - 0.5) / f, -1.0}, dir[3];
    m3mulv(dir, cm, dc);
    ProbeHit h;
    probe_trace(e, cp, dir, &h);
    gid[i] = h.g;
    if (h.g >= 0) {
      if (h.second - h.t <= PROBE_REL_TIE * h.t) fl |= 2;
      for (int k = 0; k < 3; k++) if (fabs(h.v[k] - floor(h.v[k] + 0.5)) <= 1e-9 * h.v[k]) fl |= 4;
      float lo = nextafterf(h.depth, -INFINITY), hi = nextafterf(h.depth, INFINITY);
      double mlo = 0.5 * ((double)h.depth + lo), mhi = 0.5 * ((double)h.depth + hi);
      if (fabs(h.t - mlo) <= PROBE_REL_F32 * h.t || fabs(h.t - mhi) <= PROBE_REL_F32 * h.t) fl |= 8;
      if (m->geom_type[h.g] == G_PLANE)
        for (int k = 0; k < 2; k++) if (fabs(h.hit[k] - 0.25 * floor(h.hit[k] / 0.25 + 0.5)) <= 1e-9) fl |= 16;
    }
    for (int p = 0; p < 10; p++) {
      double o2[3] = {cp[0], cp[1], cp[2]}, dc2[3] = {dc[0], dc[1], dc[2]}, dir2[3], s = (p & 1) ? -1.0 : 1.0;
      if (p < 4) dc2[p >> 1] = (0.5 * (p < 2 ? W : H) - (p < 2 ? c : r) - 0.5 + s * eps_px) / f;
      else o2[(p - 4) >> 1] += s * eps_m;
      m3mulv(dir2, cm, dc2);
      ProbeHit q;
      probe_trace(e, o2, dir2, &q);
      int moved = q.g != h.g;
      if (!moved && h.g >= 0) {
        for (int k = 0; k < 3; k++) moved |= fabs(q.n[k] - h.n[k]) > 1e-6 || q.rgb[k] != h.rgb[k];
        moved |= q.depth != h.depth;
      }
      if (moved) { fl |= 1; break; }
    }
    flags[i] = fl;
  }
}

/* ------------------------------------------------------------------ accessors for tests */
double* orc_qpos(Env* e) { return e->qpos; }
double* orc_qvel(Env* e) { return e->qvel; }
double* orc_qacc_ws(Env* e) { return e->qacc_ws; }
double* orc_ctrl(Env* e) { return e->ctrl; }
double* orc_target(Env* e) { return e->target; }
double* orc_kp(Env* e) { return e->kp; }
double* orc_last_input(Env* e) { return e->last_input; }
long orc_substeps(Env* e) { return e->substeps; }
void orc_set_dt_pid(Env* e, double dt) { e->dt_pid = dt; }
void orc_set_solver(Env* e, int solver) { e->solver = solver; }
/* contact capacity: the list keeps the first n contacts of its emission order (analytic pairs, then MPR pairs, both in pair order),
 * like the CUDA engine's list of `maxcon` contacts; clamped to [0, MAXCON] */
void orc_set_maxcon(Env* e, int n) { e->maxcon = n < 0 ? 0 : (n > MAXCON ? MAXCON : n); }
/* simple-row capacity: make_constraint keeps the equality rows and then the first limit rows (joint order, lower side first) up to
 * n rows in all, like the CUDA engine's GE_MAXSR slots; n < 0 restores the default (no cap) */
void orc_set_maxsr(Env* e, int n) { e->maxsr = n < 0 ? e->nefc_max : n; }
/* 1 if the last make_constraint dropped limit rows at the simple-row capacity */
int orc_sr_overflow(Env* e) { return e->sr_overflow; }
/* rows of the last make_constraint: out[0] equality, out[1] joint limit, out[2] contact */
void orc_efc_split(Env* e, int* out) { out[0] = e->ne; out[1] = e->nl; out[2] = e->nefc - e->ne - e->nl; }
/* 1 if the last collision stage found more contacts than the capacity */
int orc_con_overflow(Env* e) { return e->con_overflow; }
/* the most contacts one collision stage found (capacity or not) since the previous call with reset != 0 */
int orc_ncon_peak(Env* e, int reset) { int p = e->ncon_peak; if (reset) e->ncon_peak = 0; return p; }
/* broad-phase survivors of the last collision stage (the engine's "ncand") */
int orc_ncand(Env* e) { return e->ncand; }
/* set_state + controller re-sync as GraspEnv.reset_model does (GraspingEnv.py:466-470) */
void orc_reset(Env* e, const double* qpos, const double* qvel) {
  const Model* m = e->m;
  memcpy(e->qpos, qpos, sizeof(double) * m->nq);
  if (qvel) memcpy(e->qvel, qvel, sizeof(double) * m->nv); else memset(e->qvel, 0, sizeof(double) * m->nv);
  memset(e->qacc_ws, 0, sizeof(double) * m->nv);
  for (int i = 0; i < NU; i++) {
    e->kp[i] = m->pid_kp[i]; e->ctrl[i] = 0;
    e->target[i] = e->qpos[m->jnt_qposadr[m->actuator_jntid[i]]];
    e->last_input[i] = e->target[i]; /* DECISION: no derivative kick on the first call after reset */
  }
  fk(e);
}
void orc_fk(Env* e) { fk(e); }
const double* orc_field(Env* e, const char* name, int* n) {
  const Model* m = e->m;
#define F(nm, ptr, cnt) if (!strcmp(name, nm)) { if (n) *n = (cnt); return ptr; }
  F("xpos", e->xpos, 3 * m->nbody) F("xquat", e->xquat, 4 * m->nbody) F("xmat", e->xmat, 9 * m->nbody) F("xipos", e->xipos, 3 * m->nbody)
  F("cdof", e->cdof, 6 * m->nv) F("qM", e->qM, m->nM) F("qLD", e->qLD, m->nM) F("qfrc_bias", e->qfrc_bias, m->nv)
  F("qfrc_smooth", e->qfrc_smooth, m->nv) F("qacc_smooth", e->qacc_smooth, m->nv) F("qacc", e->qacc, m->nv)
  F("qfrc_constraint", e->qfrc_constraint, m->nv) F("efc_force", e->efc_force, e->nefc) F("efc_aref", e->efc_aref, e->nefc)
  F("efc_R", e->efc_R, e->nefc) F("efc_J", e->efc_J, e->nefc * m->nv) F("efc_pos", e->efc_pos, e->nefc)
  F("gpos", e->gpos, 3 * m->ngeom) F("gmat", e->gmat, 9 * m->ngeom) F("boxbox", e->bbx, BBX_W * e->nbbx)
#undef F
  if (n) *n = 0;
  return NULL;
}
int orc_ncon(Env* e) { return e->ncon; }
int orc_nefc(Env* e) { return e->nefc; }
int orc_solver_iter(Env* e) { return e->solver_iter; }
/* contact i -> out[0]=dist, out[1..3]=pos, out[4..12]=frame, out[13]=geom1, out[14]=geom2, out[15]=dim */
void orc_contact(Env* e, int i, double* out) {
  const Contact* c = &e->con[i];
  out[0] = c->dist; v3copy(out + 1, c->pos); memcpy(out + 4, c->frame, 72); out[13] = c->geom1; out[14] = c->geom2; out[15] = c->dim;
}

/* ------------------------------------------------------------------ camera math (MujocoController.py:729-806), pinned by tests/golden/camera_math.json */
/* pixel_2_world: pos_w = R^-1 (K^-1 [x, y, 1] * (-depth) + cam_pos), K = [[f,0,W/2],[0,f,H/2],[0,0,1]], f = 0.5 H / tan(fovy pi/360) */
void orc_pixel_2_world(const Model* m, int cam, int W, int H, double px, double py, double depth, double* out) {
  double f = 0.5 * H / tan(m->cam_fovy[cam] * M_PI / 360.0), d = -depth;
  double pc[3] = {(px * d - 0.5 * W * d) / f, (py * d - 0.5 * H * d) / f, d}, t[3];
  v3add(t, pc, m->cam_pos0 + 3 * cam);
  m3Tmulv(out, m->cam_mat0 + 9 * cam, t);
}
/* depth_2_meters: near / (1 - d (1 - near/far)), near = znear * extent, far = zfar * extent */
double orc_depth_2_meters(const Model* m, double gl_depth) {
  double near = m->znear * m->extent, far = m->zfar * m->extent;
  return near / (1.0 - gl_depth * (1.0 - near / far));
}
Model* orc_env_model(Env* e) { return e->m; }

long orc_mpr_calls(void) { return g_mpr_calls; }
