// Device-side view of the compiled scene (read-only, shared by all environments) and the per-warp
// shared-memory workspace layout.  One warp simulates one environment; all per-step intermediates live in
// that warp's shared-memory slice, only the state rows (qpos, qvel, warm start, controller) round-trip HBM.
#pragma once
#include <stdint.h>

#define GE_NU 7          // actuators of the UR5 + 2-finger gripper scenes (MujocoController.py:157-235)
// contacts kept per environment / narrow-phase candidate pairs: Layout::maxcon, Layout::maxcand (chosen per scene at ge_create;
// overflow is flagged in the status word)
#define GE_MAXSR 16      // "simple" constraint rows: joint equality + joint limits (<= 2 non-zeros each)
#define GE_MAXCHAIN 24   // longest dof list of one contact (both kinematic chains)

enum { G_PLANE = 0, G_SPHERE = 2, G_CAPSULE = 3, G_CYLINDER = 5, G_BOX = 6, G_MESH = 7 };
enum { J_FREE = 0, J_BALL = 1, J_SLIDE = 2, J_HINGE = 3 };

struct DevModel {
  int nbody, njnt, nq, nv, nu, ngeom, neq, npair, nmesh, nM, ntree, maxdim;
  double timestep, gravity[3], tolerance, impratio, mpr_tol, meaninertia, extent, zfar;
  int iterations, mpr_iter, any_damping, ik_base_body, ee_body;
  const double *qpos0, *body_pos, *body_quat, *body_mass, *body_ipos, *body_inertia, *body_invweight0;
  const int *body_parentid, *body_jntadr, *body_jntnum, *body_lastdof, *body_subtreenum, *body_chainmask;
  const int *jnt_type, *jnt_bodyid, *jnt_qposadr, *jnt_dofadr, *jnt_limited;
  const double *jnt_pos, *jnt_axis, *jnt_range, *jnt_margin, *jnt_solref, *jnt_solimp;
  const int *dof_bodyid, *dof_jntid, *dof_parentid, *dof_Madr, *dof_subtreenum, *dof_depth, *dof_treeindex, *tree_dofadr, *tree_dofnum, *tree_simple;
  const double *dof_armature, *dof_damping, *dof_invweight0, *tree_Minv;
  // [nv][GE_GROUP]: index in qM of entry (i, tree_dofadr + j) of dof i's row of its tree's mass block, -1 where that entry is zero
  // (derived at ge_create from dof_parentid / dof_Madr; used by the register Hessian blocks of ge_hessian.cuh)
  const int* dof_Mcol;
  const int *geom_type, *geom_bodyid, *geom_meshid;
  const double *geom_pos, *geom_lmat, *geom_size, *geom_rbound, *geom_obbcenter, *geom_obbhalf, *geom_rgba;
  const int *mesh_vertadr, *mesh_vertnum, *mesh_faceadr, *mesh_facenum;
  const double *mesh_vert, *mesh_center, *mesh_faceplane;
  const int *pair_geom, *pair_condim, *pair_rec;
  const double *pair_friction, *pair_margin, *pair_solref, *pair_solimp, *pair_rsum;
  const int* actuator_jntid;
  const double *actuator_gear, *actuator_ctrlrange;
  const int *eq_jnt1, *eq_jnt2;
  const double *eq_polycoef, *eq_solref, *eq_solimp;
  const double *cam_pos0, *cam_mat0, *cam_fovy;
  const double *pid_kp, *pid_kd, *pid_lim, *ik_chain, *ik_lower, *ik_upper, *ik_offset;
};

// workspace offsets, in doubles (ints live behind the doubles, offsets in ints from the int base)
struct Layout {
  int qpos, qvel, qaccws, ctl;  // ctl: target[8] last_input[8] kp[8] ctrl[8]
  int cdof, qM;
  int qfrc_smooth, qacc_smooth, qfrc_constraint, qacc, Ma, grad, search, Mv;
  int con, cstride;             // contact records
  int sr;                       // simple rows: coefA coefB D aref jar jv  (6 x GE_MAXSR)
  int scratch;                  // phase-aliased region, see below
  int total_doubles;
  // --- aliases inside scratch: kinematics / dynamics phase
  int lpos, lquat, janchor, jaxis, xpos, xmat, cinert, gpos, gmat, gcen;  // FK phase
  int cvel, cacc, cfrc, cdofdot;                                          // RNE phase (over lpos.. janchor.. xpos..)
  // --- aliases inside scratch: solver phase
  int H, Vb, Wb;
  // --- ints
  int i_cb1, i_cb2, i_ct1, i_ct2, i_cdim, i_cpair, i_cact, i_srA, i_srB, i_srtype, i_sract, i_cand, i_first, i_tcoupled, i_tcount, i_tlist, i_island;
  int total_ints;
  int total_bytes;
  int maxcon, maxcand;          // capacity of the contact / candidate lists
  int fk_bytes;                 // bytes of the workspace prefix the kinematics stage touches (kinematics-only kernels)
  int hcap;                     // doubles of the Hessian block region at L.H (= nv (nv + 1) / 2 when everything always fits)
  int hfull;                    // nv (nv + 1) / 2: size of the overflow row
  int i_hflag;                  // int slot: 1 while the Hessian blocks of the current build live in the overflow row
  unsigned long long* hovf_builds;  // [1] on the device: Hessian builds of this engine that used the overflow row (ge_size 13)
};

// per-environment state in HBM, row-major [N, ...]
struct EnvArrays {
  double *qpos, *qvel, *qaccws;   // [N,nq] [N,nv] [N,nv]
  double* ctl;                    // [N,32]: target[8] last_input[8] kp[8] ctrl[8]
  // movement command (MJ_Controller.move_group_to_joint_target arguments + loop counters)
  int *cmd_mask, *cmd_maxsteps, *cmd_steps, *cmd_result, *cmd_active;  // [N]
  double* cmd_tol;                // [N]
  // grasp program (GraspEnv.move_and_grasp state machine)
  int *prog_phase, *prog_rot, *prog_grasp, *prog_aux, *prog_info;  // [N] [N] [N] [N] [N,12]
  double *prog_coords, *prog_table;  // [N,3] [N]
  unsigned char* reward;          // [N]
  int* status;                    // [N]
  long long* substeps;            // [N]
  int* busy_count;                // [1]
  int* lock;                      // [N] 1 while a warp of k_run holds the env (dynamic env -> warp assignment)
  int* owed;                      // [N] visits of the env drawn in this launch and not yet run (k_run: a drawer never drops a visit)
  int* done;                      // [N] iterations the env has been given in this launch (reset before every launch)
  unsigned long long* ticket;     // [1] monotonically increasing task counter of k_run (never reset: launches subtract their base)
  double* gws;                    // [N, hfull] Hessian overflow rows (when hcap < hfull), else NULL
};
