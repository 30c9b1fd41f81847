/* grasp_engine.h — C-ABI of the H100 batched grasp-simulation engine (libgrasp_engine.so).
 *
 * The reference has no FFI layer: its boundary is two Python classes (GraspEnv, MJ_Controller) that poke
 * mujoco_py attributes.  Each entry point below names the reference interface it stands in for (file:line in
 * /root/reference).  All functions return 0 on success or a negative error code; ge_last_error() gives the message
 * of the last failure on the calling thread.  No exceptions cross the ABI.  Every pointer marked [dev] is a CUDA
 * device pointer owned by the caller (e.g. torch tensor storage); [host] pointers are ordinary host memory.
 * One handle per device; a handle is not thread-safe; launches go to the stream given at creation time
 * (0 = the legacy default stream).  N = number of environments of the handle.
 *
 * The library holds two builds of the engine (one environment per warp / one environment per CTA of 4 warps, for scenes whose
 * per-env workspace the warp-per-env build cannot hold); ge_create picks one from the scene's size (ge_size(h, 9) tells which), every
 * other entry point forwards through the handle.  Handles of different scenes may coexist in one process.
 */
#ifndef GRASP_ENGINE_H
#define GRASP_ENGINE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ge_engine* ge_handle;

enum { GE_OK = 0, GE_ERR_ARG = -1, GE_ERR_CUDA = -2, GE_ERR_MODEL = -3, GE_ERR_STATE = -4 };

/* result codes of a movement, mirroring the reference's result strings (MujocoController.py:362,376,463) */
enum { GE_MOVE_RUNNING = 0, GE_MOVE_SUCCESS = 1 /* "success" */, GE_MOVE_MAXSTEPS = 2 /* "max. steps reached: n" */,
       GE_MOVE_NO_IK = 3 /* "No valid joint angles received, could not move EE to position." */ };

/* per-environment status bits (ge_get_status); ROW_OVERFLOW: more equality + joint-limit rows than the 16 simple-row slots, the
 * later limit rows were dropped.  Bits 8..15 are the GE_NANCHECK probes. */
enum { GE_STATUS_CONTACT_OVERFLOW = 1, GE_STATUS_NONFINITE = 2, GE_STATUS_SOLVER_MAXITER = 4, GE_STATUS_ROW_OVERFLOW = 8 };

const char* ge_last_error(void);
/* library / build identification: returns e.g. "grasp_engine 0.1 sm_90a fp64" */
const char* ge_version(void);

/* mujoco_py.load_model_from_path + MjSim (MujocoController.py:33-36) + MJ_Controller.create_lists (:136-254):
 * model_blob = compiled scene (mujoco_rl_ur5_b200/model/blob.py), copied to the device; n_envs independent copies of the
 * scene are created at qpos0 with the reference PID gains.  stream: cudaStream_t cast to void* (NULL = default).
 * GE_ERR_MODEL for a scene with more than 256 geoms (the renderer's per-tile geom list), and for a kinematic tree that is not a
 * single free body and has more than 8 dofs (the mass solve gives such a tree one 8-lane group; ge_last_error names the tree).  This
 * check reads the host blob only and fails before any CUDA call.  Engines of one scene with different workspace sizes (e.g.
 * GE_MAXCON) may live side by side. */
int ge_create(const void* model_blob /*[host]*/, size_t nbytes, int n_envs, int device, void* stream, ge_handle* out);
int ge_destroy(ge_handle h);

/* model sizes: what = 0 nq, 1 nv, 2 nbody, 3 ngeom, 4 nu, 5 n_envs, 6 max contacts per env, 7 shared-memory bytes per env,
 * 8 environments per CTA of the sub-step kernel, 9 build (0 warp-per-env, 1 CTA-per-env: scenes whose warp-per-env workspace would
 * exceed 227 KB, e.g. the 40-object scene), 10 hcap = doubles of the Newton Hessian block region in the workspace, 11 hfull =
 * nv (nv + 1) / 2 = doubles of one env's Hessian overflow row in HBM (a Hessian build whose blocks add up to more than hcap goes
 * there), 12 environments of the sub-step kernel resident per SM as granted by the occupancy API, 13 Hessian builds that used the
 * overflow row since ge_create (synchronises the engine's stream; saturates at INT_MAX).  Both builds read GE_HCAP at ge_create (hcap,
 * CTA-per-env build: from Σ tree blocks + 6 maxcon + 64 up to hfull; warp-per-env build: from the larger of Σ tree blocks and
 * 6 maxcon + 6 nbody up to hfull); both also read GE_MAXCON (contact capacity, 16..512; the default hcap and the smallest GE_HCAP
 * follow it).  A value outside its range is ignored, so size 6 / 10 tell what was used.  14 bytes R of one environment state record
 * (ge_snapshot, below). */
int ge_size(ge_handle h, int what);

/* MujocoEnv.set_state + controller re-sync, as GraspEnv.reset_model does (GraspingEnv.py:466-470):
 * qpos [N,nq], qvel [N,nv] (NULL = zeros) [dev, f64]; env_mask [N] u8 (NULL = all) selects which envs are reset.
 * Warm-start is cleared, PID gains return to their initial values, PID set-points := current actuated joint angles. */
int ge_set_state(ge_handle h, const double* qpos, const double* qvel, const uint8_t* env_mask);
/* sim.data.qpos / qvel (MujocoController.py:319, GraspingEnv.py:415-416): copy out to [dev] buffers (either may be NULL) */
int ge_get_state(ge_handle h, double* qpos, double* qvel);
/* sim.data.body_xpos (MujocoController.py:341,488): xpos [N,nbody,3] [dev] after forward kinematics of the current qpos */
int ge_get_body_xpos(ge_handle h, double* xpos);

/* controller.actuators[i][4].Kp = value (GraspingEnv.py:282,347): kp [N] [dev] or NULL with scalar `value` for all envs */
int ge_set_gain(ge_handle h, int actuator, const double* kp, double value);

/* controller.current_target_joint_values / PID set-points for ALL 7 actuators (MujocoController.py:313-316): target [N,7] [dev] */
int ge_set_targets(ge_handle h, const double* target);
/* reads them back: target [N,7] [dev] */
int ge_get_targets(ge_handle h, double* target);

/* MJ_Controller.move_group_to_joint_target (MujocoController.py:269-393) set-up half: group_mask bit i = actuator i in
 * the group; target [N,7] [dev] (entries of non-members ignored; NULL = keep current targets); tolerance/max_steps scalars.
 * env_mask [N] u8 [dev] or NULL.  The movement runs inside ge_run. */
int ge_move_group(ge_handle h, int group_mask, const double* target, double tolerance, int max_steps, const uint8_t* env_mask);
/* MJ_Controller.move_ee (MujocoController.py:446-465): xyz [N,3] [dev]; IK on device then the "Arm" group movement;
 * envs whose IK fails finish immediately with GE_MOVE_NO_IK */
int ge_move_ee(ge_handle h, const double* xyz, double tolerance, int max_steps, const uint8_t* env_mask);
/* MJ_Controller.stay (MujocoController.py:621-637), deterministic: duration_ms/2 sub-steps in chunks of 10 */
int ge_stay(ge_handle h, int duration_ms, const uint8_t* env_mask);
/* GraspEnv.move_and_grasp (GraspingEnv.py:205-386): whole 11-phase attempt on device. coords [N,3] world target from
 * pixel_2_world, rot [N] int32 rotation index 0..5, table_height as GraspEnv.TABLE_HEIGHT (0.91). reward readable after ge_run */
int ge_grasp(ge_handle h, const double* coords, const int32_t* rot, double table_height, const uint8_t* env_mask);

/* Executes the pending movements / programs: the sub-step loop `pid -> sim.step()` (MujocoController.py:318-382).
 * Launches the sub-step kernel in chunks until every env is idle or `max_substeps` sub-steps per env were done
 * (max_substeps <= 0: no limit).  Returns the number of envs still busy in *n_busy (may be NULL). Synchronises the stream. */
int ge_run(ge_handle h, int max_substeps, int* n_busy);
/* one launch of exactly `substeps` sub-step iterations per busy env, no host synchronisation (for benchmarking / graphs) */
int ge_run_async(ge_handle h, int substeps);

/* results of the last movement / program, [N] each [dev], any may be NULL:
 * result (GE_MOVE_*), steps = controller.last_steps (MujocoController.py:827-829), reward u8 = grasped_something,
 * total_substeps int64 = sim.step() calls since creation */
int ge_get_results(ge_handle h, int32_t* result, int32_t* steps, uint8_t* reward, int64_t* total_substeps);
/* per-phase step counts of the last ge_grasp program: info [N,12] int32 [dev] (same layout as the oracle's info[]) */
int ge_get_grasp_info(ge_handle h, int32_t* info);
int ge_get_status(ge_handle h, int32_t* status /*[N] dev*/);
/* busy [N] u8 [dev]: 1 while the env still has a movement or program pending (i.e. ge_run would advance it) */
int ge_get_busy(ge_handle h, uint8_t* busy);

/* MJ_Controller.actuate_joint_group (MujocoController.py:256-267) writes sim.data.ctrl; ge_set_ctrl is that write for all 7
 * actuators: ctrl [N,7] f64 [dev], env_mask [N] u8 [dev] or NULL.  ge_get_ctrl reads sim.data.ctrl back ([N,7] [dev]): after a
 * movement it holds the last PID outputs (MujocoController.py:327). */
int ge_set_ctrl(ge_handle h, const double* ctrl, const uint8_t* env_mask);
int ge_get_ctrl(ge_handle h, double* ctrl);
/* `substeps` bare sim.step() calls (MujocoController.py:379, :611) with the controls as they stand - no PID evaluation, no
 * movement bookkeeping: the open-loop counterpart of ge_run for callers that drive sim.data.ctrl themselves. */
int ge_step_open_loop(ge_handle h, int substeps, const uint8_t* env_mask);

/* MJ_Controller.ik (MujocoController.py:467-517): xyz [N,3] -> q5 [N,5], ok [N] u8 (all [dev]) */
int ge_ik(ge_handle h, const double* xyz, double* q5, uint8_t* ok);
/* MJ_Controller.pixel_2_world (MujocoController.py:783-806): pixel_x, pixel_y [N] int32, depth [N] f32 -> xyz [N,3] f64;
 * GE_ERR_ARG for a camera outside [0, ncam) */
int ge_pixel_2_world(ge_handle h, int cam, int width, int height, const int32_t* px, const int32_t* py, const float* depth, double* xyz);

/* MJ_Controller.get_image_data + depth_2_meters (MujocoController.py:708-740): rgb [N,H,W,3] u8, depth_m [N,H,W] f32 [dev],
 * already flipped U/D + L/R like the reference; depth in metres.  GE_ERR_ARG for a camera outside [0, ncam) and for width or height
 * outside [1, 32767] (the screen-space boxes of the geoms are 16-bit). */
int ge_render(ge_handle h, int cam, int width, int height, uint8_t* rgb, float* depth_m);

/* diagnostics for parity tests: copies one internal per-env field of env `env` to a host buffer after running the
 * forward pipeline once on the current state (no integration).  field: "xpos","xmat","cdof","qM","qfrc_bias",
 * "qacc_smooth","qacc","qfrc_constraint","contact" (16 doubles per contact: dist,pos3,frame9,geom1,geom2,dim), "ncon","niter","nsr",
 * "status" (the status word this forward pass produced, bits as for ge_get_status), "ncand" (broad-phase survivors, counted before
 * the candidate list is cut at 2 x max contacts), "nmpr" (MPR pairs among the kept candidates),
 * "hlayout" (the last Newton Hessian build; nothing when the solve had no constraint rows): [hflag (1: blocks in the HBM overflow row),
 * total block doubles, ntree, then per tree: coupled (0/1), island label (smallest member tree; own index when uncoupled), owner warp
 * (CTA-per-env build, coupled trees; else -1), block offset, rows of its block (tree dofs, or island dofs when coupled)].
 * Returns the number of doubles written (<= cap) or a negative error. */
int ge_debug_forward(ge_handle h, int env, const char* field, double* out /*[host]*/, int cap);

/* counters: kernels launched by this handle since creation, and sub-step kernel launches among them */
int ge_counters(ge_handle h, int64_t* kernel_launches, int64_t* substep_launches);

/* Environment state records: save, restore and copy the whole state of environments, mid-movement or mid-program included.  The
 * reference's counterpart is pickling an MjSim together with its controller and GraspEnv objects; ge_set_state is its reset_model and
 * clears the warm start, the gains and any pending command, so it cannot resume a trajectory.
 *
 * One record per env, R = ge_size(h, 14) bytes, a multiple of 128; records of one call are packed back to back ([n, R]).  Format "GES1",
 * little-endian, offsets in bytes:
 *   0   u32  magic 0x31534547 ("GES1")        4  u32  R        8  u64  model fingerprint = FNV-1a-64 of the model blob bytes
 *   16  f64  qpos[nq], qvel[nv], qaccws[nv] (the Newton warm start), ctl[32] (PID target[8] last_input[8] kp[8] ctrl[8]),
 *            cmd_tol, prog_coords[3], prog_table
 *   then i64 substeps (sim.step() calls since creation: the env's clock, MuJoCo's `time`)
 *   then i32 cmd_active, cmd_mask, cmd_maxsteps, cmd_steps, cmd_result, prog_phase, prog_rot, prog_grasp, prog_aux, prog_info[12],
 *            status, reward (u8 widened), then zeros up to R.
 * Not part of a record, on purpose:
 *   - the scheduling words of the sub-step kernel (lock, owed, done, ticket) and ge_run's busy counter: they belong to one launch.  Between
 *     launches every lock and owed count is 0, done is reset at the start of each launch and ticket only orders the tasks of a launch
 *     (relative to a base the host keeps), so they carry nothing about an env from one call to the next;
 *   - the Hessian overflow rows and the workspace flag that says a build uses them: scratch of one Newton Hessian build, written before
 *     they are read within that build;
 *   - the engine's count of builds that used the overflow row (ge_size 13): a statistic of the engine, not of an environment.
 * A record does not depend on the workspace layout, so it restores across GE_MAXCON / GE_HCAP settings and both library builds of one
 * scene; it does depend on the model (fingerprint) and is refused by an engine of another scene.
 *
 * ge_snapshot: record i <- env envs[i] (envs [n] int32 [dev], or NULL for envs 0..N-1 with n = N); rec [n, R] [dev].  An index outside
 * [0, N) gives an all-zero record, which ge_restore refuses.  Stream-ordered, no synchronisation.
 * ge_restore: env e <- record row[e] of rec [n_rec, R] [dev] (row [N] int32 [dev]; -1 leaves env e alone; NULL = record e for env e).  A
 * gather, so no env is written twice.  Checks every row and every record a row selects, synchronises the stream once, and returns
 * GE_ERR_ARG (a row outside [-1, n_rec)) or GE_ERR_STATE (wrong magic, R or fingerprint) before writing anything: an engine that refuses
 * a call is left bit for bit as it was.  A restored env continues exactly where the saved one stood, busy or not, with its saved substeps.
 * ge_clone: env e <- the state env src[e] had before the call (src [N] int32 [dev], -1 = keep), so overlapping and permuting maps are
 * fine.  Goes through an engine-owned scratch of N records (allocated at the first call, freed by ge_destroy); refuses like ge_restore. */
int ge_snapshot(ge_handle h, const int32_t* envs, int n, void* rec);
int ge_restore(ge_handle h, const void* rec, int n_rec, const int32_t* row);
int ge_clone(ge_handle h, const int32_t* src);

#ifdef __cplusplus
}
#endif
#endif
