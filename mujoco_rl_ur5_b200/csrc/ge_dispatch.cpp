// libgrasp_engine.so — the public C-ABI of include/grasp_engine.h.  The engine source (grasp_engine.cu) is compiled twice
// (ge_variant.h): "smem" keeps each environment's workspace in shared memory, "hbm" keeps it in HBM rows for scenes that do not
// fit (the reference's default 40-object scene).  ge_create picks the variant; every other call forwards through the handle.
#include <stdlib.h>

#include "../../include/grasp_engine.h"

#define GE_ERR_TOO_LARGE (-100)
typedef void* vh;
#define DECL(suffix)                                                                                                               \
  extern "C" {                                                                                                                     \
  const char* ge_last_error_##suffix(void);                                                                                        \
  const char* ge_version_##suffix(void);                                                                                           \
  int ge_create_##suffix(const void*, size_t, int, int, void*, vh*);                                                               \
  int ge_destroy_##suffix(vh);                                                                                                     \
  int ge_size_##suffix(vh, int);                                                                                                   \
  int ge_set_state_##suffix(vh, const double*, const double*, const uint8_t*);                                                     \
  int ge_get_state_##suffix(vh, double*, double*);                                                                                 \
  int ge_get_body_xpos_##suffix(vh, double*);                                                                                      \
  int ge_set_gain_##suffix(vh, int, const double*, double);                                                                        \
  int ge_set_targets_##suffix(vh, const double*);                                                                                  \
  int ge_get_targets_##suffix(vh, double*);                                                                                        \
  int ge_move_group_##suffix(vh, int, const double*, double, int, const uint8_t*);                                                 \
  int ge_move_ee_##suffix(vh, const double*, double, int, const uint8_t*);                                                         \
  int ge_stay_##suffix(vh, int, const uint8_t*);                                                                                   \
  int ge_grasp_##suffix(vh, const double*, const int32_t*, double, const uint8_t*);                                                \
  int ge_run_##suffix(vh, int, int*);                                                                                              \
  int ge_run_async_##suffix(vh, int);                                                                                              \
  int ge_get_results_##suffix(vh, int32_t*, int32_t*, uint8_t*, int64_t*);                                                         \
  int ge_get_grasp_info_##suffix(vh, int32_t*);                                                                                    \
  int ge_get_status_##suffix(vh, int32_t*);                                                                                        \
  int ge_get_busy_##suffix(vh, uint8_t*);                                                                                          \
  int ge_set_ctrl_##suffix(vh, const double*, const uint8_t*);                                                                     \
  int ge_get_ctrl_##suffix(vh, double*);                                                                                           \
  int ge_step_open_loop_##suffix(vh, int, const uint8_t*);                                                                         \
  int ge_ik_##suffix(vh, const double*, double*, uint8_t*);                                                                        \
  int ge_pixel_2_world_##suffix(vh, int, int, int, const int32_t*, const int32_t*, const float*, double*);                         \
  int ge_render_##suffix(vh, int, int, int, uint8_t*, float*);                                                                     \
  int ge_debug_forward_##suffix(vh, int, const char*, double*, int);                                                               \
  int ge_counters_##suffix(vh, int64_t*, int64_t*);                                                                                \
  }
DECL(smem)
DECL(hbm)

struct ge_engine { int variant; vh h; };
static thread_local int g_last_variant = 0;

#define FWD(call_smem, call_hbm) (g_last_variant = h->variant, h->variant ? (call_hbm) : (call_smem))
#define CHECK_H if (!h) return GE_ERR_ARG

extern "C" {

const char* ge_last_error(void) { return g_last_variant ? ge_last_error_hbm() : ge_last_error_smem(); }
const char* ge_version(void) { return "grasp_engine 0.2 sm_90a fp64 warp-per-env (variants: shared-memory workspace, HBM workspace)"; }

int ge_create(const void* blob, size_t nbytes, int n_envs, int device, void* stream, ge_handle* out) {
  if (!out) return GE_ERR_ARG;
  vh h = nullptr;
  int variant = 0, r = GE_ERR_TOO_LARGE;
  const char* ev = getenv("GE_WS_GLOBAL");  // =1 forces the HBM-workspace variant (tests cover that path with the small scene)
  if (!(ev && atoi(ev) != 0)) r = ge_create_smem(blob, nbytes, n_envs, device, stream, &h);
  if (r == GE_ERR_TOO_LARGE) { variant = 1; r = ge_create_hbm(blob, nbytes, n_envs, device, stream, &h); }
  g_last_variant = variant;
  if (r != GE_OK) return r;
  ge_engine* e = new ge_engine{variant, h};
  *out = e;
  return GE_OK;
}
int ge_destroy(ge_handle h) {
  if (!h) return GE_OK;
  int r = FWD(ge_destroy_smem(h->h), ge_destroy_hbm(h->h));
  delete h;
  return r;
}
int ge_size(ge_handle h, int what) { CHECK_H; return FWD(ge_size_smem(h->h, what), ge_size_hbm(h->h, what)); }
int ge_set_state(ge_handle h, const double* qpos, const double* qvel, const uint8_t* m) { CHECK_H; return FWD(ge_set_state_smem(h->h, qpos, qvel, m), ge_set_state_hbm(h->h, qpos, qvel, m)); }
int ge_get_state(ge_handle h, double* qpos, double* qvel) { CHECK_H; return FWD(ge_get_state_smem(h->h, qpos, qvel), ge_get_state_hbm(h->h, qpos, qvel)); }
int ge_get_body_xpos(ge_handle h, double* x) { CHECK_H; return FWD(ge_get_body_xpos_smem(h->h, x), ge_get_body_xpos_hbm(h->h, x)); }
int ge_set_gain(ge_handle h, int a, const double* kp, double v) { CHECK_H; return FWD(ge_set_gain_smem(h->h, a, kp, v), ge_set_gain_hbm(h->h, a, kp, v)); }
int ge_set_targets(ge_handle h, const double* t) { CHECK_H; return FWD(ge_set_targets_smem(h->h, t), ge_set_targets_hbm(h->h, t)); }
int ge_get_targets(ge_handle h, double* t) { CHECK_H; return FWD(ge_get_targets_smem(h->h, t), ge_get_targets_hbm(h->h, t)); }
int ge_move_group(ge_handle h, int g, const double* t, double tol, int ms, const uint8_t* m) { CHECK_H; return FWD(ge_move_group_smem(h->h, g, t, tol, ms, m), ge_move_group_hbm(h->h, g, t, tol, ms, m)); }
int ge_move_ee(ge_handle h, const double* x, double tol, int ms, const uint8_t* m) { CHECK_H; return FWD(ge_move_ee_smem(h->h, x, tol, ms, m), ge_move_ee_hbm(h->h, x, tol, ms, m)); }
int ge_stay(ge_handle h, int d, const uint8_t* m) { CHECK_H; return FWD(ge_stay_smem(h->h, d, m), ge_stay_hbm(h->h, d, m)); }
int ge_grasp(ge_handle h, const double* c, const int32_t* rot, double th, const uint8_t* m) { CHECK_H; return FWD(ge_grasp_smem(h->h, c, rot, th, m), ge_grasp_hbm(h->h, c, rot, th, m)); }
int ge_run(ge_handle h, int ms, int* nb) { CHECK_H; return FWD(ge_run_smem(h->h, ms, nb), ge_run_hbm(h->h, ms, nb)); }
int ge_run_async(ge_handle h, int n) { CHECK_H; return FWD(ge_run_async_smem(h->h, n), ge_run_async_hbm(h->h, n)); }
int ge_get_results(ge_handle h, int32_t* r, int32_t* s, uint8_t* rw, int64_t* t) { CHECK_H; return FWD(ge_get_results_smem(h->h, r, s, rw, t), ge_get_results_hbm(h->h, r, s, rw, t)); }
int ge_get_grasp_info(ge_handle h, int32_t* i) { CHECK_H; return FWD(ge_get_grasp_info_smem(h->h, i), ge_get_grasp_info_hbm(h->h, i)); }
int ge_get_status(ge_handle h, int32_t* s) { CHECK_H; return FWD(ge_get_status_smem(h->h, s), ge_get_status_hbm(h->h, s)); }
int ge_get_busy(ge_handle h, uint8_t* b) { CHECK_H; return FWD(ge_get_busy_smem(h->h, b), ge_get_busy_hbm(h->h, b)); }
int ge_set_ctrl(ge_handle h, const double* c, const uint8_t* m) { CHECK_H; return FWD(ge_set_ctrl_smem(h->h, c, m), ge_set_ctrl_hbm(h->h, c, m)); }
int ge_get_ctrl(ge_handle h, double* c) { CHECK_H; return FWD(ge_get_ctrl_smem(h->h, c), ge_get_ctrl_hbm(h->h, c)); }
int ge_step_open_loop(ge_handle h, int n, const uint8_t* m) { CHECK_H; return FWD(ge_step_open_loop_smem(h->h, n, m), ge_step_open_loop_hbm(h->h, n, m)); }
int ge_ik(ge_handle h, const double* x, double* q, uint8_t* ok) { CHECK_H; return FWD(ge_ik_smem(h->h, x, q, ok), ge_ik_hbm(h->h, x, q, ok)); }
int ge_pixel_2_world(ge_handle h, int cam, int w, int hh, const int32_t* px, const int32_t* py, const float* d, double* xyz) {
  CHECK_H;
  return FWD(ge_pixel_2_world_smem(h->h, cam, w, hh, px, py, d, xyz), ge_pixel_2_world_hbm(h->h, cam, w, hh, px, py, d, xyz));
}
int ge_render(ge_handle h, int cam, int w, int hh, uint8_t* rgb, float* d) { CHECK_H; return FWD(ge_render_smem(h->h, cam, w, hh, rgb, d), ge_render_hbm(h->h, cam, w, hh, rgb, d)); }
int ge_debug_forward(ge_handle h, int env, const char* f, double* out, int cap) { CHECK_H; return FWD(ge_debug_forward_smem(h->h, env, f, out, cap), ge_debug_forward_hbm(h->h, env, f, out, cap)); }
int ge_counters(ge_handle h, int64_t* a, int64_t* b) { CHECK_H; return FWD(ge_counters_smem(h->h, a, b), ge_counters_hbm(h->h, a, b)); }

}  // extern "C"
