// libgrasp_engine.so — the public C-ABI of include/grasp_engine.h.  The engine source (grasp_engine.cu) is compiled twice
// (ge_variant.h): "warp" runs one environment per warp, "cta" one environment per CTA of 4 warps for scenes whose workspace the
// warp-per-env build cannot hold (the reference's default 40-object scene).  ge_create picks the variant; every other call forwards
// through the handle.
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
  int ge_snapshot_##suffix(vh, const int32_t*, int, void*);                                                                        \
  int ge_restore_##suffix(vh, const void*, int, const int32_t*);                                                                   \
  int ge_clone_##suffix(vh, const int32_t*);                                                                                       \
  }
DECL(warp)
DECL(cta)

struct ge_engine { int variant; vh h; };
static thread_local int g_last_variant = 0;

#define FWD(call_warp, call_cta) (g_last_variant = h->variant, h->variant ? (call_cta) : (call_warp))
#define CHECK_H if (!h) return GE_ERR_ARG

extern "C" {

const char* ge_last_error(void) { return g_last_variant ? ge_last_error_cta() : ge_last_error_warp(); }
const char* ge_version(void) { return "grasp_engine 0.3 sm_90a fp64 (builds: warp-per-env, CTA-per-env)"; }

int ge_create(const void* blob, size_t nbytes, int n_envs, int device, void* stream, ge_handle* out) {
  if (!out) return GE_ERR_ARG;
  vh h = nullptr;
  int variant = 0, r = GE_ERR_TOO_LARGE;
  const char* ev = getenv("GE_CTA_PER_ENV");  // =1 forces the CTA-per-env variant (tests cover that path with the small scene)
  if (!(ev && atoi(ev) != 0)) r = ge_create_warp(blob, nbytes, n_envs, device, stream, &h);
  if (r == GE_ERR_TOO_LARGE) { variant = 1; r = ge_create_cta(blob, nbytes, n_envs, device, stream, &h); }
  g_last_variant = variant;
  if (r != GE_OK) return r;
  ge_engine* e = new ge_engine{variant, h};
  *out = e;
  return GE_OK;
}
int ge_destroy(ge_handle h) {
  if (!h) return GE_OK;
  int r = FWD(ge_destroy_warp(h->h), ge_destroy_cta(h->h));
  delete h;
  return r;
}
int ge_size(ge_handle h, int what) { CHECK_H; return FWD(ge_size_warp(h->h, what), ge_size_cta(h->h, what)); }
int ge_set_state(ge_handle h, const double* qpos, const double* qvel, const uint8_t* m) { CHECK_H; return FWD(ge_set_state_warp(h->h, qpos, qvel, m), ge_set_state_cta(h->h, qpos, qvel, m)); }
int ge_get_state(ge_handle h, double* qpos, double* qvel) { CHECK_H; return FWD(ge_get_state_warp(h->h, qpos, qvel), ge_get_state_cta(h->h, qpos, qvel)); }
int ge_get_body_xpos(ge_handle h, double* x) { CHECK_H; return FWD(ge_get_body_xpos_warp(h->h, x), ge_get_body_xpos_cta(h->h, x)); }
int ge_set_gain(ge_handle h, int a, const double* kp, double v) { CHECK_H; return FWD(ge_set_gain_warp(h->h, a, kp, v), ge_set_gain_cta(h->h, a, kp, v)); }
int ge_set_targets(ge_handle h, const double* t) { CHECK_H; return FWD(ge_set_targets_warp(h->h, t), ge_set_targets_cta(h->h, t)); }
int ge_get_targets(ge_handle h, double* t) { CHECK_H; return FWD(ge_get_targets_warp(h->h, t), ge_get_targets_cta(h->h, t)); }
int ge_move_group(ge_handle h, int g, const double* t, double tol, int ms, const uint8_t* m) { CHECK_H; return FWD(ge_move_group_warp(h->h, g, t, tol, ms, m), ge_move_group_cta(h->h, g, t, tol, ms, m)); }
int ge_move_ee(ge_handle h, const double* x, double tol, int ms, const uint8_t* m) { CHECK_H; return FWD(ge_move_ee_warp(h->h, x, tol, ms, m), ge_move_ee_cta(h->h, x, tol, ms, m)); }
int ge_stay(ge_handle h, int d, const uint8_t* m) { CHECK_H; return FWD(ge_stay_warp(h->h, d, m), ge_stay_cta(h->h, d, m)); }
int ge_grasp(ge_handle h, const double* c, const int32_t* rot, double th, const uint8_t* m) { CHECK_H; return FWD(ge_grasp_warp(h->h, c, rot, th, m), ge_grasp_cta(h->h, c, rot, th, m)); }
int ge_run(ge_handle h, int ms, int* nb) { CHECK_H; return FWD(ge_run_warp(h->h, ms, nb), ge_run_cta(h->h, ms, nb)); }
int ge_run_async(ge_handle h, int n) { CHECK_H; return FWD(ge_run_async_warp(h->h, n), ge_run_async_cta(h->h, n)); }
int ge_get_results(ge_handle h, int32_t* r, int32_t* s, uint8_t* rw, int64_t* t) { CHECK_H; return FWD(ge_get_results_warp(h->h, r, s, rw, t), ge_get_results_cta(h->h, r, s, rw, t)); }
int ge_get_grasp_info(ge_handle h, int32_t* i) { CHECK_H; return FWD(ge_get_grasp_info_warp(h->h, i), ge_get_grasp_info_cta(h->h, i)); }
int ge_get_status(ge_handle h, int32_t* s) { CHECK_H; return FWD(ge_get_status_warp(h->h, s), ge_get_status_cta(h->h, s)); }
int ge_get_busy(ge_handle h, uint8_t* b) { CHECK_H; return FWD(ge_get_busy_warp(h->h, b), ge_get_busy_cta(h->h, b)); }
int ge_set_ctrl(ge_handle h, const double* c, const uint8_t* m) { CHECK_H; return FWD(ge_set_ctrl_warp(h->h, c, m), ge_set_ctrl_cta(h->h, c, m)); }
int ge_get_ctrl(ge_handle h, double* c) { CHECK_H; return FWD(ge_get_ctrl_warp(h->h, c), ge_get_ctrl_cta(h->h, c)); }
int ge_step_open_loop(ge_handle h, int n, const uint8_t* m) { CHECK_H; return FWD(ge_step_open_loop_warp(h->h, n, m), ge_step_open_loop_cta(h->h, n, m)); }
int ge_ik(ge_handle h, const double* x, double* q, uint8_t* ok) { CHECK_H; return FWD(ge_ik_warp(h->h, x, q, ok), ge_ik_cta(h->h, x, q, ok)); }
int ge_pixel_2_world(ge_handle h, int cam, int w, int hh, const int32_t* px, const int32_t* py, const float* d, double* xyz) {
  CHECK_H;
  return FWD(ge_pixel_2_world_warp(h->h, cam, w, hh, px, py, d, xyz), ge_pixel_2_world_cta(h->h, cam, w, hh, px, py, d, xyz));
}
int ge_render(ge_handle h, int cam, int w, int hh, uint8_t* rgb, float* d) { CHECK_H; return FWD(ge_render_warp(h->h, cam, w, hh, rgb, d), ge_render_cta(h->h, cam, w, hh, rgb, d)); }
int ge_debug_forward(ge_handle h, int env, const char* f, double* out, int cap) { CHECK_H; return FWD(ge_debug_forward_warp(h->h, env, f, out, cap), ge_debug_forward_cta(h->h, env, f, out, cap)); }
int ge_counters(ge_handle h, int64_t* a, int64_t* b) { CHECK_H; return FWD(ge_counters_warp(h->h, a, b), ge_counters_cta(h->h, a, b)); }
int ge_snapshot(ge_handle h, const int32_t* e, int n, void* r) { CHECK_H; return FWD(ge_snapshot_warp(h->h, e, n, r), ge_snapshot_cta(h->h, e, n, r)); }
int ge_restore(ge_handle h, const void* r, int n, const int32_t* row) { CHECK_H; return FWD(ge_restore_warp(h->h, r, n, row), ge_restore_cta(h->h, r, n, row)); }
int ge_clone(ge_handle h, const int32_t* src) { CHECK_H; return FWD(ge_clone_warp(h->h, src), ge_clone_cta(h->h, src)); }

}  // extern "C"
