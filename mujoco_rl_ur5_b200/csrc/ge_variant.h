// Two builds of the same engine source live in libgrasp_engine.so, selected per scene by ge_dispatch.cpp.  Both keep each
// environment's workspace in shared memory (every workspace pointer provably derives from the shared window, so the compiler emits
// LDS/STS in all stage functions: 13 % fewer instructions than generic loads, measured r01):
//   variant 0 "warp": one warp per environment, up to ten environments per SM;
//   variant 1 "cta":  a whole CTA of 4 warps per environment, for scenes that variant 0 cannot hold in 227 KB per environment (the
//                     40-object scene: the packed Newton Hessian alone is 247 KB).  The stage code is the same source: lane loops
//                     stride by GE_LANES, `gsync()` is __syncthreads(), reductions go through shared memory, and the pieces that are
//                     inherently warp-shaped (MPR on one geom pair, the 8-lane tree groups, one dense island factorisation) are dealt
//                     out to the 4 warps.
// The variant's namespace and its C entry points get a suffix; the public names of include/grasp_engine.h are the dispatcher's.
#pragma once
#ifndef GE_VARIANT
#define GE_VARIANT 0
#endif
#if GE_VARIANT == 0
#define ge ge_warp
#define GE_API(n) n##_warp
#define GE_LANES 32   // threads that cooperate on one environment: one warp
#else
#define ge ge_cta
#define GE_API(n) n##_cta
#define GE_LANES 128  // threads that cooperate on one environment: one CTA of 4 warps
#endif
#define GE_NW (GE_LANES / 32)
#define GE_ERR_TOO_LARGE (-100)  // internal: variant 0 cannot hold the scene, the dispatcher then creates variant 1

#define ge_last_error GE_API(ge_last_error)
#define ge_version GE_API(ge_version)
#define ge_create GE_API(ge_create)
#define ge_destroy GE_API(ge_destroy)
#define ge_size GE_API(ge_size)
#define ge_set_state GE_API(ge_set_state)
#define ge_get_state GE_API(ge_get_state)
#define ge_get_body_xpos GE_API(ge_get_body_xpos)
#define ge_set_gain GE_API(ge_set_gain)
#define ge_set_targets GE_API(ge_set_targets)
#define ge_get_targets GE_API(ge_get_targets)
#define ge_move_group GE_API(ge_move_group)
#define ge_move_ee GE_API(ge_move_ee)
#define ge_stay GE_API(ge_stay)
#define ge_grasp GE_API(ge_grasp)
#define ge_run GE_API(ge_run)
#define ge_run_async GE_API(ge_run_async)
#define ge_get_results GE_API(ge_get_results)
#define ge_get_grasp_info GE_API(ge_get_grasp_info)
#define ge_get_status GE_API(ge_get_status)
#define ge_get_busy GE_API(ge_get_busy)
#define ge_set_ctrl GE_API(ge_set_ctrl)
#define ge_get_ctrl GE_API(ge_get_ctrl)
#define ge_step_open_loop GE_API(ge_step_open_loop)
#define ge_ik GE_API(ge_ik)
#define ge_pixel_2_world GE_API(ge_pixel_2_world)
#define ge_render GE_API(ge_render)
#define ge_debug_forward GE_API(ge_debug_forward)
#define ge_counters GE_API(ge_counters)
#define ge_snapshot GE_API(ge_snapshot)
#define ge_restore GE_API(ge_restore)
#define ge_clone GE_API(ge_clone)
#define ge_engine GE_API(ge_engine)
