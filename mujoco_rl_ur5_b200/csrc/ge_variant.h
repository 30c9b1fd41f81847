// Two builds of the same engine source live in libgrasp_engine.so, selected per scene by ge_dispatch.cpp:
//   variant 0 "smem": the per-env workspace is a slice of the CTA's shared memory.  Every workspace pointer provably derives
//                     from the shared window, so the compiler emits LDS/STS in all stage functions (13 % fewer instructions
//                     than generic loads, measured r01);
//   variant 1 "hbm":  one workspace row per env in HBM (L1/L2-cached) for scenes whose workspace exceeds 227 KB (the 40-object
//                     scene: the packed Newton Hessian alone is 247 KB).
// The variant's namespace and its C entry points get a suffix; the public names of include/grasp_engine.h are the dispatcher's.
#pragma once
#ifndef GE_VARIANT
#define GE_VARIANT 0
#endif
#if GE_VARIANT == 0
#define ge ge_smem
#define GE_API(n) n##_smem
#define GE_WS_IN_HBM 0
#define GE_LANES 32   // threads that cooperate on one environment: one warp
#else
#define ge ge_hbm
#define GE_API(n) n##_hbm
#define GE_WS_IN_HBM 0  // (r02: the big-scene build keeps its workspace in shared memory too; only oversized Hessian builds overflow to HBM)
// r02: the big-scene variant gives every environment a whole CTA of 4 warps.  The stage code is the same source: lane loops stride
// by GE_LANES, `gsync()` is __syncthreads(), reductions go through shared memory, and the pieces that are inherently warp-shaped
// (MPR on one geom pair, the 8-lane tree groups, one dense island factorisation) are dealt out to the 4 warps.
#ifndef GE_BIG_LANES
#define GE_BIG_LANES 128  // (-DGE_BIG_LANES=64 / 256: experiments with 2 / 8 warps per environment, tools/build_exp_libs.sh)
#endif
#define GE_LANES GE_BIG_LANES
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
