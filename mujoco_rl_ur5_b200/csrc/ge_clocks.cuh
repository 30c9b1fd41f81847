// Per-stage cycle profile of the sub-step kernel (-DGE_STAGE_CLOCKS; tools/build_profile_libs.sh, tools/k_run_stage_profile.py).
// Thread 0 of every environment group keeps, per warp slot (CTA x warp of the grid), the clock64() value of its last mark;
// GE_CLK(stage) charges the cycles since that mark to `stage` and starts the next interval.  Every cycle of k_run therefore lands in
// exactly one stage.  The counters belong to k_run alone: it arms its slot on entry (GE_CLK_START) and disarms it on exit
// (GE_CLK_STOP), and a mark on a disarmed slot counts nothing, so the other kernels that share the stage code (k_step_open, k_debug)
// leave the profile alone.  With -DGE_STAGE_WARM the pure stages (stage_fk, stage_rne + stage_crb, mul_M) are run a second time right
// after the first pass, on unchanged inputs; that pass is charged to its own WARM_* slot, so cold minus warm is what fetching the
// stage's code (and its first touch of the model constants) costs.  Both are off in the product build, where the macros are empty.
#pragma once

namespace ge {

// The Newton Hessian build is split into its four parts: per-tree bookkeeping (coupling, contact membership, islands, block offsets),
// the rows of M, the accumulation of the uncoupled trees' blocks and that of the island blocks.  SC_HESS_BUILDS / SC_HESS_COUPLED
// count the builds, and those with at least one coupled tree (the island path).
enum StageClock {
  SC_PID, SC_FK, SC_COLLISION, SC_MPR, SC_RNE_CRB, SC_MASS, SC_CONSTRAINTS, SC_NEWTON, SC_HESS_LISTS, SC_HESS_MROWS, SC_HESS_TREES,
  SC_HESS_ISLANDS, SC_CHOL, SC_LINESEARCH, SC_NT_UPDATE, SC_EULER, SC_SCHED, SC_BARRIER, SC_SUBSTEPS, SC_WARM_FK, SC_WARM_RNE_CRB,
  SC_WARM_MULM, SC_MULM_COLD, SC_HESS_BUILDS, SC_HESS_COUPLED, SC_NUM
};
#define GE_CLK_SLOTS 4096

#ifdef GE_STAGE_CLOCKS
__device__ unsigned long long g_stage_clk[GE_CLK_SLOTS][SC_NUM];
__device__ long long g_stage_last[GE_CLK_SLOTS];
__device__ __forceinline__ int clk_slot() { return (blockIdx.x * blockDim.y + threadIdx.y) % GE_CLK_SLOTS; }
__device__ __forceinline__ void clk_mark(int stage) {
  const int s = clk_slot();
  if (threadIdx.x == 0 && g_stage_last[s] != 0) {  // 0: slot not armed by k_run
    const long long now = clock64();
    g_stage_clk[s][stage] += now - g_stage_last[s];
    g_stage_last[s] = now;
  }
}
__device__ __forceinline__ void clk_start() { if (threadIdx.x == 0) g_stage_last[clk_slot()] = clock64(); }
__device__ __forceinline__ void clk_stop() { if (threadIdx.x == 0) g_stage_last[clk_slot()] = 0; }
__device__ __forceinline__ void clk_count(int stage) { const int s = clk_slot(); if (threadIdx.x == 0 && g_stage_last[s] != 0) g_stage_clk[s][stage]++; }
#define GE_CLK(stage) clk_mark(stage)
#define GE_CLK_START() clk_start()
#define GE_CLK_STOP() clk_stop()
#define GE_CLK_COUNT(stage) clk_count(stage)
#else
#define GE_CLK(stage) ((void)0)
#define GE_CLK_START() ((void)0)
#define GE_CLK_STOP() ((void)0)
#define GE_CLK_COUNT(stage) ((void)0)
#endif

// GE_WARM(cold, warm, code): charge the interval just ended (the first pass) to `cold`, run `code` again and charge it to `warm`
#if defined(GE_STAGE_CLOCKS) && defined(GE_STAGE_WARM)
#define GE_WARM(cold, warm, ...) do { GE_CLK(cold); __VA_ARGS__; GE_CLK(warm); } while (0)
#else
#define GE_WARM(cold, warm, ...) ((void)0)
#endif

}  // namespace ge
