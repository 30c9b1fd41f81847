#!/bin/bash
# Profile builds of the engine library (ge_clocks.cuh) into the git-ignored exp_libs/, selected with GE_LIB=<path>:
#   exp_libs/libgrasp_engine_<tag>_clk.so    per-stage clock64() counters of k_run (-DGE_STAGE_CLOCKS)
#   exp_libs/libgrasp_engine_<tag>_warm.so   the same, plus a second (warm) pass of the pure stages (-DGE_STAGE_WARM)
#   exp_libs/libgrasp_engine_<tag>.so        the product build of the same source (no counters)
# usage: tools/build_profile_libs.sh TAG [SOURCE_ROOT]   (SOURCE_ROOT: a checkout holding mujoco_rl_ur5_b200/csrc; default this one)
set -e
cd "$(dirname "$0")/.."
TAG=${1:?tag}
SRC=${2:-.}
CS=$SRC/mujoco_rl_ur5_b200/csrc
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -diag-suppress 550"
O=exp_libs/obj/$TAG
mkdir -p $O
build() {  # name extra-flags
  rm -f $O/v0$1.o $O/v1$1.o $O/d$1.o  # a failed compile must not leave an older object to link
  nvcc $FLAGS -DGE_VARIANT=0 $2 -c -o $O/v0$1.o $CS/grasp_engine.cu & p0=$!
  nvcc $FLAGS -DGE_VARIANT=1 $2 -c -o $O/v1$1.o $CS/grasp_engine.cu & p1=$!
  nvcc $FLAGS -x cu -c -o $O/d$1.o $CS/ge_dispatch.cpp & p2=$!
  wait $p0 && wait $p1 && wait $p2 || { echo "nvcc failed for exp_libs/libgrasp_engine_$TAG$1.so" >&2; exit 1; }
  nvcc -gencode arch=compute_90a,code=sm_90a -shared -o exp_libs/libgrasp_engine_$TAG$1.so $O/v0$1.o $O/v1$1.o $O/d$1.o
  echo built exp_libs/libgrasp_engine_$TAG$1.so
}
build "" ""
build _clk "-DGE_STAGE_CLOCKS"
build _warm "-DGE_STAGE_CLOCKS -DGE_STAGE_WARM"
