#!/bin/bash
# Experimental builds of the engine library with a different number of lanes per environment in the big-scene variant
# (ge_variant.h: GE_BIG_LANES); V0FLAGS=-DGE_V0_CAP_REGS builds the warp-per-env variant with the old 128-register budget.  Output: exp_libs/libgrasp_engine_l<lanes>.so (git-ignored; travels with gpurun); use with GE_LIB=<path>.
set -e
cd "$(dirname "$0")/.."
CS=mujoco_rl_ur5_b200/csrc
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -diag-suppress 550"
mkdir -p exp_libs/obj
for L in "$@"; do
  nvcc $FLAGS -DGE_VARIANT=0 $V0FLAGS -c -o exp_libs/obj/v0.o $CS/grasp_engine.cu &
  nvcc $FLAGS -DGE_VARIANT=1 -DGE_BIG_LANES=$L $V1FLAGS -c -o exp_libs/obj/v1_$L.o $CS/grasp_engine.cu &
  nvcc $FLAGS -x cu -c -o exp_libs/obj/d.o $CS/ge_dispatch.cpp &
  wait
  nvcc -gencode arch=compute_90a,code=sm_90a -shared -o exp_libs/libgrasp_engine_l$L.so exp_libs/obj/v0.o exp_libs/obj/v1_$L.o exp_libs/obj/d.o
  echo built exp_libs/libgrasp_engine_l$L.so
done
