#!/bin/bash
# builds trace_harness binaries of lutgemv_kernels.cu with different compile-time knobs (run from the repo root)
set -e
B="nvcc -O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -I include tests/perf/trace_harness.cu squeezellm_b200/csrc/lutgemv_kernels.cu"
build() { name=$1; shift; echo "== $name $*"; $B "$@" -Xptxas=-v -o tests/perf/th_$name 2>&1 | grep -E "lutgemv_kernelILi4ELb1|registers|spill" | grep -A2 "ILi4ELb1" | grep -E "registers|spill" | head -3; }
build base
build tma14 -DSQLLM_LDG=0 -DSQLLM_NW=14 -DSQLLM_MINB4=2 -DSQLLM_MINB3=2
build cpa14 -DSQLLM_LDG=2 -DSQLLM_NW=14 -DSQLLM_MINB4=2 -DSQLLM_MINB3=2
build ldg14 -DSQLLM_LDG=1 -DSQLLM_NW=14 -DSQLLM_MINB4=2 -DSQLLM_MINB3=2 -DSQLLM_PF4=6
build cpa16 -DSQLLM_LDG=2 -DSQLLM_NW=16 -DSQLLM_MINB4=1 -DSQLLM_MINB3=1 -DSQLLM_PF4=12
build tma22 -DSQLLM_LDG=0 -DSQLLM_NW=22 -DSQLLM_MINB4=1 -DSQLLM_MINB3=1
build ldg22 -DSQLLM_LDG=1 -DSQLLM_NW=22 -DSQLLM_MINB4=1 -DSQLLM_MINB3=1 -DSQLLM_PF4=8
