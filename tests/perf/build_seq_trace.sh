#!/bin/bash
# builds tests/perf/seq_trace[_variant] binaries: $1 = suffix, rest = extra nvcc flags
suf=$1; shift
nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -I include "$@" -o tests/perf/seq_trace$suf tests/perf/seq_trace.cu squeezellm_b200/csrc/*.cu 2>&1 | grep -i "error" 
