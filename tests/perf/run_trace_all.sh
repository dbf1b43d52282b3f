#!/bin/bash
# full per-CTA timelines (every CTA) of one steady-state launch, exact and fp16, the four 7B shapes, with outliers
# (tests/perf/trace_harness: the -DSQLLM_TRACE build that its header describes)
for sh in "4096 12288" "4096 4096" "11008 4096" "4096 22016"; do
  for mode in exact fp16; do
    echo "=== $sh $mode"
    TRACE_ALL=1 SQLLM_LUT_MODE=$mode timeout 120 ./tests/perf/trace_harness 4 $sh 16 1 2 2>&1 | awk '/per-CTA/{p=1} p||NR==1'
  done
done
