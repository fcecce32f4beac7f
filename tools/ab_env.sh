#!/bin/bash
# tools/ab_env.sh VAR "v1 v2 ..." [bench args] — on the GPU box: the bench workload (c2 and c3 maps) under each value of an
# environment switch of the library (e.g. DTS_BIN_WARPS), per-kernel times from the bench line
cd "$(dirname "$0")/.."
export DTS_NO_REBUILD=1
var=$1; vals=$2; shift 2
for v in $vals; do
  for m in small_loop loop_obstacles; do
    env $var=$v python bench.py --no-cpu-baseline --configs none --steps 20 --warmup 5 --map $m "$@" 2>>"${TMPDIR:-/tmp}/ab_err.log" | tail -1 | python -c "
import json,sys
d=json.loads(sys.stdin.read()); k=d['kernel_ms']
print('$var=$v $m', round(d['value']), 'env-steps/s', ' '.join(f'{n}={v*1000:.0f}us' for n,v in k.items()))"
  done
done
