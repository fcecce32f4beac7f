#!/bin/bash
# tools/ab_all.sh [bench args] — on the GPU box: time every gym-duckietown_b200/variants/libdtsim_*.so on the bench workload
cd "$(dirname "$0")/.."
export DTS_NO_REBUILD=1
cp gym-duckietown_b200/libdtsim.so /tmp/libdtsim_keep.so
for v in gym-duckietown_b200/variants/libdtsim_*.so; do
  tag=$(basename "$v" .so | sed 's/libdtsim_//')
  cp "$v" gym-duckietown_b200/libdtsim.so
  for m in small_loop loop_obstacles; do
    python bench.py --no-cpu-baseline --configs none --steps 20 --warmup 5 --map $m "$@" 2>>"${TMPDIR:-/tmp}/ab_err.log" | tail -1 | python -c "
import json,sys
d=json.loads(sys.stdin.read()); k=d['kernel_ms']
print('$tag $m', round(d['value']), 'env-steps/s', ' '.join(f'{n}={v*1000:.0f}us' for n,v in k.items()))"
  done
done
cp /tmp/libdtsim_keep.so gym-duckietown_b200/libdtsim.so
