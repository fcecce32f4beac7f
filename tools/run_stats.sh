#!/bin/bash
# tools/run_stats.sh — on a GPU machine with nvcc: tools/raster_stats.py for the c2 and c3 maps on a -DDTS_STATS=1 build of
# libdtsim.so, then the normal build is restored
cd "$(dirname "$0")/.."
build() { python -c "import sys; sys.path.insert(0, 'gym-duckietown_b200'); import build; build.build(force=True)"; }
trap build EXIT
DTS_NVCC_EXTRA=-DDTS_STATS=1 build || exit 1
export DTS_NO_REBUILD=1
for m in small_loop loop_obstacles; do echo "== $m"; python tools/raster_stats.py $m 2>&1 | grep -v Warn; done
