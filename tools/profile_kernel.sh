#!/bin/bash
mkdir -p tools/runs
# ncu --set full capture of one kernel of the bench step (run from the repo root): tools/profile_kernel.sh k_tile
k=${1:-k_tile}
timeout 900 ncu --set full --import-source on --clock-control none -k regex:$k -s 1 -c 1 -f -o tools/runs/prof_$k \
    python bench.py --steps 1 --warmup 1 --e2e-steps 1 --no-cpu-baseline > tools/runs/ncu_$k.log 2>&1
tail -1 tools/runs/ncu_$k.log
