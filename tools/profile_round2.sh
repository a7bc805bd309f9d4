#!/bin/bash
mkdir -p tools/runs
# round-2 profile set (run on the GPU box): launch list of the bench command + full captures of the tile kernel (all 8 levels),
# the LM kernel (one batch of 32 different windows) and the IMMA K-list kernel
ncu --metrics gpu__time_duration.sum --clock-control none -c 2500 --csv --log-file tools/runs/r2_launches_bench_final.csv python bench.py --steps 2 --warmup 3 --no-cpu-baseline --e2e-lanes 1 > tools/runs/r2_launches_bench_final.log 2>&1
timeout 900 ncu --set full --import-source on --clock-control none -k regex:k_tile -s 8 -c 8 -f -o tools/runs/r2_prof_k_tile_final python tools/extract_time.py 320 2 > tools/runs/ncu_tile_all.log 2>&1
tail -1 tools/runs/ncu_tile_all.log
timeout 600 ncu --set full --import-source on --clock-control none -k regex:k_local_ba -s 1 -c 1 -f -o tools/runs/r2_prof_k_local_ba_final python tools/ba_prof2.py > tools/runs/ncu_ba.log 2>&1
tail -1 tools/runs/ncu_ba.log
timeout 600 ncu --set full --import-source on --clock-control none -k regex:k_bow_topk_imma -s 2 -c 1 -f -o tools/runs/r2_prof_k_bow_topk_imma_final python tools/bow_time.py > tools/runs/ncu_bow.log 2>&1
tail -1 tools/runs/ncu_bow.log
