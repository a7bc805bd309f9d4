#!/bin/bash
mkdir -p tools/runs
# bench.py (GPU arm only) for several SM budgets of the balanced LocalBA launch: tools/sweep_ba_sms.sh "48 64 80" [extra bench args]
for s in $1; do
  timeout 300 python bench.py --no-cpu-baseline --ba-sms $s ${@:2} > tools/runs/sweep_sms$s.json 2> tools/runs/sweep_err.log
  python - "$s" <<'PY'
import json, sys
s = sys.argv[1]
try:
    d = json.loads(open("tools/runs/sweep_sms%s.json" % s).read().strip().splitlines()[-1])
    print("SMS", s, "value %.0f ms/step %.2f e2e %.0f r1 %.0f ba_kernel %.2f" % (d["value"], d["ms_per_step"], d["e2e"]["value"], d["phase_ms"]["round1_workload_frames_per_s"], d.get("roofline_local_ba", {}).get("launch_ms", 0)))
except Exception as e:
    print("SMS", s, "failed", e)
PY
done
