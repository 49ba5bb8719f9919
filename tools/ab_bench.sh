#!/bin/bash
# A/B of environment settings (the variables bench.py only sets by default, such as CUDA_DEVICE_MAX_CONNECTIONS, and AB_INFLIGHT)
# inside ONE GPU-box session (boxes differ by a few per cent, so only same-box numbers compare).
# usage: tools/ab_bench.sh "<ENV=.. ENV=..>" "<...>" ...   prints ms/step of the headline path and the e2e figure per variant
for v in "$@"; do
  AB_INFLIGHT=$(echo "$v" | sed -n 's/.*AB_INFLIGHT=\([0-9]*\).*/\1/p'); AB_INFLIGHT=${AB_INFLIGHT:-16}
  env $v timeout 300 python bench.py --steps 48 --warmup 3 --inflight ${AB_INFLIGHT:-16} --no-configs --no-cpu --no-extra > /tmp/ab.json 2>/tmp/ab.err
  python - "$v" <<'PY'
import json, sys
try:
    d = json.loads(open("/tmp/ab.json").read().strip().splitlines()[-1])
    print("%-60s ms/step %.3f  frames/s %.0f  e2e ms %.3f" % (sys.argv[1], d["ms_per_step"], d["frames_per_s"], d["e2e"]["ms_per_step"]), flush=True)
except Exception as e:
    print(sys.argv[1], "FAILED", e, open("/tmp/ab.err").read()[-500:])
PY
done
