#!/bin/bash
# N = 2 A/B of environment settings (the variables bench.py only sets by default, such as NCCL_MAX_NCHANNELS, and AB_INFLIGHT) in one 2-GPU box session:
# tools/ab_bench_n2.sh "<ENV=..>" ...
port=29520
for v in "$@"; do
  port=$((port+1))
  AB_INFLIGHT=$(echo "$v" | sed -n 's/.*AB_INFLIGHT=\([0-9]*\).*/\1/p'); AB_INFLIGHT=${AB_INFLIGHT:-24}
  env $v timeout 400 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port $port bench.py --gpus 2 --steps 48 --warmup 3 --inflight $AB_INFLIGHT --no-configs --no-extra --no-cpu > /tmp/abn2.json 2>/tmp/abn2.err
  python - "$v" <<'PY'
import json, sys
try:
    d = json.loads(open("/tmp/abn2.json").read().strip().splitlines()[-1])
    print("%-50s ms/step %.3f  frames/s %.0f  e2e ms %.3f e2e frames/s %.0f" % (sys.argv[1], d["ms_per_step"], d["frames_per_s"], d["e2e"]["ms_per_step"], d["e2e"]["frames_per_s"]), flush=True)
except Exception as e:
    print(sys.argv[1], "FAILED", e, open("/tmp/abn2.err").read()[-600:])
PY
done
