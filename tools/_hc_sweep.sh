#!/bin/bash
# Development helper (run on a GPU): MobileNetV2 e2e inside bench.py's process environment (NUMA binding, clock sampler)
# against the host-copy thread count (DFQ_HOST_COPY_THREADS) and the number of upload parts (DFQ_UPLOAD_PARTS).
#   CFGS="0:1 1:1" bash tools/_hc_sweep.sh
for cfg in ${CFGS:-0:1 0:1 1:1}; do
  t=${cfg%%:*}; p=${cfg##*:}
  echo "== DFQ_HOST_COPY_THREADS=$t DFQ_UPLOAD_PARTS=$p"
  DFQ_HOST_COPY_THREADS=$t DFQ_UPLOAD_PARTS=$p timeout -k 5 200 python bench.py --layers 256 --no-e2e --no-cpu-baseline --steps 3 --warmup 3 2>/dev/null | python -c "
import json,sys
for l in sys.stdin:
    if l.startswith('{'):
        d=json.loads(l); m=d['mobilenetv2']; print(m['e2e_ms'], m['device_ms'], m['e2e_parts_ms'])"
done
