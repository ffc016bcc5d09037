#!/bin/bash
# Development helper (run on a GPU): the end-to-end arm of bench.py against chunk size (pairs) and arena slots.
#   CFGS="32:4 16:6" bash tools/_e2e_sweep.sh
for cfg in ${CFGS:-32:4 16:4 16:6 64:4}; do
  c=${cfg%%:*}; s=${cfg##*:}
  echo "== e2e-chunk $c pairs, $s slots"
  timeout -k 5 300 python bench.py --no-mbv2 --no-cpu-baseline --no-parity-check --steps 5 --warmup 3 --e2e-chunk $c --e2e-slots $s 2>/dev/null | python -c "
import json,sys
for l in sys.stdin:
    if l.startswith('{'):
        d=json.loads(l); e=d['e2e']; print(e['value'], e['ms_per_step'], e['pcie_GBps_each_way'], e['copy_only']['GBps_each_way'])"
done
