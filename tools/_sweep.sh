#!/bin/bash
# Development helper (run on a GPU): phase timings of the stack bench for alternative builds of the library.
#   LIBS="libdfq_sm90 libdfq_variant" bash tools/_sweep.sh [pairs]
# Build a variant here first:  DFQ_NVCC_DEFS="-DDFQ_TILE_BLOCK=128" DFQ_LIB_OUT=$PWD/dfq_b200/libdfq_variant.so python -m dfq_b200._build
for lib in ${LIBS:-libdfq_sm90}; do
  echo "== $lib"
  DFQ_LIB=$PWD/dfq_b200/$lib.so timeout -k 5 200 python bench.py --steps 3 --layers ${1:-2048} --no-cpu-baseline --no-e2e --no-mbv2 2>/dev/null | python -c "import sys,json; d=json.loads(sys.stdin.read().strip().splitlines()[-1]); print(d['phases_ms'], d['parity_check']['ok'] if d.get('parity_check') else None)"
done
