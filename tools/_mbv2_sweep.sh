#!/bin/bash
# Development helper (run on a GPU): MobileNetV2 device-resident calibration time for grid caps of the equalization kernel.
for g in ${GRIDS:-444 296 148 96}; do
  echo "== DFQ_CLE_GRID=$g"
  DFQ_CLE_GRID=$g timeout -k 5 120 python tools/mbv2_profile.py 2>&1 | tail -2
done
