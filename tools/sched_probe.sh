#!/bin/bash
# schedule comparison on the headline policy mix (tools/mix_probe.py): event schedule, chained, chained + persistent rows
for e in "FAA_CHAIN=0" "FAA_PERSIST=0" "FAA_PERSIST=1" "FAA_PERSIST=1 FAA_ROWS_MID=66" "FAA_PERSIST=1 FAA_ROWS_MID=99" "FAA_PERSIST=1 FAA_ROWS_LIGHT=37" "FAA_PERSIST=1 FAA_ROWS_LIGHT=75"; do
  env $e timeout 120 python tools/mix_probe.py
done
