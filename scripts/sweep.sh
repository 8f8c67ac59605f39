#!/bin/bash
# dev tool: decode-loop timing of the persistent kernel vs the per-kernel graph chain, and of the experiment bits
# (CAR_EXP: 1/2 pre-poll variants, bits 8-11 pre-poll back-off; see csrc/decode_persistent.cuh)
for cfg in "CAR_MEGA=1" "CAR_MEGA=1 CAR_EXP=1" "CAR_MEGA=0"; do
  echo "== $cfg"
  env $cfg N=1024 timeout 120 python scripts/quick_xl.py 2>&1 | grep -E "iter 2|prefill|Error|error" | head -5
  env $cfg N=256 timeout 120 python scripts/quick_xl.py 2>&1 | grep -E "iter 2"
done
