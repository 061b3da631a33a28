#!/bin/bash
# Is a fast block coder bound by one block's serial chain or by the SM's instruction throughput?
# ht_encode / ht_decode stage times (CUDA events, tools/profile_once.py) against the number of code-blocks
# in one launch: 1/4, 1/2, 1, 2 and 4 8K frames (more frames are stacked as tiles of one canvas).  Nearly
# flat up to one frame means chain-bound (ILP and occupancy pay); linear means throughput-bound (the
# instruction count pays).  Then the existing coder switches, once each, against the default.
# usage: tools/coder_probe.sh [LABEL]     OJB_LIB_PATH picks the library.  One result line per run, prefixed with LABEL.
L=${1:-default}
nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv,noheader
run() {      # run NAME ENV... : one profile_once.py call, stage times of the last of PN frames
  local name=$1; shift
  env "$@" PN=3 timeout 600 python tools/profile_once.py 2>&1 | tail -1 | python -c "
import ast, sys
line = sys.stdin.read().strip()
try:
    n, e, d = ast.literal_eval('(' + line.replace(' {', ', {') + ')')     # '<bytes> {encoder} {decoder}'
    print('%-10s %-22s ht_encode %7.3f ms  ht_decode %7.3f ms  sum %7.3f ms' % ('$L', '$name', e['ht_encode'], d['ht_decode'], e['ht_encode'] + d['ht_decode']))
except Exception:
    print('%-10s %-22s unparsed: %s' % ('$L', '$name', line[-300:]))
"
}
run "blocks x1/4" PH=2048
run "blocks x1/2" PH=4096
run "blocks x1" PH=8192
run "blocks x2" PH=16384 PTILE=8192
run "blocks x4" PH=32768 PTILE=8192
run "encoder=warp" OJB_BLOCK_ENCODER=warp
run "carveout=25" OJB_SMEM_CARVEOUT=25
run "carveout=75" OJB_SMEM_CARVEOUT=75
