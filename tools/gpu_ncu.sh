#!/bin/bash
# one ncu --set full capture of the hot kernels on a single 8K encode+decode (never a bench number)
mkdir -p gpurun_out
NAME=${PROF_NAME:-prof_r01b}
timeout 1500 ncu --set full --clock-control none --import-source on \
   -k regex:"${PROF_KERNELS:-ht_encode|ht_decode|ht_dec_fill|dwt_fwd_stream|dwt_inv_stream|gather_blocks|assemble}" -c 20 \
   -o gpurun_out/$NAME python tools/profile_once.py > gpurun_out/ncu_full.log 2>&1
tail -3 gpurun_out/ncu_full.log; ls -la gpurun_out/
