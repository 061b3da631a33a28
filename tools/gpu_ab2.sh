#!/bin/bash
# A/B of environment switches on one 8K frame: stage times (CUDA events) per variant, then ncu counters of the default
# usage: AB_VARIANTS="OJB_BLOCK_ENCODER=warp;OJB_NO_FAST_BLOCKS=1" bash tools/gpu_ab2.sh
mkdir -p gpurun_out
: > gpurun_out/ab2.log
IFS=';' read -ra VARS <<< "default;${AB_VARIANTS}"
for v in "${VARS[@]}"; do
  [ -z "$v" ] && continue
  for prev in 1 ${AB_IRV:+0}; do
    echo "== $v PREV=$prev" >> gpurun_out/ab2.log
    if [ "$v" = "default" ]; then PREV=$prev PN=4 python tools/profile_once.py >> gpurun_out/ab2.log 2>&1
    else env $v PREV=$prev PN=4 python tools/profile_once.py >> gpurun_out/ab2.log 2>&1; fi
  done
done
timeout 600 ncu --metrics gpu__time_duration.sum,smsp__inst_executed.sum,smsp__issue_active.avg.pct_of_peak_sustained_active,sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active,sm__warps_active.avg.pct_of_peak_sustained_active \
  --clock-control none -k regex:"ht_" --csv --log-file gpurun_out/ab2_ncu.csv python tools/profile_once.py > gpurun_out/ab2_ncu.log 2>&1
python - <<'PY'
import re
for ln in open('gpurun_out/ab2.log'):
    if ln.startswith('=='): print(ln.strip()); continue
    m = re.findall(r"'(dwt|ht_encode|assemble|ht_decode|dwt_inv|host_parse|host_ms)': ([0-9.]+)", ln)
    if m: print('   ', ' '.join('%s=%.3f' % (k, float(v)) for k, v in m))
import csv
rows=[r for r in csv.reader(open('gpurun_out/ab2_ncu.csv')) if len(r)>10]
h=rows[0]; ki=h.index("Kernel Name"); mi=h.index("Metric Name"); vi=h.index("Metric Value"); ii=h.index("ID")
d={}
for r in rows[1:]:
    d.setdefault((r[ii], r[ki][:44]),{})[r[mi]]=r[vi]
for (i,k),m in d.items():
    print(i,k, " ".join("%s=%s"%(a.split('.')[0].replace('smsp__','').replace('sm__',''),b) for a,b in m.items()))
PY
