#!/bin/bash
# quick A/B of the block coders on one 8K frame: CUDA-event stage times (fast kernels vs the general ones) and the
# ncu instruction counts / durations of the coder kernels.  Never a bench number.
mkdir -p gpurun_out
echo "== fast" > gpurun_out/ab.log
PN=4 python tools/profile_once.py >> gpurun_out/ab.log 2>&1
echo "== general (OJB_NO_FAST_BLOCKS=1)" >> gpurun_out/ab.log
OJB_NO_FAST_BLOCKS=1 PN=4 python tools/profile_once.py >> gpurun_out/ab.log 2>&1
if [ -n "$AB_IRV" ]; then
echo "== fast, 9/7" >> gpurun_out/ab.log
PREV=0 PN=4 python tools/profile_once.py >> gpurun_out/ab.log 2>&1
fi
timeout 600 ncu --metrics gpu__time_duration.sum,smsp__inst_executed.sum,smsp__issue_active.avg.pct_of_peak_sustained_active,sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active,sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active,dram__bytes_read.sum,dram__bytes_write.sum \
  --clock-control none -k regex:"ht_|dwt_|gather|assemble" --csv --log-file gpurun_out/ab_ncu.csv python tools/profile_once.py > gpurun_out/ab_ncu.log 2>&1
cat gpurun_out/ab.log
python - <<'PY'
import csv
rows=[r for r in csv.reader(open('gpurun_out/ab_ncu.csv')) if len(r)>10]
h=rows[0]; ki=h.index("Kernel Name"); mi=h.index("Metric Name"); vi=h.index("Metric Value"); ii=h.index("ID")
d={}
for r in rows[1:]:
    d.setdefault((r[ii], r[ki][:40]),{})[r[mi]]=r[vi]
for (i,k),m in d.items():
    print(i,k, " ".join("%s=%s"%(a.split('.')[0].replace('smsp__','').replace('sm__',''),b) for a,b in m.items()))
PY
