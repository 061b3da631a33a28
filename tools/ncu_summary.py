#!/usr/bin/env python3
"""Summarise an `ncu --set full` report (tools/gpu_ncu.sh) into a small JSON:
per kernel family: launches, time, DRAM bytes, instructions, issue-active %, achieved occupancy,
top stall reasons.  Usage: ncu_summary.py prof_X.ncu-rep X_kernels.json"""
import csv, json, subprocess, sys

rep, out = sys.argv[1], sys.argv[2]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
h = rows[0]
ki = h.index("Kernel Name")
stall = [i for i, c in enumerate(h) if c.startswith("smsp__pcsamp_warps_issue_stalled_") and not c.endswith("_not_issued")]


units = rows[1]
SCALE = {"ns": 1e-6, "us": 1e-3, "usecond": 1e-3, "ms": 1.0, "msecond": 1.0, "s": 1e3, "second": 1e3,           # -> ms
         "byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}                                               # -> MB


def g(r, n):
    """metric value; times come back in ms and byte counts in MB whatever unit ncu chose for the report"""
    try:
        i = h.index(n)
        return float(r[i]) * SCALE.get(units[i], 1.0)
    except Exception:
        return 0.0


fam = (("hdr_trees", "hdr_trees"), ("hdr_items", "hdr_items"), ("hdr_groups", "hdr_groups"), ("hdr_chain", "hdr_chain"), ("hdr_expand", "hdr_expand"), ("hdr_write", "hdr_write"), ("hdr_layout", "hdr_layout"), ("hdr_place", "hdr_place"), ("hdr_copy", "hdr_copy"), ("ht_encode_split", "ht_encode_split"), ("ht_decode_split", "ht_decode_split"), ("dec_merge", "dec_merge"), ("ht_encode_serial", "ht_encode_serial"), ("ht_encode", "ht_encode"), ("ht_decode_serial", "ht_decode_serial"), ("ht_dec_fill", "ht_dec_fill"),
       ("gather_blocks", "gather_blocks"), ("assemble_kernel", "assemble"), ("ctrl_copy", "ctrl_copy"),
       ("dwt_fwd_stream", "dwt_fwd"), ("dwt_inv_stream", "dwt_inv"))
res = {}
for r in rows[2:]:
    key = next((k for pat, k in fam if pat in r[ki]), None)
    if key is None:
        continue
    d = res.setdefault(key, dict(launches=0, time_ms=0.0, dram_read_MB=0.0, dram_write_MB=0.0, inst_executed=0,
                                 per_launch=[]))
    t = g(r, "gpu__time_duration.sum")
    d["launches"] += 1; d["time_ms"] += t
    d["dram_read_MB"] += g(r, "dram__bytes_read.sum"); d["dram_write_MB"] += g(r, "dram__bytes_write.sum")
    d["inst_executed"] += int(g(r, "smsp__inst_executed.sum"))
    vals = sorted(((float(r[i] or 0), h[i].replace("smsp__pcsamp_warps_issue_stalled_", "")) for i in stall), reverse=True)
    tot = sum(v for v, _ in vals) or 1.0
    d["per_launch"].append(dict(kernel=r[ki][:64], time_ms=round(t, 4), regs=int(g(r, "launch__registers_per_thread")),
                                grid=int(g(r, "launch__grid_size")),
                                issue_active_pct=round(g(r, "smsp__issue_active.avg.pct_of_peak_sustained_active"), 1),
                                warps_active_pct=round(g(r, "sm__warps_active.avg.pct_of_peak_sustained_active"), 1),
                                dram_pct_of_peak=round(g(r, "dram__throughput.avg.pct_of_peak_sustained_elapsed"), 1),
                                stalls_pct={n: round(100 * v / tot) for v, n in vals[:4]}))
for d in res.values():
    d["traffic_bytes"] = int((d["dram_read_MB"] + d["dram_write_MB"]) * 1e6)
    for k in ("time_ms", "dram_read_MB", "dram_write_MB"):
        d[k] = round(d[k], 3)
res["_note"] = ("ncu --set full --clock-control none --import-source on, one 8192x8192x3 12-bit 5/3 encode + decode "
                "(tools/profile_once.py); cold-cache single launches under the profiler, never bench values; dwt_* sum the "
                "five level launches; report: " + rep)
json.dump(res, open(out, "w"), indent=1)
print(json.dumps({k: (v["time_ms"], v["traffic_bytes"]) for k, v in res.items() if k != "_note"}))
