#!/usr/bin/env python
"""Summarise an .ncu-rep (read here, no GPU needed): per-kernel key metrics + top SASS stall lines.
usage: python scripts/ncu_summary.py prof.ncu-rep [kernel-regex] [--json profiles/ncu_traffic.json WORKLOAD]
--json merges {WORKLOAD: {"source": rep, "kernels": {name: {dram_bytes, time_us, inst, regs}}}} into the file bench.py reads
for roofline.traffic (dram__bytes_read.sum + dram__bytes_write.sum per launch of the CURRENT kernels)."""
import csv, subprocess, sys, collections, io, re, json, os
args = sys.argv[1:]
jpath = jwl = None
if "--json" in args:
    i = args.index("--json")
    jpath, jwl = args[i + 1], args[i + 2]
    del args[i:i + 3]
rep = args[0]
pat = args[1] if len(args) > 1 else None
jrec = {}
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
idx = {h: i for i, h in enumerate(hdr)}
want = ['gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum', 'lts__t_bytes.sum', 'lts__t_sector_hit_rate.pct',
        'sm__warps_active.avg.pct_of_peak_sustained_active', 'launch__registers_per_thread', 'launch__grid_size',
        'launch__occupancy_limit_registers', 'launch__occupancy_limit_shared_mem', 'sm__throughput.avg.pct_of_peak_sustained_elapsed',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'smsp__inst_executed.sum', 'sm__cycles_active.avg',
        'smsp__issue_active.avg.pct_of_peak_sustained_active', 'l1tex__t_sector_hit_rate.pct']
stall = [h for h in hdr if h.startswith('smsp__average_warps_issue_stalled') and h.endswith('_per_issue_active.ratio')]
seen = set()
for r in rows[2:]:
    name = r[idx['Kernel Name']]
    short = name.split('(')[0][-60:]
    if pat and not re.search(pat, name): continue
    if short in seen: continue
    seen.add(short)
    print("====", short)
    def _num(key):
        try:
            v = float(r[idx[key]].replace(",", ""))
        except Exception:
            return None
        u = units[idx[key]].lower()
        scale = {"gbyte": 1e9, "mbyte": 1e6, "kbyte": 1e3, "byte": 1, "ms": 1e3, "us": 1, "ns": 1e-3, "msecond": 1e3, "usecond": 1, "nsecond": 1e-3}.get(u, 1)
        return v * scale
    if jpath:
        rd, wr = _num('dram__bytes_read.sum'), _num('dram__bytes_write.sum')
        jrec[short.strip()] = {"dram_bytes": (rd or 0) + (wr or 0), "time_us": _num('gpu__time_duration.sum'),
                               "inst": _num('smsp__inst_executed.sum'), "regs": _num('launch__registers_per_thread')}
    for w in want:
        if w in idx: print("   %-62s %s %s" % (w, r[idx[w]], units[idx[w]]))
    st = sorted(((float(r[idx[h]] or 0), h) for h in stall), reverse=True)[:6]
    for v, h in st:
        print("   stall %-40s %.2f" % (h.replace('smsp__average_warps_issue_stalled_', '').replace('_per_issue_active.ratio', ''), v))

if jpath:
    d = json.load(open(jpath)) if os.path.exists(jpath) else {}
    d[jwl] = {"source": os.path.basename(rep), "kernels": jrec}
    json.dump(d, open(jpath, "w"), indent=1, sort_keys=True)
