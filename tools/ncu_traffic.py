#!/usr/bin/env python
"""profiles/ncu_traffic.json from `ncu --set full` captures of single launches at known shapes (no GPU needed).
usage: python tools/ncu_traffic.py prof_out/prof_<tag>_<kernel>_Sq<..>_Sk<..>_H<..>_c<0|1>.ncu-rep [...]
The launch shape is in the file name (tools/profile.sh writes it); every entry keeps where it came from.
bench.py reads this table for `roofline.traffic` -- a shape that was never captured yields null."""
import csv
import io
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "profiles", "ncu_traffic.json")
tab = json.load(open(OUT)) if os.path.exists(OUT) else {}
for rep in sys.argv[1:]:
    m = re.search(r"_(fwd|bwd)_Sq(\d+)_Sk(\d+)_H(\d+)_c([01])", os.path.basename(rep))
    if not m:
        print("skip (no shape in name):", rep)
        continue
    kern, Sq, Sk, Hh, c = m.group(1) + "_chunk_kernel", int(m.group(2)), int(m.group(3)), int(m.group(4)), int(m.group(5))
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    col = lambda name: hdr.index(name)  # noqa: E731

    def to_bytes(row, name):
        u = units[col(name)].lower()
        f = {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9, "tbyte": 1e12}[u]
        return float(row[col(name)].replace(",", "")) * f

    for r in rows[2:]:
        if kern not in r[col("Kernel Name")]:
            continue
        rd, wr = to_bytes(r, "dram__bytes_read.sum"), to_bytes(r, "dram__bytes_write.sum")
        key = f"{kern}:Sq={Sq}:Sk={Sk}:H={Hh}:causal={c}"
        tab[key] = {"dram_bytes": rd + wr, "dram_bytes_read": rd, "dram_bytes_write": wr,
                    "duration_ms_under_ncu": float(r[col("gpu__time_duration.sum")].replace(",", "")) *
                    {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}[units[col("gpu__time_duration.sum")].lower()],
                    "tensor_active_pct": float(r[col("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active")]),
                    "source": os.path.basename(rep)}
        print(key, tab[key])
        break
json.dump(tab, open(OUT, "w"), indent=1, sort_keys=True)
