#!/usr/bin/env python3
"""Regenerate profiles/ncu_traffic.json (read by bench.py for `roofline.traffic`) from an ncu capture of ONE 2^20 x 100 LDE step.

    ncu --set full --clock-control none -k regex:'ntt_(pass|lde_mid)_' -s 3 -c 3 -o ntt python tools/run_lde_once.py 2 100
    python tools/ncu_traffic.py ntt.ncu-rep profiles/ntt_pass_kernels.txt

dram__bytes_read.sum + dram__bytes_write.sum per launch, summed over the 3 launches of the step.  Also writes the per-launch
summary table (tools/ncu_summary.py) next to it."""
import csv
import json
import pathlib
import subprocess
import sys

rep = sys.argv[1]
summary = pathlib.Path(sys.argv[2]) if len(sys.argv) > 2 else None
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units = rows[0], rows[1]
scale = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0}
per = []
for r in rows[2:]:
    d, u = dict(zip(hdr, r)), dict(zip(hdr, units))
    tot = 0.0
    for k in ("dram__bytes_read.sum", "dram__bytes_write.sum"):
        tot += float(d[k]) * scale.get(u[k], 1.0)
    per.append(tot)
out = {"lde_step_dram_bytes": sum(per), "per_launch_dram_bytes": per,
       "source": f"{summary or rep} (ncu --set full --clock-control none, {len(per)} launches of one 2^20x100 LDE step; regenerate with tools/ncu_traffic.py)"}
root = pathlib.Path(__file__).resolve().parent.parent
(root / "profiles").mkdir(exist_ok=True)
(root / "profiles" / "ncu_traffic.json").write_text(json.dumps(out))
print(out)
if summary:
    txt = subprocess.run([sys.executable, str(root / "tools" / "ncu_summary.py"), rep], capture_output=True, text=True).stdout
    summary.write_text(txt)
    print(txt)
