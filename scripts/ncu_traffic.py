"""Extracts duration / DRAM traffic / key metrics of one kernel from an `ncu --set full` report into a small JSON under
profiles/ (bench.py reads roofline.traffic from profiles/convexify_ncu.json).
usage: ncu_traffic.py report.ncu-rep cfg2 profiles/convexify_ncu.json"""
import csv
import io
import json
import subprocess
import sys

rep, cfg, out = sys.argv[1], sys.argv[2], sys.argv[3]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units, vals = rows[0], rows[1], rows[2]
m = dict(zip(hdr, vals))
u = dict(zip(hdr, units))


def num(k):
    try:
        return float(m[k].replace(",", ""))
    except (KeyError, ValueError):
        return None


def to_bytes(k):
    v = num(k)
    if v is None:
        return None
    return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u.get(k, "byte"), 1)


rd, wr = to_bytes("dram__bytes_read.sum"), to_bytes("dram__bytes_write.sum")
keys = ["gpu__time_duration.sum", "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct",
        "launch__registers_per_thread", "launch__occupancy_limit_shared_mem", "launch__grid_size",
        "smsp__inst_executed_op_local_ld.sum", "smsp__inst_executed_op_local_st.sum",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smsp__inst_executed.sum"]
entry = {"kernel": m.get("Kernel Name"), "dram_bytes_read": rd, "dram_bytes_write": wr,
         "dram_bytes": None if rd is None or wr is None else rd + wr}
for k in keys:
    entry[k] = num(k)
    if k in u:
        entry[k + ".unit"] = u[k]
try:
    data = json.load(open(out))
except (OSError, ValueError):
    data = {}
data[cfg] = entry
json.dump(data, open(out, "w"), indent=1)
print(json.dumps(entry, indent=1))
