#!/usr/bin/env python
"""profiles/scan_traffic.json from an `ncu --set full` capture of ivfpq_scan_kernel at the BASELINE configuration
(`ncu --set full -k regex:ivfpq_scan_kernel -o scan python bench.py ...`).  The file is stamped with the hash of the scan kernel's
sources (bench.py::scan_source_hash): bench.py reports `roofline.traffic` only while that hash still matches the tree.

    python scripts/make_scan_traffic.py scan.ncu-rep
"""
import csv
import io
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units, vals = rows[0], rows[1], rows[2]


def get(name):
    i = hdr.index(name)
    v = float(vals[i].replace(",", ""))
    scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12, "ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3,
             "%": 1, "": 1}.get(units[i], 1)
    return v * scale


import importlib.util
spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
bench = importlib.util.module_from_spec(spec)
sys.argv = ["bench.py"]
spec.loader.exec_module(bench)
out = {
    "config": {"n": 100_000_000, "nq": 10_000, "nlist": 16384, "M": 64, "nprobe": 32, "k": 100},
    "kernel": vals[hdr.index("Kernel Name")].split("(")[0],
    "dram_bytes_read": get("dram__bytes_read.sum"), "dram_bytes_write": get("dram__bytes_write.sum"),
    "dram_bytes_per_launch": get("dram__bytes_read.sum") + get("dram__bytes_write.sum"),
    "duration_ms_under_ncu": get("gpu__time_duration.sum"),
    "dram_throughput_pct": get("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"),
    "l1tex_throughput_pct": get("l1tex__throughput.avg.pct_of_peak_sustained_elapsed"),
    "lts_throughput_pct": get("lts__throughput.avg.pct_of_peak_sustained_elapsed"),
    "registers_per_thread": get("launch__registers_per_thread"),
    "kernel_source_sha16": bench.scan_source_hash(),
    "source": f"ncu --set full --clock-control none -k regex:ivfpq_scan -s 4 -c 1 python bench.py ... ({os.path.basename(rep)})",
}
os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
json.dump(out, open(os.path.join(ROOT, "profiles", "scan_traffic.json"), "w"), indent=1)
print(json.dumps(out, indent=1))
