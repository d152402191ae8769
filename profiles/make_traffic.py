#!/usr/bin/env python
"""profiles/r2_traffic.json from an `ncu --set full` capture: DRAM bytes (read + write) per field of the line kernel, tagged
with the hash of the kernel sources the capture was taken from.  bench.py reports `roofline.traffic` only when that hash
equals the hash of the sources it runs (bench.py: library_source_hash), so a stale capture can never be quoted for a newer
build.

    python profiles/make_traffic.py <rep>.ncu-rep <variant> <fields per launch> "<what the capture was>"
"""
import csv
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    rep, variant, fields, note = sys.argv[1], sys.argv[2], int(sys.argv[3]), sys.argv[4]
    import bench
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], stdout=subprocess.PIPE, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units, data = rows[0], rows[1], rows[2:]
    col = {h: i for i, h in enumerate(hdr)}
    best = None
    for r in data:
        name = r[col["Kernel Name"]]
        if "k_lines" not in name:
            continue
        def val(key):
            v, u = float(r[col[key]].replace(",", "")), units[col[key]]
            return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}[u]
        tot = val("dram__bytes_read.sum") + val("dram__bytes_write.sum")
        dur = float(r[col["gpu__time_duration.sum"]].replace(",", ""))
        if best is None or tot > best[1]:
            best = (name.split("(")[0], tot, dur, r[col["Grid Size"]])
    assert best, "no line kernel in the capture"
    path = os.path.join(ROOT, "profiles", "r2_traffic.json")
    try:
        table = json.load(open(path))
    except Exception:
        table = {}
    table[variant] = {"kernel": best[0], "dram_bytes_per_launch": best[1], "fields_per_launch": fields,
                      "dram_bytes_per_field": best[1] / fields, "duration_us_under_ncu": best[2], "grid": best[3],
                      "src_sha": bench.library_source_hash(), "capture": note}
    json.dump(table, open(path, "w"), indent=1, sort_keys=True)
    print(json.dumps(table[variant], indent=1))


if __name__ == "__main__":
    main()
