#!/usr/bin/env python
"""Top source lines by stall samples for one kernel of an ncu report.

usage: tools/line_hotspots.py <report.ncu-rep> <cubin stem, e.g. aac_kernel> <kernel name substring> [top N]
Joins ncu's SASS source page with nvdisasm -g line info of the in-tree libsymgpu.so."""
import collections
import csv
import io
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sass_lines(so, stem, kernel):
    tmp = tempfile.mkdtemp()
    subprocess.check_call(["cuobjdump", "-xelf", "all", os.path.abspath(so)], cwd=tmp, stdout=subprocess.DEVNULL)
    sass = subprocess.run(["nvdisasm", "-g", "-c", os.path.join(tmp, stem + ".sm_90a.cubin")], capture_output=True, text=True).stdout
    out, cur, infn = [], 0, False
    for ln in sass.splitlines():
        if ln.strip().startswith(".section") and ".text." in ln:
            infn = kernel in ln
        m = re.search(r'//## File "([^"]*)", line (\d+)', ln)
        if m:
            cur = (os.path.basename(m.group(1)), int(m.group(2)))
        if infn and re.match(r"^\s*/\*[0-9a-f]{4,6}\*/", ln):
            out.append((cur, ln.split("*/", 1)[1].strip()))
    return out


def main():
    rep, stem, kernel = sys.argv[1:4]
    top = int(sys.argv[4]) if len(sys.argv) > 4 else 25
    lines = sass_lines(os.path.join(ROOT, "symphonia_b200/libsymgpu.so"), stem, kernel)
    txt = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(txt)))
    # one block per profiled kernel: a "Kernel Name" row, a header row, then the instructions
    blocks, i = [], 0
    while i < len(rows):
        if rows[i] and rows[i][0] == "Kernel Name":
            name, hdr, j = rows[i][1], rows[i + 1], i + 2
            while j < len(rows) and not (rows[j] and rows[j][0] == "Kernel Name"):
                j += 1
            blocks.append((name, hdr, rows[i + 2:j]))
            i = j
        else:
            i += 1
    for name, hdr, body in blocks:
        if kernel not in name:
            continue
        if len(body) != len(lines):
            print(f"{name}: instruction count mismatch (report {len(body)}, cubin {len(lines)})")
            continue
        col = {n: k for k, n in enumerate(hdr)}
        stalls = [h for h in hdr if h.startswith("stall_") and "Not Issued" not in h]
        agg = collections.defaultdict(lambda: collections.Counter())
        for (where, _), r in zip(lines, body):
            a = agg[where]
            a["samples"] += int(r[col["# Samples"]])
            a["inst"] += int(r[col["Instructions Executed"]])
            for s in stalls:
                a[s] += int(r[col[s]])
        ts = sum(a["samples"] for a in agg.values())
        ti = sum(a["inst"] for a in agg.values())
        print(f"{name[:70]}: {ts} samples, {ti} warp-instructions")
        for where, a in sorted(agg.items(), key=lambda kv: -kv[1]["samples"])[:top]:
            tops = " ".join(f"{s[6:]}:{100 * a[s] / max(a['samples'], 1):.0f}%" for s in sorted(stalls, key=lambda s: -a[s])[:3])
            print(f"  {where[0]}:{where[1]:<5d} {100 * a['samples'] / ts:5.1f}% samples {100 * a['inst'] / ti:5.1f}% inst  {tops}")
        break
    return 0


if __name__ == "__main__":
    sys.exit(main())
