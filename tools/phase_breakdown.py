#!/usr/bin/env python
"""Per-phase instruction / stall-sample breakdown of the MP3 kernel from an ncu report.

usage: tools/phase_breakdown.py <report.ncu-rep> [libsymgpu.so]
Joins the SASS listing of ncu's source page (per-instruction executed counts and stall samples) with
nvdisasm -g line info of the same cubin, and buckets source lines of mp3_kernel.cu by the markers
`// PHASE: name` found in it (falls back to function-name heuristics when absent)."""
import csv
import io
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def line_of_each_instruction(so, variant=None):
    tmp = tempfile.mkdtemp()
    subprocess.check_call(["cuobjdump", "-xelf", "all", os.path.abspath(so)], cwd=tmp, stdout=subprocess.DEVNULL)
    sass = subprocess.run(["nvdisasm", "-g", "-c", os.path.join(tmp, "mp3_kernel.sm_90a.cubin")],
                          capture_output=True, text=True).stdout
    out, cur, infn = [], 0, False
    for ln in sass.splitlines():
        if ln.startswith("\t.text.") or ".text." in ln and ln.strip().startswith(".section"):
            infn = "mp3_synth_kernel" in ln and (variant is None or variant in ln)
        m = re.search(r'//## File ".*mp3_kernel.cu", line (\d+)', ln)
        if m:
            cur = int(m.group(1))
        elif "//## File" in ln:
            cur = -1
        if infn and re.match(r"^\s*/\*[0-9a-f]{4,6}\*/", ln):
            out.append((cur, ln.split("*/", 1)[1].strip()))
    return out


def phase_table(src):
    """[(first_line, name)] from `// PHASE: name` markers, else built-in ranges by content."""
    marks = []
    for i, ln in enumerate(open(src).read().splitlines(), 1):
        m = re.search(r"// PHASE: (.+)$", ln)
        if m:
            marks.append((i, m.group(1).strip()))
    return marks


def main():
    rep = sys.argv[1]
    so = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "symphonia_b200/libsymgpu.so")
    txt = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(txt)))
    # the kernel has a single-tile-group and a multi-tile-group instantiation (last template argument)
    name = next((r[1] for r in rows if r and r[0] == "Kernel Name"), "")
    # "mp3_synth_kernel<16, 16, 0>" -> the mangled template argument list ILi16ELi16ELb0EE
    targs = re.sub(r"\((int|bool)\)", "", re.search(r"<([^>]*)>", name).group(1)).replace(" ", "").split(",")
    variant = "I" + "".join(f"Li{a}E" for a in targs[:2]) + "".join("Lb1E" if a in ("1", "true") else "Lb0E" for a in targs[2:]) + "E"
    lines = line_of_each_instruction(so, variant)
    hdr_i = next(i for i, r in enumerate(rows) if r and r[0] == "Address")
    hdr = rows[hdr_i]
    body = rows[hdr_i + 1:]
    if len(body) != len(lines):
        print(f"instruction count mismatch: report {len(body)} vs cubin {len(lines)} (different build?)")
        return 1
    col = {n: hdr.index(n) for n in hdr}
    marks = phase_table(os.path.join(ROOT, "symphonia_b200/csrc/mp3_kernel.cu"))
    if not marks:
        print("no // PHASE: markers in mp3_kernel.cu")
        return 1

    def phase(line):
        name = "?"
        for first, nm in marks:
            if line >= first:
                name = nm
        return name

    stalls = [h for h in hdr if h.startswith("stall_") and "Not Issued" not in h]
    agg = {}
    for (line, _), r in zip(lines, body):
        p = phase(line)
        a = agg.setdefault(p, {"inst": 0, "samples": 0, **{s: 0 for s in stalls}})
        a["inst"] += int(r[col["Instructions Executed"]])
        a["samples"] += int(r[col["# Samples"]])
        for s in stalls:
            a[s] += int(r[col[s]])
    ti = sum(a["inst"] for a in agg.values())
    ts = sum(a["samples"] for a in agg.values())
    print(f"{'phase':28s} {'inst':>10s} {'%':>5s} {'samples':>8s} {'%':>5s}  top stalls")
    for p, a in sorted(agg.items(), key=lambda kv: -kv[1]["samples"]):
        top = sorted(((a[s], s[6:]) for s in stalls), reverse=True)[:4]
        tops = " ".join(f"{n}:{100 * v / max(a['samples'], 1):.0f}%" for v, n in top)
        print(f"{p:28s} {a['inst']:10d} {100 * a['inst'] / ti:5.1f} {a['samples']:8d} {100 * a['samples'] / ts:5.1f}  {tops}")
    print(f"{'total':28s} {ti:10d}       {ts:8d}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
