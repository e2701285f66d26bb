"""Packets per second and frames per launch of 64 AAC and 64 Vorbis decoder threads on ONE context (`shared_context_host files`), against
the shape before shared submission for those codecs: one context per decoder thread (`shared_context_host files-apart`, every decode() one
launch of its own).  Prints one JSON object with the card's name and power limit; the numbers in DESIGN.md §9 come from it.

    python tools/measure_shared_context.py [--files 64] [--packets 200] [--repeats 3]

Needs an H100 (the library has no CPU path).  Writes its input files to a temporary directory."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _gpu():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=64)
    ap.add_argument("--packets", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    from tests import test_zz_adts_aac_to_pcm as adts
    from tests.test_cpp_shared_context_gpu import _build_shared, _ogg_vorbis_file
    exe = _build_shared()
    # eight distinct streams per codec, repeated: every decoder is independent, so copies cost what distinct files cost
    distinct = 8
    make = {
        "aac": lambda k: adts._file(8000 + k, 44100, 2, n=a.packets)[0],
        "vorbis": lambda k: _ogg_vorbis_file(8100 + k, [(8, 11), (7, 9)][k % 2], 2, n_packets=a.packets),
    }
    result = {"gpu": _gpu(), "files": a.files, "packets_per_file": a.packets, "runs": {}}
    with tempfile.TemporaryDirectory() as d:
        args = {}
        for codec, fn in make.items():
            blobs = [fn(k) for k in range(distinct)]
            args[codec] = []
            for i in range(a.files):
                p = os.path.join(d, f"{codec}{i:03d}")
                with open(p, "wb") as f:
                    f.write(blobs[i % distinct])
                args[codec].append(f"{codec}:{p}")
        for rep in range(a.repeats):  # the two shapes alternate, so drift on a shared machine hits both
            for codec in make:
                for mode in ("files", "files-apart"):
                    res = subprocess.run([exe, mode] + args[codec], capture_output=True, text=True, timeout=1200)
                    if res.returncode != 0:
                        raise SystemExit(f"{mode} {codec} failed: {res.stdout}{res.stderr}")
                    m = re.search(r"packets (\d+) decoded (\d+) seconds ([\d.]+) packets_per_s (\d+)", res.stdout)
                    b = re.search(r"codec \w+ batches (\d+) frames (\d+)", res.stdout)
                    run = {"packets": int(m.group(1)), "seconds": float(m.group(3)), "packets_per_s": int(m.group(4))}
                    if b:
                        run["batches"], run["frames_per_batch"] = int(b.group(1)), round(int(b.group(2)) / int(b.group(1)), 2)
                    result["runs"].setdefault(f"{codec} {mode}", []).append(run)
    result["median_packets_per_s"] = {k: sorted(r["packets_per_s"] for r in v)[len(v) // 2] for k, v in result["runs"].items()}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
