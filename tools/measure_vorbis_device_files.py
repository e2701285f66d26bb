"""Time of decode.decode_vorbis_files_dev (Ogg Vorbis files already in device memory: pages indexed, headers chosen and jobs built
on the device) against decode.decode_vorbis_files(device=True), which indexes every file on the host, in one invocation.

Corpus: the 256-file writer corpus of tools/measure_vorbis_files.py (4 distinct 64-packet streams repeated, 44.1 kHz stereo,
blocks of 256 / 2048 samples), once per residue type (0, 1, 2), and one long file of 4000 packets.  The files are uploaded
once; the device call starts from resident bytes.

Reports, with the card name and power limit read in the same run:
  dev_ms       decode_vorbis_files_dev end to end, by a host clock around the call (it ends in a device synchronise and the
               read-back of its results): median of --reps calls after 2 warm-up calls
  phases_ms    one call split by CUDA events on the engine's stream: index (two symgpu_ogg_index_dev calls and the host wait
               between them), heads, setup (host wait, header read-back, header checks, setup / group build), jobs, decode
               (including its stream / floor registration); median over --reps calls
  host_ms      decode_vorbis_files(device=True) on the same files' bytes, same clock, median of --reps calls
  read_back_bytes, and whether every file's samples equal the host-indexed path's

usage: python tools/measure_vorbis_device_files.py [--reps 5] [--out FILE.json]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import symphonia_b200 as sb  # noqa: E402
from symphonia_b200 import _native as nat  # noqa: E402
from symphonia_b200 import decode  # noqa: E402
from tests import _vorbis_corpus as corpus  # noqa: E402

from measure_vorbis_files import card, writer_files  # noqa: E402

PHASES = ("start", "index", "heads", "setup", "jobs", "decode")


def upload(files):
    import torch
    ranges, at = [], 0
    for f in files:
        ranges.append((at, len(f)))
        at += len(f)
    return torch.from_numpy(np.frombuffer(b"".join(files), dtype=np.uint8).copy()).cuda(), ranges


def clock(fn, reps):
    fn()
    fn()
    times = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t) * 1e3)
    return statistics.median(times)


def phases(eng, data_t, ranges, reps):
    import torch
    stream = torch.cuda.ExternalStream(eng.cuda_stream, device=data_t.device)
    runs = []
    for _ in range(reps):
        ev = {}

        def mark(phase, state):
            ev[phase] = torch.cuda.Event(enable_timing=True)
            ev[phase].record(stream)
        decode._vorbis_files_dev(eng, data_t, ranges, nat.FMT_S16, None, None, mark=mark)
        ev["decode"].synchronize()
        runs.append({b: ev[a].elapsed_time(ev[b]) for a, b in zip(PHASES, PHASES[1:])})
    return {k: statistics.median(r[k] for r in runs) for k in PHASES[1:]}


def measure(eng, files, reps):
    data_t, ranges = upload(files)
    stats = {}
    got = decode.decode_vorbis_files_dev(eng, data_t, ranges, stats=stats)
    want = decode.decode_vorbis_files(eng, files, device=True)
    same = all(g.shape == w.shape and bool((g == w).all()) for (g, _), (w, _) in zip(got, want))
    return dict(files=len(files), bytes=sum(len(f) for f in files), jobs=len(stats["status"]), same_as_host=same,
                read_back_bytes=stats["read_back_bytes"],
                dev_ms=clock(lambda: decode.decode_vorbis_files_dev(eng, data_t, ranges), reps),
                phases_ms=phases(eng, data_t, ranges, reps),
                host_ms=clock(lambda: decode.decode_vorbis_files(eng, files, device=True), reps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    report = dict(card=card())
    with sb.Engine(0) as eng:
        for rtype in (0, 1, 2):
            report[f"residue_type_{rtype}"] = r = measure(eng, writer_files(256, 64, rtype), a.reps)
            print(rtype, json.dumps(r), flush=True)
        s, pk = corpus.writer(1302, 100, channels=2, bs_exp=(8, 11))
        report["long_file"] = r = measure(eng, [corpus.ogg(s, pk * 40, 1303)], a.reps)
        print("long", json.dumps(r), flush=True)
    print(json.dumps(report))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
