"""Time of decode.decode_alac_files_dev (CAF files already in device memory: chunks and packet tables read on the device, the job
table decoded in place) against the host-indexed path, decode.decode_alac_files(device=True), in one invocation.

Inputs (seeded): 256 files of about 30 s (323 packets of 4096 frames at 44.1 kHz), half stereo 16-bit and half stereo 24-bit,
and one long file of about 10 minutes (6 460 packets, stereo 16-bit).  Each file's packets are drawn from a pool of 24 packets
per depth written by tests/_alac_bitstream.py (order-8 prediction of a few sinusoids and noise), so that the corpus is quick to
make; the decoder does the same work on every packet.  The files are uploaded once, back to back.

Checks before timing: Engine.caf_index_dev equals packetizer.caf_index for every file (records byte for byte, packets), and the
resident output equals the host-indexed output.  Reports, with the card name and power limit read in the same run (medians of
--reps calls after one warm-up call, the two calls taken in turn):
  dev_ms / host_ms            end to end, host clock (both end in a device synchronise and their read-backs)
  audio_s_per_s, files_per_s  the corpus's audio seconds and files over those times
  read_back_bytes             of decode_alac_files_dev
  oracle                      oracle/oracle_alac.cpp decoding 8 of the 30 s files' packets on one CPU thread: audio-s/s

usage: python tools/measure_alac_files.py [--reps 3] [--out FILE.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import symphonia_b200 as sb  # noqa: E402
from symphonia_b200 import _native as nat  # noqa: E402
from symphonia_b200 import decode, packetizer  # noqa: E402
from tests import _alac_bitstream as ab  # noqa: E402
from tests import _alac_cases as cases  # noqa: E402
from tests import _caf_corpus  # noqa: E402

FRAMES = 4096


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def pool(rng, bit_depth, n=24):
    ck = cases.cookie(channels=2, bit_depth=bit_depth, frame_length=FRAMES)
    el = [dict(kind="cpe", order=8, coeffs=[900, -400, 200, -100, 50, -25, 12, -6], lpc_shift=9, ms_weight=2, ms_shift=1,
               shift=8 if bit_depth == 24 else 0)]
    return ck, [ab.encode_packet(ab.signal(rng, FRAMES, 2, bit_depth, amp=0.4), ck, el) for _ in range(n)]


def caf_file(ck, packets):
    return _caf_corpus.caf([_caf_corpus.desc(ck), _caf_corpus.chunk(b"kuki", ab.cookie_bytes(ck)), _caf_corpus.pakt([len(p) for p in packets], ck),
                            _caf_corpus.chunk(b"data", bytes(4) + b"".join(packets))])


def corpus():
    rng = np.random.default_rng(2026)
    pools = [pool(rng, 16), pool(rng, 24)]
    files = []
    for k in range(256):
        ck, pk = pools[k % 2]
        files.append(caf_file(ck, [pk[(k + j) % len(pk)] for j in range(323)]))
    ck, pk = pools[0]
    files.append(caf_file(ck, [pk[j % len(pk)] for j in range(6460)]))
    return files


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    files = corpus()
    infos = [packetizer.caf_index(f) for f in files]
    audio_s = sum(int(i["n_packets"]) * FRAMES / 44100 for i, _ in infos)
    ranges, at = [], 0
    for f in files:
        ranges.append((at, len(f)))
        at += len(f)
    report = dict(card=card(), files=len(files), audio_seconds=round(audio_s, 1), bytes=at)
    with sb.Engine(0) as eng:
        data_t = torch.from_numpy(np.frombuffer(b"".join(files), dtype=np.uint8).copy()).cuda()
        torch.cuda.synchronize()
        dinfos, first, packets_t, _, _ = eng.caf_index_dev(data_t, ranges)
        packets = packets_t.cpu().numpy().view(nat.CAF_PACKET_DTYPE)
        same_index = all(dinfos[i:i + 1].tobytes() == np.array([info], dtype=nat.CAF_INFO_DTYPE).tobytes()
                         and packets[int(first[i]):int(first[i]) + len(p)].tobytes() == p.tobytes() for i, (info, p) in enumerate(infos))
        stats = {}
        got = decode.decode_alac_files_dev(eng, data_t, ranges, stats=stats)
        want = decode.decode_alac_files(eng, files, device=True)
        same_out = all(ra == rb and x.shape == y.shape and bool((x == y).all()) for (x, ra), (y, rb) in zip(got, want))
        del got, want
        report.update(same_index=same_index, same_as_host=same_out, read_back_bytes=int(stats["read_back_bytes"]))
        times = {"dev": [], "host": []}
        for rep in range(a.reps + 1):
            for name, call in (("dev", lambda: decode.decode_alac_files_dev(eng, data_t, ranges)),
                               ("host", lambda: decode.decode_alac_files(eng, files, device=True))):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                r = call()
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                del r
                if rep:
                    times[name].append(dt)
        for name, ts in times.items():
            ms = statistics.median(ts) * 1e3
            report[f"{name}_ms"] = round(ms, 2)
            report[f"{name}_audio_s_per_s"] = round(audio_s / (ms / 1e3), 0)
            report[f"{name}_files_per_s"] = round(len(files) / (ms / 1e3), 1)
    # the oracle on one CPU thread, over 8 of the 30 s files
    orc = cases.oracle_lib()
    t0, secs = time.perf_counter(), 0.0
    for k in range(8):
        info, pk = infos[k]
        ck = {f: int(info[f]) for f in ("frame_length", "bit_depth", "pb", "mb", "kb", "channels")}
        for p in pk:
            cases.oracle_packet(orc, files[k][int(p["offset"]):int(p["offset"]) + int(p["size"])], ck)
        secs += len(pk) * FRAMES / 44100
    report["oracle_one_thread_audio_s_per_s"] = round(secs / (time.perf_counter() - t0), 0)
    print(json.dumps(report))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
