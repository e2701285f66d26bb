"""Throughput of device Ogg Vorbis decoding (symgpu_vorbis_decode_*, decode.decode_vorbis_files) against today's paths, in one
invocation.

Corpus: tests/_vorbis_bitstream.py writer streams at 44.1 kHz stereo (blocks of 256 / 2048 samples), seeded, paginated by
tests/_vorbis_corpus.py; 256 files x 64 packets, once per residue type (0, 1, 2).  The writer is pure Python, so 4 distinct
streams are written once and repeated.  Its codebooks are random, not libvorbis output: real encoder files have other book
shapes, and nothing here can produce them.

Reports, with the card name and power limit read in the same run:
  device-resident bytes -> interleaved s16 samples in HBM: ms per call by CUDA events over --iters calls after 3 warm-up calls
    (a call's host work -- setup build, stream / floor registration -- lies between the events), packets/s and audio-s/s, at
    1, 8 and 256 files per call
  decode_vorbis_files through host memory, end to end (indexing, copies, decoding)
  decode_files on the same files (host front-end, GPU synthesis and output stage)
  ogg_vorbis_index + symgpu_vorbis_fe_decode_packets alone, one file per host thread on 16 host threads
  symgpu_vorbis_fe_decode_packets alone on files indexed beforehand, 16 host threads (the same work as the device call)

usage: python tools/measure_vorbis_files.py [--iters 20] [--out FILE.json]
"""
import argparse
import concurrent.futures
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import symphonia_b200 as sb  # noqa: E402
from symphonia_b200 import _native as nat  # noqa: E402
from symphonia_b200 import decode  # noqa: E402
from tests import _vorbis_corpus as corpus  # noqa: E402

RATE = 44100


def writer_files(n_files, n_packets, residue_type, distinct=4, seed=1):
    out = []
    for d in range(distinct):
        s, pk = corpus.writer(seed + 10 * residue_type + d, n_packets, channels=2, bs_exp=(8, 11), residue_type=residue_type)
        out.append(corpus.ogg(s, pk, seed + d))
    return [out[i % distinct] for i in range(n_files)]


def device_resident(eng, files, iters):
    import torch
    plan = decode.vorbis_files_plan(files)
    dev = torch.device("cuda", eng.device)
    as_t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to(dev)  # noqa: E731
    data_t, jobs_t = as_t(plan["data"]), as_t(plan["jobs"])
    out = torch.empty(plan["out_samples"], dtype=torch.int16, device=dev)
    results = torch.empty(len(files) * nat.VORBIS_RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    status = torch.empty(len(plan["jobs"]), dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    stream = torch.cuda.ExternalStream(eng.cuda_stream, device=dev)
    call = lambda: eng.vorbis_decode_dev(plan["headers"], plan["setups"], data_t, jobs_t, plan["groups"], nat.FMT_S16, out, results, status)  # noqa: E731
    for _ in range(3):
        call()
    eng.sync()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record(stream)
    for _ in range(iters):
        call()
    end.record(stream)
    end.synchronize()
    ms = start.elapsed_time(end) / iters
    r = results.cpu().numpy().view(nat.VORBIS_RESULT_DTYPE)
    packets, frames = int(r["packets"].sum()), int(r["frames"].sum())
    return dict(ms_per_call=ms, packets_per_s=packets / ms * 1e3, audio_s_per_s=frames / RATE / ms * 1e3, packets=packets,
                decoded_fraction=packets / max(len(plan["jobs"]), 1))


def wall(fn, reps=3):
    fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps


def host_frontend_16(files):
    def one(f):
        ix = decode.ogg_vorbis_index(f)
        ix["fe"].decode_packets(ix["blob"], ix["table"])
        ix["fe"].close()
    with concurrent.futures.ThreadPoolExecutor(16) as pool:
        return wall(lambda: list(pool.map(one, files)), reps=2)


def host_frontend_16_indexed(files):
    """symgpu_vorbis_fe_decode_packets alone, on files indexed beforehand: the host work the device call replaces."""
    ix = [decode.ogg_vorbis_index(f) for f in files]
    with concurrent.futures.ThreadPoolExecutor(16) as pool:
        t = wall(lambda: list(pool.map(lambda x: x["fe"].decode_packets(x["blob"], x["table"]), ix)), reps=2)
    for x in ix:
        x["fe"].close()
    return t


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    report = dict(card=card())
    with sb.Engine(0) as eng:
        for rtype in (0, 1, 2):
            files = writer_files(256, 64, rtype)
            got = decode.decode_vorbis_files(eng, files)
            audio = sum(len(x) for x, _ in got) / RATE
            packets = sum(len(decode.ogg_vorbis_index(f)["table"]) for f in files[:4]) * len(files) // 4
            r = dict(files=len(files), packets=packets, audio_s=audio, device=device_resident(eng, files, a.iters))
            r["device_1_file"] = device_resident(eng, files[:1], a.iters)
            r["device_8_files"] = device_resident(eng, files[:8], a.iters)
            t = wall(lambda: decode.decode_vorbis_files(eng, files), reps=2)
            r["decode_vorbis_files_host"] = dict(s=t, audio_s_per_s=audio / t)
            t = wall(lambda: decode.decode_files(eng, files), reps=2)
            r["decode_files"] = dict(s=t, audio_s_per_s=audio / t)
            t = host_frontend_16(files)
            r["host_frontend_16_threads"] = dict(s=t, audio_s_per_s=audio / t, packets_per_s=packets / t)
            t = host_frontend_16_indexed(files)
            r["host_frontend_16_threads_indexed"] = dict(s=t, audio_s_per_s=audio / t, packets_per_s=packets / t)
            report[f"residue_type_{rtype}"] = r
            print(rtype, json.dumps(r), flush=True)
    print(json.dumps(report))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
