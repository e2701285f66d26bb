"""Throughput of device AAC-LC decoding (symgpu_aac_decode_*, decode.decode_aac_files) against today's paths, in one invocation.

Corpus: tests/_aac_bitstream.py streams at 44.1 kHz stereo, seeded, wrapped in ADTS.  The writer picks every section's book at
random, noise (PNS) included, so nearly every packet draws noise and pass B re-decodes it; the "quiet" corpus has no noise bands
(hand-built mono packets, pass B idle).  The writer is pure Python, so a few distinct packet lists are written once and reused:
  writer   256 files x 64 frames
  quiet    256 files x 64 frames
  long     4 files x 10 000 frames (the serial per-file walk)

Reports, with the card name and power limit read in the same run:
  device-resident bytes -> interleaved s16 samples in HBM (CUDA events over --iters calls after 3 warm-up calls): ms per call,
    frames/s and audio-s/s, also at 1 and 8 files per call, and n_redecoded
  decode_aac_files through host memory, end to end (indexing, copies, decoding)
  decode_files on the same files (host front-end, GPU synthesis and output stage)
  adts index + symgpu_aac_fe_decode_packets alone, one file per host thread on 16 host threads

usage: python tools/measure_aac_files.py [--iters 20] [--out FILE.json]
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
from symphonia_b200 import decode, frontend  # noqa: E402
from tests import _aac_bitstream as ab  # noqa: E402
from tests import _aac_corpus as corpus  # noqa: E402

RATE = 44100


def writer_files(n_files, n_frames, distinct=8, seed=1):
    out = []
    for d in range(distinct):
        s = ab.Stream(np.random.default_rng(seed + d), rate=RATE, channels=2)
        out.append(corpus.adts([s.packet()[0] for _ in range(n_frames)], RATE, 2, seed=d))
    return [out[i % distinct] for i in range(n_files)], 2


def quiet_files(n_files, n_frames):
    return [corpus.adts(corpus.quiet(n_frames), RATE, 1)] * n_files, 1


def long_files(n_files, n_frames, distinct=200):
    s = ab.Stream(np.random.default_rng(99), rate=RATE, channels=2)
    pk = [s.packet()[0] for _ in range(distinct)]
    return [corpus.adts([pk[k % distinct] for k in range(n_frames)], RATE, 2, seed=i) for i in range(n_files)], 2


def device_resident(eng, files, iters):
    import torch
    plan = decode.aac_files_plan(files)
    eng.aac_streams_alloc(max(len(files), 1))
    dev = torch.device("cuda", eng.device)
    as_t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to(dev)  # noqa: E731
    data_t, jobs_t = as_t(plan["data"]), as_t(plan["jobs"])
    out = torch.empty(plan["out_samples"], dtype=torch.int16, device=dev)
    results = torch.empty(len(files) * nat.AAC_RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    status = torch.empty(len(plan["jobs"]), dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    stream = torch.cuda.ExternalStream(eng.cuda_stream, device=dev)
    redone = 0
    for _ in range(3):
        redone = eng.aac_decode_dev(data_t, jobs_t, plan["groups"], nat.FMT_S16, out, results, status)
    eng.sync()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record(stream)
    for _ in range(iters):
        eng.aac_decode_dev(data_t, jobs_t, plan["groups"], nat.FMT_S16, out, results, status)
    end.record(stream)
    end.synchronize()
    ms = start.elapsed_time(end) / iters
    frames = len(plan["jobs"])
    return dict(ms_per_call=ms, frames_per_s=frames / ms * 1e3, audio_s_per_s=frames * 1024 / RATE / ms * 1e3, n_redecoded=redone)


def wall(fn, reps=3):
    fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps


def host_frontend_16(files):
    def one(f):
        packets, rate, ch = decode.adts_aac_index(f)
        table = np.zeros(len(packets), dtype=nat.PIECE_DTYPE)
        table["offset"], table["len"] = packets["offset"], packets["size"]
        fe = frontend.AacFrontend(rate, ch)
        fe.decode_packets(f, table)
        fe.close()
    with concurrent.futures.ThreadPoolExecutor(16) as pool:
        return wall(lambda: list(pool.map(one, files)), reps=2)


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
        for name, (files, ch) in (("writer", writer_files(256, 64)), ("quiet", quiet_files(256, 64)), ("long", long_files(4, 10000))):
            frames = sum(len(decode.adts_aac_index(f)[0]) for f in files)
            audio = frames * 1024 / RATE
            r = dict(files=len(files), frames=frames, device=device_resident(eng, files, a.iters))
            if name != "long":
                r["device_1_file"] = device_resident(eng, files[:1], a.iters)
                r["device_8_files"] = device_resident(eng, files[:8], a.iters)
            t = wall(lambda: decode.decode_aac_files(eng, files), reps=2)
            r["decode_aac_files_host"] = dict(s=t, audio_s_per_s=audio / t)
            t = wall(lambda: decode.decode_files(eng, files), reps=2)
            r["decode_files"] = dict(s=t, audio_s_per_s=audio / t)
            t = host_frontend_16(files)
            r["host_frontend_16_threads"] = dict(s=t, audio_s_per_s=audio / t, frames_per_s=frames / t)
            report[name] = r
            print(name, json.dumps(r), flush=True)
    print(json.dumps(report))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
