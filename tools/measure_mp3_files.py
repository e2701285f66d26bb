"""Throughput of device Layer III decoding (symgpu_mp3_decode_*, decode.decode_mp3_files) against today's paths, in one invocation.

Corpus: tests/_mp3_bitstream.py streams at 44.1 kHz, seeded -- 256 files x 64 frames at 128 kbit/s joint stereo and at 320 kbit/s
stereo, plus 4 files x 10 000 frames at 128 kbit/s joint stereo (the serial reservoir walk of a long file).  The writer is pure
Python, so a few distinct streams are written once and reused: a file is one of them, or one repeated back to back (a stream's
first frame never reaches back into the reservoir, so the joints decode as cleanly as the rest).

Reports, with the card name and power limit read in the same run:
  device-resident bytes -> interleaved s16 samples in HBM (CUDA events over many calls after warm-up): frames/s and audio-s/s, also
    at 1 and 8 files per call, and the rounds a call takes
  decode_mp3_files through host memory, end to end (indexing, copies, decoding)
  decode_files on the same files (host front-end, GPU synthesis and output stage)
  symgpu_mpa_index + symgpu_mp3_fe_decode_packets alone, one file per host thread on 16 host threads

usage: python tools/measure_mp3_files.py [--files 256] [--frames 64] [--iters 20] [--out FILE.json]
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
from symphonia_b200 import decode, frontend, packetizer  # noqa: E402
from tests import _mp3_bitstream as bw  # noqa: E402

RATE = 44100


def streams(n, n_frames, mode, bitrate_idx, seed):
    rng = np.random.default_rng(seed)
    return [b"".join(bw.gen_stream(rng, n_frames, version="1", mode=mode, rate_idx=0, bitrate_idx=bitrate_idx, pair_blocks=True, fill=(0.6, 1.0))[0])
            for _ in range(n)]


def device_resident(eng, files, iters, warmup=3):
    """(seconds per call from CUDA events, packets, PCM frames, rounds) of mp3_decode_dev on resident bytes."""
    import torch
    plan = decode.mp3_files_plan(files)
    eng.mp3_streams_alloc(len(files))
    dev = torch.device("cuda", eng.device)
    as_t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to(dev)  # noqa: E731
    data_t, jobs_t = as_t(plan["data"]), as_t(plan["jobs"])
    out = torch.empty(plan["out_samples"], dtype=torch.int16, device=dev)
    res = torch.empty(len(files) * nat.MP3_RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    st = torch.empty(len(plan["jobs"]), dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    stream = torch.cuda.ExternalStream(eng.cuda_stream, device=dev)
    for _ in range(warmup):
        rounds = eng.mp3_decode_dev(data_t, jobs_t, plan["groups"], nat.FMT_S16, out, res, st)
    eng.sync()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(stream)
    for _ in range(iters):
        eng.mp3_decode_dev(data_t, jobs_t, plan["groups"], nat.FMT_S16, out, res, st)
    t1.record(stream)
    t1.synchronize()
    assert (st.cpu().numpy() == nat.MP3_JOB_DECODED).all()
    results = res.cpu().numpy().view(nat.MP3_RESULT_DTYPE)
    return t0.elapsed_time(t1) / 1e3 / iters, len(plan["jobs"]), int(results["frames"].sum()), rounds


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = float(subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                                     timeout=60).stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001 -- reported as unknown
        limit = None
    return name, limit


def rate(n, sec):
    return round(n / sec) if sec > 0 else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=256)
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--long-files", type=int, default=4)
    ap.add_argument("--long-frames", type=int, default=10000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    res = dict(card=name, power_limit_w=limit, sample_rate=RATE, host_threads=16)
    t = time.perf_counter()
    js = streams(a.distinct, a.frames, 1, 9, 9500)
    st320 = streams(a.distinct, a.frames, 0, 14, 9600)
    piece = streams(1, 500, 1, 9, 9700)[0]
    reps = -(-a.long_frames // 500)
    sets = {"joint_stereo_128k": [js[f % a.distinct] for f in range(a.files)], "stereo_320k": [st320[f % a.distinct] for f in range(a.files)],
            "long_joint_stereo_128k": [piece * reps for _ in range(a.long_files)]}
    res["corpus_write_s"] = round(time.perf_counter() - t, 1)
    with sb.Engine(0) as eng:
        for label, files in sets.items():
            r = {"files": len(files), "frames_per_file": len(packetizer.mpa_index(files[0])[1]), "file_MB": round(sum(map(len, files)) / 1e6, 2)}
            sec, packets, pcm_frames, rounds = device_resident(eng, files, a.iters if len(files) > 4 else max(3, a.iters // 4))
            audio_s = pcm_frames / RATE
            r["device_resident"] = dict(ms_per_call=round(sec * 1e3, 3), frames_per_s=rate(packets, sec), audio_s_per_s=rate(audio_s, sec), rounds=rounds)
            for n in (1, 8):
                if n < len(files):
                    s1, k1, p1, _ = device_resident(eng, files[:n], a.iters)
                    r[f"device_resident_{n}_files"] = dict(ms_per_call=round(s1 * 1e3, 3), frames_per_s=rate(k1, s1), audio_s_per_s=rate(p1 / RATE, s1))
            decode.decode_mp3_files(eng, files[:2])
            t = time.perf_counter()
            got = decode.decode_mp3_files(eng, files)
            e2e = time.perf_counter() - t
            r["decode_mp3_files_host_e2e"] = dict(s=round(e2e, 3), frames_per_s=rate(packets, e2e), audio_s_per_s=rate(audio_s, e2e))
            decode.decode_files(eng, files[:2])
            t = time.perf_counter()
            want = decode.decode_files(eng, files)
            df = time.perf_counter() - t
            r["decode_files"] = dict(s=round(df, 3), frames_per_s=rate(packets, df), audio_s_per_s=rate(audio_s, df))
            assert all(g[1] == w[1] and g[0].tobytes() == w[0].tobytes() for g, w in zip(got, want))

            def fe(f):
                _, pk = packetizer.mpa_index(f)
                return frontend.Mp3Frontend().decode_packets(f, pk)
            with concurrent.futures.ThreadPoolExecutor(max_workers=16) as pool:
                list(pool.map(fe, files[:2]))
                t = time.perf_counter()
                list(pool.map(fe, files))
                hf = time.perf_counter() - t
            r["index_and_host_front_end_16_threads"] = dict(s=round(hf, 3), frames_per_s=rate(packets, hf), audio_s_per_s=rate(audio_s, hf))
            res[label] = r
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
