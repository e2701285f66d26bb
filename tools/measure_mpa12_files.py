"""Throughput of device Layer I / II decoding (symgpu_mpa12_decode_*, decode.decode_mpa12_files) against today's path, in one invocation.

Corpus: tests/_mpa12_bitstream.py, seeded -- Layer II 48 kHz stereo 256 kbit/s (768-byte frames, Table 3-B.2a), plus a Layer I corpus
at 48 kHz stereo 384 kbit/s.  The writer is pure Python, so a pool of distinct frames is written once and repeated: file f's frame k
is pool[(f + 7 k) % pool size].

Reports, with the card name and power limit read in the same run:
  device-resident bytes -> interleaved s16 samples in HBM (CUDA events over many calls after warm-up): frames/s and audio-s/s, also
    at 1 and 8 files per call
  decode_mpa12_files through host memory, end to end (indexing, copies, decoding)
  decode_files on the same files (host front-end, GPU synthesis and output stage)
  symgpu_mpa12_fe_decode_packets alone, one file per host thread on all host threads

usage: python tools/measure_mpa12_files.py [--files 256] [--frames 64] [--iters 20] [--out FILE.json]
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
from tests import _mpa12_bitstream as bw  # noqa: E402


def corpus(n_files, n_frames, layer, bitrate_idx, pool_size, seed):
    rng = np.random.default_rng(seed)
    gen = bw.gen_layer1_frame if layer == 1 else bw.gen_layer2_frame
    pool = [gen(rng, "1", bitrate_idx, 1, 0, density=0.9)[0] for _ in range(pool_size)]
    return [b"".join(pool[(f + 7 * k) % pool_size] for k in range(n_frames)) for f in range(n_files)]


def device_resident(eng, files, iters, warmup=3):
    """(seconds per call from CUDA events, packets, PCM frames) of mpa12_decode_dev on resident bytes."""
    import torch
    plan = decode.mpa12_files_plan(files)
    eng.mp3_streams_alloc(len(files))
    dev = torch.device("cuda", eng.device)
    as_t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to(dev)  # noqa: E731
    data_t, jobs_t = as_t(plan["data"]), as_t(plan["jobs"])
    out = torch.empty(plan["out_samples"], dtype=torch.int16, device=dev)
    res = torch.empty(len(files) * nat.MPA12_RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    st = torch.empty(len(plan["jobs"]), dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    stream = torch.cuda.ExternalStream(eng.cuda_stream, device=dev)
    for _ in range(warmup):
        eng.mpa12_decode_dev(data_t, jobs_t, plan["groups"], nat.FMT_S16, out, res, st)
    eng.sync()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(stream)
    for _ in range(iters):
        eng.mpa12_decode_dev(data_t, jobs_t, plan["groups"], nat.FMT_S16, out, res, st)
    t1.record(stream)
    t1.synchronize()
    assert (st.cpu().numpy() == nat.MPA12_JOB_DECODED).all()
    results = res.cpu().numpy().view(nat.MPA12_RESULT_DTYPE)
    return t0.elapsed_time(t1) / 1e3 / iters, len(plan["jobs"]), int(results["frames"].sum())


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = float(subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                                     timeout=60).stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001 -- reported as unknown
        limit = None
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=256)
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--pool", type=int, default=48)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    res = dict(card=name, power_limit_w=limit, files=a.files, frames_per_file=a.frames, sample_rate=48000, channels=2, host_threads=os.cpu_count())
    t = time.perf_counter()
    sets = {"layer2_256k": corpus(a.files, a.frames, 2, 12, a.pool, 9300), "layer1_384k": corpus(a.files, a.frames, 1, 12, a.pool, 9400)}
    res["corpus_write_s"] = round(time.perf_counter() - t, 1)
    with sb.Engine(0) as eng:
        for label, files in sets.items():
            r = {"files": len(files), "file_MB": round(sum(map(len, files)) / 1e6, 2)}
            sec, packets, pcm_frames = device_resident(eng, files, a.iters)
            audio_s = pcm_frames / 48000
            r["device_resident"] = dict(ms_per_call=round(sec * 1e3, 3), frames_per_s=round(packets / sec), audio_s_per_s=round(audio_s / sec))
            for n in (1, 8):
                s1, k1, p1 = device_resident(eng, files[:n], a.iters)
                r[f"device_resident_{n}_files"] = dict(ms_per_call=round(s1 * 1e3, 3), frames_per_s=round(k1 / s1), audio_s_per_s=round(p1 / 48000 / s1))
            decode.decode_mpa12_files(eng, files[:4])
            t = time.perf_counter()
            got = decode.decode_mpa12_files(eng, files)
            e2e = time.perf_counter() - t
            r["decode_mpa12_files_host_e2e"] = dict(s=round(e2e, 3), frames_per_s=round(packets / e2e), audio_s_per_s=round(audio_s / e2e))
            decode.decode_files(eng, files[:4])
            t = time.perf_counter()
            want = decode.decode_files(eng, files)
            df = time.perf_counter() - t
            r["decode_files"] = dict(s=round(df, 3), frames_per_s=round(packets / df), audio_s_per_s=round(audio_s / df))
            assert all(g[1] == w[1] and g[0].tobytes() == w[0].tobytes() for g, w in zip(got, want))

            def fe(f):
                track, pk = packetizer.mpa_index(f)
                return frontend.mpa12_decode_packets(f, pk, int(track["layer"]))
            with concurrent.futures.ThreadPoolExecutor(max_workers=os.cpu_count()) as pool:
                list(pool.map(fe, files[:8]))
                t = time.perf_counter()
                list(pool.map(fe, files))
                hf = time.perf_counter() - t
            r["host_front_end_all_threads"] = dict(s=round(hf, 3), frames_per_s=round(packets / hf), audio_s_per_s=round(audio_s / hf))
            res[label] = r
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
