"""Throughput of device FLAC decoding (symgpu_flac_decode_*, decode.decode_flac_files) against today's path, in one invocation.

Corpus: tests/_flac_bitstream.py over workloads.flac_batch, seeded -- 16-bit stereo 44.1 kHz frames of 4096 samples, plus a 24-bit
variant.  The writer is pure Python (tens of ms per frame), so a few hundred distinct frames are written and repeated: file f's
frame k is one of a few frames written with frame number k.  The encoder picks sub-frame types at random, VERBATIM included, so
this corpus is heavier per sample than typical encoder output.

Reports, with the card name and power limit read in the same run:
  device-resident bytes -> interleaved int32 PCM in HBM (CUDA events over many launches after warm-up): frames/s, audio-s/s,
    and algorithmic bytes (file bytes in + PCM out) over that time against 3.35 TB/s; also at 1 and 8 files per call
  decode_flac_files through host memory, end to end (indexing, copies, decoding)
  today's path on the same corpus: decode_flac file by file, and the host front-end alone on all host threads

usage: python tools/measure_flac_files.py [--files 256] [--frames 64] [--iters 20] [--out FILE.json]
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
from symphonia_b200 import decode, frontend, packetizer, workloads  # noqa: E402
from tests import _flac_bitstream as fw  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def corpus(n_files, n_frames, bps, per_number, seed):
    """n_files files of n_frames full 4096-sample stereo frames; per_number distinct frames per frame number."""
    need = n_frames * per_number
    frames, subs, samples = workloads.flac_batch(need + need // 6 + 7, 4096, seed=seed, bps=bps, channels=2)
    full = [f for f in range(len(frames)) if f % 7][:need]
    rng = np.random.default_rng(seed)
    pool = [[fw.write_frame(rng, frames[f], subs[2 * f:2 * f + 2], samples, k, stream_bps=bps) for f in full[k * per_number:(k + 1) * per_number]]
            for k in range(n_frames)]
    files = []
    for i in range(n_files):
        pk = [pool[k][(i + k) % per_number] for k in range(n_frames)]
        files.append(fw.native_file(pk, fw.stream_info_block(4096, 4096, 44100, 2, bps, 4096 * n_frames, min(map(len, pk)), max(map(len, pk)))))
    return files


def device_resident(eng, files, iters, warmup=3):
    """(seconds per call from CUDA events, FLAC frames, PCM frames, file bytes, PCM bytes) of flac_decode_dev on resident bytes."""
    import torch
    plan = decode.flac_files_plan(files)
    dev = torch.device("cuda", eng.device)
    as_t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to(dev)  # noqa: E731
    data_t, jobs_t, groups_t = as_t(plan["data"]), as_t(plan["jobs"]), as_t(plan["groups"])
    out = torch.empty(plan["out_cap"], dtype=torch.int32, device=dev)
    gf = torch.empty(len(files), dtype=torch.int64, device=dev)
    st = torch.empty(len(plan["jobs"]), dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    stream = torch.cuda.ExternalStream(eng.cuda_stream, device=dev)
    for _ in range(warmup):
        eng.flac_decode_dev(data_t, jobs_t, groups_t, out, gf, st)
    eng.sync()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(stream)
    for _ in range(iters):
        eng.flac_decode_dev(data_t, jobs_t, groups_t, out, gf, st)
    t1.record(stream)
    t1.synchronize()
    assert (st.cpu().numpy() == nat.FLAC_JOB_DECODED).all()
    pcm_frames = int(gf.sum().item())
    return t0.elapsed_time(t1) / 1e3 / iters, len(plan["jobs"]), pcm_frames, int(plan["data"].size), pcm_frames * 2 * 4


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
    ap.add_argument("--per-number", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    res = dict(card=name, power_limit_w=limit, files=a.files, frames_per_file=a.frames, block=4096, channels=2, host_threads=os.cpu_count())
    t = time.perf_counter()
    sets = {"16-bit": corpus(a.files, a.frames, 16, a.per_number, 9100), "24-bit": corpus(a.files // 4, a.frames, 24, 2, 9200)}
    res["corpus_write_s"] = round(time.perf_counter() - t, 1)
    with sb.Engine(0) as eng:
        for label, files in sets.items():
            r = {"files": len(files), "file_MB": round(sum(map(len, files)) / 1e6, 1)}
            sec, frames, pcm_frames, fbytes, pbytes = device_resident(eng, files, a.iters)
            audio_s = pcm_frames / 44100
            r["device_resident"] = dict(ms_per_call=round(sec * 1e3, 3), frames_per_s=round(frames / sec), audio_s_per_s=round(audio_s / sec),
                                        bytes_per_s=round((fbytes + pbytes) / sec / 1e9, 2), share_of_hbm=round((fbytes + pbytes) / sec / HBM_BYTES_PER_S, 4))
            for n in (1, 8):
                s1, _, p1, _, _ = device_resident(eng, files[:n], a.iters)
                r[f"device_resident_{n}_files"] = dict(ms_per_call=round(s1 * 1e3, 3), audio_s_per_s=round(p1 / 44100 / s1))
            decode.decode_flac_files(eng, files[:4])
            t = time.perf_counter()
            got = decode.decode_flac_files(eng, files)
            e2e = time.perf_counter() - t
            r["decode_flac_files_host_e2e"] = dict(s=round(e2e, 3), frames_per_s=round(frames / e2e), audio_s_per_s=round(audio_s / e2e))
            t = time.perf_counter()
            for k, f in enumerate(files):
                want, _ = decode.decode_flac(eng, f)
                assert (want == got[k][0]).all()
            per_file = time.perf_counter() - t
            r["decode_flac_file_by_file"] = dict(s=round(per_file, 3), frames_per_s=round(frames / per_file), audio_s_per_s=round(audio_s / per_file))

            def fe(f):
                info, packets = packetizer.flac_index(f)
                table = np.zeros(len(packets), dtype=nat.PIECE_DTYPE)
                table["offset"], table["len"] = packets["offset"], packets["size"]
                return frontend.flac_decode_packets(f, table, int(info["bits_per_sample"]), int(info["channels"]), int(info["block_max"]))
            with concurrent.futures.ThreadPoolExecutor(max_workers=os.cpu_count()) as pool:
                list(pool.map(fe, files[:8]))
                t = time.perf_counter()
                list(pool.map(fe, files))
                hf = time.perf_counter() - t
            r["host_front_end_all_threads"] = dict(s=round(hf, 3), frames_per_s=round(frames / hf), audio_s_per_s=round(audio_s / hf))
            res[label] = r
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
