"""Time of the device MPEG index (symgpu_mpa_index_dev) and of decode.decode_mpeg_files_dev (MPEG audio files already in device
memory: frames, tags and trims found on the device, decoded from the job table in place) against the host-indexed path,
decode.decode_mpeg_files(device=True), in one invocation.

Inputs: 256 decodable files -- 192 Layer III (MPEG-1 joint stereo and MPEG-2 mono, 32 frames each) and 64 Layer I / II (32 frames
each), 16 + 8 distinct streams repeated -- and one Layer III file of 10 000 frames (a 500-frame stream whose first frame needs no
reservoir, 20 times over).  The files are uploaded once, back to back; the device calls start from resident bytes.

Reports, with the card name and power limit read in the same run (every time a median of --reps calls after 2 warm-up calls,
the four kinds of call taken in turn):
  index_dev_ms    symgpu_mpa_index_dev alone (jobs only, sized by the lengths // 24 bound), CUDA events on the engine's stream
                  around the call; this includes its one host wait, for the candidate count
  index_host_ms   packetizer.mpa_index of every file on 16 host threads, host clock (the index phase of the host-indexed path)
  dev_ms          decode_mpeg_files_dev end to end, host clock (it ends in a device synchronise and the read-back of its results)
  host_ms         decode_mpeg_files(device=True) on the same files' bytes, host clock
  read_back_bytes of decode_mpeg_files_dev, and whether its samples, errors and stats equal the host-indexed path's and the device
  index's tracks and packets equal the host index's (checked before timing)
The Layer III decode walks each file's bit reservoir in one thread (DESIGN §10.8), which can dominate a long file: that is why the
index phase is reported on its own.

usage: python tools/measure_mpeg_device_files.py [--reps 5] [--out FILE.json]
"""
import argparse
import concurrent.futures
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
from symphonia_b200 import decode, packetizer  # noqa: E402
from tests import _mp3_bitstream as bw  # noqa: E402
from tests import _mpa12_bitstream as b12  # noqa: E402

from measure_aac_files import card  # noqa: E402


def many_files(seed=5):
    rng = np.random.default_rng(seed)
    mp3 = [b"".join(bw.gen_stream(rng, 32, version=v, mode=m, bitrate_idx=b, pair_blocks=True)[0])
           for v, m, b in [("1", 1, 9), ("2", 3, 8)] * 8]
    l12 = [b"".join((b12.gen_layer1_frame if k % 2 else b12.gen_layer2_frame)(rng, "1", 9 if k % 2 else 8, 0, k % 4 if k % 4 != 3 else 0)[0]
                    for _ in range(32)) for k in range(8)]
    return [mp3[k % len(mp3)] for k in range(192)] + [l12[k % len(l12)] for k in range(64)]


def one_long(seed=6):
    frames, _ = bw.gen_stream(np.random.default_rng(seed), 500, version="1", mode=1, bitrate_idx=9, pair_blocks=True)
    return [b"".join(frames) * 20]


def upload(files):
    import torch
    ranges, at = [], 0
    for f in files:
        ranges.append((at, len(f)))
        at += len(f)
    return torch.from_numpy(np.frombuffer(b"".join(files), dtype=np.uint8).copy()).cuda(), ranges


def check(eng, files, data_t, ranges, pool):
    """Device index == host index per file; decode_mpeg_files_dev == decode_mpeg_files(device=True).  Returns its read_back_bytes."""
    packets_t, _, index, tracks = eng.mpa_index_dev(data_t, ranges)
    packets = packets_t.cpu().numpy().view(nat.MPA_PACKET_DTYPE)
    for i, (track, want) in enumerate(pool.map(packetizer.mpa_index, files)):
        a = int(index[i]["first_packet"])
        assert packets[a:a + len(want)].tobytes() == want.tobytes() and int(index[i]["n_packets"]) == len(want)
        assert tracks[i].tobytes() == np.asarray(track).tobytes()
    e_d, s_d, e_h, s_h = {}, {}, {}, {}
    got = decode.decode_mpeg_files_dev(eng, data_t, ranges, errors=e_d, stats=s_d)
    want = decode.decode_mpeg_files(eng, files, device=True, errors=e_h, stats=s_h)
    assert e_d == e_h and s_d["status"].tobytes() == s_h["status"].tobytes() and s_d["rounds"] == s_h["rounds"]
    assert all(gr == wr and g.shape == w.shape and bool((g == w).all()) for (g, gr), (w, wr) in zip(got, want))
    return s_d["read_back_bytes"]


def measure(eng, files, reps, pool):
    import torch
    data_t, ranges = upload(files)
    read_back = check(eng, files, data_t, ranges, pool)
    r = np.array(ranges, dtype=np.uint64)
    cap = int((r[:, 1] // nat.MPA_MIN_FRAME).sum())
    jobs_t = torch.empty(cap * nat.MP3_JOB_DTYPE.itemsize, dtype=torch.uint8, device=data_t.device)
    index_t = torch.empty(len(files) * nat.MPA_FILE_INDEX_DTYPE.itemsize, dtype=torch.uint8, device=data_t.device)
    tracks_t = torch.empty(len(files) * nat.MPA_TRACK_DTYPE.itemsize, dtype=torch.uint8, device=data_t.device)
    stream = torch.cuda.ExternalStream(eng.cuda_stream, device=data_t.device)
    torch.cuda.synchronize(data_t.device)

    def index_dev():
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record(stream)
        eng.mpa_index_dev_queue(data_t, ranges, cap, None, jobs_t, index_t, tracks_t)
        end.record(stream)
        end.synchronize()
        return start.elapsed_time(end)

    def clocked(fn):
        def run():
            t = time.perf_counter()
            fn()
            return (time.perf_counter() - t) * 1e3
        return run
    calls = dict(index_dev_ms=index_dev,
                 index_host_ms=clocked(lambda: list(pool.map(packetizer.mpa_index, files))),
                 dev_ms=clocked(lambda: decode.decode_mpeg_files_dev(eng, data_t, ranges)),
                 host_ms=clocked(lambda: decode.decode_mpeg_files(eng, files, device=True)))
    times = {k: [] for k in calls}
    for rep in range(reps + 2):
        for k, fn in calls.items():
            t = fn()
            if rep >= 2:
                times[k].append(t)
    frames = int(index_t.cpu().numpy().view(nat.MPA_FILE_INDEX_DTYPE)["n_packets"].sum())
    out = dict(files=len(files), bytes=int(data_t.numel()), frames=frames, same_as_host=True, read_back_bytes=read_back)
    out.update({k: statistics.median(v) for k, v in times.items()})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    assert a.reps >= 5
    report = dict(card=card())
    print("card", report["card"], flush=True)
    with sb.Engine(0) as eng, concurrent.futures.ThreadPoolExecutor(16) as pool:
        for name, make in (("files_256", many_files), ("one_10000", one_long)):
            report[name] = r = measure(eng, make(), a.reps, pool)
            print(name, json.dumps(r), flush=True)
    print(json.dumps(report))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
