"""Time of the device FLAC index (symgpu_flac_index_dev) and of decode.decode_flac_files_dev (native FLAC files already in device
memory: frames found on the device, decoded from the job table in place) against the host-indexed path,
decode.decode_flac_files(device=True), in one invocation.

Inputs: 256 decodable files of 64 frames (16-bit stereo, 576-sample blocks; 16 distinct streams repeated), and one stream of
100 000 small frames (random bodies behind valid headers and CRC-16s, so only its index is timed: it shows that no file is walked
by one thread).  The files are uploaded once, back to back; the device calls start from resident bytes.

Reports, with the card name and power limit read in the same run (every time a median of --reps calls after 2 warm-up calls,
the kinds of call taken in turn):
  index_dev_ms    symgpu_flac_index_dev alone (jobs only, sized by the lengths // 8 bound), CUDA events on the engine's stream
                  around the call; this includes its one host wait, for the node count
  index_host_ms   packetizer.flac_index of every file on 16 host threads, host clock (the index phase of the host-indexed path)
  dev_ms          decode_flac_files_dev end to end, host clock (it ends in a device synchronise and the read-back of its results)
  host_ms         decode_flac_files(device=True) on the same files' bytes, host clock
  read_back_bytes of decode_flac_files_dev, and same_as_host: its samples and errors equal the host-indexed path's and the device
  index's infos and packets equal the host index's (checked before timing)

usage: python tools/measure_flac_device_files.py [--reps 5] [--out FILE.json]
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
from tests import _flac_corpus  # noqa: E402
from tests.test_flac_decode_gpu import _file, _frames  # noqa: E402

from measure_aac_files import card  # noqa: E402


def many_files():
    streams = []
    for k in range(16):
        pk, pcm = _frames(600 + k, 16, 2, 576, 64)
        streams.append(_file(pk, pcm, 16, 2, 576, 576)[0])
    return [streams[k % len(streams)] for k in range(256)]


def one_long():
    return [_flac_corpus.hundred_thousand()]


def upload(files):
    import torch
    ranges, at = [], 0
    for f in files:
        ranges.append((at, len(f)))
        at += len(f)
    return torch.from_numpy(np.frombuffer(b"".join(files), dtype=np.uint8).copy()).cuda(), ranges


def check(eng, files, data_t, ranges, pool, decodes):
    """Device index == host index per file; decode_flac_files_dev == decode_flac_files(device=True).  Returns its read_back_bytes."""
    packets_t, _, index, infos = eng.flac_index_dev(data_t, ranges)
    packets = packets_t.cpu().numpy().view(nat.FLAC_PACKET_DTYPE)
    for i, (info, want) in enumerate(pool.map(packetizer.flac_index, files)):
        a = int(index[i]["first_packet"])
        assert packets[a:a + len(want)].tobytes() == want.tobytes() and int(index[i]["n_packets"]) == len(want)
        assert infos[i].tobytes() == np.asarray(info).tobytes()
    if not decodes:
        return None
    e_d, s_d, e_h = {}, {}, {}
    got = decode.decode_flac_files_dev(eng, data_t, ranges, errors=e_d, stats=s_d)
    want = decode.decode_flac_files(eng, files, device=True, errors=e_h)
    assert e_d == e_h
    assert all(gr == wr and g.shape == w.shape and bool((g == w).all()) for (g, gr), (w, wr) in zip(got, want))
    return s_d["read_back_bytes"]


def measure(eng, files, reps, pool, decodes):
    import torch
    data_t, ranges = upload(files)
    read_back = check(eng, files, data_t, ranges, pool, decodes)
    r = np.array(ranges, dtype=np.uint64)
    cap = int((r[:, 1] // nat.FLAC_MIN_FRAME).sum())
    jobs_t = torch.empty(cap * nat.FLAC_JOB_DTYPE.itemsize, dtype=torch.uint8, device=data_t.device)
    index_t = torch.empty(len(files) * nat.FLAC_FILE_INDEX_DTYPE.itemsize, dtype=torch.uint8, device=data_t.device)
    infos_t = torch.empty(len(files) * nat.FLAC_STREAM_INFO_DTYPE.itemsize, dtype=torch.uint8, device=data_t.device)
    stream = torch.cuda.ExternalStream(eng.cuda_stream, device=data_t.device)
    torch.cuda.synchronize(data_t.device)

    def index_dev():
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record(stream)
        eng.flac_index_dev_queue(data_t, ranges, cap, None, jobs_t, index_t, infos_t)
        end.record(stream)
        end.synchronize()
        return start.elapsed_time(end)

    def clocked(fn):
        def run():
            t = time.perf_counter()
            fn()
            return (time.perf_counter() - t) * 1e3
        return run
    calls = dict(index_dev_ms=index_dev, index_host_ms=clocked(lambda: list(pool.map(packetizer.flac_index, files))))
    if decodes:
        calls.update(dev_ms=clocked(lambda: decode.decode_flac_files_dev(eng, data_t, ranges)),
                     host_ms=clocked(lambda: decode.decode_flac_files(eng, files, device=True)))
    times = {k: [] for k in calls}
    for rep in range(reps + 2):
        for k, fn in calls.items():
            t = fn()
            if rep >= 2:
                times[k].append(t)
    frames = int(index_t.cpu().numpy().view(nat.FLAC_FILE_INDEX_DTYPE)["n_packets"].sum())
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
        for name, make, decodes in (("files_256", many_files, True), ("one_100000", one_long, False)):
            report[name] = r = measure(eng, make(), a.reps, pool, decodes)
            print(name, json.dumps(r), flush=True)
    print(json.dumps(report))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
