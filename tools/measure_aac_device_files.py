"""Time of the device ADTS index (symgpu_adts_index_dev) and of decode.decode_aac_files_dev (ADTS AAC-LC files already in device
memory: frames indexed on the device, decoded from the job table in place) against the host-indexed paths, in one invocation.

Corpora: those of tools/measure_aac_files.py -- writer 256 files x 64 frames, quiet 256 x 64, long 4 x 10 000 -- and one file of
40 000 frames.  The files are uploaded once, back to back; the device calls start from resident bytes.

Reports, with the card name and power limit read in the same run (every time a median of --reps calls after 2 warm-up calls,
the four kinds of call taken in turn):
  index_dev_ms    symgpu_adts_index_dev alone (jobs only, sized by the lengths // 7 bound), CUDA events on the engine's stream
                  around the call; this includes its one host wait, for the candidate count
  index_host_ms   packetizer.adts_index of every file on 16 host threads, host clock
  dev_ms          decode_aac_files_dev end to end, host clock (it ends in a device synchronise and the read-back of its results)
  host_ms         decode_aac_files(device=True) on the same files' bytes, host clock
  read_back_bytes of decode_aac_files_dev, and whether its samples, errors and status equal the host-indexed path's and the
  device index's packets equal the host index's (checked before timing)

usage: python tools/measure_aac_device_files.py [--reps 5] [--out FILE.json]
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

from measure_aac_files import card, long_files, quiet_files, writer_files  # noqa: E402


def upload(files):
    import torch
    ranges, at = [], 0
    for f in files:
        ranges.append((at, len(f)))
        at += len(f)
    return torch.from_numpy(np.frombuffer(b"".join(files), dtype=np.uint8).copy()).cuda(), ranges


def check(eng, files, data_t, ranges, pool):
    """Device index == host index per file; decode_aac_files_dev == decode_aac_files(device=True).  Returns its read_back_bytes."""
    packets_t, _, index = eng.adts_index_dev(data_t, ranges)
    packets = packets_t.cpu().numpy().view(nat.ADTS_PACKET_DTYPE)
    for i, (want, stop) in enumerate(pool.map(packetizer.adts_index, files)):
        a = int(index[i]["first_packet"])
        assert packets[a:a + len(want)].tobytes() == want.tobytes() and int(index[i]["n_packets"]) == len(want) and int(index[i]["stop"]) == stop
    e_d, s_d, e_h, s_h = {}, {}, {}, {}
    got = decode.decode_aac_files_dev(eng, data_t, ranges, errors=e_d, stats=s_d)
    want = decode.decode_aac_files(eng, files, device=True, errors=e_h, stats=s_h)
    assert e_d == e_h and s_d["status"].tobytes() == s_h["status"].tobytes() and s_d["n_redecoded"] == s_h["n_redecoded"]
    assert all(gr == wr and g.shape == w.shape and bool((g == w).all()) for (g, gr), (w, wr) in zip(got, want))
    return s_d["read_back_bytes"]


def measure(eng, files, reps, pool):
    import torch
    data_t, ranges = upload(files)
    read_back = check(eng, files, data_t, ranges, pool)
    r = np.array(ranges, dtype=np.uint64)
    cap = int((r[:, 1] // 7).sum())
    jobs_t = torch.empty(cap * nat.PIECE_DTYPE.itemsize, dtype=torch.uint8, device=data_t.device)
    index_t = torch.empty(len(files) * nat.ADTS_FILE_INDEX_DTYPE.itemsize, dtype=torch.uint8, device=data_t.device)
    stream = torch.cuda.ExternalStream(eng.cuda_stream, device=data_t.device)
    torch.cuda.synchronize(data_t.device)

    def index_dev():
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record(stream)
        eng.adts_index_dev_queue(data_t, ranges, cap, None, jobs_t, index_t)
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
                 index_host_ms=clocked(lambda: list(pool.map(packetizer.adts_index, files))),
                 dev_ms=clocked(lambda: decode.decode_aac_files_dev(eng, data_t, ranges)),
                 host_ms=clocked(lambda: decode.decode_aac_files(eng, files, device=True)))
    times = {k: [] for k in calls}
    for rep in range(reps + 2):
        for k, fn in calls.items():
            t = fn()
            if rep >= 2:
                times[k].append(t)
    frames = int(index_t.cpu().numpy().view(nat.ADTS_FILE_INDEX_DTYPE)["n_packets"].sum())
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
    corpora = (("writer", lambda: writer_files(256, 64)[0]), ("quiet", lambda: quiet_files(256, 64)[0]),
               ("long", lambda: long_files(4, 10000)[0]), ("one_40000", lambda: long_files(1, 40000)[0]))
    with sb.Engine(0) as eng, concurrent.futures.ThreadPoolExecutor(16) as pool:
        for name, make in corpora:
            report[name] = r = measure(eng, make(), a.reps, pool)
            print(name, json.dumps(r), flush=True)
    print(json.dumps(report))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
