"""Time of the FLAC-in-Ogg many-file calls against native FLAC twins holding the same frames, in one invocation:
decode.decode_ogg_flac_files(device=True) (host index) and decode.decode_ogg_flac_files_dev (pages, identification packets and jobs
on the device), against decode.decode_flac_files(device=True) and decode.decode_flac_files_dev on the twins.

Inputs: 256 decodable Ogg FLAC files of 54 frames (16-bit stereo, 576-sample blocks, a comment packet, pages of random fill; 16
distinct streams repeated) and their native twins (tests/_ogg_flac_corpus.py).  Each set is uploaded once, back to back; the
resident calls start from resident bytes.

Reports, with the card name and power limit read in the same run (every time a median of --reps calls after 2 warm-up calls,
the kinds of call taken in turn; each a host clock around the whole call, which ends in a device synchronise and the read-back
of its results):
  ogg_host_ms     decode_ogg_flac_files(device=True) on the Ogg files
  ogg_dev_ms      decode_ogg_flac_files_dev on the resident Ogg files
  flac_host_ms    decode_flac_files(device=True) on the twins
  flac_dev_ms     decode_flac_files_dev on the resident twins
  ogg_dev_kernel_ms   CUDA events on the engine's stream around decode_ogg_flac_files_dev (its host waits included)
  ogg_plan_ms     decode.ogg_flac_files_plan alone: the host index of the host-indexed call (pages, gather, the FLAC rules, the job
                  table), on the default host threads
  flac_plan_ms    decode.flac_files_plan alone on the twins: the same phase of decode_flac_files
  read_back_bytes of decode_ogg_flac_files_dev, launches per call, and same_as_twins: every call's samples equal the twins'
  (checked before timing)

usage: python tools/measure_ogg_flac_files.py [--reps 5] [--out FILE.json]
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
from symphonia_b200 import decode  # noqa: E402
from tests import _ogg_flac_corpus as oc  # noqa: E402

from measure_aac_files import card  # noqa: E402


def files():
    ogg, twins = [], []
    for k in range(16):
        frames = oc.frames(700 + k, 16, 2, 576, 63)
        data = oc.ogg([oc.ident(oc.info_block(576, 2, 16)), oc.comment()] + frames, 700 + k)
        ogg.append(data)
        twins.append(oc.twin(data))
    return [ogg[k % 16] for k in range(256)], [twins[k % 16] for k in range(256)]


def upload(fs):
    import torch
    ranges, at = [], 0
    for f in fs:
        ranges.append((at, len(f)))
        at += len(f)
    return torch.from_numpy(np.frombuffer(b"".join(fs), dtype=np.uint8).copy()).cuda(), ranges


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    assert a.reps >= 5
    report = dict(card=card())
    print("card", report["card"], flush=True)
    ogg, twins = files()
    with sb.Engine(0) as eng:
        ogg_t, ogg_r = upload(ogg)
        twin_t, twin_r = upload(twins)
        want = decode.decode_flac_files(eng, twins, device=True)
        stats = {}
        before = eng.launch_count
        got = [decode.decode_ogg_flac_files(eng, ogg, device=True), decode.decode_ogg_flac_files_dev(eng, ogg_t, ogg_r, stats=stats),
               decode.decode_flac_files_dev(eng, twin_t, twin_r)]
        launches = eng.launch_count - before
        for g in got:
            assert all(gr == wr and g_.shape == w.shape and bool((g_ == w).all()) for (g_, gr), (w, wr) in zip(g, want))
        stream = torch.cuda.ExternalStream(eng.cuda_stream, device=ogg_t.device)

        def events():
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record(stream)
            decode.decode_ogg_flac_files_dev(eng, ogg_t, ogg_r)
            end.record(stream)
            end.synchronize()
            return start.elapsed_time(end)

        def clocked(fn):
            def run():
                t = time.perf_counter()
                fn()
                return (time.perf_counter() - t) * 1e3
            return run
        calls = dict(ogg_host_ms=clocked(lambda: decode.decode_ogg_flac_files(eng, ogg, device=True)),
                     ogg_dev_ms=clocked(lambda: decode.decode_ogg_flac_files_dev(eng, ogg_t, ogg_r)),
                     flac_host_ms=clocked(lambda: decode.decode_flac_files(eng, twins, device=True)),
                     flac_dev_ms=clocked(lambda: decode.decode_flac_files_dev(eng, twin_t, twin_r)),
                     ogg_dev_kernel_ms=events,
                     ogg_plan_ms=clocked(lambda: decode.ogg_flac_files_plan(ogg)),
                     flac_plan_ms=clocked(lambda: decode.flac_files_plan(twins)))
        times = {k: [] for k in calls}
        for rep in range(a.reps + 2):
            for k, fn in calls.items():
                t = fn()
                if rep >= 2:
                    times[k].append(t)
    report.update(files=len(ogg), ogg_bytes=int(ogg_t.numel()), twin_bytes=int(twin_t.numel()), frames=int(sum(len(w) for w, _ in want) // 576),
                  same_as_twins=True, read_back_bytes=stats["read_back_bytes"], launches_three_calls=launches)
    report.update({k: statistics.median(v) for k, v in times.items()})
    print(json.dumps(report))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
