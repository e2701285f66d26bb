"""Throughput of the device Ogg page index (symgpu_ogg_index_dev, Engine.ogg_index_dev) against the host index
(symgpu_ogg_index, packetizer.ogg_index) on the same files, in one invocation.

Corpus: 256 Ogg Vorbis writer files (tests/_vorbis_corpus.py, 44.1 kHz stereo, blocks of 256 / 2048 samples, 64 packets each);
4 distinct streams written once and repeated, as tools/measure_vorbis_files.py does.  Reports, with the card name and power
limit read in the same run, the median and min-max over --iters alternating repeats of:
  device: one symgpu_ogg_index_dev call with the tables' capacities known, files already resident, by CUDA events; GB/s of
    file bytes
  host: packetizer.ogg_index of every file on 16 host threads, by the host clock
  many streams: Engine.ogg_index_dev (capacities known, one call and its readback) on one 3 MB file of 37 500 small pages that
    announce 30 000 serials (tests/_ogg_corpus.many_serials), by the host clock, against packetizer.ogg_index of that file
Both tables are checked equal, file by file, before anything is timed.

usage: python tools/measure_ogg_device_files.py [--iters 20] [--out FILE.json]
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
from symphonia_b200 import packetizer  # noqa: E402
from tests import _ogg_corpus  # noqa: E402
from tests import _vorbis_corpus as corpus  # noqa: E402


def writer_files(n_files, n_packets, distinct=4, seed=1):
    out = []
    for d in range(distinct):
        s, pk = corpus.writer(seed + d, n_packets, channels=2, bs_exp=(8, 11))
        out.append(corpus.ogg(s, pk, seed + d))
    return [out[i % distinct] for i in range(n_files)]


def stats(xs):
    return dict(median=float(np.median(xs)), min=float(np.min(xs)), max=float(np.max(xs)))


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--files", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    files = writer_files(a.files, 64)
    n_bytes = sum(len(f) for f in files)
    buf = np.frombuffer(b"".join(files), dtype=np.uint8)
    offs = np.concatenate([[0], np.cumsum([len(f) for f in files])[:-1]])
    ranges = np.stack([offs, [len(f) for f in files]], axis=1).astype(np.uint64)
    with sb.Engine(0) as eng:
        dev = torch.device("cuda", eng.device)
        data_t = torch.from_numpy(buf.copy()).to(dev)
        packets_t, pieces_t, index = eng.ogg_index_dev(data_t, ranges)
        cap_p, cap_q = packets_t.numel() // nat.OGG_PACKET_DTYPE.itemsize, pieces_t.numel() // nat.PIECE_DTYPE.itemsize
        pk = packets_t.cpu().numpy().view(nat.OGG_PACKET_DTYPE)
        pc = pieces_t.cpu().numpy().view(nat.PIECE_DTYPE)
        for i, f in enumerate(files):
            wp, wq = packetizer.ogg_index(f)
            r = index[i]
            assert pk[int(r["first_packet"]):int(r["first_packet"]) + int(r["n_packets"])].tobytes() == wp.tobytes()
            assert pc[int(r["first_piece"]):int(r["first_piece"]) + int(r["n_pieces"])].tobytes() == wq.tobytes()
        stream = torch.cuda.ExternalStream(eng.cuda_stream, device=dev)
        index_t = torch.empty(len(files) * nat.OGG_FILE_INDEX_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        rr = np.ascontiguousarray(ranges).view(nat.FILE_RANGE_DTYPE).reshape(-1)
        L = nat.lib()
        import ctypes
        torch.cuda.current_stream(dev).synchronize()   # index_t was allocated on torch's stream, the calls run on the engine's

        def device_call():
            rc = L.symgpu_ogg_index_dev(eng._ctx, ctypes.c_void_p(data_t.data_ptr()), data_t.numel(), ctypes.c_void_p(rr.ctypes.data), len(rr),
                                        ctypes.c_void_p(packets_t.data_ptr()), cap_p, ctypes.c_void_p(pieces_t.data_ptr()), cap_q,
                                        ctypes.c_void_p(index_t.data_ptr()))
            assert rc == 0
        pool = concurrent.futures.ThreadPoolExecutor(16)
        for _ in range(3):
            device_call()
            list(pool.map(packetizer.ogg_index, files))
        eng.sync()
        dev_ms, host_ms = [], []
        for _ in range(a.iters):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            device_call()
            e1.record(stream)
            e1.synchronize()
            dev_ms.append(e0.elapsed_time(e1))
            t = time.perf_counter()
            list(pool.map(packetizer.ogg_index, files))
            host_ms.append((time.perf_counter() - t) * 1e3)
        pool.shutdown()
        many = _ogg_corpus.many_serials(30000, seed=36)
        many_t = torch.from_numpy(np.frombuffer(many, dtype=np.uint8).copy()).to(dev)
        mp, mq, mix = eng.ogg_index_dev(many_t, [(0, len(many))])
        assert mp.cpu().numpy().tobytes() == packetizer.ogg_index(many)[0].tobytes()
        many_dev, many_host = [], []
        for _ in range(5):
            t = time.perf_counter()
            eng.ogg_index_dev(many_t, [(0, len(many))], int(mix["n_packets"][0]), int(mix["n_pieces"][0]))
            many_dev.append((time.perf_counter() - t) * 1e3)
            t = time.perf_counter()
            packetizer.ogg_index(many)
            many_host.append((time.perf_counter() - t) * 1e3)
    res = dict(gpu=gpu, files=len(files), bytes=n_bytes, packets=int(index["n_packets"].sum()), iters=a.iters,
               device_index_ms=stats(dev_ms), device_index_gbps=n_bytes / (float(np.median(dev_ms)) * 1e-3) / 1e9,
               host_index_16_threads_ms=stats(host_ms),
               many_streams=dict(bytes=len(many), serials=int(len(np.unique(mp.cpu().numpy().view(nat.OGG_PACKET_DTYPE)["serial"]))),
                                 device_call_ms=stats(many_dev), host_index_ms=stats(many_host)))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
