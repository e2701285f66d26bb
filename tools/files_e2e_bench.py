#!/usr/bin/env python3
"""End to end from FILE BYTES for all three codecs of the north star (SURVEY §8f N1 + N2 in front of the synthesis kernels): a corpus
of MP3, ADTS AAC-LC and Ogg Vorbis files through `symphonia_b200.decode.decode_files` -- front-ends on host threads, one synthesis
launch per codec, output stage per file -- host wall clock around the whole call, and the plan (CPU) share on its own.

NOT part of the headline measurement (bench.py is).  `--plan-only` runs the CPU half without a GPU.  One JSON line."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from symphonia_b200 import _native as nat  # noqa: E402
from symphonia_b200 import decode  # noqa: E402
from tests import _mp3_bitstream as bw  # noqa: E402
from tests import test_zz_adts_aac_to_pcm as ta  # noqa: E402
from tests import test_zz_ogg_vorbis_to_pcm as tv  # noqa: E402


def corpus(n_each, frames):
    """A few distinct files per codec (the Python writers are slow), reused round-robin; every file is still a stream of its own."""
    rng = np.random.default_rng(11)
    mp3 = [b"".join(bw.gen_stream(rng, frames, version="1", mode=1, bitrate_idx=9, fill=(0.85, 1.0), pair_blocks=True)[0]) for _ in range(3)]
    aac = [ta._file(40 + k, 44100, 2, n=frames)[0] for k in range(3)]
    vor = [tv._file(40 + k, n_packets=frames)[0] for k in range(3)]
    return [src[k % 3] for src in (mp3, aac, vor) for k in range(n_each)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files-per-codec", type=int, default=64)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    ap.add_argument("--plan-only", action="store_true")
    args = ap.parse_args()
    files = corpus(args.files_per_codec, args.frames)
    out = {"workload": f"{args.files_per_codec} files each of MP3 128k joint stereo, ADTS AAC-LC stereo, Ogg Vorbis; {args.frames} packets per file",
           "file_bytes": sum(map(len, files)), "threads": args.threads, "host_cores_total": os.cpu_count()}
    best = 1e9
    for _ in range(3):
        t0 = time.perf_counter()
        plans, batches = decode.plan_files(files, threads=args.threads)
        best = min(best, time.perf_counter() - t0)
    audio = sum(p["total_frames"] / p["sample_rate"] for p in plans)
    out.update(audio_seconds=audio, plan_s=best, plan_audio_s_per_s=audio / best,
               units={k: int(len(b["runs"]) and sum(int(r["n_packets" if k == "vorbis" else "n_frames"]) for r in b["runs"])) for k, b in batches.items()})
    if not args.plan_only:
        import symphonia_b200 as sb
        with sb.Engine(0) as eng:
            decode.decode_files(eng, files, nat.FMT_S16, threads=args.threads)   # warm-up: tables, allocations
            best = 1e9
            for _ in range(5):
                t0 = time.perf_counter()
                res = decode.decode_files(eng, files, nat.FMT_S16, threads=args.threads)
                best = min(best, time.perf_counter() - t0)
            out.update(decode_files_s=best, e2e_audio_s_per_s=audio / best, output_bytes=int(sum(r[0].nbytes for r in res)))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
