#!/usr/bin/env python3
"""A mixed corpus through `symphonia_b200.decode.decode_any_files`: MP3, MPEG Layer II, ADTS AAC-LC, Ogg Vorbis and native FLAC files
from the test writers (seeded; a few distinct files per kind reused round-robin, shuffled, every file a stream of its own), decoded
in one call to interleaved samples of one format.

Measured, each as a host clock around a call that ends in engine.sync(), after every shape has run once, `--repeats` times with the
variants alternating inside every repeat (median, min and max printed):
  any_host / any_device            the whole corpus, device=False / device=True
  any_resident                     the whole corpus already in device memory (uploaded once before timing), through
                                   decode_any_files_dev: sniffed, indexed and decoded on the device
  any_host_lossy / any_device_lossy / decode_files_lossy
                                   the corpus without its FLAC files (decode_files does not take them) through decode_any_files
                                   and through decode_files (front-ends on host threads, one synthesis launch per codec)
  flac_host_s32 / flac_host_<fmt>  the FLAC files alone through decode_flac_files: what the narrower output saves on the way back
The card's name and power limit are read in the same run.  Needs a GPU; `--plan-only` runs the host halves (`*_files_plan`) and
reports counts -- files, jobs, bytes in, bytes out per format -- and no time.  NOT the headline measurement (bench.py is).
One JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from symphonia_b200 import _native as nat  # noqa: E402
from symphonia_b200 import decode  # noqa: E402
from tests import _mp3_bitstream as bw  # noqa: E402
from tests import _mpa12_bitstream as b12  # noqa: E402
from tests import test_flac_decode_gpu as tf  # noqa: E402
from tests import test_zz_adts_aac_to_pcm as ta  # noqa: E402
from tests import test_zz_ogg_vorbis_to_pcm as tv  # noqa: E402

FORMATS = {"f32": nat.FMT_F32, "s16": nat.FMT_S16, "s24": nat.FMT_S24, "s32": nat.FMT_S32, "u8": nat.FMT_U8}
DISTINCT = 3   # the Python writers are slow


def corpus(n_each, packets, seed=11):
    """{kind: n_each files of at least `packets` packets} and the shuffled list of all of them."""
    rng = np.random.default_rng(seed)
    mp3 = [b"".join(bw.gen_stream(rng, packets, version="1", mode=1, bitrate_idx=9, fill=(0.85, 1.0), pair_blocks=True)[0]) for _ in range(DISTINCT)]
    mp2 = [b"".join(b12.gen_layer2_frame(rng, "1", 12, 0, 1, mode_ext=k % 4)[0] for k in range(packets)) for _ in range(DISTINCT)]
    aac = [ta._file(40 + k, 44100, 2, n=packets)[0] for k in range(DISTINCT)]
    vorbis = [tv._file(40 + k, n_packets=packets)[0] for k in range(DISTINCT)]
    flac = []
    for k in range(DISTINCT):      # 16-bit stereo, 1152-sample blocks (the writer keeps 6 frames of 7 and one short block)
        pk, pcm = tf._frames(seed + k, 16, 2, 1152, packets * 7 // 6 + 2)
        flac.append(tf._file(pk, pcm, 16, 2, 1152, 1152)[0])
    by_kind = {name: [src[k % DISTINCT] for k in range(n_each)] for name, src in (("mp3", mp3), ("mp2", mp2), ("aac", aac), ("vorbis", vorbis), ("flac", flac))}
    files = [f for fs in by_kind.values() for f in fs]
    order = np.random.default_rng(seed + 1).permutation(len(files))
    return by_kind, [files[i] for i in order]


def plan_counts(by_kind, threads):
    """Per kind, from the host halves of the device decoders: files, jobs, bytes in, and output samples (the capacity the call reserves)."""
    plans = {"mp3": decode.mp3_files_plan(by_kind["mp3"], threads), "mp2": decode.mpa12_files_plan(by_kind["mp2"], threads),
             "aac": decode.aac_files_plan(by_kind["aac"], threads), "vorbis": decode.vorbis_files_plan(by_kind["vorbis"], threads),
             "flac": decode.flac_files_plan(by_kind["flac"], threads)}
    counts = {}
    for kind, p in plans.items():
        samples = int(p["out_cap"] if kind == "flac" else p["out_samples"])
        counts[kind] = dict(files=len(by_kind[kind]), failed=len(p["failed"]), jobs=len(p["jobs"]), bytes_in=int(p["data"].size), out_samples=samples,
                            bytes_out={name: samples * np.dtype(nat.FMT_NUMPY[f]).itemsize for name, f in FORMATS.items()})
    return counts


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True, check=True)
    name, limit = [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]
    return dict(name=name, power_limit_w=float(limit))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files-per-kind", type=int, default=64)
    ap.add_argument("--packets", type=int, default=100)
    ap.add_argument("--format", choices=sorted(FORMATS), default="s16")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    ap.add_argument("--plan-only", action="store_true")
    args = ap.parse_args()
    fmt = FORMATS[args.format]
    by_kind, files = corpus(args.files_per_kind, args.packets)
    lossy = [f for f in files if decode.sniff(f) != "flac"]
    out = {"workload": f"{args.files_per_kind} files each of MP3 128k joint stereo, Layer II 256k joint stereo, ADTS AAC-LC stereo, Ogg Vorbis, "
                       f"FLAC 16-bit stereo; at least {args.packets} packets per file; output {args.format}",
           "files": len(files), "file_bytes": sum(map(len, files)), "threads": args.threads, "host_cores_total": os.cpu_count(),
           "plan": plan_counts(by_kind, args.threads)}
    if args.plan_only:
        print(json.dumps(out))
        return
    import torch
    import symphonia_b200 as sb
    if not torch.cuda.is_available():
        sys.exit("any_files_bench: no CUDA device; the timings need one (--plan-only counts without)")
    out["device"] = card()
    # the corpus resident on the device, back to back, for decode_any_files_dev
    ranges, at = [], 0
    for f in files:
        ranges.append((at, len(f)))
        at += len(f)
    resident = torch.from_numpy(np.frombuffer(b"".join(files), dtype=np.uint8).copy()).cuda()
    with sb.Engine(0) as eng:
        kw = dict(threads=args.threads)
        variants = {"any_host": lambda: decode.decode_any_files(eng, files, fmt, **kw),
                    "any_device": lambda: decode.decode_any_files(eng, files, fmt, device=True, **kw),
                    "any_resident": lambda: decode.decode_any_files_dev(eng, resident, ranges, fmt),
                    "any_host_lossy": lambda: decode.decode_any_files(eng, lossy, fmt, **kw),
                    "any_device_lossy": lambda: decode.decode_any_files(eng, lossy, fmt, device=True, **kw),
                    "decode_files_lossy": lambda: decode.decode_files(eng, lossy, fmt, **kw),
                    "flac_host_s32": lambda: decode.decode_flac_files(eng, by_kind["flac"], fmt=nat.FMT_S32, **kw)}
        if fmt != nat.FMT_S32:
            variants["flac_host_" + args.format] = lambda: decode.decode_flac_files(eng, by_kind["flac"], fmt=fmt, **kw)
        results = {name: fn() for name, fn in variants.items()}            # warm-up: every shape once
        eng.sync()
        audio = {name: sum(r[0].shape[0] / r[1] for r in res if r[1]) for name, res in results.items()}
        nbytes = {name: int(sum(r[0].numel() * r[0].element_size() if hasattr(r[0], "numel") else r[0].nbytes for r in res)) for name, res in results.items()}
        for (a, ra), (b, rb) in zip(results["any_host_lossy"], results["decode_files_lossy"]):
            assert ra == rb and a.shape == b.shape and a.tobytes() == b.tobytes(), "decode_any_files and decode_files disagree on the lossy files"
        del results
        times = {name: [] for name in variants}
        for _ in range(args.repeats):
            for name, fn in variants.items():
                t0 = time.perf_counter()
                fn()
                eng.sync()
                times[name].append(time.perf_counter() - t0)
    out["repeats"] = args.repeats
    out["timing"] = "host clock around one call ended by engine.sync(); seconds"
    for name, ts in times.items():
        med = statistics.median(ts)
        out[name] = dict(median_s=med, min_s=min(ts), max_s=max(ts), audio_seconds=audio[name], audio_s_per_s=audio[name] / med, output_bytes=nbytes[name])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
