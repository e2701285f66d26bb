#!/usr/bin/env python
"""Secondary measurements: BASELINE configs[2] (AAC-LC 48 kHz stereo, 8192 frames) and configs[3]
(Vorbis 44.1 kHz stereo long/short mix, 8192 packets) on one GPU, device-resident inputs.
Prints one JSON line per codec with the same roofline arithmetic as bench.py (the headline metric
and the driver contract live in bench.py; this script feeds profiles/ and DESIGN.md)."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def _time_steps(eng, fn, steps, warmup):
    import torch
    ext = torch.cuda.ExternalStream(eng.cuda_stream)
    for i in range(warmup):
        fn(i)
    eng.sync()
    with torch.cuda.stream(ext):
        evs = []
        for i in range(steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn(warmup + i)
            b.record()
            evs.append((a, b))
    eng.sync()
    torch.cuda.synchronize()
    return float(np.mean([a.elapsed_time(b) for a, b in evs]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--codec", default="both", choices=["aac", "vorbis", "both", "mp3-short", "mixed", "mpa2", "flac", "all"])
    ap.add_argument("--tns", type=float, default=0.2)
    args = ap.parse_args()
    import torch
    import symphonia_b200 as sb
    from symphonia_b200 import workloads
    dev = torch.device("cuda", 0)
    eng = sb.Engine(0)
    peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]) if os.path.exists(
        os.path.join(ROOT, "MEASURED_PEAKS.json")) else 6650.0
    S, F, SETS = 64, 128, 4
    if args.codec in ("mp3-short", "all"):
        # SURVEY 8d worst case: 8192 streams x 1 frame -- every tile loads and stores its stream's state, which is
        # therefore counted in the algorithmic bytes (overlap 4608 B + 15 history slots 3840 B, read + written).
        S1 = 8192
        units, spectra, runs = workloads.mp3_batch(S1, 1, seed=workloads.SEED_BASE + 11)
        eng.mp3_streams_alloc(S1)
        sets = []
        for _ in range(SETS):
            sets.append((torch.from_numpy(units.view(np.uint8).reshape(-1).copy()).to(dev), torch.from_numpy(spectra).to(dev),
                         torch.empty((S1, 2, 1152), dtype=torch.float32, device=dev)))
        ms = _time_steps(eng, lambda i: eng.mp3_synth_dev(sets[i % SETS][0], sets[i % SETS][1], runs, sets[i % SETS][2]),
                         args.steps, args.warmup)
        algo = S1 * (workloads.MP3_ALGO_BYTES_PER_FRAME + 2 * (4608 + 3840))
        audio = workloads.mp3_audio_seconds(S1)
        ach = algo / (ms * 1e-3) / 1e9
        print(json.dumps({"codec": "mp3", "workload": "MP3 44.1kHz stereo, 8192 streams x 1 frame (state in and out of HBM for every frame)",
                          "value": audio / (ms * 1e-3), "unit": "audio-s/s", "kernel_ms": ms,
                          "roofline": {"bound": "hbm", "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak,
                                       "algorithmic_bytes_per_launch": algo}}), flush=True)
    if args.codec in ("mpa2", "all"):
        # SURVEY 8f N4: MPEG Layer II, 8192 frames (64 streams x 128), polyphase synthesis of the decoder's sub-band samples
        x, r2 = workloads.mpa12_batch(S, F, layer=2)
        eng.mp3_streams_alloc(S)
        sets = [(torch.from_numpy(x).to(dev), torch.empty((S * F, 2, 1152), dtype=torch.float32, device=dev)) for _ in range(SETS)]
        ms = _time_steps(eng, lambda i: eng.mpa12_synth_dev(sets[i % SETS][0], r2, 36, sets[i % SETS][1]), args.steps, args.warmup)
        algo = S * F * (2 * 32 * 36 * 4 + 2 * 1152 * 4)
        audio = S * F * 1152 / 44100.0
        ach = algo / (ms * 1e-3) / 1e9
        print(json.dumps({"codec": "mp2", "workload": "MPEG Layer II 44.1kHz stereo, 8192 frames (64 streams x 128), polyphase synthesis",
                          "value": audio / (ms * 1e-3), "unit": "audio-s/s", "kernel_ms": ms,
                          "roofline": {"bound": "hbm", "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak,
                                       "algorithmic_bytes_per_launch": algo}}), flush=True)
    if args.codec == "flac":  # not part of "all": the kernel's last fix has not been re-run on a GPU yet
        # SURVEY 8f N4: FLAC 16-bit stereo, 2048 frames of 4096 samples: prediction + decorrelation + scaling, in place
        NF, BS = 2048, 4096
        frames, subs, samples = workloads.flac_batch(64, BS, seed=workloads.SEED_BASE + 6)
        reps = NF // 64  # the 64 generated frames repeated (the generator's exact-integer encoder is slow)
        fr = np.tile(frames, reps)
        sb_ = np.tile(subs, reps)
        fr["first_subframe"] = np.arange(NF) * 2
        sb_["offset"] = np.arange(NF * 2, dtype=np.uint64) * BS
        smp = np.tile(samples, reps)
        d_fr = torch.from_numpy(fr.view(np.uint8).reshape(-1).copy()).to(dev)
        d_sb = torch.from_numpy(sb_.view(np.uint8).reshape(-1).copy()).to(dev)
        src = torch.from_numpy(smp).to(dev)
        work = [torch.empty_like(src) for _ in range(SETS)]

        for w in work:  # restoration is in place: every step starts from the residuals again
            w.copy_(src)
        # time copy alone, then copy + restore; the difference is the restoration
        ext = torch.cuda.ExternalStream(eng.cuda_stream)
        def timed(fn, n):
            with torch.cuda.stream(ext):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for i in range(n):
                    fn(i)
                b.record()
            eng.sync()
            torch.cuda.synchronize()
            return a.elapsed_time(b) / n
        def both(i):
            with torch.cuda.stream(ext):
                work[i % SETS].copy_(src)
            eng.flac_restore_dev(d_fr, NF, d_sb, NF * 2, work[i % SETS])
        def copy_only(i):
            with torch.cuda.stream(ext):
                work[i % SETS].copy_(src)
        timed(both, 3)
        ms = timed(both, args.steps) - timed(copy_only, args.steps)
        n_samples = int(sb_["n"].sum())
        algo = n_samples * 8 + NF * 2 * 144
        audio = float(sb_["n"][0::2].sum()) / 44100.0
        ach = algo / (ms * 1e-3) / 1e9
        print(json.dumps({"codec": "flac", "workload": "FLAC 16-bit stereo, 2048 frames x 4096 samples: prediction, decorrelation, scaling (in place)",
                          "value": audio / (ms * 1e-3), "unit": "audio-s/s", "kernel_ms": ms,
                          "roofline": {"bound": "hbm", "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak,
                                       "algorithmic_bytes_per_launch": algo}}), flush=True)
    if args.codec in ("mixed", "all"):
        # SURVEY 8d config 5 at 1/16 scale: 4096 streams x 16 frames, 50 % MP3 / 30 % AAC / 20 % Vorbis, on ONE context;
        # a step = the three launches back to back.
        Fm = 16
        n_mp3, n_aac, n_vor = 2048, 1229, 819
        mu, ms_, mr = workloads.mp3_batch(n_mp3, Fm, seed=workloads.SEED_BASE + 51)
        au, at, ac, ar = workloads.aac_batch(n_aac, Fm, seed=workloads.SEED_BASE + 52)
        wl = workloads.vorbis_batch(n_vor, Fm, seed=workloads.SEED_BASE + 53)
        eng.mp3_streams_alloc(n_mp3)
        eng.aac_streams_alloc(n_aac)
        eng.vorbis_streams_set(wl["streams"])
        eng.vorbis_floors_set(wl["floors"])
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        d_mu, d_ms, d_mp = t(mu.view(np.uint8).reshape(-1)), t(ms_), torch.empty((n_mp3 * Fm, 2, 1152), dtype=torch.float32, device=dev)
        d_au, d_at, d_ac = t(au.view(np.uint8).reshape(-1)), t(at.view(np.uint8).reshape(-1)), t(ac)
        d_ap = torch.empty((n_aac * Fm, 2, 1024), dtype=torch.float32, device=dev)
        d_vu, d_vy, d_vr = t(wl["units"].view(np.uint8).reshape(-1)), t(wl["floor_y"].view(np.int16)), t(wl["residue"])
        d_vp = torch.zeros((n_vor * Fm, 2, wl["slot"]), dtype=torch.float32, device=dev)

        def step(i):
            eng.mp3_synth_dev(d_mu, d_ms, mr, d_mp)
            eng.aac_synth_dev(d_au, d_at, len(at), d_ac, ar, d_ap)
            eng.vorbis_synth_dev(d_vu, d_vy, d_vr, wl["runs"], wl["slot"], d_vp)
        ms = _time_steps(eng, step, args.steps, args.warmup)
        audio = (workloads.mp3_audio_seconds(n_mp3 * Fm) + n_aac * Fm * 1024 / 48000.0 + float(wl["out_len"].sum()) / 44100.0)
        print(json.dumps({"codec": "mixed", "workload": "4096 streams x 16 frames on one context: 2048 MP3 + 1229 AAC-LC + 819 Vorbis "
                          "(SURVEY config 5 at 1/16 scale; 0.57 GB in + 0.57 GB out per step, far beyond the 50 MB L2 of an H100)",
                          "value": audio / (ms * 1e-3), "unit": "audio-s/s", "step_ms": ms, "audio_s_per_step": audio}), flush=True)
    if args.codec in ("aac", "both", "all"):
        units, tns, coeffs, runs = workloads.aac_batch(S, F, tns_prob=args.tns)
        eng.aac_streams_alloc(S)
        sets = []
        for _ in range(SETS):
            sets.append((torch.from_numpy(units.view(np.uint8).reshape(-1).copy()).to(dev),
                         torch.from_numpy(tns.view(np.uint8).reshape(-1).copy()).to(dev) if len(tns) else torch.zeros(8, device=dev),
                         torch.from_numpy(coeffs).to(dev), torch.empty((S * F, 2, 1024), dtype=torch.float32, device=dev)))
        ms = _time_steps(eng, lambda i: eng.aac_synth_dev(sets[i % SETS][0], sets[i % SETS][1], len(tns), sets[i % SETS][2],
                                                          runs, sets[i % SETS][3]), args.steps, args.warmup)
        algo = S * F * workloads.AAC_ALGO_BYTES_PER_FRAME
        audio = S * F * 1024 / 48000.0
        ach = algo / (ms * 1e-3) / 1e9
        print(json.dumps({"codec": "aac-lc", "workload": "AAC-LC 48kHz stereo, 8192 frames, TNS in %.0f%% of channel-frames" % (100 * args.tns),
                          "value": audio / (ms * 1e-3), "unit": "audio-s/s", "kernel_ms": ms, "n_tns_filters": int(len(tns)),
                          "roofline": {"bound": "hbm", "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak,
                                       "algorithmic_bytes_per_launch": algo}}), flush=True)
    if args.codec in ("vorbis", "both", "all"):
        wl = workloads.vorbis_batch(S, F)
        eng.vorbis_streams_set(wl["streams"])
        eng.vorbis_floors_set(wl["floors"])
        slot = wl["slot"]
        sets = []
        for _ in range(SETS):
            sets.append((torch.from_numpy(wl["units"].view(np.uint8).reshape(-1).copy()).to(dev),
                         torch.from_numpy(wl["floor_y"].view(np.int16).copy()).to(dev), torch.from_numpy(wl["residue"]).to(dev),
                         torch.zeros((S * F, 2, slot), dtype=torch.float32, device=dev)))
        ms = _time_steps(eng, lambda i: eng.vorbis_synth_dev(sets[i % SETS][0], sets[i % SETS][1], sets[i % SETS][2],
                                                             wl["runs"], slot, sets[i % SETS][3]), args.steps, args.warmup)
        n2 = np.where(wl["units"]["block_flag"] == 1, 1024, 128)
        algo = int((n2 * 4 * 2 + 2 * 65 * 2 + 16 + wl["out_len"] * 4 * 2).sum())
        audio = float(wl["out_len"].sum()) / 44100.0
        ach = algo / (ms * 1e-3) / 1e9
        print(json.dumps({"codec": "vorbis", "workload": "Vorbis 44.1kHz stereo coupled, blocksizes 256/2048, 8192 packets "
                          "(%.0f%% long)" % (100 * float((n2 == 1024).mean())),
                          "value": audio / (ms * 1e-3), "unit": "audio-s/s", "kernel_ms": ms,
                          "roofline": {"bound": "hbm", "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak,
                                       "algorithmic_bytes_per_launch": algo}}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
