#!/usr/bin/env python
"""A/B of the MP3 kernel variants on the bench shape (8192 frames, 64 streams x 128): device-resident inputs, rotating
buffer sets, CUDA events; every variant's PCM is compared bit for bit with the first-generation kernel's.
usage: tools/mp3_variant_bench.py [variant ...]     variant = v1 | <warps>:<mode>"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import symphonia_b200 as sb  # noqa: E402
from symphonia_b200 import workloads  # noqa: E402

variants = sys.argv[1:] or ["v1", "auto", "12:33", "12:81"]
dev = torch.device("cuda", 0)
S, F = 64, 128
shapes = {"bench": (S, F), "serving": (8192, 1)}
lib = sb.lib()
res = {}
ref = {}
for shape, (s_, f_) in shapes.items():
    units, spectra, runs = workloads.mp3_batch(s_, f_, seed=workloads.SEED_BASE + 1)
    for v in variants:
        if v in ("v1", "auto"):
            os.environ["SYMGPU_MP3_KERNEL"] = v
        else:
            os.environ["SYMGPU_MP3_KERNEL"] = "v2"
            nw, mode = (int(x) for x in v.split(":"))
            assert lib.symgpu_debug_mp3_v2_variant(nw, mode) == 1, v
        eng = sb.Engine(0)
        eng.mp3_streams_alloc(s_)
        ext = torch.cuda.ExternalStream(eng.cuda_stream)
        sets = [(torch.from_numpy(units.view(np.uint8).reshape(-1).copy()).to(dev), torch.from_numpy(spectra).to(dev),
                 torch.zeros((s_ * f_, 2, 1152), dtype=torch.float32, device=dev)) for _ in range(4)]
        eng.mp3_synth_dev(sets[0][0], sets[0][1], runs, sets[0][2])
        eng.sync()
        pcm = sets[0][2].cpu().numpy().view(np.uint32)
        if shape not in ref:
            ref[shape] = pcm
        same = bool((pcm == ref[shape]).all())
        for i in range(5):
            eng.mp3_synth_dev(sets[i % 4][0], sets[i % 4][1], runs, sets[i % 4][2])
        eng.sync()
        with torch.cuda.stream(ext):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(100):
                eng.mp3_synth_dev(sets[i % 4][0], sets[i % 4][1], runs, sets[i % 4][2])
            b.record()
        eng.sync()
        torch.cuda.synchronize()
        res[f"{shape}/{v}"] = {"us": round(a.elapsed_time(b) * 10.0, 1), "same_as_first": same}
        print(shape, v, res[f"{shape}/{v}"], flush=True)
        del sets
        eng.close()
print(json.dumps(res))
