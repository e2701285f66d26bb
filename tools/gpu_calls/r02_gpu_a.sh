#!/bin/bash
# Round 2, GPU call A: parity of the v2 MP3 kernel + every previously gated test, A/B bench v2 vs v1, ncu of v2.
cd "$(dirname "$0")/../.."
tag=${1:-r02a}
out=gpurun_out
mkdir -p $out
python -c "import __graft_entry__ as g; g.build()" > $out/${tag}_build.log 2>&1 || { tail -20 $out/${tag}_build.log; exit 1; }
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,power.draw --format=csv > $out/${tag}_smi.txt
# 1. MP3 parity first (the new kernel), stop at first failure to keep the log short
timeout 900 python -m pytest tests/test_mp3_parity_gpu.py -m gpu -x -q 2>&1 | tail -25 | tee $out/${tag}_pytest_mp3.txt
# 2. the whole GPU suite, no -x
timeout 1500 python -m pytest tests -m gpu -q 2>&1 | tail -60 | tee $out/${tag}_pytest_gpu.txt
# 4. A/B bench
timeout 400 python bench.py --steps 20 --warmup 5 > $out/${tag}_bench_v2.json 2>$out/${tag}_bench_v2.err
SYMGPU_MP3_KERNEL=v1 timeout 400 python bench.py --steps 20 --warmup 5 --no-cpu-baseline > $out/${tag}_bench_v1.json 2>$out/${tag}_bench_v1.err
python - <<PY
import json
for v in ("v2","v1"):
    try:
        d=json.load(open("$out/${tag}_bench_%s.json" % v))
        print(v, "value", round(d["value"]), "kernel_ms", round(d["roofline"]["kernel_ms"],4), "frac", round(d["roofline"]["frac"],4), "e2e_ms", round(d["e2e"]["ms_per_step"],3), d["clocks"])
    except Exception as e:
        print(v, "failed", e)
PY
# 5. launch list + full capture of the v2 kernel
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -c 200 --csv --log-file $out/${tag}_mp3_launches.csv python bench.py --steps 10 --warmup 3 --no-cpu-baseline > /dev/null 2>&1
timeout 400 ncu --set full --clock-control none --import-source on -k regex:mp3v2_synth -c 1 -s 4 -o $out/${tag}_prof_mp3 -f python bench.py --steps 3 --warmup 3 --no-cpu-baseline > $out/${tag}_prof_mp3.log 2>&1
tail -2 $out/${tag}_prof_mp3.log
ls -la $out | tail -20
