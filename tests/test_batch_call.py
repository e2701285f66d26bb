"""The host-side rules every many-file device decoder shares (symphonia_b200/csrc/batch_call.h), on the CPU.

tests/cpp/batch_call_driver.cpp runs the group rules and the merge of written output ranges; it is built plainly and once more
with AddressSanitizer + UndefinedBehaviorSanitizer.  The group cases are the ones the GPU argument-error tests pin for each codec;
the merge is checked against a numpy model of the written bytes."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "symphonia_b200", "csrc")
OK, LIMIT, ARG = 0, 3, 6


@pytest.fixture(scope="module", params=["plain", "sanitized"])
def run(request, tmp_path_factory):
    d = tmp_path_factory.mktemp("batch_call")
    exe = str(d / request.param)
    cmd = ["g++", "-std=c++17", "-Wall", "-I/usr/local/cuda/include", f"-I{CSRC}", "-o", exe, os.path.join(ROOT, "tests", "cpp", "batch_call_driver.cpp")]
    cmd += ["-O2"] if request.param == "plain" else ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"]
    subprocess.check_call(cmd)

    def go(lines):
        res = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=600,
                             env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=1"))
        assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
        return res.stdout.splitlines()
    return go


def _ranges(n_jobs, groups):
    return f"ranges {n_jobs} {len(groups)} " + " ".join(f"{f} {n}" for f, n in groups)


def _slots(n_allocated, slots):
    return f"slots {n_allocated} {len(slots)} " + " ".join(map(str, slots))


def test_group_rules(run):
    cases = [
        (_ranges(4, [(0, 2), (2, 2)]), OK),
        (_ranges(4, [(0, 3), (2, 2)]), ARG),                  # overlapping groups
        (_ranges(4, [(2, 2), (0, 3)]), ARG),                  # the same, out of table order
        (_ranges(4, [(0, 4), (2, 0), (4, 0)]), OK),           # empty groups may sit anywhere inside the table
        (_ranges(4, [(0, 4), (5, 0)]), ARG),                  # ... but not past its end
        (_ranges(4, [(3, 2)]), ARG),                          # jobs beyond the table
        (_ranges(8, [(4, 4), (0, 4), (8, 0)]), OK),
        (_ranges(2**32, [(2**32 - 1, 1), (0, 2**32 - 1)]), OK),
        (_ranges(0, []), OK),
        (_slots(4, [0, 1]), OK),
        (_slots(4, [1, 1]), ARG),                             # duplicate slot
        (_slots(4, [0, 4]), LIMIT),                           # slot not allocated
        (_slots(4, [4, 4]), ARG),                             # a duplicate is reported before the allocation
        (_slots(0, []), OK),
        ("region 0 9216 9216", OK),
        ("region 2 9216 9216", LIMIT),                        # region beyond out
        ("region 9216 0 9216", OK),
        ("region 9217 0 9216", LIMIT),                        # out_offset > out_samples
        (f"region {2**64 - 1} 1 9216", LIMIT),                # no wrap-around in out_samples - out_offset
        (f"region 1 {2**64 - 1} 9216", LIMIT),
        (f"region 0 {2**64 - 1} {2**64 - 1}", OK),
    ]
    got = run([c for c, _ in cases])
    assert [int(g) for g in got] == [want for _, want in cases], [(c, g) for (c, _), g in zip(cases, got)]


def test_jobs_in_bytes(run):
    n = 1000
    cases = [
        (f"jobs {n} 4 0 250 250 250 500 250 750 250", 1),
        (f"jobs {n} 4 0 250 250 250 500 250 750 {n}", 0),     # job outside bytes
        (f"jobs {n} 1 {n} 0", 1),
        (f"jobs {n} 1 {n + 1} 0", 0),
        (f"jobs {n} 1 {2**64 - 1} 2", 0),                     # no wrap-around in offset + len
        ("jobs 0 0", 1),
    ]
    assert [int(g) for g in run([c for c, _ in cases])] == [want for _, want in cases]


def _model(ranges, size):
    written = np.zeros(size, dtype=bool)
    for b, e in ranges:
        written[b:e] = True
    return written


@pytest.mark.parametrize("seed", range(4))
def test_merge_equals_the_written_bytes(run, seed):
    rng = np.random.default_rng(seed)
    tables, lines = [], []
    for t in range(300):
        k = int(rng.integers(0, 24))
        size = int(rng.choice([16, 64, 4096]))
        b = rng.integers(0, size, k)
        e = np.minimum(b + rng.integers(0, size // 4 + 1, k), size)
        pick = rng.random(k)
        e = np.where(pick < 0.15, b, e)                                    # empty ranges
        if k > 1:
            b[1] = np.where(pick[1] < 0.5, e[0], b[1])                     # one touching its neighbour
            b[-1], e[-1] = (b[0], max(b[0], e[0] - 1)) if pick[-1] < 0.5 else (b[-1], e[-1])   # one nested
        r = list(zip(b.tolist(), e.tolist()))
        tables.append((r, size))
        lines.append(f"merge {k} " + " ".join(f"{x} {y}" for x, y in r))
    for (r, size), out in zip(tables, run(lines)):
        v = [int(x) for x in out.split()]
        m = list(zip(v[1::2], v[2::2]))
        assert len(m) == v[0]
        assert all(x < y for x, y in m), (r, m)                            # no empty range
        assert all(m[i][1] < m[i + 1][0] for i in range(len(m) - 1)), (r, m)   # sorted, disjoint and not touching
        assert (_model(m, size) == _model(r, size)).all(), (r, m)
