"""The schedule of the device Ogg page index (symphonia_b200/csrc/ogg_index_kernel.cu), on the CPU.

tests/cpp/ogg_index_driver.cpp runs its steps -- a successor for every capture pattern found on its own, the chain from byte 0,
the logical streams walked one serial after another -- through the shared functions of include/symgpu/packetizer.hpp, and must
give the packets and pieces of symgpu_ogg_index on every file of tests/_ogg_corpus.  It is built plainly and once more with
AddressSanitizer + UndefinedBehaviorSanitizer.  The shared page end trims and Vorbis packet timer are checked against the C
entry points."""
import os
import subprocess

import numpy as np
import pytest

from tests import _ogg_corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", params=["plain", "sanitized"])
def run(request, tmp_path_factory):
    d = tmp_path_factory.mktemp("ogg_index")
    exe = str(d / request.param)
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "ogg_index_driver.cpp")]
    cmd += ["-O2"] if request.param == "plain" else ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"]
    subprocess.check_call(cmd)

    def go(lines):
        res = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=600,
                             env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=1"))
        assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
        blocks, cur = [], []
        for line in res.stdout.splitlines():
            if line == "end":
                blocks.append(cur)
                cur = []
            else:
                cur.append(line)
        return blocks
    go.dir = d
    return go


def host_lines(data):
    import ctypes

    from symphonia_b200 import _native as nat
    from symphonia_b200 import packetizer
    packets, pieces = packetizer.ogg_index(data)
    a = np.frombuffer(data, dtype=np.uint8)
    n, m = ctypes.c_size_t(0), ctypes.c_size_t(0)
    rc = nat.lib().symgpu_ogg_index(ctypes.c_void_p(a.ctypes.data) if a.size else None, a.size, None, 0, ctypes.byref(n), None, 0, ctypes.byref(m))
    lines = [f"P {p['serial']} {p['page_sequence']} {p['page_absgp']} {p['len']} {p['first_piece']} {p['n_pieces']} {p['last_on_page']}" for p in packets]
    lines += [f"Q {q['offset']} {q['len']}" for q in pieces]
    return lines + [f"S {1 if rc == 1 else 0}"]


def test_schedule_equals_the_host_index(run):
    files = _ogg_corpus.files()
    paths = []
    for k, (_, data) in enumerate(files):
        p = run.dir / f"f{k}.ogg"
        p.write_bytes(data)
        paths.append(f"index {p}")
    got = run(paths)
    assert len(got) == len(files)
    n_packets = 0
    for (name, data), lines in zip(files, got):
        want = host_lines(data)
        assert lines == want, name
        n_packets += sum(line.startswith("P") for line in want)
    assert n_packets > 2500


def test_trims_and_durations_equal_the_c_entry_points(run):
    from symphonia_b200 import packetizer
    rng = np.random.default_rng(41)
    reqs, want = [], []
    for trial in range(60):
        n = int(rng.integers(0, 40))
        seq = np.sort(rng.integers(0, 12, n)).astype(np.uint32)
        if trial % 3 == 0:
            seq[:] = 3                                 # every packet on one page
        gp = np.zeros(n, dtype=np.uint64)
        for s in np.unique(seq):
            gp[seq == s] = int(rng.integers(0, 40000))
        dur = rng.choice([0, 64, 128, 576, 1024, 2048], n).astype(np.uint32)
        disc = np.where(rng.integers(0, 4, n) == 0, dur // 2, 0).astype(np.uint32)
        reqs.append(f"trims {n} " + " ".join(f"{a} {b} {c} {e}" for a, b, c, e in zip(seq, gp, dur, disc)))
        want.append([str(v) for v in packetizer.ogg_page_end_trims(seq, gp, dur, disc)])
        ident = np.zeros(1, dtype=[("sample_rate", "<u4"), ("channels", "u1"), ("bs0_exp", "u1"), ("bs1_exp", "u1"), ("reserved", "u1")])[0]
        bs0 = int(rng.integers(6, 12))
        ident["sample_rate"], ident["channels"], ident["bs0_exp"], ident["bs1_exp"] = 44100, 2, bs0, int(rng.integers(bs0, 14))
        n_modes, mask = int(rng.integers(1, 65)), int(rng.integers(0, 2**63))
        heads = rng.integers(0, 65536, n).astype(np.uint16)
        lens = rng.integers(0, 3, n).astype(np.uint8)
        d, c, _ = packetizer.vorbis_packet_durations(ident, n_modes, mask, None, heads=heads, lens=lens)
        reqs.append(f"durs {ident['bs0_exp']} {ident['bs1_exp']} {n_modes} {mask} {n} " + " ".join(f"{h} {ln}" for h, ln in zip(heads, lens)))
        want.append([f"{a} {b}" for a, b in zip(d, c)])
    assert run(reqs) == want
