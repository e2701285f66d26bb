"""The Vorbis job build on the device (symphonia_b200/csrc/vorbis_jobs_kernel.cu), on the CPU.

tests/cpp/ogg_vorbis_jobs_driver.cpp runs its rules -- the header choice, the audio packets, each packet's block exponent, the
previous-exponent scan and the page end trims run by run from prefix sums -- through the shared functions of
include/symgpu/packetizer.hpp, and must give what decode.ogg_vorbis_index gives on every Vorbis and Ogg corpus file: the
headers, the audio packets' lengths, their discard and end trim, and which files fail.  On random streams, several to a job
table, it must give what symgpu_ogg_page_end_trims and symgpu_vorbis_packet_durations give stream by stream.  It is built plainly
and once more with AddressSanitizer + UndefinedBehaviorSanitizer."""
import os
import subprocess

import numpy as np
import pytest

from tests import _ogg_corpus, _vorbis_corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", params=["plain", "sanitized"])
def run(request, tmp_path_factory):
    d = tmp_path_factory.mktemp("ogg_vorbis_jobs")
    exe = str(d / request.param)
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "ogg_vorbis_jobs_driver.cpp")]
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


def _host(data):
    """ogg_vorbis_index of the file: (headers, audio lens, discard, trim_end) or its failure message."""
    from symphonia_b200 import decode
    try:
        ix = decode.ogg_vorbis_index(data)
    except Exception as e:  # noqa: BLE001 -- the message is what is compared
        return f"{type(e).__name__}: {e}"
    ix["fe"].close()
    return ix["headers"], [int(v) for v in ix["table"]["len"]], [int(v) for v in ix["discard"]], [int(v) for v in ix["trim_end"]]


def _shared(data, lines):
    """The driver's answer for the file, its headers checked on the host as the device path checks them."""
    from symphonia_b200 import decode, packetizer
    head = [int(v) for v in lines[0].split()[1:]]
    n_stream, setup = head[0], head[1]
    if n_stream == 0:
        return "ValueError: no Ogg packets"
    packets, pieces = packetizer.ogg_index(data)
    ident_b = packetizer.gather(data, packets[0], pieces)
    setup_b = packetizer.gather(data, packets[setup], pieces) if setup < n_stream else None
    assert head[2] == len(ident_b) and head[3] == (len(setup_b) if setup_b is not None else 0)
    try:
        decode.vorbis_open_headers(ident_b, setup_b)[3].close()
    except Exception as e:  # noqa: BLE001
        return f"{type(e).__name__}: {e}"
    audio = [line.split() for line in lines if line.startswith("A ")]
    jobs = [line.split() for line in lines if line.startswith("J ")]
    assert len(jobs) == len(audio), lines[-1]
    return (ident_b, setup_b), [int(a[2]) for a in audio], [int(j[1]) for j in jobs], [int(j[2]) for j in jobs]


def test_jobs_equal_the_host_index_on_every_corpus_file(run):
    from symphonia_b200 import packetizer
    files = [(f"vorbis-{name}", d) for name, d in _vorbis_corpus.files()] + _ogg_corpus.files()
    reqs = []
    for k, (_, data) in enumerate(files):
        packets, pieces = packetizer.ogg_index(data)
        paths = [run.dir / f"f{k}.{ext}" for ext in ("ogg", "packets", "pieces")]
        for p, b in zip(paths, (data, packets.tobytes(), pieces.tobytes())):
            p.write_bytes(b)
        reqs.append("vorbis " + " ".join(str(p) for p in paths))
    got = run(reqs)
    assert len(got) == len(files)
    good = 0
    for (name, data), lines in zip(files, got):
        want = _host(data)
        assert _shared(data, lines) == want, name
        good += not isinstance(want, str)
    assert good >= len(_vorbis_corpus.files()) - 3 and good < len(files)


def _random_streams(rng, trial):
    """Several streams of (seq, absgp, dur, discard): sorted page numbers, some starting just below 2^32 so that they wrap, one
    page only in every third trial."""
    streams = []
    for _ in range(int(rng.integers(1, 5))):
        n = int(rng.integers(0, 40))
        seq = np.sort(rng.integers(0, 12, n)).astype(np.uint64)
        if trial % 3 == 0:
            seq[:] = 3
        if trial % 4 == 1:
            seq = (seq + 2**32 - 4) % 2**32
        gp = np.zeros(n, dtype=np.uint64)
        for s in np.unique(seq):
            gp[seq == s] = int(rng.integers(0, 40000))
        dur = rng.choice([0, 64, 128, 576, 1024, 2048], n).astype(np.uint32)
        disc = np.where(rng.integers(0, 4, n) == 0, dur // 2, 0).astype(np.uint32)
        streams.append((seq.astype(np.uint32), gp, dur, disc))
    return streams


def test_run_trims_and_scanned_durations_equal_the_c_entry_points(run):
    from symphonia_b200 import packetizer
    rng = np.random.default_rng(43)
    reqs, want = [], []
    for trial in range(80):
        streams = _random_streams(rng, trial)
        req = f"trims {len(streams)}"
        w = []
        for seq, gp, dur, disc in streams:
            req += f" {len(seq)} " + " ".join(f"{a} {b} {c} {e}" for a, b, c, e in zip(seq, gp, dur, disc))
            w += [str(v) for v in packetizer.ogg_page_end_trims(seq, gp, dur, disc)]
        reqs.append(req)
        want.append(w)
        ident = np.zeros(1, dtype=[("sample_rate", "<u4"), ("channels", "u1"), ("bs0_exp", "u1"), ("bs1_exp", "u1"), ("reserved", "u1")])[0]
        bs0 = int(rng.integers(6, 12))
        ident["sample_rate"], ident["channels"], ident["bs0_exp"], ident["bs1_exp"] = 44100, 2, bs0, int(rng.integers(bs0, 14))
        n_modes, mask = int(rng.integers(1, 65)), int(rng.integers(0, 2**63))
        req = f"durs {ident['bs0_exp']} {ident['bs1_exp']} {n_modes} {mask} {len(streams)}"
        w = []
        for seq, *_ in streams:
            heads = rng.integers(0, 65536, len(seq)).astype(np.uint16)
            lens = rng.integers(0, 3, len(seq)).astype(np.uint8)
            d, c, _ = packetizer.vorbis_packet_durations(ident, n_modes, mask, None, heads=heads, lens=lens)
            req += f" {len(seq)} " + " ".join(f"{h} {ln}" for h, ln in zip(heads, lens))
            w += [f"{a} {b}" for a, b in zip(d, c)]
        reqs.append(req)
        want.append(w)
    assert run(reqs) == want
