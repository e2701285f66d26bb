"""The Vorbis packet rules shared by the CPU front-end and the device kernels (symphonia_b200/csrc/vorbis_entropy.h), on the CPU,
and the host half of decode_vorbis_files (decode.vorbis_files_plan).

tests/cpp/vorbis_entropy_driver.cpp runs the device's schedule -- every packet decoded with a fresh partition-class buffer in a
shuffled order, previous block flags chained over the decoded packets afterwards -- and compares every packet with
symgpu_vorbis_fe_decode_packets in stream order: status, units, floor_y and residue bits.  The driver is built with
-ffp-contract=off, and once more with AddressSanitizer + UndefinedBehaviorSanitizer.  The corpus (tests/_vorbis_corpus.py) has
residue types 0, 1 and 2, mono, coupled and uncoupled stereo, class words of 2-3 partitions with short blocks after long ones,
residues that begin beyond the short block, block sizes up to 8192, damaged packets, packets refused mid-residue by a pass that
names a codebook without VQ values, before their window flags, and empty packets."""
import os
import struct
import subprocess

import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import decode
from tests import _vorbis_corpus as corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "symphonia_b200", "csrc")


@pytest.fixture(scope="module")
def drivers(tmp_path_factory):
    d = tmp_path_factory.mktemp("vorbis_entropy")
    src = [os.path.join(ROOT, "tests", "cpp", "vorbis_entropy_driver.cpp"), os.path.join(CSRC, "vorbis_frontend.cpp"), os.path.join(CSRC, "packetizer.cpp")]
    common = ["g++", "-std=c++17", "-ffp-contract=off", "-I/usr/local/cuda/include", "-pthread"]
    plain, sanitized = str(d / "driver"), str(d / "driver_sanitized")
    subprocess.check_call(common + ["-O2", "-o", plain] + src)
    subprocess.check_call(common + ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-o", sanitized] + src)
    return d, {"plain": plain, "sanitized": sanitized}


def _run(driver, tmp, streams, seed):
    blob = struct.pack("<I", len(streams))
    for _, s, packets in streams:
        blob += struct.pack("<I", len(s.ident)) + s.ident + struct.pack("<I", len(s.setup)) + s.setup + struct.pack("<I", len(packets))
        blob += b"".join(struct.pack("<I", len(p)) + p for p in packets)
    src = str(tmp / "in.bin")
    with open(src, "wb") as f:
        f.write(blob)
    res = subprocess.run([driver, src, str(seed)], capture_output=True, text=True, timeout=900,
                         env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=1"))
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    return [int(v) for v in res.stdout.split()]


@pytest.mark.parametrize("build", ["plain", "sanitized"])
def test_device_schedule_equals_the_front_end(drivers, build):
    tmp, exes = drivers
    streams = corpus.streams()
    for seed in (1, 2):
        decoded, refused = _run(exes[build], tmp, streams, seed)
        assert decoded + refused == sum(len(p) for _, _, p in streams)
        assert decoded > 200 and refused >= 1


def test_one_stream_at_a_time_equals_all_streams_at_once(drivers):
    tmp, exes = drivers
    streams = corpus.streams()
    whole = _run(exes["plain"], tmp, streams, 3)
    parts = [_run(exes["plain"], tmp, [s], 3) for s in streams]
    assert [sum(p[i] for p in parts) for i in range(2)] == whole


def test_plan_jobs_setups_and_failures():
    files = [d for _, d in corpus.files()]
    bad = b"not an ogg file"
    errors = {}
    plan = decode.vorbis_files_plan(files + [bad], threads=4, errors=errors)
    assert set(errors) == {len(files)} and plan["failed"] == [len(files)]
    groups, jobs = plan["groups"], plan["jobs"]
    assert len(groups) == len(files) + 1 and groups["n_jobs"][-1] == 0
    # one setup per distinct header pair: only the two "shared" files share theirs
    names = [n for n, _ in corpus.files()]
    a, b = names.index("shared-a"), names.index("shared-b")
    assert len(plan["setups"]) == len(files) - 1 and groups["setup"][a] == groups["setup"][b]
    assert len(set(groups["setup"][:len(files)].tolist())) == len(files) - 1
    for k, data in enumerate(files):
        ix = decode.ogg_vorbis_index(data)
        ix["fe"].close()
        g = groups[k]
        mine = jobs[int(g["first_job"]):int(g["first_job"]) + int(g["n_jobs"])]
        assert len(mine) == len(ix["table"])
        # trims equal the reader's, packet bytes equal the gathered stream's
        assert (mine["discard"] == ix["discard"]).all() and (mine["trim_end"] == ix["trim_end"]).all()
        base = int(mine["offset"][0]) - int(ix["table"]["offset"][0])
        for j, t in zip(mine, ix["table"]):
            assert bytes(plan["data"][int(j["offset"]):int(j["offset"]) + int(j["len"])]) == \
                bytes(ix["blob"][int(t["offset"]):int(t["offset"]) + int(t["len"])])
        assert base >= 0
        r = plan["setups"][int(g["setup"])]
        h = plan["headers"]
        assert h[int(r["ident_offset"]):int(r["ident_offset"]) + int(r["ident_len"])] == ix["headers"][0]
        assert h[int(r["setup_offset"]):int(r["setup_offset"]) + int(r["setup_len"])] == ix["headers"][1]
        assert int(g["out_offset"]) % int(ix["ident"]["channels"]) == 0
    assert plan["jobs"].dtype == nat.VORBIS_JOB_DTYPE and np.all(np.diff(groups["first_job"][:len(files)].astype(np.int64)) >= 0)


@pytest.mark.parametrize("name, least", [("non-vq-pass", 3), ("forty-modes", 3), ("damaged-mono", 1)])
def test_refusals_mid_residue_and_before_the_window_flags(drivers, name, least):
    """The streams whose packets are refused where the fresh class buffer matters most: mid-residue, after class words and earlier
    passes have grown the serial front-end's class vector (a pass naming a codebook without VQ values); before the window flags
    (one-byte packets of long modes among 40 modes); before the packet-type bit (an empty packet)."""
    tmp, exes = drivers
    stream = [s for s in corpus.streams() if s[0] == name]
    for build in ("plain", "sanitized"):
        decoded, refused = _run(exes[build], tmp, stream, 4)
        assert decoded >= 3 and refused >= least
