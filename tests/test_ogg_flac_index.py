"""FLAC in Ogg on the host, and the device job build's rules on the CPU.

decode.ogg_flac_index (symgpu_ogg_flac_packets) must make the decisions oracle/ogg_flac_oracle.py restates from
symphonia-format-ogg/src/mappings/flac.rs on every file of tests/_ogg_flac_corpus.py and on mutated streams: which streams are
Ogg FLAC, their STREAMINFO, which packets carry audio, every audio packet's bytes and slot, and the failure messages.
tests/cpp/ogg_flac_jobs_driver.cpp runs the per-file, per-packet, scan and gather steps of ogg_flac_jobs_kernel.cu through the
same packetizer.hpp functions the kernels call, on all corpus files in one table; it must give what ogg_flac_index gives.  It is
built plainly and once more with AddressSanitizer + UndefinedBehaviorSanitizer."""
import os
import subprocess

import numpy as np
import pytest

from oracle import ogg_flac_oracle
from symphonia_b200 import _native as nat
from symphonia_b200 import decode, packetizer
from tests import _ogg_flac_corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def corpus():
    return _ogg_flac_corpus.files()


def _host(data):
    try:
        return decode.ogg_flac_index(data)
    except Exception as e:  # noqa: BLE001 -- the message is what is compared
        return f"{type(e).__name__}: {e}"


_STATUS = {"no packets": "ValueError: no Ogg packets", "not flac": "[2] symgpu_ogg_flac_packets", "bad streaminfo": "[1] symgpu_ogg_flac_packets"}


def _same_as_oracle(data):
    want, got = ogg_flac_oracle.read(data), _host(data)
    if want["status"] != "ok":
        assert isinstance(got, str) and got.endswith(_STATUS[want["status"]]), (want["status"], got)
        return want["status"]
    assert not isinstance(got, str), got
    info = got["info"]
    for k in ("block_min", "block_max", "frame_min", "frame_max", "sample_rate", "channels", "bits_per_sample", "n_samples"):
        assert int(info[k]) == want["info"][k], k
    assert bytes(info["md5"]) == want["info"]["md5"] and int(info["first_frame_pos"]) == 0
    blob, table = got["blob"], got["table"]
    assert [bytes(blob[int(t["offset"]):int(t["offset"]) + int(t["len"])]) for t in table] == [p for p, _ in want["audio"]]
    assert [int(s) for s in got["slot"]] == [s for _, s in want["audio"]]
    return "ok"


def test_corpus_matches_the_oracle(corpus):
    seen = {_same_as_oracle(data) for _, data, _ in corpus}
    assert seen == {"ok", "no packets", "not flac", "bad streaminfo"}
    names = {name: twin for name, _, twin in corpus}
    assert names["FLAC with a second stream of higher serial"] is not None and names["FLAC with a second stream of lower serial"] is None


def test_slots_cover_refusals(corpus):
    """A header the decoder refuses has slot 0; a valid header above STREAMINFO's maximum keeps its block (the decode refuses it)."""
    got = {name: _host(data) for name, data, _ in corpus}
    assert 0 in [int(s) for s in got["corrupt CRC-8"]["slot"]]
    assert 1152 in [int(s) for s in got["block above STREAMINFO maximum"]["slot"]]
    assert len(got["metadata packets"]["table"]) == len(got["plain stereo"]["table"])


def _mutants(data, rng, n):
    for _ in range(n):
        b = bytearray(data)
        for at in rng.integers(0, len(b), int(rng.integers(1, 4))):
            b[int(at)] ^= 1 << int(rng.integers(8))
        yield bytes(b)


def test_mutated_streams_match_the_oracle(corpus):
    rng = np.random.default_rng(91)
    seen = set()
    for name, data, _ in corpus[:12]:
        for m in _mutants(data, rng, 12):
            seen.add(_same_as_oracle(m))
    assert "ok" in seen


def test_identification_rule_byte_by_byte():
    """Every byte of a valid identification packet, flipped: the C rule and the oracle agree on Ogg FLAC or not, and on the
    STREAMINFO check."""
    head = _ogg_flac_corpus.ident(_ogg_flac_corpus.info_block(576, 2, 16))
    for at in range(len(head)):
        for bit in (0, 7):
            p = bytearray(head)
            p[at] ^= 1 << bit
            table = np.zeros(1, dtype=nat.PIECE_DTYPE)
            table["len"] = len(p)
            try:
                want = "ok" if ogg_flac_oracle.detect(bytes(p)) is not None else 2
            except Exception:  # noqa: BLE001 -- a refused STREAMINFO
                want = 1
            try:
                packetizer.ogg_flac_packets(bytes(p), table)
                got = "ok"
            except Exception as e:  # noqa: BLE001
                got = e.status
            assert got == want, (at, bit)


@pytest.fixture(scope="module", params=["plain", "sanitized"])
def driver(request, tmp_path_factory):
    d = tmp_path_factory.mktemp("ogg_flac_jobs")
    exe = str(d / request.param)
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "ogg_flac_jobs_driver.cpp")]
    cmd += ["-O2"] if request.param == "plain" else ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"]
    subprocess.check_call(cmd)
    return exe, d


def test_device_schedule_on_the_cpu(driver, corpus):
    exe, d = driver
    files = [data for _, data, _ in corpus] + [_ogg_flac_corpus.files(seed=92)[0][1]]
    args = [str(len(files))]
    for k, data in enumerate(files):
        packets, pieces = packetizer.ogg_index(data)
        for ext, blob in (("bin", data), ("pk", packets.tobytes()), ("pc", pieces.tobytes())):
            (d / f"f{k}.{ext}").write_bytes(blob)
        args += [str(d / f"f{k}.bin"), str(d / f"f{k}.pk"), str(d / f"f{k}.pc")]
    res = subprocess.run([exe], input=" ".join(args) + "\n", capture_output=True, text=True, timeout=600,
                         env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=1"))
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    lines = res.stdout.splitlines()
    heads = [[int(v) for v in ln.split()[1:]] for ln in lines if ln.startswith("F ")]
    jobs = [[int(v) for v in ln.split()[1:]] for ln in lines if ln.startswith("J ")]
    out = (d / "f0.bin.out").read_bytes()
    status = {1: "ValueError: no Ogg packets", 2: "[2] symgpu_ogg_flac_packets", 3: "[1] symgpu_ogg_flac_packets"}
    at = 0
    for i, data in enumerate(files):
        h, want = heads[i], _host(data)
        if h[0]:
            assert isinstance(want, str) and want.endswith(status[h[0]]), (i, h, want)
            assert h[7] == 0
            continue
        info = want["info"]
        assert h[2:7] == [int(info[k]) for k in ("block_min", "block_max", "sample_rate", "channels", "bits_per_sample")]
        table, slot = want["table"], [int(s) for s in want["slot"]]
        assert h[7] == len(table) and h[8] == int(table["len"].astype(np.int64).sum()) and h[9] == sum(slot)
        mine = jobs[at:at + h[7]]
        assert [j[0] for j in mine] == [i] * len(mine) and [j[2] for j in mine] == slot
        for j, t in zip(mine, table):
            assert out[j[3]:j[3] + j[1]] == bytes(want["blob"][int(t["offset"]):int(t["offset"]) + int(t["len"])])
        at += h[7]
    assert at == len(jobs)


def test_router_check_of_the_first_packet():
    """decode_any_files' test of a stream's first packet: Ogg FLAC by shape (also with a refused STREAMINFO), a Vorbis
    identification header or anything else of another length or lead-in not, without a library call."""
    head = _ogg_flac_corpus.ident(_ogg_flac_corpus.info_block(576, 2, 16))
    assert decode._is_ogg_flac_ident(head) and decode._is_ogg_flac_ident(np.frombuffer(head, dtype=np.uint8))
    assert decode._is_ogg_flac_ident(_ogg_flac_corpus.ident(_ogg_flac_corpus.info_block(576, 2, 16, block_min=8)))
    assert not decode._is_ogg_flac_ident(_ogg_flac_corpus.ident(_ogg_flac_corpus.info_block(576, 2, 16), major=2))
    assert not decode._is_ogg_flac_ident(b"\x01vorbis" + bytes(23)) and not decode._is_ogg_flac_ident(head[:50])
    assert not decode._is_ogg_flac_ident(b"\x00" + head[1:])
