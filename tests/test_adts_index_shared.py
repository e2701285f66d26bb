"""The schedule of the device ADTS index (symphonia_b200/csrc/adts_index_kernel.cu), on the CPU.

tests/cpp/adts_index_driver.cpp runs its steps over many files in one buffer -- the candidates, their successors, the doubling
rounds, the records from each chain's end, the packets -- through the shared functions of include/symgpu/packetizer.hpp, and
every file's packets and stop must equal symgpu_adts_index of that file's bytes alone.  It is built plainly and once more with
AddressSanitizer + UndefinedBehaviorSanitizer."""
import os
import subprocess

import pytest

from tests import _adts_corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", params=["plain", "sanitized"])
def run(request, tmp_path_factory):
    d = tmp_path_factory.mktemp("adts_index")
    exe = str(d / request.param)
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "adts_index_driver.cpp")]
    cmd += ["-O2"] if request.param == "plain" else ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"]
    subprocess.check_call(cmd)

    def go(mode, buf, ranges, rounds=None):
        path = d / "buf.bin"
        path.write_bytes(buf.tobytes())
        args = [mode, str(path)] + ([] if rounds is None else [str(rounds)]) + [str(len(ranges))] + [f"{o} {n}" for o, n in ranges]
        res = subprocess.run([exe], input=" ".join(args) + "\n", capture_output=True, text=True, timeout=600,
                             env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=1"))
        assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
        lines = res.stdout.splitlines()
        assert lines[-1] == "end"
        return lines[:-1]
    return go


def _per_file(lines, n_files):
    """("K k", then per file its P lines and an S line) -> (k, [(P lines, S fields)])."""
    assert lines[0].startswith("K ")
    out, cur = [], []
    for line in lines[1:]:
        if line.startswith("S "):
            out.append((cur, [int(x) for x in line.split()[1:]]))
            cur = []
        else:
            cur.append(line)
    assert len(out) == n_files and not cur
    return int(lines[0].split()[1]), out


def _host(data):
    from symphonia_b200 import packetizer
    packets, stop = packetizer.adts_index(data)
    lines = [f"P {p['offset']} {p['size']} {p['sample_rate']} {p['pts']} {p['channels']} {p['profile']}" for p in packets]
    first = packets[0] if len(packets) else None
    head = [int(first["sample_rate"]), int(first["channels"]), int(first["profile"])] if first is not None else [0, 0, 0]
    return lines, [stop] + head


def _check(run, files, seed, rounds=-1):
    buf, ranges = _adts_corpus.pack(files, seed)
    k, got = _per_file(run("index", buf, ranges, rounds), len(files))
    assert k == (max(n for _, n in ranges) // 2).bit_length()
    n_packets = 0
    for f, (lines, fields) in zip(files, got):
        want_lines, want_fields = _host(f)
        assert lines == want_lines and fields == want_fields
        n_packets += len(want_lines)
    return n_packets


def test_schedule_equals_the_host_index_per_file(run):
    files = [d for _, d in _adts_corpus.files()]
    stops = {_host(f)[1][0] for f in files}
    assert stops == {0, 1, 2, 3}
    assert _check(run, files, 31) > 900
    assert _check(run, files[::-1], 32) > 900


def test_dense_sync_and_a_long_file_need_the_rounds_the_ranges_give(run):
    dense, long = _adts_corpus.dense_sync(), _adts_corpus.long_file()
    want_frames = len(_host(long)[0])
    assert want_frames == 30000
    for files in ([dense], [long], [dense, long, b""]):
        _check(run, files, 33)
        buf, ranges = _adts_corpus.pack(files, 34)
        assert run("extra", buf, ranges) == ["X 0"]   # the K rounds ranked every chain node: a further round adds nothing
    # and the rounds matter: the long chain needs bit_length(30000 - 1) = 15 of them, so 14 leave its tail unranked
    buf, ranges = _adts_corpus.pack([long], 35)
    _, got = _per_file(run("index", buf, ranges, 14), 1)
    assert len(got[0][0]) < want_frames
    _, got = _per_file(run("index", buf, ranges, 15), 1)
    assert got[0][0] == _host(long)[0]
