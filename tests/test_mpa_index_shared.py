"""The schedule of the device MPEG index (symphonia_b200/csrc/mpa_index_kernel.cu), on the CPU.

tests/cpp/mpa_index_driver.cpp runs its steps over many files in one buffer -- the candidates, their successors and hunt steps, the
jumping rounds, each file's first frame and track, the doubling rounds, the scans, the packets -- through the shared functions of
include/symgpu/packetizer.hpp, and every file's track and packets must equal symgpu_mpa_index of that file's bytes alone, seekable or
not.  It is built plainly and once more with AddressSanitizer + UndefinedBehaviorSanitizer."""
import os
import subprocess

import pytest

from tests import _mpa_corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", params=["plain", "sanitized"])
def run(request, tmp_path_factory):
    d = tmp_path_factory.mktemp("mpa_index")
    exe = str(d / request.param)
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "mpa_index_driver.cpp")]
    cmd += ["-O2"] if request.param == "plain" else ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"]
    subprocess.check_call(cmd)

    def go(mode, buf=None, ranges=(), *extra):
        args = [mode]
        if buf is not None:
            path = d / "buf.bin"
            path.write_bytes(buf.tobytes())
            args += [str(path)] + [str(x) for x in extra] + [str(len(ranges))] + [f"{o} {n}" for o, n in ranges]
        res = subprocess.run([exe], input=" ".join(args) + "\n", capture_output=True, text=True, timeout=900,
                             env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=1"))
        assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
        lines = res.stdout.splitlines()
        assert lines[-1] == "end"
        return lines[:-1]
    return go


def _per_file(lines, n_files):
    """("R h k", then per file its P lines and a T line) -> ((h, k), [(P lines, T line)])."""
    assert lines[0].startswith("R ")
    out, cur = [], []
    for line in lines[1:]:
        if line.startswith("T "):
            out.append((cur, line))
            cur = []
        else:
            cur.append(line)
    assert len(out) == n_files and not cur
    return tuple(int(x) for x in lines[0].split()[1:]), out


def _host(data, seekable):
    """symgpu_mpa_index of the bytes, in the driver's format."""
    from symphonia_b200 import SymgpuError, packetizer
    try:
        t, packets = packetizer.mpa_index(data, seekable)
    except SymgpuError as e:
        assert e.status == 1
        return [], "T 1 00000000 0 0 0 0 0 0 0 0 0 0 0"
    lines = [f"P {p['offset']} {p['size']} {int(p['header']):08x} {p['pts']} {p['dur']} {p['trim_start']} {p['trim_end']} {p['main_data_begin']}"
             for p in packets]
    track = (f"T 0 {int(t['first_header']):08x} {t['sample_rate']} {t['version']} {t['layer']} {t['channels']} {t['tag']} {t['has_delay']} "
             f"{t['has_num_frames']} {t['delay']} {t['padding']} {t['num_frames']} {t['first_packet_pos']}")
    return lines, track


def _check(run, files, seed, seekable=1, h=-1, k=-1):
    """Every file's result equals the host index; returns (stated rounds, packets in all)."""
    buf, ranges = _mpa_corpus.pack(files, seed)
    rounds, got = _per_file(run("index", buf, ranges, seekable, h, k), len(files))
    longest = max(n for _, n in ranges)
    assert rounds == (longest.bit_length(), (longest // 4).bit_length())
    n_packets = 0
    for i, (f, (lines, track)) in enumerate(zip(files, got)):
        want_lines, want_track = _host(f, bool(seekable))
        assert track == want_track, i
        assert lines == want_lines, i
        n_packets += len(want_lines)
    return n_packets


def _same(run, files, seed, seekable=1, h=-1, k=-1):
    try:
        _check(run, files, seed, seekable, h, k)
        return True
    except AssertionError:
        return False


def test_schedule_equals_the_host_index_per_file(run):
    named = _mpa_corpus.files()
    files = [d for _, d in named]
    tracks = [_host(f, True)[1] for f in files]
    assert sum(t.startswith("T 1 ") for t in tracks) >= 6                     # frameless files
    assert {t.split()[7] for t in tracks if t.startswith("T 0 ")} == {"0", "1", "2", "3"}   # no tag, Xing, Info, VBRI
    for seekable in (1, 0):
        assert _check(run, files, 31 + seekable, seekable) > 4000
    assert _check(run, files[::-1], 33) > 4000


def test_decodable_files(run):
    files = [d for _, d in _mpa_corpus.decodable()]
    for seekable in (1, 0):
        assert _check(run, files, 34, seekable) > 150


def test_long_files_need_the_rounds_the_ranges_give(run):
    dense, hunt, long = _mpa_corpus.dense_skip(), _mpa_corpus.long_hunt(), _mpa_corpus.long_file()
    assert len(_host(long, True)[0]) == 30000
    assert _host(dense, True)[1].startswith("T 1 ")
    assert _host(hunt, True)[1].endswith(f" {36 * 10000}") and len(_host(hunt, True)[0]) == 3
    for files in ([dense], [hunt], [long], [dense, hunt, long, b""]):
        _check(run, files, 35)
        buf, ranges = _mpa_corpus.pack(files, 36)
        assert run("extra", buf, ranges) == ["X 0 0"]   # the stated rounds finished every hunt and ranked every chain node
    # and the rounds matter: the hunt passes 10 000 rejected frames, so 2^13 = 8192 jumps do not reach its end; the chain has
    # 30 000 nodes, so 14 doubling rounds leave its tail unranked
    assert not _same(run, [hunt], 37, h=13) and _same(run, [hunt], 37, h=14)
    assert not _same(run, [long], 38, k=14) and _same(run, [long], 38, k=15)


def test_the_capacity_bound_holds_for_every_header_word(run):
    assert run("minframe") == ["M 24"]
    files = [d for _, d in _mpa_corpus.files()] + [_mpa_corpus.long_file()]
    for f in files:
        assert len(_host(f, True)[0]) <= len(f) // 24


def test_the_estimate_in_integers_equals_the_double_arithmetic(run):
    """mpa_estimate_frames divides in integers (the device has no double division without fused multiply-adds): every count and
    average frame length it can meet, totals that make the quotient exact included, must give what the host's doubles give."""
    checked, differ = (int(x) for x in run("extrapolate")[0].split()[1:])
    assert checked > 4_000_000 and differ == 0
