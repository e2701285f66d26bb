"""The schedule of the device FLAC index (symphonia_b200/csrc/flac_index_kernel.cu), on the CPU.

tests/cpp/flac_index_driver.cpp runs its steps over many files in one buffer -- open(), the tiles and their CRC keys, each node's
header, the radix sort by key, the end search, the successors, the doubling rounds, the scans, the packets -- through the shared
functions of include/symgpu/packetizer.hpp, and every file's stream info and packets must equal symgpu_flac_index of that file's
bytes alone.  It is built plainly and once more with AddressSanitizer + UndefinedBehaviorSanitizer."""
import os
import subprocess

import pytest

from tests import _flac_corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", params=["plain", "sanitized"])
def run(request, tmp_path_factory):
    d = tmp_path_factory.mktemp("flac_index")
    exe = str(d / request.param)
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "flac_index_driver.cpp")]
    cmd += ["-O2"] if request.param == "plain" else ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"]
    subprocess.check_call(cmd)

    def go(mode, buf=None, ranges=(), *extra):
        args = [mode]
        if buf is not None:
            path = d / "buf.bin"
            path.write_bytes(buf.tobytes())
            args += [str(path)] + [str(x) for x in extra] + [str(len(ranges))] + [f"{o} {n}" for o, n in ranges]
        else:
            args += [str(x) for x in extra]
        res = subprocess.run([exe], input=" ".join(args) + "\n", capture_output=True, text=True, timeout=1800,
                             env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=1"))
        assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
        lines = res.stdout.splitlines()
        assert lines[-1] == "end"
        return lines[:-1]
    return go


def _per_file(lines, n_files):
    """("R t k", then per file its P lines and an I line) -> ((t, k), [(P lines, I line)])."""
    assert lines[0].startswith("R ")
    out, cur = [], []
    for line in lines[1:]:
        if line.startswith("I "):
            out.append((cur, line))
            cur = []
        else:
            cur.append(line)
    assert len(out) == n_files and not cur
    return tuple(int(x) for x in lines[0].split()[1:]), out


def host(data):
    """symgpu_flac_index of the bytes, in the driver's format."""
    from symphonia_b200 import SymgpuError, packetizer
    try:
        info, packets = packetizer.flac_index(data)
    except SymgpuError as e:
        assert e.status in (1, 2)
        return [], f"I {e.status} " + " ".join(["0"] * 26)
    lines = [f"P {p['offset']} {p['ts']} {p['size']} {p['dur']}" for p in packets]
    fields = [info[k] for k in ("n_samples", "first_frame_pos", "sample_rate", "frame_min", "frame_max", "block_min", "block_max", "channels",
                                "bits_per_sample", "has_md5")]
    return lines, "I 0 " + " ".join(str(int(x)) for x in fields) + " " + " ".join(str(int(x)) for x in info["md5"])


def _check(run, files, seed, k=-1):
    """Every file's result equals the host index; returns the packets in all."""
    buf, ranges = _flac_corpus.pack(files, seed)
    rounds, got = _per_file(run("index", buf, ranges, k), len(files))
    longest = max(n for _, n in ranges)
    assert rounds == ((longest // 2).bit_length(), (longest // 8).bit_length())
    n_packets = 0
    for i, (f, (lines, info)) in enumerate(zip(files, got)):
        want_lines, want_info = host(f)
        assert info == want_info, i
        assert lines == want_lines, i
        n_packets += len(want_lines)
    return n_packets


def _same(run, files, seed, k=-1):
    try:
        _check(run, files, seed, k)
        return True
    except AssertionError:
        return False


def test_schedule_equals_the_host_index_per_file(run):
    named = _flac_corpus.files()
    files = [d for _, d in named]
    infos = {name: host(d)[1] for name, d in named}
    assert sum(i.startswith("I 2 ") for i in infos.values()) >= 5 and sum(i.startswith("I 1 ") for i in infos.values()) >= 8
    counts = {name: len(host(d)[0]) for name, d in named}
    # the cases do what their names say (host side): a corrupted frame is dropped, the false syncs are not frames, a cut last frame
    # is dropped, and repeated / decreasing numbers lose frames to the sequence rule
    assert counts["corrupted frame"] < 12 and counts["false syncs"] == 30 and counts["cut last frame"] == 9 and counts["ends at the end"] == 10
    assert counts["repeated sequence numbers"] < 8 and counts["decreasing sequence numbers"] < 8 and counts["sync-dense junk"] == 0
    assert counts["sync-dense frames"] == 20 and 0 < counts["one key"] < 600
    assert _check(run, files, 81) > 450
    assert _check(run, files[::-1], 82) > 450


def test_decodable_files(run):
    from tests.test_flac_decode_gpu import _corpus
    files = [d for _, d, _ in _corpus()]
    assert _check(run, files, 83) > 100


def test_the_crc_key_combine_equals_the_plain_crc(run):
    checked, differ = (int(x) for x in run("crc", None, (), 5, 20000)[0].split()[1:])
    assert checked == 20000 and differ == 0


def test_long_files_need_the_rounds_the_ranges_give(run):
    chain = _flac_corpus.long_chain()
    n = (1 << 15) - 8
    assert len(host(chain)[0]) == n and (len(chain) // 8).bit_length() == 15
    for files in ([chain], [chain, _flac_corpus.files()[0][1], b""]):
        _check(run, files, 84)
        buf, ranges = _flac_corpus.pack(files, 85)
        assert run("extra", buf, ranges) == ["X 0"]   # the stated rounds ranked every chain node
    # and the rounds matter: the chain has 32 760 nodes, so 14 doubling rounds leave its tail unranked
    assert not _same(run, [chain], 86, k=14) and _same(run, [chain], 86, k=15)


def test_the_end_search_window(run):
    """A frame whose CRC-valid end lies past the 16 MiB window behind another sync word is no frame; without that sync word the
    next frame past the window is examined and the big frame is found."""
    past, within = _flac_corpus.past_window(), _flac_corpus.within_window()
    assert len(host(past)[0]) == 5 and host(past)[0][0].split()[1] != str(int(host(past)[1].split()[3]))
    assert len(host(within)[0]) == 4 and int(host(within)[0][0].split()[3]) > 16 << 20
    _check(run, [past, within], 87)


def test_the_capacity_bound(run):
    files = [d for _, d in _flac_corpus.files()] + [_flac_corpus.long_chain()]
    for f in files:
        assert len(host(f)[0]) <= len(f) // 8
    assert all(int(line.split()[3]) >= 8 for f in files for line in host(f)[0])
