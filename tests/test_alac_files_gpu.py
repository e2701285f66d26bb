"""ALAC in CAF decoded on the device: every corpus file through decode_alac_files, host-indexed into host memory and into device
memory, equals the oracle's packet-by-packet decode bit for bit in all five sample formats, with the same per-packet status."""
import numpy as np
import pytest

import symphonia_b200 as sb
import symphonia_b200._native as nat
from symphonia_b200 import decode
from tests import _alac_bitstream as ab
from tests import _alac_cases as cases
from tests import _caf_corpus

pytestmark = pytest.mark.gpu

CORPUS = _caf_corpus.corpus()
FORMATS = [nat.FMT_S32, nat.FMT_S24, nat.FMT_S16, nat.FMT_U8, nat.FMT_F32]


def convert(s, fmt):
    """FromSample<i32> of the 32-bit-scaled samples (include/symgpu.h, symgpu_flac_decode_fmt_*)."""
    s = s.astype(np.int32)
    if fmt == nat.FMT_S32:
        return s
    if fmt == nat.FMT_S24:
        return s >> 8
    if fmt == nat.FMT_S16:
        return (s >> 16).astype(np.int16)
    if fmt == nat.FMT_U8:
        return ((s.view(np.uint32).astype(np.uint64) + 0x80000000) % (1 << 32) >> 24).astype(np.uint8)
    return (s.astype(np.float64) / 2147483648.0).astype(np.float32)


@pytest.fixture(scope="module")
def eng():
    with sb.Engine(0) as e:
        yield e


@pytest.fixture(scope="module")
def orc():
    return cases.oracle_lib()


def expected(orc, data):
    """(samples [frames, channels] int32, per-packet status) the oracle gives for a file, or None when it does not open."""
    try:
        info, packets = sb.packetizer.caf_index(data)
    except sb.engine.SymgpuError:
        return None
    ck = {k: int(info[k]) for k in ("frame_length", "bit_depth", "pb", "mb", "kb", "channels")}
    parts, status = [np.zeros((0, ck["channels"]), dtype=np.int32)], []
    for p in packets:
        refused, s = cases.oracle_packet(orc, data[int(p["offset"]):int(p["offset"]) + int(p["size"])], ck)
        status.append(1 if refused else 0)
        parts.append(s)
    return np.concatenate(parts), np.array(status, dtype=np.uint8)


def damaged_corpus():
    rng = np.random.default_rng(21)
    out = [c[1] for c in CORPUS]
    for name, data, expect in CORPUS:
        if expect is None or not expect["packets"]:
            continue
        b = bytearray(data)
        start = len(data) - sum(len(p) for p in expect["packets"]) - (3 if name == "cut_last_packet" else 0)
        for _ in range(8):
            k = int(rng.integers(start * 8, len(b) * 8))
            b[k // 8] ^= 0x80 >> (k % 8)
        out.append(bytes(b))
    return out


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("device", [False, True])
def test_every_file_equals_the_oracle(eng, orc, fmt, device):
    files = damaged_corpus()
    errors, stats = {}, {}
    got = decode.decode_alac_files(eng, files, fmt=fmt, device=device, errors=errors, stats=stats)
    status_at, refused_seen = 0, 0
    for i, data in enumerate(files):
        want = expected(orc, data)
        samples, rate = got[i]
        samples = samples.cpu().numpy() if device else samples
        if want is None:
            assert i in errors and samples.size == 0 and rate == 0
            continue
        w, st = want
        assert i not in errors
        assert samples.shape == w.shape
        assert samples.dtype == convert(w, fmt).dtype and (samples.view(np.uint8) == convert(w, fmt).view(np.uint8)).all(), i
        assert (stats["status"][status_at:status_at + len(st)] == st).all()
        status_at += len(st)
        refused_seen += int(st.sum())
    assert status_at == len(stats["status"]) and refused_seen > 0


def _caf_of(packets, ck):
    return _caf_corpus.caf([_caf_corpus.desc(ck), _caf_corpus.chunk(b"kuki", ab.cookie_bytes(ck)), _caf_corpus.pakt([len(p) for p in packets], ck),
                            _caf_corpus.chunk(b"data", bytes(4) + b"".join(packets))])


def test_256_files_more_packets_than_a_grid_row(eng):
    """256 files holding 69 376 packets in all: more jobs than the 65 535 blocks of a grid's y or z row."""
    rng = np.random.default_rng(8)
    ck = cases.cookie(channels=2, frame_length=64)
    pool = [ab.signal(rng, 64, 2, 16) for _ in range(40)]
    enc = [ab.encode_packet(x, ck) for x in pool]
    files, wants = [], []
    for k in range(256):
        idx = [(k + j) % len(pool) for j in range(1 + (k % 7) * 90)]
        files.append(_caf_of([enc[i] for i in idx], ck))
        wants.append((np.concatenate([pool[i] for i in idx]).astype(np.int64) << 16).astype(np.int32))
    assert sum(len(w) for w in wants) // 64 > 65535
    got = decode.decode_alac_files(eng, files, device=True)
    for (s, rate), w in zip(got, wants):
        assert rate == 44100 and (s.cpu().numpy() == w).all()
    blob, ranges = _resident(files)
    got_dev = decode.decode_alac_files_dev(eng, blob, ranges)
    for (s, rate), w in zip(got_dev, wants):
        assert rate == 44100 and (s.cpu().numpy() == w).all()


def _resident(files):
    import torch
    ranges, at = [], 0
    for f in files:
        ranges.append((at, len(f)))
        at += len(f)
    return torch.from_numpy(np.frombuffer(b"".join(files), dtype=np.uint8).copy()).cuda(), ranges


def test_device_index_equals_host_index(eng):
    from tests.test_caf_index import _mutants
    files = damaged_corpus() + _mutants()
    blob, ranges = _resident(files)
    infos, first, packets_t, jobs_t, _ = eng.caf_index_dev(blob, ranges)
    packets = packets_t.cpu().numpy().view(nat.CAF_PACKET_DTYPE)
    jobs = jobs_t.cpu().numpy().view(nat.FLAC_JOB_DTYPE)
    at = 0
    for i, f in enumerate(files):
        want_info = np.zeros(1, dtype=nat.CAF_INFO_DTYPE)
        try:
            want_info[0], want_packets = sb.packetizer.caf_index(f)
        except sb.engine.SymgpuError:
            want_packets = np.zeros(0, dtype=nat.CAF_PACKET_DTYPE)
            import ctypes
            n = ctypes.c_size_t(0)
            a = np.frombuffer(f, dtype=np.uint8) if f else np.zeros(1, dtype=np.uint8)
            nat.lib().symgpu_caf_index(ctypes.c_void_p(a.ctypes.data), len(f), ctypes.c_void_p(want_info.ctypes.data), None, 0, ctypes.byref(n))
        assert infos[i:i + 1].tobytes() == want_info.tobytes(), i
        assert int(first[i]) == at
        k = int(infos["n_packets"][i])
        assert packets[at:at + k].tobytes() == want_packets.tobytes()
        assert (jobs["offset"][at:at + k] == want_packets["offset"] + ranges[i][0]).all() and (jobs["len"][at:at + k] == want_packets["size"]).all()
        assert (jobs["group"][at:at + k] == i).all() and (jobs["slot"][at:at + k] == infos["frame_length"][i]).all()
        at += k


@pytest.mark.parametrize("fmt", [nat.FMT_S32, nat.FMT_S16, nat.FMT_F32])
def test_resident_equals_host_indexed(eng, fmt):
    files = damaged_corpus()
    blob, ranges = _resident(files)
    e_dev, s_dev, e_host, s_host = {}, {}, {}, {}
    got = decode.decode_alac_files_dev(eng, blob, ranges, fmt=fmt, errors=e_dev, stats=s_dev)
    want = decode.decode_alac_files(eng, files, fmt=fmt, device=True, errors=e_host, stats=s_host)
    assert e_dev == e_host and (np.asarray(s_dev["status"]) == np.asarray(s_host["status"])).all()
    assert s_dev["read_back_bytes"] < len(blob)
    for (a, ra), (b, rb) in zip(got, want):
        assert ra == rb and a.shape == b.shape and bool((a == b).all())


def test_any_files_routes_caf(eng, orc):
    files = [c[1] for c in CORPUS if c[1][:4] == b"caff"]
    errors, stats = {}, {}
    got = decode.decode_any_files(eng, files, fmt=nat.FMT_S32, errors=errors, stats=stats)
    assert stats["calls"] == ["alac"]
    want = decode.decode_alac_files(eng, files, fmt=nat.FMT_S32)
    for (a, ra), (b, rb) in zip(got, want):
        assert ra == rb and a.shape == b.shape and (a == b).all()


def test_any_files_dev_takes_caf(eng):
    files = [c[1] for c in CORPUS if c[1][:4] == b"caff"]
    blob, ranges = _resident(files)
    errors, stats = {}, {}
    got = decode.decode_any_files_dev(eng, blob, ranges, fmt=nat.FMT_S16, errors=errors, stats=stats)
    want_errors, want_stats = {}, {}
    want = decode.decode_alac_files_dev(eng, blob, ranges, fmt=nat.FMT_S16, errors=want_errors, stats=want_stats)
    assert stats["calls"] == ["alac"] and stats["read_back_bytes"] == 4 * len(files) + want_stats["read_back_bytes"]
    assert (np.asarray(stats["alac"]["status"]) == np.asarray(want_stats["status"])).all()
    assert errors == want_errors
    for (a, ra), (b, rb) in zip(got, want):
        assert ra == rb and a.shape == b.shape and bool((a == b).all())


def test_lists_without_caf_make_the_same_calls(eng):
    """A list without CAF files: the kinds' calls only, and read-back of the heads plus each kind's own."""
    from tests import _flac_corpus
    files = [f for _, f in _flac_corpus.files()[:6]]
    blob, ranges = _resident(files)
    stats, flac_stats = {}, {}
    decode.decode_any_files_dev(eng, blob, ranges, fmt=nat.FMT_S32, stats=stats)
    decode.decode_flac_files_dev(eng, blob, ranges, fmt=nat.FMT_S32, stats=flac_stats)
    assert stats["calls"] == ["flac"] and stats["read_back_bytes"] == 4 * len(files) + flac_stats["read_back_bytes"]
    host_stats = {}
    decode.decode_any_files(eng, files, fmt=nat.FMT_S32, stats=host_stats)
    assert host_stats["calls"] == ["flac"]
