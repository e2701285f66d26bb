"""decode.decode_any_files_dev: a shuffled mixed list of native FLAC, ADTS AAC-LC, Ogg Vorbis and MPEG audio files already in
device memory, with failing files of every kind, against decode.decode_any_files(device=True) of the same bytes: results at their
input positions, the same messages and the same per-kind stats."""
import numpy as np
import pytest

import symphonia_b200 as sb
from symphonia_b200 import _native as nat
from symphonia_b200 import decode
from tests import _flac_corpus
from tests import test_zz_many_files as many
from tests.test_flac_decode_gpu import _corpus as flac_corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    with sb.Engine(0) as e:
        yield e


@pytest.fixture(scope="module")
def mixed():
    flac = [d for _, d, _ in flac_corpus()]
    rng = np.random.default_rng(141)
    garbage = b"\x00" + rng.integers(0, 255, 900, dtype=np.uint8).tobytes()
    lossy = many._files()
    vorbis = next(f for f in lossy if decode.sniff(f) == "vorbis")
    aac = next(f for f in lossy if decode.sniff(f) == "aac")
    bad = [garbage, vorbis[:20], b"fLaC" + bytes(5), b"", aac[:5], b"fL", b"\xff\xf1"]
    files = lossy + flac[:6] + flac[13:16] + flac[-1:] + bad
    order = np.random.default_rng(142).permutation(len(files))
    return [files[i] for i in order]


def _same(got, want):
    assert len(got) == len(want)
    for k, ((g, gr), (w, wr)) in enumerate(zip(got, want)):
        assert gr == wr and tuple(g.shape) == tuple(w.shape) and g.dtype == w.dtype, k
        assert g.is_cuda and (g.cpu().numpy().view(np.uint8) == w.cpu().numpy().view(np.uint8)).all(), k


def _without_reads(stats):
    return {k: ({kk: vv for kk, vv in v.items() if kk != "read_back_bytes"} if isinstance(v, dict) else v) for k, v in stats.items() if k != "read_back_bytes"}


def _equal_stats(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], dict):
            assert a[k].keys() == b[k].keys(), k
            for kk in a[k]:
                x, y = a[k][kk], b[k][kk]
                assert (np.asarray(x) == np.asarray(y)).all() if isinstance(x, np.ndarray) else x == y, (k, kk)
        else:
            assert a[k] == b[k], k


@pytest.mark.parametrize("fmt", (nat.FMT_S16, nat.FMT_F32))
def test_same_as_the_host_sniffed_path(eng, mixed, fmt):
    import torch
    buf, ranges = _flac_corpus.pack(mixed, 143)
    data_t = torch.from_numpy(buf).cuda()
    errors, stats = {}, {}
    want = decode.decode_any_files(eng, mixed, fmt, threads=4, device=True, errors=errors, stats=stats)
    errors_dev, stats_dev = {}, {}
    got = decode.decode_any_files_dev(eng, data_t, ranges, fmt, errors=errors_dev, stats=stats_dev)
    _same(got, want)
    assert errors_dev == errors and len(errors) >= 6
    assert stats_dev["calls"] == stats["calls"] == ["flac", "aac", "vorbis", "mpa"]
    _equal_stats(_without_reads(stats_dev), stats)
    kinds = stats_dev["calls"]
    assert stats_dev["read_back_bytes"] == 4 * len(mixed) + sum(stats_dev[k]["read_back_bytes"] for k in kinds)


def test_only_present_kinds_and_no_file(eng, mixed):
    import torch
    flac = [f for f in mixed if decode.sniff(f) == "flac"]
    buf, ranges = _flac_corpus.pack(flac, 144)
    stats = {}
    got = decode.decode_any_files_dev(eng, torch.from_numpy(buf).cuda(), ranges, nat.FMT_S32, stats=stats)
    _same(got, decode.decode_flac_files(eng, flac, device=True, fmt=nat.FMT_S32))
    assert stats["calls"] == ["flac"]
    stats = {}
    assert decode.decode_any_files_dev(eng, torch.from_numpy(buf).cuda(), [], stats=stats) == [] and stats["calls"] == []
