"""FLAC in Ogg inside mixed lists: decode.decode_any_files and decode.decode_any_files_dev route an Ogg file to 'oggflac' when its
chosen stream's first packet is an Ogg FLAC identification packet, and every other Ogg file to 'vorbis'.  Host and resident
calls must agree on results, messages and calls; the resident call's read-back identity must hold; and taking the Ogg FLAC files
out of a list must leave every other kind's results and stats -- its read-back count included -- as they were."""
import numpy as np
import pytest
import torch

import symphonia_b200 as sb
from symphonia_b200 import _native as nat
from oracle import ogg_flac_oracle
from symphonia_b200 import decode
from tests import _flac_corpus, _ogg_flac_corpus
from tests import test_zz_many_files as many
from tests.test_flac_decode_gpu import _corpus as flac_corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    with sb.Engine(0) as e:
        yield e


@pytest.fixture(scope="module")
def lists():
    """(mixed list, the positions of its Ogg FLAC files, the same list without them).  The corpus files whose stream is not Ogg
    FLAC stay in both lists: they are Vorbis files to the router."""
    corpus = [d for _, d, _ in _ogg_flac_corpus.files()]
    oggflac = [d for d in corpus if ogg_flac_oracle.read(d)["status"] in ("ok", "bad streaminfo")]
    not_flac = [d for d in corpus if not any(d is o for o in oggflac)]
    lossy = many._files()
    vorbis = next(f for f in lossy if decode.sniff(f) == "vorbis")
    bad = [b"\x00" * 50, vorbis[:20], b"fLaC" + bytes(5), b""]
    files = lossy + [d for _, d, _ in flac_corpus()][:4] + bad + not_flac + oggflac
    order = np.random.default_rng(151).permutation(len(files))
    files = [files[i] for i in order]
    flac_at = [i for i, f in enumerate(files) if any(f is o for o in oggflac)]
    return files, flac_at, [f for i, f in enumerate(files) if i not in set(flac_at)]


def _np(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else x


def _same(a, b):
    a, b = np.ascontiguousarray(_np(a)), np.ascontiguousarray(_np(b))
    return a.shape == b.shape and a.dtype == b.dtype and (a.view(np.uint8) == b.view(np.uint8)).all()


def _same_stats(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        if isinstance(a[k], np.ndarray):
            assert _same(a[k], b[k]), k
        else:
            assert a[k] == b[k], k


def _dev(eng, files, fmt, seed):
    buf, ranges = _flac_corpus.pack(files, seed)
    errors, stats = {}, {}
    got = decode.decode_any_files_dev(eng, torch.from_numpy(buf).cuda(), ranges, fmt, errors=errors, stats=stats)
    return got, errors, stats


@pytest.mark.parametrize("fmt", (nat.FMT_S16, nat.FMT_F32, nat.FMT_S32))
def test_mixed_list_host_and_resident(eng, lists, fmt):
    files, flac_at, _ = lists
    errors, stats = {}, {}
    host = decode.decode_any_files(eng, files, fmt, threads=4, device=True, errors=errors, stats=stats)
    got, errors_dev, stats_dev = _dev(eng, files, fmt, 152)
    assert stats["calls"] == stats_dev["calls"] == ["flac", "aac", "vorbis", "oggflac", "mpa"]
    assert errors == errors_dev
    for (g, gr), (w, wr) in zip(got, host):
        assert gr == wr and _same(g, w)
    mine = decode.decode_ogg_flac_files(eng, [files[i] for i in flac_at], fmt=fmt, device=True)
    for i, (w, wr) in zip(flac_at, mine):
        assert host[i][1] == wr and _same(host[i][0], w)
    assert _same(stats["oggflac"]["status"], stats_dev["oggflac"]["status"])
    assert stats_dev["read_back_bytes"] == 4 * len(files) + sum(stats_dev[k]["read_back_bytes"] for k in stats_dev["calls"])


def test_removing_the_ogg_flac_files_changes_nothing_else(eng, lists):
    files, flac_at, rest = lists
    keep = [i for i in range(len(files)) if i not in set(flac_at)]
    for fmt in (nat.FMT_S16, nat.FMT_F32):
        full, errors_full, stats_full = _dev(eng, files, fmt, 153)
        got, errors, stats = _dev(eng, rest, fmt, 153)
        assert stats["calls"] == ["flac", "aac", "vorbis", "mpa"]
        assert errors == {keep.index(i): m for i, m in errors_full.items() if i in set(keep)}
        for k, i in enumerate(keep):
            assert got[k][1] == full[i][1] and _same(got[k][0], full[i][0])
        for kind in stats["calls"]:
            _same_stats(stats[kind], stats_full[kind])
        assert stats["read_back_bytes"] == 4 * len(rest) + sum(stats[k]["read_back_bytes"] for k in stats["calls"])
        host_errors, host_stats = {}, {}
        host = decode.decode_any_files(eng, rest, fmt, threads=4, errors=host_errors, stats=host_stats)
        assert host_stats["calls"] == stats["calls"] and host_errors == errors
        for (g, gr), (w, wr) in zip(got, host):
            assert gr == wr and _same(g, w)


def test_an_ogg_flac_file_alone_and_a_lower_serial_vorbis_stream(eng):
    corpus = {n: d for n, d, _ in _ogg_flac_corpus.files()}
    files = [corpus["plain stereo"], corpus["FLAC with a second stream of lower serial"], corpus["major version 2"]]
    for run in (lambda: decode.decode_any_files(eng, files, nat.FMT_S16, errors=errors, stats=stats),
                lambda: _dev(eng, files, nat.FMT_S16, 154)):
        errors, stats = {}, {}
        got = run()
        if isinstance(got, tuple):
            got, errors, stats = got
        assert stats["calls"] == ["vorbis", "oggflac"]
        assert sorted(errors) == [1, 2] and len(got[0][0]) > 0


def test_many_ogg_files_and_the_shared_ogg_limit(eng):
    """A list of 8 192 Ogg files, half FLAC in Ogg, through decode_any_files_dev equals decode_any_files; and the Ogg files of a
    resident list share one limit, named as such, checked before anything is launched."""
    corpus = _ogg_flac_corpus.files()
    files = [d for _, d, _ in corpus] * (8192 // len(corpus) + 1)
    files = files[:8192]
    got, errors, stats = _dev(eng, files, nat.FMT_S16, 155)
    host_errors, host_stats = {}, {}
    host = decode.decode_any_files(eng, files, nat.FMT_S16, errors=host_errors, stats=host_stats)
    assert stats["calls"] == host_stats["calls"] == ["vorbis", "oggflac"] and errors == host_errors
    for (g, gr), (w, wr) in zip(got, host):
        assert gr == wr and _same(g, w)
    one = corpus[0][1]
    data_t = torch.from_numpy(np.frombuffer(one, dtype=np.uint8).copy()).cuda()
    before = eng.launch_count
    with pytest.raises(ValueError, match="65536 Ogg files"):
        decode.decode_any_files_dev(eng, data_t, [(0, len(one))] * (nat.OGG_MAX_FILES + 1))
    assert eng.launch_count == before
