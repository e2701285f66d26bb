"""decode.decode_any_files: a mixed list of native FLAC, ADTS AAC-LC, Ogg Vorbis and MPEG audio files in one call, every file
decoded by the device decoder of its kind.  The call is routing, so the test is about places: every result at its input position
and equal to what the file's own decoder returns, errors keyed by input position, one sub-call per kind present and none for a
kind that is absent."""
import numpy as np
import pytest

import symphonia_b200 as sb
from symphonia_b200 import _native as nat
from symphonia_b200 import decode
from tests import test_zz_many_files as many
from tests.test_flac_decode_gpu import _corpus as flac_corpus

pytestmark = pytest.mark.gpu

ALONE = {"flac": lambda eng, f, fmt, device: decode.decode_flac_files(eng, [f], device=device, fmt=fmt)[0],
         "aac": lambda eng, f, fmt, device: decode.decode_aac_files(eng, [f], fmt, device=device)[0],
         "vorbis": lambda eng, f, fmt, device: decode.decode_vorbis_files(eng, [f], fmt, device=device)[0],
         "mpa": lambda eng, f, fmt, device: decode.decode_mpeg_files(eng, [f], fmt, device=device)[0]}


@pytest.fixture(scope="module")
def eng():
    with sb.Engine(0) as e:
        yield e


@pytest.fixture(scope="module")
def mixed():
    """(files, the positions of the files no decoder can open): the lossy corpus of test_zz_many_files, FLAC files of several bit
    depths, channel counts and block sizes, and four files that fail -- garbage, an Ogg page cut short, a FLAC marker without
    STREAMINFO, an empty file -- shuffled."""
    flac = [d for _, d, _ in flac_corpus()]
    rng = np.random.default_rng(41)
    garbage = b"\x00" + rng.integers(0, 255, 900, dtype=np.uint8).tobytes()     # (255 left out: no MPEG sync word by chance)
    vorbis = next(f for f in many._files() if decode.sniff(f) == "vorbis")
    bad = [garbage, vorbis[:20], b"fLaC" + bytes(5), b""]
    files = many._files() + flac[:6] + flac[13:16] + flac[-1:] + bad
    order = np.random.default_rng(42).permutation(len(files))
    files = [files[i] for i in order]
    return files, sorted(i for i, f in enumerate(files) if any(f is b for b in bad))


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and (np.ascontiguousarray(a).view(np.uint8) == np.ascontiguousarray(b).view(np.uint8)).all()


def test_every_file_as_its_own_decoder_decodes_it(eng, mixed):
    files, bad = mixed
    kinds = [decode.sniff(f) for f in files]
    assert set(kinds) == {"flac", "aac", "vorbis", "mpa"}
    lossy = [i for i, k in enumerate(kinds) if k != "flac" and i not in bad]
    for fmt in (nat.FMT_S16, nat.FMT_F32):
        errors, stats = {}, {}
        got = decode.decode_any_files(eng, files, fmt, threads=4, errors=errors, stats=stats)
        assert len(got) == len(files) and sorted(errors) == bad and all(errors[i] for i in bad)
        assert stats["calls"] == ["flac", "aac", "vorbis", "mpa"]
        assert stats["vorbis"]["n_setups"] >= 2 and "n_redecoded" in stats["aac"] and stats["mpa"]["rounds"] >= 1 and stats["flac"] == {}
        assert len(stats["aac"]["status"]) > 0 and len(stats["vorbis"]["status"]) > 0 and len(stats["mpa"]["status"]) > 0
        old = decode.decode_files(eng, [files[i] for i in lossy], fmt, threads=4)
        for i, (pcm, rate) in enumerate(got):
            assert isinstance(pcm, np.ndarray) and pcm.dtype == np.dtype(nat.FMT_NUMPY[fmt]), i
            if i in bad:
                assert pcm.shape == (0, 0) and rate == 0, i
                continue
            alone, alone_rate = ALONE[kinds[i]](eng, files[i], fmt, False)
            assert rate == alone_rate and rate > 0 and _same(pcm, alone), (i, kinds[i], fmt)
            if kinds[i] == "flac":
                host, host_rate = decode.decode_flac(eng, files[i], fmt)
                assert rate == host_rate and _same(pcm, host), (i, fmt)
            else:
                want, want_rate = old[lossy.index(i)]
                assert rate == want_rate and _same(pcm, want), (i, kinds[i], fmt)


def test_device_results_equal_host_results(eng, mixed):
    import torch
    files, bad = mixed
    for fmt in (nat.FMT_S16, nat.FMT_F32):
        host = decode.decode_any_files(eng, files, fmt)
        errors = {}
        dev = decode.decode_any_files(eng, files, fmt, device=True, errors=errors)
        assert sorted(errors) == bad
        for i, ((a, ra), (b, rb)) in enumerate(zip(host, dev)):
            assert b.is_cuda and b.dtype == getattr(torch, decode._TORCH_DTYPES[fmt]) and ra == rb, i
            assert tuple(b.shape) == a.shape and _same(b.cpu().numpy().reshape(a.shape), a), i


def test_only_the_kinds_present_are_called(eng, mixed):
    files, _ = mixed
    flac = [f for f in files if decode.sniff(f) == "flac"]
    before = eng.launch_count
    decode.decode_flac_files(eng, flac, fmt=nat.FMT_S16)
    flac_launches = eng.launch_count - before
    stats = {}
    before = eng.launch_count
    got = decode.decode_any_files(eng, flac, nat.FMT_S16, stats=stats)
    assert eng.launch_count - before == flac_launches and stats == {"calls": ["flac"], "flac": {}}
    assert len(got) == len(flac)
    vorbis_and_aac = [f for f in files if decode.sniff(f) in ("vorbis", "aac")]
    stats = {}
    decode.decode_any_files(eng, vorbis_and_aac, stats=stats)
    assert stats["calls"] == ["aac", "vorbis"] and "flac" not in stats and "mpa" not in stats
    stats = {}
    before = eng.launch_count
    assert decode.decode_any_files(eng, [], stats=stats) == [] and stats == {"calls": []} and eng.launch_count == before


def test_limits_hold_per_kind(eng):
    adts = b"\xff\xf1" + bytes(6)
    with pytest.raises(ValueError, match="decode_aac_files takes at most 65536 files"):
        decode.decode_any_files(eng, [adts] * ((1 << 16) + 1))
