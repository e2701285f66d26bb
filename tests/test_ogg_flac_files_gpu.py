"""FLAC in Ogg decoded on the device, many files per call: decode.decode_ogg_flac_files (host index, device=False and True) and
decode.decode_ogg_flac_files_dev (pages, identification packets and jobs on the device).  Every file of
tests/_ogg_flac_corpus.py must come out bit-identical to decode_flac_files of its native twin, in every sample format, through
all three calls, with the same messages, the same results for failed files and the same per-packet status."""
import numpy as np
import pytest
import torch

import symphonia_b200 as sb
from symphonia_b200 import _native as nat
from symphonia_b200 import decode
from tests import _flac_corpus, _ogg_flac_corpus

pytestmark = pytest.mark.gpu

FMTS = (nat.FMT_S32, nat.FMT_S24, nat.FMT_S16, nat.FMT_U8, nat.FMT_F32)


@pytest.fixture(scope="module")
def eng():
    with sb.Engine(0) as e:
        yield e


@pytest.fixture(scope="module")
def corpus():
    return _ogg_flac_corpus.files()


def _np(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else x


def _same(a, b):
    a, b = np.ascontiguousarray(_np(a)), np.ascontiguousarray(_np(b))
    return a.shape == b.shape and a.dtype == b.dtype and (a.view(np.uint8) == b.view(np.uint8)).all()


def _resident(files, seed):
    buf, ranges = _flac_corpus.pack(files, seed)
    return torch.from_numpy(buf).cuda(), ranges


def _three(eng, files, fmt, seed=1):
    """[(results, errors, status)] of the host-indexed call (device False / True) and the resident call."""
    out = []
    for device in (False, True):
        errors, stats = {}, {}
        out.append((decode.decode_ogg_flac_files(eng, files, threads=4, device=device, errors=errors, fmt=fmt, stats=stats), errors, stats["status"]))
    data_t, ranges = _resident(files, seed)
    errors, stats = {}, {}
    out.append((decode.decode_ogg_flac_files_dev(eng, data_t, ranges, fmt, errors=errors, stats=stats), errors, stats["status"]))
    return out


@pytest.mark.parametrize("fmt", FMTS)
def test_equal_to_the_native_twins(eng, corpus, fmt):
    files = [d for _, d, _ in corpus]
    twins = [t for _, _, t in corpus]
    good = [i for i, t in enumerate(twins) if t is not None]
    want = decode.decode_flac_files(eng, [twins[i] for i in good], fmt=fmt)
    runs = _three(eng, files, fmt)
    for got, errors, status in runs:
        assert sorted(errors) == [i for i, t in enumerate(twins) if t is None]
        for k, i in enumerate(good):
            assert got[i][1] == want[k][1] and _same(got[i][0], want[k][0]), corpus[i][0]
            assert len(got[i][0]) > 0 or corpus[i][0] == "frames the decoder refuses"
        for i in errors:
            assert tuple(got[i][0].shape) == (0, 0) and got[i][1] == 0
    (_, e0, s0), (_, e1, s1), (_, e2, s2) = runs
    assert e0 == e1 == e2 and _same(s0, s1) and _same(s0, s2)
    assert (s0 != 0).any() and (s0 == 0).any()       # refused packets are in the corpus


def test_failure_messages(eng, corpus):
    errors = {}
    decode.decode_ogg_flac_files(eng, [d for _, d, _ in corpus], errors=errors)
    names = {corpus[i][0]: m for i, m in errors.items()}
    assert names["no packets"] == "ValueError: no Ogg packets"
    assert names["STREAMINFO refused"].endswith("[1] symgpu_ogg_flac_packets")
    for n in ("identification packet of 50 bytes", "identification packet of 52 bytes", "major version 2", "wrong fLaC",
              "first block not STREAMINFO", "FLAC with a second stream of lower serial"):
        assert names[n].endswith("[2] symgpu_ogg_flac_packets"), n


def test_launches_do_not_grow_with_the_files(eng, corpus):
    files = [d for _, d, _ in corpus]
    counts = []
    for n in (len(files), 8 * len(files)):
        data_t, ranges = _resident((files * 8)[:n], 5)
        before = eng.launch_count
        decode.decode_ogg_flac_files_dev(eng, data_t, ranges)
        counts.append(eng.launch_count - before)
    assert counts[0] == counts[1] > 0


def test_one_long_file(eng):
    data, twin = _ogg_flac_corpus.long_file()
    want = decode.decode_flac_files(eng, [twin], fmt=nat.FMT_S16)[0]
    assert len(want[0]) > 1000 * 576
    got = decode.decode_ogg_flac_files(eng, [data], fmt=nat.FMT_S16)[0]
    assert got[1] == want[1] and _same(got[0], want[0])
    data_t, ranges = _resident([data], 6)
    got = decode.decode_ogg_flac_files_dev(eng, data_t, ranges, nat.FMT_S16)[0]
    assert got[1] == want[1] and _same(got[0], want[0])


def test_several_thousand_files(eng, corpus):
    files = [d for _, d, _ in corpus] * 150
    twins = [t for _, _, t in corpus] * 150
    good = [i for i, t in enumerate(twins) if t is not None]
    assert len(files) > 4000
    want = decode.decode_flac_files(eng, [twins[i] for i in good], fmt=nat.FMT_S32, device=True)
    data_t, ranges = _resident(files, 7)
    errors, stats = {}, {}
    got = decode.decode_ogg_flac_files_dev(eng, data_t, ranges, nat.FMT_S32, errors=errors, stats=stats)
    assert len(errors) == len(files) - len(good)
    for k, i in enumerate(good):
        assert got[i][1] == want[k][1] and torch.equal(got[i][0], want[k][0])
    host = {}
    decode.decode_ogg_flac_files(eng, files, errors=host)
    assert host == errors and stats["read_back_bytes"] > 0
