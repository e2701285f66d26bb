"""decode.decode_mpeg_files_dev: MPEG audio files of every layer already in device memory, indexed on the device and decoded from
the job table in place, against decode.decode_mpeg_files(device=True) of the same bytes."""
import numpy as np
import pytest

from symphonia_b200 import _native as nat
from tests import _mpa_corpus
from tests import _streams as st

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import symphonia_b200 as sb
    e = sb.Engine(0)
    yield e
    e.close()


def _upload(files, seed):
    import torch
    buf, ranges = _mpa_corpus.pack(files, seed)
    return torch.from_numpy(buf).cuda(), ranges


def _corpus():
    """The decodable files (every layer, gapless, tag-only, over-reading), junk and frameless files."""
    files = [d for _, d in _mpa_corpus.decodable()]
    rng = np.random.default_rng(71)
    files += [st.mpa_junk(rng, 3000), b"", bytes(500), b"junk" * 40]
    return files


def _same(got, want):
    assert len(got) == len(want)
    for k, ((g, gr), (w, wr)) in enumerate(zip(got, want)):
        assert gr == wr and tuple(g.shape) == tuple(w.shape) and g.dtype == w.dtype, k
        assert g.is_cuda and (g.cpu().numpy().view(np.uint8) == w.cpu().numpy().view(np.uint8)).all(), k


def _both(eng, files, fmt, seed=7):
    from symphonia_b200 import decode
    e_h, s_h, e_d, s_d = {}, {}, {}, {}
    want = decode.decode_mpeg_files(eng, files, fmt, device=True, errors=e_h, stats=s_h)
    data_t, ranges = _upload(files, seed)
    got = decode.decode_mpeg_files_dev(eng, data_t, ranges, fmt, errors=e_d, stats=s_d)
    _same(got, want)
    assert e_d == e_h
    assert set(s_d) == set(s_h) | {"read_back_bytes"}
    if "rounds" in s_h:
        assert s_d["rounds"] == s_h["rounds"] and s_d["status"].tobytes() == s_h["status"].tobytes()
    return got, e_d, s_d


def test_corpus_equals_the_host_indexed_path(eng):
    files = _corpus()
    for fmt in (nat.FMT_S16, nat.FMT_F32):
        got, errors, stats = _both(eng, files, fmt)
        assert len(errors) >= 3 and all(v.startswith("SymgpuError: ") and v.endswith("[1] symgpu_mpa_index") for v in errors.values())
        assert sum(len(g) > 0 for g, _ in got) >= 12
        assert stats["rounds"] > 1 and (stats["status"] != 0).any()   # the over-reading file took extra rounds


def test_one_layer_family_only(eng):
    named = dict(_mpa_corpus.decodable())
    for names in (["layer1-0", "layer2-1", "layer1-2"], ["mp3-0", "tag-only", "gapless"], ["tag-only"]):
        _both(eng, [named[k] for k in names], nat.FMT_S16, seed=8)


def test_only_records_results_and_status_are_read_back(eng):
    from symphonia_b200 import packetizer
    files = _corpus()
    _, _, stats = _both(eng, files, nat.FMT_S16, seed=9)
    n_packets = 0
    for f in files:
        try:
            n_packets += len(packetizer.mpa_index(f)[1])
        except Exception:  # noqa: BLE001 -- a frameless file has no packet
            pass
    per_file = nat.MPA_FILE_INDEX_DTYPE.itemsize + nat.MPA_TRACK_DTYPE.itemsize + nat.MP3_RESULT_DTYPE.itemsize
    assert stats["read_back_bytes"] <= len(files) * per_file + n_packets
    assert stats["read_back_bytes"] < sum(len(f) for f in files) // 4


def test_argument_errors_launch_nothing(eng):
    import torch

    from symphonia_b200 import decode
    data_t, ranges = _upload(_corpus()[:2], 10)
    before = eng.launch_count
    for bad in ([(0, data_t.numel() + 1)], [(data_t.numel(), 1)], [(2**63, 2**63)], [(0, 1)] * (nat.MPA_MAX_FILES + 1)):
        with pytest.raises(ValueError):
            decode.decode_mpeg_files_dev(eng, data_t, bad)
    with pytest.raises(ValueError):
        decode.decode_mpeg_files_dev(eng, data_t.cpu(), ranges)
    with pytest.raises(ValueError):
        decode.decode_mpeg_files_dev(eng, data_t.view(torch.int8), ranges)
    assert eng.launch_count == before
    assert decode.decode_mpeg_files_dev(eng, data_t, []) == [] and eng.launch_count == before
