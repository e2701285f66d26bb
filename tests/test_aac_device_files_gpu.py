"""decode.decode_aac_files_dev: ADTS AAC-LC files already in device memory, indexed on the device and decoded from the job table
in place, against decode.decode_aac_files(device=True) of the same bytes."""
import numpy as np
import pytest

from tests import _aac_corpus, _adts_corpus
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
    buf, ranges = _adts_corpus.pack(files, seed)
    return torch.from_numpy(buf).cuda(), ranges


def _corpus():
    """The _aac_corpus files, junk, frameless files and a 3-channel file."""
    files = [d for _, d in _adts_corpus.aac_files()]
    rng = np.random.default_rng(51)
    files.append(st.mpa_junk(rng, 3000))                                              # junk: no ADTS frame, or a bad one
    files += [b"", bytes(500)]                                                        # frameless
    files.append(_aac_corpus.adts(_aac_corpus.quiet(4), 44100, 1, seed=3)[:-3])       # cut payload: three frames
    files.append(b"".join(st.adts_frame(rng, 60, channels=3) for _ in range(5)))      # 3 channels
    return files


def _same(got, want):
    assert len(got) == len(want)
    for k, ((g, gr), (w, wr)) in enumerate(zip(got, want)):
        assert gr == wr and tuple(g.shape) == tuple(w.shape) and g.dtype == w.dtype, k
        assert g.is_cuda and (g.cpu().numpy().view(np.uint8) == w.cpu().numpy().view(np.uint8)).all(), k


def _both(eng, files, fmt, seed=7):
    from symphonia_b200 import decode
    e_h, s_h, e_d, s_d = {}, {}, {}, {}
    want = decode.decode_aac_files(eng, files, fmt, device=True, errors=e_h, stats=s_h)
    data_t, ranges = _upload(files, seed)
    got = decode.decode_aac_files_dev(eng, data_t, ranges, fmt, errors=e_d, stats=s_d)
    _same(got, want)
    assert e_d == e_h
    assert s_d["n_redecoded"] == s_h["n_redecoded"] and s_d["status"].tobytes() == s_h["status"].tobytes()
    return got, e_d, s_d


def test_corpus_equals_the_host_indexed_path(eng):
    from symphonia_b200 import _native as nat
    files = _corpus()
    for fmt in (nat.FMT_S16, nat.FMT_F32):
        got, errors, stats = _both(eng, files, fmt)
        assert sum(len(g) > 0 for g, _ in got) >= len(_adts_corpus.aac_files())
        assert set(errors.values()) == {"ValueError: no ADTS frames", "ValueError: channel configuration outside AAC-LC mono / stereo"}
        assert stats["n_redecoded"] > 0 and (stats["status"] != 0).any()


def test_launches_do_not_grow_with_the_files(eng):
    from symphonia_b200 import _native as nat
    from symphonia_b200 import decode
    files = [d for _, d in _adts_corpus.aac_files()][:8]   # the same files, so the same index rounds, in both calls
    counts = []
    for n in (8, 64):
        data_t, ranges = _upload([files[k % len(files)] for k in range(n)], n)
        decode.decode_aac_files_dev(eng, data_t, ranges, nat.FMT_S16)
        before = eng.launch_count
        decode.decode_aac_files_dev(eng, data_t, ranges, nat.FMT_S16)
        counts.append(eng.launch_count - before)
    assert counts[0] == counts[1]


def test_only_records_results_and_status_are_read_back(eng):
    from symphonia_b200 import _native as nat
    from symphonia_b200 import packetizer
    files = _corpus()
    _, _, stats = _both(eng, files, nat.FMT_S16, seed=9)
    n_packets = sum(len(packetizer.adts_index(f)[0]) for f in files)
    assert stats["read_back_bytes"] <= len(files) * (nat.ADTS_FILE_INDEX_DTYPE.itemsize + nat.AAC_RESULT_DTYPE.itemsize) + n_packets
    assert stats["read_back_bytes"] < sum(len(f) for f in files) // 4


def test_argument_errors_launch_nothing(eng):
    import torch
    from symphonia_b200 import _native as nat
    from symphonia_b200 import decode
    data_t, ranges = _upload([d for _, d in _adts_corpus.aac_files()][:2], 10)
    before = eng.launch_count
    for bad in ([(0, data_t.numel() + 1)], [(data_t.numel(), 1)], [(2**63, 2**63)], [(0, 1)] * (nat.ADTS_MAX_FILES + 1)):
        with pytest.raises(ValueError):
            decode.decode_aac_files_dev(eng, data_t, bad)
    with pytest.raises(ValueError):
        decode.decode_aac_files_dev(eng, data_t.cpu(), ranges)
    with pytest.raises(ValueError):
        decode.decode_aac_files_dev(eng, data_t.view(torch.int8), ranges)
    assert eng.launch_count == before
    assert decode.decode_aac_files_dev(eng, data_t, []) == [] and eng.launch_count == before
