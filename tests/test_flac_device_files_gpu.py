"""decode.decode_flac_files_dev: native FLAC files already in device memory, indexed on the device and decoded from the job table
in place, against decode.decode_flac_files(device=True) of the same bytes, in every output format."""
import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import decode
from tests import _flac_corpus

pytestmark = pytest.mark.gpu

FORMATS = (nat.FMT_S32, nat.FMT_S24, nat.FMT_S16, nat.FMT_U8, nat.FMT_F32)


@pytest.fixture(scope="module")
def eng():
    import symphonia_b200 as sb
    e = sb.Engine(0)
    yield e
    e.close()


def _corpus():
    """The decodable files of every depth, channel count, block size and blocking strategy, plus files that fail to open (empty, a
    marker without STREAMINFO, no marker, frames without the marker), one that opens without frames and one with a cut last
    frame."""
    from tests.test_flac_decode_gpu import _corpus as decodable
    files = [d for _, d, _ in decodable()]
    files += [b"", b"fLaC" + bytes(5), b"junk" * 30, _flac_corpus.files()[-12][1], files[2][:len(files[2]) - 9],
              b"\xff\xf8\x00" * 10 + files[3] + b"\xff\xf8junk"]
    return files


def _upload(files, seed):
    import torch
    buf, ranges = _flac_corpus.pack(files, seed)
    return torch.from_numpy(buf).cuda(), ranges


def _same(got, want):
    assert len(got) == len(want)
    for k, ((g, gr), (w, wr)) in enumerate(zip(got, want)):
        assert gr == wr and tuple(g.shape) == tuple(w.shape) and g.dtype == w.dtype, k
        assert g.is_cuda and (g.cpu().numpy().view(np.uint8) == w.cpu().numpy().view(np.uint8)).all(), k


@pytest.mark.parametrize("fmt", FORMATS)
def test_bit_identical_to_the_host_indexed_path(eng, fmt):
    files = _corpus()
    data_t, ranges = _upload(files, 101)
    errors, errors_dev, stats = {}, {}, {}
    want = decode.decode_flac_files(eng, files, threads=4, device=True, errors=errors, fmt=fmt)
    got = decode.decode_flac_files_dev(eng, data_t, ranges, fmt, errors=errors_dev, stats=stats)
    _same(got, want)
    assert errors_dev == errors and len(errors) >= 3
    assert sum(int(r[0].shape[0]) for r in got) > 10000


def test_error_texts_and_read_back_bytes(eng):
    files = _corpus()
    data_t, ranges = _upload(files, 102)
    errors, stats = {}, {}
    got = decode.decode_flac_files_dev(eng, data_t, ranges, errors=errors, stats=stats)
    from symphonia_b200 import SymgpuError
    n = len(files) - 6
    assert errors[n + 1] == f"SymgpuError: {SymgpuError(1, 'symgpu_flac_index')}"      # a marker without STREAMINFO
    assert errors[n] == errors[n + 2] == errors[n + 5] == f"SymgpuError: {SymgpuError(2, 'symgpu_flac_index')}"   # no marker
    assert all(got[i][1] == 0 and tuple(got[i][0].shape) == (0, 0) for i in errors)
    n_jobs = sum(len(decode.packetizer.flac_index(f)[1]) for i, f in enumerate(files) if i not in errors)
    # the index records and stream infos, the frames per file and a status byte per packet: nothing else comes back
    assert stats["read_back_bytes"] == len(files) * (nat.FLAC_FILE_INDEX_DTYPE.itemsize + nat.FLAC_STREAM_INFO_DTYPE.itemsize + 8) + n_jobs


def test_no_file_and_argument_checks(eng):
    import torch
    data_t = torch.zeros(16, dtype=torch.uint8, device="cuda")
    assert decode.decode_flac_files_dev(eng, data_t, []) == []
    with pytest.raises(ValueError):
        decode.decode_flac_files_dev(eng, data_t, [(8, 9)])
    with pytest.raises(ValueError):
        decode.decode_flac_files_dev(eng, data_t.cpu(), [(0, 4)])
