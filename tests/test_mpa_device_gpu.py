"""symgpu_mpa_index_dev (Engine.mpa_index_dev): the MPEG audio frame index of many files in device memory, against
symgpu_mpa_index of each file's bytes alone -- tracks, packets, jobs and status -- plus the launch count, capacities that are too
small, argument errors and the long files."""
import time

import numpy as np
import pytest

from symphonia_b200 import _native as nat
from tests import _mpa_corpus

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


def _host(data, seekable=True):
    from symphonia_b200 import SymgpuError, packetizer
    try:
        return packetizer.mpa_index(data, seekable)
    except SymgpuError as e:
        assert e.status == 1
        return None


def _check(eng, files, seed, seekable=True):
    """Every file's index equals the host index of its bytes; returns the packets in all."""
    data_t, ranges = _upload(files, seed)
    packets_t, jobs_t, index, tracks = eng.mpa_index_dev(data_t, ranges, seekable=seekable)
    packets = packets_t.cpu().numpy().view(nat.MPA_PACKET_DTYPE)
    jobs = jobs_t.cpu().numpy().view(nat.MP3_JOB_DTYPE)
    total = 0
    for i, f in enumerate(files):
        want = _host(f, seekable)
        ix = index[i]
        if want is None:
            assert ix["status"] == nat.MPA_NO_FRAME and ix["n_packets"] == 0 and tracks[i].tobytes() == bytes(48), i
            continue
        track, want_packets = want
        assert ix["status"] == 0 and ix["n_packets"] == len(want_packets), i
        assert tracks[i].tobytes() == np.asarray(track).tobytes(), i
        got = packets[int(ix["first_packet"]):][:len(want_packets)]
        assert got.tobytes() == want_packets.tobytes(), i
        j = jobs[int(ix["first_packet"]):][:len(want_packets)]
        assert (j["offset"] == want_packets["offset"] + np.uint64(ranges[i][0])).all() and (j["len"] == want_packets["size"]).all(), i
        assert (j["trim_start"] == want_packets["trim_start"]).all(), i
        assert (j["trim_end"] == np.minimum(want_packets["trim_end"], np.uint64(0xFFFFFFFF))).all(), i
        total += len(want_packets)
    return total


def test_corpus_equals_the_host_index(eng):
    files = [d for _, d in _mpa_corpus.files()] + [d for _, d in _mpa_corpus.decodable()]
    for seekable in (True, False):
        assert _check(eng, files, 61, seekable) > 4000


def test_long_files(eng):
    for files in ([_mpa_corpus.long_file()], [_mpa_corpus.dense_skip()], [_mpa_corpus.long_hunt()],
                  [_mpa_corpus.long_file(), _mpa_corpus.dense_skip(), _mpa_corpus.long_hunt(), b""]):
        data_t, ranges = _upload(files, 62)
        eng.mpa_index_dev(data_t, ranges)   # warm
        t0 = time.perf_counter()
        eng.mpa_index_dev(data_t, ranges)
        assert time.perf_counter() - t0 < 5.0   # a loose sanity bound on the host clock: no file is walked by one thread
        assert _check(eng, files, 62) >= (30000 if len(files[0]) == 30000 * 32 else 0)


def test_launches_do_not_grow_with_the_files(eng):
    files = [d for _, d in _mpa_corpus.decodable()][:8]   # the same files, so the same longest file, in both calls
    counts = []
    for n in (8, 64):
        data_t, ranges = _upload([files[k % len(files)] for k in range(n)], n)
        before = eng.launch_count
        eng.mpa_index_dev(data_t, ranges)
        counts.append(eng.launch_count - before)
    longest = max(len(f) for f in files)
    assert counts[0] == counts[1] == 10 + longest.bit_length() + (longest // 4).bit_length()


def test_a_small_capacity_leaves_out_the_files_that_do_not_fit(eng):
    files = [d for _, d in _mpa_corpus.decodable()]
    data_t, ranges = _upload(files, 63)
    n = [0 if _host(f) is None else len(_host(f)[1]) for f in files]
    first = np.concatenate([[0], np.cumsum(n)[:-1]])
    for cap in (0, 1, sum(n) // 2, sum(n) - 1, sum(n)):
        packets_t, jobs_t, index, _ = eng.mpa_index_dev(data_t, ranges, cap=cap)
        assert (index["first_packet"] == first).all() and (index["n_packets"] == n).all()
        over = (first + np.asarray(n)) > cap
        assert ((index["status"] & nat.MPA_NOT_WRITTEN) != 0).tolist() == over.tolist()
        packets = packets_t.cpu().numpy().view(nat.MPA_PACKET_DTYPE)
        for i in np.nonzero(~over)[0]:
            if n[i]:
                assert packets[first[i]:first[i] + n[i]].tobytes() == _host(files[i])[1].tobytes()


def test_argument_errors_and_no_file_launch_nothing(eng):
    import torch

    from symphonia_b200 import SymgpuError
    data_t, ranges = _upload([d for _, d in _mpa_corpus.decodable()][:2], 64)
    idx, trk = torch.empty(16 * 70000, dtype=torch.uint8, device="cuda"), torch.empty(48 * 70000, dtype=torch.uint8, device="cuda")
    before = eng.launch_count
    for bad, status in (([(0, data_t.numel() + 1)], 6), ([(data_t.numel(), 1)], 6), ([(2**63, 2**63)], 6), ([(0, 1)] * (nat.MPA_MAX_FILES + 1), 3)):
        with pytest.raises(SymgpuError) as e:      # SYMGPU_ERR_ARG, SYMGPU_ERR_LIMIT
            eng.mpa_index_dev_queue(data_t, bad, 0, None, None, idx, trk)
        assert e.value.status == status
    assert eng.launch_count == before
    eng.mpa_index_dev_queue(data_t, [], 0, None, None, idx, trk)
    assert eng.launch_count == before
