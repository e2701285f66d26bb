"""symgpu_flac_index_dev (Engine.flac_index_dev): the native FLAC frame index of many files in device memory, against
symgpu_flac_index of each file's bytes alone -- stream infos, packets, jobs and the open status -- plus the launch count, capacities
that are too small, argument errors and the long files."""
import numpy as np
import pytest

from symphonia_b200 import _native as nat
from tests import _flac_corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import symphonia_b200 as sb
    e = sb.Engine(0)
    yield e
    e.close()


def _upload(files, seed):
    import torch
    buf, ranges = _flac_corpus.pack(files, seed)
    return torch.from_numpy(buf).cuda(), ranges


def _host(data):
    from symphonia_b200 import SymgpuError, packetizer
    try:
        return packetizer.flac_index(data)
    except SymgpuError as e:
        return e.status


def _check(eng, files, seed):
    """Every file's index equals the host index of its bytes; returns the packets in all."""
    data_t, ranges = _upload(files, seed)
    packets_t, jobs_t, index, infos = eng.flac_index_dev(data_t, ranges)
    packets = packets_t.cpu().numpy().view(nat.FLAC_PACKET_DTYPE)
    jobs = jobs_t.cpu().numpy().view(nat.FLAC_JOB_DTYPE)
    total = 0
    for i, f in enumerate(files):
        want = _host(f)
        ix = index[i]
        assert ix["status"] == 0, i
        if not isinstance(want, tuple):
            assert ix["open"] == want and ix["n_packets"] == 0 and ix["samples"] == 0 and infos[i].tobytes() == bytes(56), i
            continue
        info, want_packets = want
        assert ix["open"] == 0 and ix["n_packets"] == len(want_packets), i
        assert ix["samples"] == int(want_packets["dur"].astype(np.int64).sum()), i
        assert infos[i].tobytes() == np.asarray(info).tobytes(), i
        got = packets[int(ix["first_packet"]):][:len(want_packets)]
        assert got.tobytes() == want_packets.tobytes(), i
        j = jobs[int(ix["first_packet"]):][:len(want_packets)]
        assert (j["offset"] == want_packets["offset"] + np.uint64(ranges[i][0])).all() and (j["len"] == want_packets["size"]).all(), i
        assert (j["group"] == i).all() and (j["slot"] == want_packets["dur"]).all() and (j["reserved"] == 0).all(), i
        total += len(want_packets)
    return total


def test_corpus_equals_the_host_index(eng):
    from tests.test_flac_decode_gpu import _corpus
    files = [d for _, d in _flac_corpus.files()] + [d for _, d, _ in _corpus()]
    assert _check(eng, files, 91) > 600
    assert _check(eng, files[::-1], 92) > 600


def test_long_files(eng):
    chain, past, within, big = _flac_corpus.long_chain(), _flac_corpus.past_window(), _flac_corpus.within_window(), _flac_corpus.hundred_thousand()
    assert _check(eng, [chain], 93) == (1 << 15) - 8
    assert _check(eng, [past, within], 94) == 9
    assert _check(eng, [big, chain, b""], 95) == 100000 + (1 << 15) - 8


def test_launches_do_not_grow_with_the_files(eng):
    from tests.test_flac_decode_gpu import _corpus
    files = [d for _, d, _ in _corpus()][:8]   # the same files, so the same longest file, in both calls
    counts = []
    for n in (8, 64):
        data_t, ranges = _upload([files[k % len(files)] for k in range(n)], n)
        before = eng.launch_count
        eng.flac_index_dev(data_t, ranges)
        counts.append(eng.launch_count - before)
    longest = max(len(f) for f in files)
    assert counts[0] == counts[1] == 28 + 2 * (longest // 2).bit_length() + (longest // 8).bit_length()


def test_a_small_capacity_leaves_out_the_files_that_do_not_fit(eng):
    files = [d for _, d in _flac_corpus.files()]
    data_t, ranges = _upload(files, 96)
    n = [0 if not isinstance(_host(f), tuple) else len(_host(f)[1]) for f in files]
    first = np.concatenate([[0], np.cumsum(n)[:-1]])
    for cap in (0, 1, sum(n) // 2, sum(n) - 1, sum(n)):
        packets_t, jobs_t, index, _ = eng.flac_index_dev(data_t, ranges, cap=cap)
        assert (index["first_packet"] == first).all() and (index["n_packets"] == n).all()
        over = (first + np.asarray(n)) > cap
        assert ((index["status"] & nat.FLAC_NOT_WRITTEN) != 0).tolist() == over.tolist()
        packets = packets_t.cpu().numpy().view(nat.FLAC_PACKET_DTYPE)
        for i in np.nonzero(~over)[0]:
            if n[i]:
                assert packets[first[i]:first[i] + n[i]].tobytes() == _host(files[i])[1].tobytes()


def test_argument_errors_and_no_file_launch_nothing(eng):
    import torch

    from symphonia_b200 import SymgpuError
    data_t, ranges = _upload([d for _, d in _flac_corpus.files()][:2], 97)
    idx, inf = torch.empty(24 * 70000, dtype=torch.uint8, device="cuda"), torch.empty(56 * 70000, dtype=torch.uint8, device="cuda")
    before = eng.launch_count
    for bad, status in (([(0, data_t.numel() + 1)], 6), ([(data_t.numel(), 1)], 6), ([(2**63, 2**63)], 6), ([(0, 1)] * (nat.FLAC_MAX_FILES + 1), 3)):
        with pytest.raises(SymgpuError) as e:      # SYMGPU_ERR_ARG, SYMGPU_ERR_LIMIT
            eng.flac_index_dev_queue(data_t, bad, 0, None, None, idx, inf)
        assert e.value.status == status
    assert eng._lib.symgpu_flac_index_dev(eng._ctx, None, 0, None, 1, None, None, 0, None, None) == 6   # no file table
    assert eng.launch_count == before
    eng.flac_index_dev_queue(data_t, [], 0, None, None, idx, inf)
    assert eng.launch_count == before
