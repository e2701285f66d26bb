"""symgpu_adts_index_dev: ADTS files already in device memory indexed by one call, against packetizer.adts_index of each file's
bytes."""
import numpy as np
import pytest

from tests import _adts_corpus

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


def _packets(packets_t, jobs_t, index, i):
    from symphonia_b200 import _native as nat
    packets = packets_t.cpu().numpy().view(nat.ADTS_PACKET_DTYPE)
    jobs = jobs_t.cpu().numpy().view(nat.PIECE_DTYPE)
    a, n = int(index[i]["first_packet"]), int(index[i]["n_packets"])
    return packets[a:a + n], jobs[a:a + n]


def _same_as_host(files, ranges, packets_t, jobs_t, index, only=None):
    from symphonia_b200 import packetizer
    total = 0
    for i, f in enumerate(files):
        if only is not None and i not in only:
            continue
        want, stop = packetizer.adts_index(f)
        got, jobs = _packets(packets_t, jobs_t, index, i)
        assert got.tobytes() == want.tobytes(), i
        assert int(index[i]["stop"]) == stop, i
        head = (int(want[0]["sample_rate"]), int(want[0]["channels"]), int(want[0]["profile"])) if len(want) else (0, 0, 0)
        assert (int(index[i]["sample_rate"]), int(index[i]["channels"]), int(index[i]["profile"])) == head, i
        assert (jobs["offset"] == want["offset"] + np.uint64(ranges[i][0])).all() and (jobs["len"] == want["size"]).all(), i
        total += len(want)
    return total


def test_index_equals_the_host_index_per_file(eng):
    files = [d for _, d in _adts_corpus.files()]
    data_t, ranges = _upload(files, 41)
    packets_t, jobs_t, index = eng.adts_index_dev(data_t, ranges)
    assert not index["status"].any()
    assert _same_as_host(files, ranges, packets_t, jobs_t, index) > 900
    assert set(int(s) for s in index["stop"]) == {0, 1, 2, 3}


def test_launches_do_not_grow_with_the_files(eng):
    files = [d for _, d in _adts_corpus.aac_files()][:8]   # the same files, so the same longest file, in both calls
    counts = []
    for n in (8, 64):
        data_t, ranges = _upload([files[k % len(files)] for k in range(n)], n)
        eng.adts_index_dev(data_t, ranges)
        before = eng.launch_count
        eng.adts_index_dev(data_t, ranges)
        counts.append(eng.launch_count - before)
    k = (max(len(f) for f in files) // 2).bit_length()
    assert counts[0] == counts[1] == 7 + k


def test_a_capacity_below_the_total_writes_the_files_that_fit(eng):
    from symphonia_b200 import _native as nat
    files = [d for _, d in _adts_corpus.aac_files()][:6]
    data_t, ranges = _upload(files, 42)
    _, _, full = eng.adts_index_dev(data_t, ranges)
    order = np.argsort(full["first_packet"], kind="stable")
    cap = int(full["first_packet"][order[3]])          # the files before the fourth in the table fit
    packets_t, jobs_t, index = eng.adts_index_dev(data_t, ranges, cap)
    fits = full["first_packet"] + full["n_packets"] <= cap
    assert fits.sum() == 3
    assert (((index["status"] & nat.ADTS_NOT_WRITTEN) != 0) == ~fits).all()
    assert (index["n_packets"] == full["n_packets"]).all() and (index["first_packet"] == full["first_packet"]).all()
    _same_as_host(files, ranges, packets_t, jobs_t, index, only=set(np.nonzero(fits)[0]))


def test_argument_errors_launch_nothing(eng):
    import symphonia_b200 as sb
    from symphonia_b200 import _native as nat
    data_t, _ = _upload([_adts_corpus.ends()[0][1]], 43)
    before = eng.launch_count
    for bad, status in (([(0, data_t.numel() + 1)], 6), ([(data_t.numel(), 1)], 6), ([(2**63, 2**63)], 6),
                        ([(0, 1)] * (nat.ADTS_MAX_FILES + 1), 3)):
        with pytest.raises(sb.SymgpuError) as e:
            eng.adts_index_dev(data_t, bad, 0)
        assert e.value.status == status
    assert eng.launch_count == before
    _, _, index = eng.adts_index_dev(data_t, [], 0)         # no file: no launch
    assert len(index) == 0 and eng.launch_count == before


def test_a_long_file(eng):
    """30 000 frames in one file: the chain is ranked in K rounds, not walked, and the call is quick (a loose host-clock bound, a
    sanity check rather than a measurement)."""
    import time
    long = _adts_corpus.long_file()
    data_t, ranges = _upload([long, _adts_corpus.dense_sync()], 44)
    eng.adts_index_dev(data_t, ranges)
    t = time.perf_counter()
    packets_t, jobs_t, index = eng.adts_index_dev(data_t, ranges)
    assert time.perf_counter() - t < 1.0
    assert int(index[0]["n_packets"]) == 30000
    _same_as_host([long, _adts_corpus.dense_sync()], ranges, packets_t, jobs_t, index)
