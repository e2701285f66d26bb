"""symgpu_ogg_index_dev: Ogg files already in device memory indexed by one call, against packetizer.ogg_index of each file's bytes."""
import ctypes

import numpy as np
import pytest

from tests import _ogg_corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import symphonia_b200 as sb
    e = sb.Engine(0)
    yield e
    e.close()


def _upload(files, gap=5):
    """The files back to back in one CUDA tensor, `gap` junk bytes between them; (tensor, ranges)."""
    import torch
    parts, ranges, at = [], [], 0
    for k, f in enumerate(files):
        parts += [np.frombuffer(f, dtype=np.uint8), np.full(gap, 0x4f, dtype=np.uint8)]   # 'O': a file's last bytes never see the next
        ranges.append((at, len(f)))
        at += len(f) + gap
    buf = np.concatenate(parts) if parts else np.zeros(0, dtype=np.uint8)
    return torch.from_numpy(buf).cuda(), ranges


def _tables(packets_t, pieces_t, index, i):
    from symphonia_b200 import _native as nat
    packets = packets_t.cpu().numpy().view(nat.OGG_PACKET_DTYPE)
    pieces = pieces_t.cpu().numpy().view(nat.PIECE_DTYPE)
    r = index[i]
    return (packets[int(r["first_packet"]):int(r["first_packet"]) + int(r["n_packets"])],
            pieces[int(r["first_piece"]):int(r["first_piece"]) + int(r["n_pieces"])])


def _host_status(data):
    from symphonia_b200 import _native as nat
    a = np.frombuffer(data, dtype=np.uint8)
    n, m = ctypes.c_size_t(0), ctypes.c_size_t(0)
    rc = nat.lib().symgpu_ogg_index(ctypes.c_void_p(a.ctypes.data) if a.size else None, a.size, None, 0, ctypes.byref(n), None, 0, ctypes.byref(m))
    return 1 if rc == 1 else 0


def test_index_equals_the_host_index_per_file(eng):
    from symphonia_b200 import packetizer
    files = [d for _, d in _ogg_corpus.files()]
    files += [b"", bytes(300), np.random.default_rng(5).integers(0, 256, 3000, dtype=np.uint8).tobytes(), files[0][:len(files[0]) // 2 + 3]]
    order = np.random.default_rng(6).permutation(len(files))
    files = [files[i] for i in order]
    data_t, ranges = _upload(files)
    packets_t, pieces_t, index = eng.ogg_index_dev(data_t, ranges)
    total = 0
    for i, f in enumerate(files):
        want_packets, want_pieces = packetizer.ogg_index(f)
        got_packets, got_pieces = _tables(packets_t, pieces_t, index, i)
        assert got_packets.tobytes() == want_packets.tobytes(), i
        assert got_pieces.tobytes() == want_pieces.tobytes(), i
        assert int(index[i]["status"]) == _host_status(f), i
        assert int(index[i]["packet_bytes"]) == int(want_packets["len"].sum())
        assert int(index[i]["max_packet_len"]) == (int(want_packets["len"].max()) if len(want_packets) else 0)
        total += len(want_packets)
    assert total > 2500


def test_launches_do_not_grow_with_the_files(eng):
    from symphonia_b200 import _native as nat
    files = [d for name, d in _ogg_corpus.files() if name.startswith("vorbis-")]
    counts = []
    for n in (8, 64):
        data_t, ranges = _upload([files[k % len(files)] for k in range(n)])
        packets_t, pieces_t, _ = eng.ogg_index_dev(data_t, ranges)
        before = eng.launch_count
        _, _, index = eng.ogg_index_dev(data_t, ranges, packets_t.numel() // nat.OGG_PACKET_DTYPE.itemsize, pieces_t.numel() // nat.PIECE_DTYPE.itemsize)
        counts.append(eng.launch_count - before)
        assert not (index["status"] & nat.OGG_NOT_WRITTEN).any()
    assert counts[0] == counts[1] == 5


def test_capacities_below_the_totals_write_nothing_for_the_files_past_them(eng):
    import torch
    from symphonia_b200 import _native as nat
    from symphonia_b200 import packetizer
    files = [d for name, d in _ogg_corpus.files() if name.startswith("vorbis-")][:6]
    data_t, ranges = _upload(files)
    _, _, full = eng.ogg_index_dev(data_t, ranges)
    cap = int(full["first_packet"][3])                 # the first three files fit
    packets_t, pieces_t, index = eng.ogg_index_dev(data_t, ranges, cap, int(full["first_piece"][-1] + full["n_pieces"][-1]))
    assert (index["status"][:3] & nat.OGG_NOT_WRITTEN == 0).all() and (index["status"][3:] & nat.OGG_NOT_WRITTEN != 0).all()
    for i in range(3):
        assert _tables(packets_t, pieces_t, index, i)[0].tobytes() == packetizer.ogg_index(files[i])[0].tobytes()
    assert packets_t.numel() == cap * nat.OGG_PACKET_DTYPE.itemsize and torch.cuda.is_available()


def test_argument_errors_launch_nothing(eng):
    import symphonia_b200 as sb
    from symphonia_b200 import _native as nat
    data_t, ranges = _upload([b"OggS" * 10])
    before = eng.launch_count
    for bad, status in (([(0, len(data_t) + 1)], 6), ([(len(data_t), 1)], 6), ([(2**63, 2**63)], 6), ([(0, 1)] * (nat.OGG_MAX_FILES + 1), 3)):
        with pytest.raises(sb.SymgpuError) as e:
            eng.ogg_index_dev(data_t, bad, 0, 0)
        assert e.value.status == status
    assert eng.launch_count == before
    _, _, index = eng.ogg_index_dev(data_t, [], 0, 0)       # no file: no launch
    assert len(index) == 0 and eng.launch_count == before


def test_many_logical_streams_cost_linear_time(eng):
    """A 3 MB file of 37 500 small pages, 30 000 of them announcing a serial of their own: the walk is linear in the pages, so a
    call takes milliseconds, and the tables equal the host's."""
    import time

    from symphonia_b200 import packetizer
    data = _ogg_corpus.many_serials(30000, seed=36)
    assert len(data) > 1_000_000
    data_t, ranges = _upload([data])
    eng.ogg_index_dev(data_t, ranges)
    t = time.perf_counter()
    packets_t, pieces_t, index = eng.ogg_index_dev(data_t, ranges)
    assert time.perf_counter() - t < 2.0
    want_packets, want_pieces = packetizer.ogg_index(data)
    got_packets, got_pieces = _tables(packets_t, pieces_t, index, 0)
    assert len(want_packets) == 30000 and len(np.unique(want_packets["serial"])) == 30000
    assert got_packets.tobytes() == want_packets.tobytes() and got_pieces.tobytes() == want_pieces.tobytes()
