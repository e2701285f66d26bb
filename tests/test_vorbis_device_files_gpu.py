"""decode.decode_vorbis_files_dev: Ogg Vorbis files already in device memory, indexed, given their jobs and decoded on the device,
against decode.decode_vorbis_files(device=True) of the same bytes."""
import numpy as np
import pytest

from tests import _ogg_corpus, _vorbis_corpus
from tests import _streams as st

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import symphonia_b200 as sb
    e = sb.Engine(0)
    yield e
    e.close()


def _upload(files, seed):
    """The files in one CUDA tensor, in a shuffled order with random junk (0 to 40 bytes) between them; (tensor, ranges)."""
    import torch
    rng = np.random.default_rng(seed)
    order = rng.permutation(len(files))
    parts, ranges, at = [], [None] * len(files), 0
    for i in order:
        gap = rng.integers(0, 256, int(rng.integers(0, 41)), dtype=np.uint8)
        parts += [gap, np.frombuffer(files[i], dtype=np.uint8)]
        at += gap.size
        ranges[i] = (at, len(files[i]))
        at += len(files[i])
    buf = np.concatenate(parts) if parts else np.zeros(0, dtype=np.uint8)
    return torch.from_numpy(buf).cuda(), ranges


def _corpus():
    files = [d for _, d in _vorbis_corpus.files()]
    files += [d for name, d in _ogg_corpus.files() if name.split("-")[0] in ("mux", "damage", "cut", "junk", "empty", "one")]
    whole = files[0]
    files.append(whole[:len(whole) // 2 + 11])   # cut mid-page
    files.append(whole[:58])                     # the identification page alone: no setup header
    return files


def _same(got, want):
    assert len(got) == len(want)
    for k, ((g, gr), (w, wr)) in enumerate(zip(got, want)):
        assert gr == wr and tuple(g.shape) == tuple(w.shape) and g.dtype == w.dtype, k
        assert g.is_cuda and (g.cpu().numpy().view(np.uint8) == w.cpu().numpy().view(np.uint8)).all(), k


def _both(eng, files, fmt, seed=7):
    from symphonia_b200 import decode
    e_h, s_h, e_d, s_d = {}, {}, {}, {}
    want = decode.decode_vorbis_files(eng, files, fmt, device=True, errors=e_h, stats=s_h)
    data_t, ranges = _upload(files, seed)
    got = decode.decode_vorbis_files_dev(eng, data_t, ranges, fmt, errors=e_d, stats=s_d)
    _same(got, want)
    assert e_d == e_h
    assert s_d["n_setups"] == s_h["n_setups"] and (s_d["status"] == s_h["status"]).all()
    return got, e_d, s_d


def test_whole_corpus_equals_the_host_indexed_path(eng):
    from symphonia_b200 import _native as nat
    files = _corpus()
    for fmt in (nat.FMT_S16, nat.FMT_F32):
        got, errors, stats = _both(eng, files, fmt)
        assert sum(len(g) > 0 for g, _ in got) >= 12 and len(errors) >= 20
        assert any(m == "ValueError: no Ogg packets" for m in errors.values())
        assert any(m == "ValueError: no Vorbis setup header" for m in errors.values())


def test_jobs_and_gathered_bytes_equal_the_host_plan(eng):
    from symphonia_b200 import _native as nat
    from symphonia_b200 import decode
    files = _corpus()
    plan = decode.vorbis_files_plan(files)
    seen = {}
    data_t, ranges = _upload(files, 8)
    decode._vorbis_files_dev(eng, data_t, ranges, nat.FMT_S16, None, None, mark=lambda phase, state: seen.update(state))
    eng.sync()
    jobs = seen["jobs"].cpu().numpy().view(nat.VORBIS_JOB_DTYPE)
    audio = seen["audio"].cpu().numpy()
    groups = seen["groups"]
    checked = 0
    for g in range(len(files)):
        hg, dg = plan["groups"][g], groups[g]
        assert hg["n_jobs"] == dg["n_jobs"] and hg["out_offset"] == dg["out_offset"] and hg["setup"] == dg["setup"], g
        hj = plan["jobs"][int(hg["first_job"]):int(hg["first_job"]) + int(hg["n_jobs"])]
        dj = jobs[int(dg["first_job"]):int(dg["first_job"]) + int(dg["n_jobs"])]
        for f in ("len", "discard", "trim_end"):
            assert (hj[f] == dj[f]).all(), (g, f)
        for a, b in zip(hj, dj):
            assert plan["data"][int(a["offset"]):int(a["offset"]) + int(a["len"])].tobytes() == audio[int(b["offset"]):int(b["offset"]) + int(b["len"])].tobytes()
        checked += len(dj)
    assert checked > 200 and (plan["jobs"]["trim_end"] > 0).any() and (plan["jobs"]["discard"] > 0).any()


def _one_segment_pages(seed, n):
    """A stream whose pages hold one lacing value each: every header and packet of 255 bytes or more spans pages."""
    s, pk = _vorbis_corpus.writer(seed, n, channels=2, bs_exp=(8, 11))
    pages = st.ogg_paginate(91, [s.ident, b"\x03vorbis" + bytes(20), s.setup] + pk, np.random.default_rng(seed), max_segments=1)
    return b"".join(pages)


def test_headers_and_packets_spanning_pages_and_a_long_file(eng):
    from symphonia_b200 import _native as nat
    from symphonia_b200 import decode, packetizer
    spanning = _one_segment_pages(1301, 12)
    s, pk = _vorbis_corpus.writer(1302, 100, channels=2, bs_exp=(8, 11))
    long = _vorbis_corpus.ogg(s, pk * 40, 1303)
    assert len(decode.ogg_vorbis_index(long)["table"]) >= 3000
    packets, _ = packetizer.ogg_index(spanning)
    assert packets["n_pieces"][2] > 1    # the setup header lies on several pages
    got, errors, _ = _both(eng, [spanning, long], nat.FMT_S16)
    assert not errors and all(len(g) > 0 for g, _ in got)


def test_launches_do_not_grow_with_the_files(eng):
    from symphonia_b200 import _native as nat
    from symphonia_b200 import decode
    files = [d for _, d in _vorbis_corpus.files()][:6]
    counts = []
    for n in (8, 64):
        data_t, ranges = _upload([files[k % len(files)] for k in range(n)], n)
        decode.decode_vorbis_files_dev(eng, data_t, ranges, nat.FMT_S16)
        before = eng.launch_count
        decode.decode_vorbis_files_dev(eng, data_t, ranges, nat.FMT_S16)
        counts.append(eng.launch_count - before)
    assert counts[0] == counts[1]


def test_only_records_and_headers_are_read_back(eng):
    from symphonia_b200 import _native as nat
    from symphonia_b200 import packetizer
    files = _corpus()
    _, _, stats = _both(eng, files, nat.FMT_S16, seed=9)
    header_bytes = 0
    for f in files:
        packets, _ = packetizer.ogg_index(f)
        if len(packets):
            lens = packets["len"][packets["serial"] == packets["serial"][0]]
            header_bytes += int(lens[0])
            setup = [packetizer.gather(f, packets[k], packetizer.ogg_index(f)[1]) for k in range(1, len(lens)) if lens[k] >= 7]
            setup = [b for b in setup if b[:7] == b"\x05vorbis"]
            header_bytes += len(setup[0]) if setup else 0
    n, n_jobs = len(files), len(stats["status"])
    records = n * (nat.OGG_FILE_INDEX_DTYPE.itemsize + nat.VORBIS_FILE_HEADS_DTYPE.itemsize + nat.VORBIS_RESULT_DTYPE.itemsize) + n_jobs
    assert stats["read_back_bytes"] <= records + header_bytes
    assert stats["read_back_bytes"] < sum(len(f) for f in files) // 4


def test_argument_errors_launch_nothing(eng):
    from symphonia_b200 import _native as nat
    from symphonia_b200 import decode
    data_t, ranges = _upload([d for _, d in _vorbis_corpus.files()][:2], 10)
    before = eng.launch_count
    for bad in ([(0, data_t.numel() + 1)], [(data_t.numel(), 1)], [(2**63, 2**63)], [(0, 1)] * (nat.VORBIS_MAX_FILES + 1)):
        with pytest.raises(ValueError):
            decode.decode_vorbis_files_dev(eng, data_t, bad)
    with pytest.raises(ValueError):
        decode.decode_vorbis_files_dev(eng, data_t.cpu(), ranges)
    assert eng.launch_count == before
    assert decode.decode_vorbis_files_dev(eng, data_t, []) == [] and eng.launch_count == before
