"""The FLAC device path's output stage in the caller's sample format (symgpu_flac_decode_fmt_*, decode.decode_flac_files(...,
fmt=...)): for every SYMGPU_FMT_* the interleaving kernel must write exactly decode.flac_convert of the int32 result -- the
reference's FromSample<i32>, pinned on the CPU in tests/test_flac_convert.py -- with the same statuses, frame counts, launch
count and region discipline as the int32 call."""
import ctypes

import numpy as np
import pytest

import symphonia_b200 as sb
from symphonia_b200 import _native as nat
from symphonia_b200 import decode
from tests.test_flac_decode_gpu import _corpus, _frames, _jobs_of
from tests.test_flac_entropy_shared import _damaged

pytestmark = pytest.mark.gpu

FORMATS = (nat.FMT_F32, nat.FMT_S16, nat.FMT_S24, nat.FMT_S32, nat.FMT_U8)
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def corpus():
    return _corpus()


@pytest.fixture(scope="module")
def eng():
    with sb.Engine(0) as e:
        yield e


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and (np.ascontiguousarray(a).view(np.uint8) == np.ascontiguousarray(b).view(np.uint8)).all()


def test_every_format_is_the_conversion_of_the_int32_result(eng, corpus):
    files = [d for _, d, _ in corpus]
    base = decode.decode_flac_files(eng, files)
    assert any(np.abs(pcm.astype(np.int64)).max() > 2 ** 24 for pcm, _ in base if pcm.size)     # f32 has something to round
    for fmt in FORMATS:
        got = decode.decode_flac_files(eng, files, fmt=fmt)
        assert len(got) == len(files)
        for (name, data, _), (pcm, rate), (pcm32, rate32) in zip(corpus, got, base):
            assert rate == rate32, name
            assert pcm.dtype == np.dtype(nat.FMT_NUMPY[fmt]) and _same(pcm, decode.flac_convert(pcm32, fmt)), (name, fmt)
            alone, alone_rate = decode.decode_flac(eng, data, fmt=fmt)
            assert alone_rate == rate and _same(pcm, alone), (name, fmt)
            if fmt == nat.FMT_S32:
                assert _same(pcm, pcm32), name


def test_device_resident_results_in_every_format(eng, corpus):
    import torch
    files = [d for _, d, _ in corpus[:14]]
    for fmt in FORMATS:
        host = decode.decode_flac_files(eng, files, fmt=fmt)
        dev = decode.decode_flac_files(eng, files, device=True, fmt=fmt)
        for (a, ra), (b, rb) in zip(host, dev):
            assert b.is_cuda and b.dtype == getattr(torch, decode._TORCH_DTYPES[fmt]) and ra == rb
            assert _same(b.cpu().numpy(), a), fmt


def test_launches_depend_on_neither_format_nor_file_count(eng, corpus):
    files = [corpus[k % len(corpus)][1] for k in range(48)]
    counts = set()
    for fmt in FORMATS:
        for some in (files, files[:2]):
            before = eng.launch_count
            decode.decode_flac_files(eng, some, fmt=fmt)
            counts.add(eng.launch_count - before)
    assert len(counts) == 1, counts


def _decode_dev(eng, data, jobs, groups, cap, fmt):
    """symgpu_flac_decode_fmt_dev over a sentinel-filled output: (out as bytes, group_frames, status)."""
    import torch
    d = torch.device("cuda", eng.device)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to(d)  # noqa: E731
    size = np.dtype(nat.FMT_NUMPY[fmt]).itemsize
    out = torch.full((cap * size,), SENTINEL, dtype=torch.uint8, device=d).view(getattr(torch, decode._TORCH_DTYPES[fmt]))
    gf = torch.zeros(len(groups), dtype=torch.int64, device=d)
    st = torch.zeros(len(jobs), dtype=torch.uint8, device=d)
    data_t, jobs_t, groups_t = t(np.frombuffer(data, dtype=np.uint8).copy()), t(jobs), t(groups)
    torch.cuda.synchronize()
    eng.flac_decode_dev(data_t, jobs_t, groups_t, out, gf, st, fmt)
    eng.sync()
    return out.view(torch.uint8).cpu().numpy(), gf.cpu().numpy(), st.cpu().numpy()


def test_damaged_packets_keep_their_statuses_and_regions(eng):
    """Two files in one call: damaged packets and one slot too small in the first, clean packets in the second.  Whatever the
    format, the statuses and frame counts are those of the int32 call, accepted packets hold the converted samples, and every byte
    outside the written frames -- the unused tail of each region included -- keeps the sentinel."""
    pk, _ = _frames(601, 16, 2, 576, 36)
    hit = _damaged(pk, 3)
    clean, _ = _frames(602, 24, 2, 576, 5)
    data, jobs = _jobs_of(hit + clean, 576)
    jobs["group"][len(hit):] = 1
    jobs["slot"][7] = 575                                    # an untouched packet whose block no longer fits
    groups = np.zeros(2, dtype=nat.FLAC_GROUP_DTYPE)
    groups["max_block"], groups["channels"] = 576, 2
    groups["bits_per_sample"] = 16, 24
    groups[1]["out_offset"] = 2 * 576 * len(hit) + 7         # an odd offset: no store may assume more than the sample's own alignment
    cap = int(groups[1]["out_offset"]) + 2 * 576 * len(clean) + 5
    out32, gf32, st32 = eng.flac_decode_host(data, jobs, groups, cap)
    assert st32[7] == nat.FLAC_JOB_NO_ROOM and (st32[len(hit):] == 0).all()
    assert 0 < (st32[:len(hit)] == nat.FLAC_JOB_REFUSED).sum() < len(hit) - 8
    written = np.zeros(cap, dtype=bool)
    for g in range(2):
        at = int(groups[g]["out_offset"])
        written[at:at + int(gf32[g]) * 2] = True
    assert 0 < written.sum() < cap - 12
    for fmt in (nat.FMT_S16, nat.FMT_U8, nat.FMT_F32, nat.FMT_S24, nat.FMT_S32):
        size = np.dtype(nat.FMT_NUMPY[fmt]).itemsize
        want = np.ascontiguousarray(decode.flac_convert(out32, fmt)).view(np.uint8).reshape(cap, size)
        # host variant: only the written frames are copied back
        host = np.full(cap * size, SENTINEL, dtype=np.uint8).view(nat.FMT_NUMPY[fmt])
        out, gf, st = eng.flac_decode_host(data, jobs, groups, cap, out=host, fmt=fmt)
        assert st.tolist() == st32.tolist() and gf.tolist() == gf32.tolist(), fmt
        got = out.view(np.uint8).reshape(cap, size)
        assert (got[written] == want[written]).all() and (got[~written] == SENTINEL).all(), fmt
        # device variant: what the kernels themselves wrote
        raw, gf, st = _decode_dev(eng, data, jobs, groups, cap, fmt)
        assert st.tolist() == st32.tolist() and gf.tolist() == [int(v) for v in gf32], fmt
        got = raw.reshape(cap, size)
        assert (got[written] == want[written]).all() and (got[~written] == SENTINEL).all(), fmt


def test_unknown_format_is_an_argument_error_before_any_launch(eng):
    import torch
    pk, _ = _frames(603, 16, 2, 576, 3)
    data, jobs = _jobs_of(pk, 576)
    groups = np.zeros(1, dtype=nat.FLAC_GROUP_DTYPE)
    groups[0]["max_block"], groups[0]["bits_per_sample"], groups[0]["channels"] = 576, 16, 2
    cap = 2 * 576 * 3
    before = eng.launch_count
    for fmt in (5, -1, 99):
        with pytest.raises(sb.SymgpuError) as e:
            eng.flac_decode_host(data, jobs, groups, cap, out=np.zeros(cap, dtype=np.int32), fmt=fmt)
        assert e.value.status == 6                          # SYMGPU_ERR_ARG
        one = torch.zeros(cap, dtype=torch.int32, device="cuda")
        p = ctypes.c_void_p(one.data_ptr())
        assert sb.lib().symgpu_flac_decode_fmt_dev(eng._ctx, p, 4, p, 1, p, 1, fmt, p, cap, p, p) == 6
    assert eng.launch_count == before
    out, gf, st = eng.flac_decode_host(data, jobs, groups, cap, fmt=nat.FMT_S16)      # and the engine is as healthy as before
    assert out.dtype == np.int16 and 2 * 576 < int(gf[0]) <= 3 * 576 and (st == 0).all()      # (the stream's last block is short)
