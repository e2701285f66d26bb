"""MPEG Layer III decoded on the device, many files per call (symgpu_mp3_decode_host / _dev, decode.decode_mp3_files): every file
must come out exactly as decode.decode_mpeg_audio gives it -- the same bytes, shape and sample rate -- whose front-end runs on the
CPU.  Plus joint-stereo window mismatches (left out whole), per-packet statuses against the CPU front-end, rounds, the oracle, the
device-resident variant, the launch count, edge cases, argument errors and the decode_mpeg_files router."""
import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import decode, frontend, packetizer
from tests import _mp3_bitstream as bw
from tests import _mpa12_bitstream as b12
from tests import _streams as st
from tests import test_zz_file_to_pcm as chain
from tests.test_mp3_entropy_shared import _p23_at, _set_bits, _table, mismatch

pytestmark = pytest.mark.gpu

FORMATS = (nat.FMT_F32, nat.FMT_S16, nat.FMT_S24, nat.FMT_S32, nat.FMT_U8)
# (version, mode, rate_idx, bitrate_idx, protected, mode_ext): stereo, joint stereo with MS / intensity / both, dual channel, mono,
# CRC, MPEG-1 / 2 / 2.5
CASES = [("1", 0, 0, 9, False, None), ("1", 1, 0, 9, False, 2), ("1", 1, 1, 11, True, 1), ("1", 1, 2, 14, False, 3), ("1", 2, 0, 10, True, None),
         ("1", 3, 0, 5, False, None), ("2", 1, 0, 8, False, 3), ("2", 3, 1, 6, True, None), ("2.5", 1, 2, 6, False, 2), ("2.5", 0, 0, 4, False, None)]


@pytest.fixture(scope="module")
def engine():
    import symphonia_b200 as sb
    eng = sb.Engine(0)
    yield eng
    eng.close()


def _file(case, seed, n=16, pair_blocks=True):
    version, mode, rate_idx, bitrate_idx, protected, mode_ext = case
    rng = np.random.default_rng(seed)
    frames, _ = bw.gen_stream(rng, n, version=version, mode=mode, rate_idx=rate_idx, bitrate_idx=bitrate_idx, protected=protected,
                              pair_blocks=pair_blocks, force_mode_ext=None if mode_ext is None else (lambda k: mode_ext))
    return frames


def _over_read(seed):
    """MPEG-1 stereo with three frames whose first part2_3_length reaches past their main data: three rounds... at least."""
    frames = _file(CASES[0], seed, n=24)
    out = [bytearray(f) for f in frames]
    for k in (4, 11, 17):
        _set_bits(out[k], 8 * 4 + _p23_at("1", 2), 12, 4095)
    return b"".join(bytes(b) for b in out)


def _tagged(seed):
    """A LAME tag with encoder delay and padding, junk in front and in the middle."""
    rng = np.random.default_rng(seed)
    frames = _file(CASES[1], seed, n=20)
    tag = st.mpa_tag_frame(rng, dict(version="1", layer=3, bitrate_idx=9, rate_idx=0, mode=1), num_frames=20)
    noise = rng.integers(0, 255, 120, dtype=np.uint8).tobytes()
    return noise + tag + b"".join(frames[:9]) + noise[:29] + b"".join(frames[9:])


def _corpus():
    files = [b"".join(_file(c, 100 + k)) for k, c in enumerate(CASES)]
    files += chain._corpus()
    files.append(_tagged(5))
    files.append(b"".join(_file(CASES[1], 7, n=30)[9:]))          # cut at the front: the first frames reach into missing bytes
    files.append(_over_read(9))
    return files


def _expect(engine, files, fmt):
    engine.mp3_streams_alloc(1)
    return [decode.decode_mpeg_audio(engine, f, fmt, stream=0) for f in files]


def _same(got, want, what):
    for k, ((g, gr), (w, wr)) in enumerate(zip(got, want)):
        g = g.cpu().numpy() if hasattr(g, "cpu") else g
        assert gr == wr and g.shape == w.shape and g.dtype == w.dtype, (what, k, gr, wr, g.shape, w.shape)
        assert g.tobytes() == w.tobytes(), (what, k)


@pytest.mark.parametrize("fmt", FORMATS)
def test_files_equal_the_one_file_decoder(engine, fmt):
    files = _corpus()
    want = _expect(engine, files, fmt)
    assert all(len(w) > 0 for w, _ in want)
    stats = {}
    _same(decode.decode_mp3_files(engine, files, fmt, stats=stats), want, f"format {fmt}")
    assert stats["rounds"] >= 2 and (stats["status"] == nat.MP3_JOB_FAILED).sum() == stats["rounds"] - 1


def test_one_file_per_version_against_the_oracle(engine, oracle):
    from tests.test_zz_file_to_pcm import _decode_expect
    for case in (CASES[1], CASES[7], CASES[8]):
        data = b"".join(_file(case, 11))
        for fmt in (nat.FMT_S16, nat.FMT_F32):
            want, rate, channels, total = _decode_expect(oracle, data, fmt)
            (got, got_rate), = decode.decode_mp3_files(engine, [data], fmt)
            assert got_rate == rate and got.shape == (total, channels) and got.tobytes() == want.tobytes()


def test_window_mismatches_are_left_out(engine):
    """A joint-stereo frame whose channels are on different window sequences is left out whole; the rest equals the serial
    front-end's batch without those frames, synthesised and packed by the host entry points."""
    files = [b"".join(_file(c, 40 + k, n=24, pair_blocks=False)) for k, c in enumerate((CASES[1], CASES[3], CASES[6]))]
    stats = {}
    got = decode.decode_mp3_files(engine, files, nat.FMT_S32, stats=stats)
    n_left = 0
    for k, data in enumerate(files):
        track, packets = packetizer.mpa_index(data)
        units, quant, frame_of, info = frontend.Mp3Frontend().decode_packets(data, packets)
        keep = ~mismatch(units)
        n_left += int((~keep).sum())
        units, quant, kept = units[keep], quant[keep], packets[frame_of[keep]]
        per, ch = 576 * int(info["granules"]), int(info["channels"])
        runs = np.zeros(1, dtype=nat.MP3_RUN_DTYPE)
        runs[0] = (0, 0, len(units), int(info["granules"]), ch, 0)
        engine.mp3_streams_alloc(1)
        engine.mp3_stream_reset(0)
        pcm = engine.mp3_synth_host_quantized(units.reshape(-1), quant, runs)
        spans = np.zeros(len(units), dtype=nat.PCM_SPAN_DTYPE)
        spans["src"] = np.arange(len(units), dtype=np.uint64) * 2304
        spans["plane_stride"], spans["frames"] = 1152, per
        spans["trim_start"] = np.minimum(kept["trim_start"], per)
        spans["trim_end"] = np.minimum(kept["trim_end"], per - spans["trim_start"])
        left = per - spans["trim_start"].astype(np.int64) - spans["trim_end"].astype(np.int64)
        spans["dst_frame"] = np.concatenate([[0], np.cumsum(left)[:-1]]).astype(np.uint64)
        want = engine.pcm_pack_host(pcm, spans, ch, nat.FMT_S32, int(left.sum()))
        assert got[k][1] == int(info["sample_rate"]) and got[k][0].tobytes() == want.tobytes(), k
    assert n_left > 0 and (stats["status"] == nat.MP3_JOB_LEFT_OUT).sum() == n_left


def _mixed(n, seed):
    rng = np.random.default_rng(seed)
    return [b"".join(_file(CASES[(seed + k) % len(CASES)], seed + k, n=int(rng.integers(3, 12)))) for k in range(n)]


def test_many_files_in_one_call_with_a_constant_launch_count(engine):
    few, many = _mixed(8, 500), _mixed(64, 600)
    for files in (few, many):
        assert {int(packetizer.mpa_index(f)[0]["channels"]) for f in files} == {1, 2}
    counts = []
    for files in (few, many):
        want = _expect(engine, files, nat.FMT_S16)
        before = engine.launch_count
        stats = {}
        got = decode.decode_mp3_files(engine, files, nat.FMT_S16, stats=stats)
        counts.append(engine.launch_count - before)
        assert stats["rounds"] == 1
        _same(got, want, f"{len(files)} files")
    assert counts[0] == counts[1] > 0, counts


def _jobs_of(packets_list):
    data = b"".join(packets_list)
    jobs = np.zeros(len(packets_list), dtype=nat.MP3_JOB_DTYPE)
    jobs["offset"] = np.cumsum([0] + [len(p) for p in packets_list[:-1]]) if packets_list else []
    jobs["len"] = [len(p) for p in packets_list]
    return data, jobs


def _group(first, n, slot, granules, channels, out_offset):
    g = np.zeros(1, dtype=nat.MP3_GROUP_DTYPE)
    g[0] = (out_offset, first, n, slot, granules, channels, (0, 0))
    return g


def test_per_packet_status_equals_the_front_end(engine):
    rng = np.random.default_rng(31)
    a = _file(CASES[1], 71, n=12, pair_blocks=False)
    b = _file(CASES[7], 72, n=10)
    over = [bytearray(f) for f in _file(CASES[0], 73, n=10)]
    _set_bits(over[3], 8 * 4 + _p23_at("1", 2), 12, 4095)
    p1 = a[:3] + [a[3][:-1], b"\x00\x01", a[4] + b"\0"] + a[5:] + [b[0]]
    p2 = [rng.integers(0, 256, 7, dtype=np.uint8).tobytes() + b[0]] + b[1:4] + [b[4][:20]] + b[5:]
    p3 = [bytes(f) for f in over]
    data, jobs = _jobs_of(p1 + p2 + p3)
    n1, n2, n3 = len(p1), len(p2), len(p3)
    groups = np.concatenate([_group(0, n1, 0, 2, 2, 0), _group(n1, n2, 1, 1, 1, 2 * n1 * 1152),
                             _group(n1 + n2, n3, 2, 2, 2, 2 * n1 * 1152 + n2 * 576), _group(n1 + n2 + n3, 0, 3, 2, 2, 0)])
    engine.mp3_streams_alloc(4)
    cap = 2 * n1 * 1152 + n2 * 576 + 2 * n3 * 1152
    out, results, status, rounds = engine.mp3_decode_host(data, jobs, groups, nat.FMT_S16, cap)
    most = 0
    for lo, n, g in ((0, n1, 0), (n1, n2, 1), (n1 + n2, n3, 2)):
        pk = _table([bytes(x) for x in (p1 + p2 + p3)[lo:lo + n]])
        chunk = b"".join((p1 + p2 + p3)[lo:lo + n])
        units, _, frame_of, _ = frontend.Mp3Frontend().decode_packets(chunk, pk)
        *_, r = frontend.entropy_decode_cpu(chunk, pk)
        most = max(most, r)
        out_ = mismatch(units)
        want = np.full(n, nat.MP3_JOB_REFUSED, np.uint8)
        want[frame_of] = np.where(out_, nat.MP3_JOB_LEFT_OUT, nat.MP3_JOB_DECODED)
        s = status[lo:lo + n]
        refused = want == nat.MP3_JOB_REFUSED
        assert (s[~refused] == want[~refused]).all(), g
        assert np.isin(s[refused], (nat.MP3_JOB_REFUSED, nat.MP3_JOB_FAILED)).all() and (s == nat.MP3_JOB_FAILED).sum() == r - 1, g
        assert int(results["packets"][g]) == int((~out_).sum()), g
    assert rounds == most >= 2
    assert results[3].tobytes() == bytes(24)                          # a group with no jobs
    # a group whose granules / channels disagree with its packets refuses them all
    _, r2, s2, _ = engine.mp3_decode_host(data, jobs[n1:n1 + n2], _group(0, n2, 0, 2, 2, 0), nat.FMT_S16, 2 * n2 * 1152)
    assert (s2 == nat.MP3_JOB_REFUSED).all() and r2["packets"][0] == 0 and r2["frames"][0] == 0


def test_device_resident_variant_equals_the_host_variant(engine):
    import torch
    files = _corpus() + [b"not an mpeg file"]
    for fmt in (nat.FMT_S16, nat.FMT_F32):
        e_host, e_dev, s_host, s_dev = {}, {}, {}, {}
        host = decode.decode_mp3_files(engine, files, fmt, errors=e_host, stats=s_host)
        dev = decode.decode_mp3_files(engine, files, fmt, device=True, errors=e_dev, stats=s_dev)
        assert sorted(e_host) == sorted(e_dev) == [len(files) - 1]
        assert s_host["rounds"] == s_dev["rounds"] and (s_host["status"] == s_dev["status"]).all()
        _same(dev, host, f"device variant, format {fmt}")
        ptrs = {t.untyped_storage().data_ptr() for t, _ in dev if t.numel()}
        assert len(ptrs) == 1 and all(isinstance(t, torch.Tensor) and t.is_cuda for t, _ in dev)


def test_other_files_do_not_stop_the_others(engine):
    rng = np.random.default_rng(61)
    layer2 = b"".join(b12.gen_layer2_frame(rng, "1", 8, 0, 0)[0] for _ in range(4))
    cut = b"".join(_file(CASES[0], 62, n=3))[:-5]                     # the last frame cut short
    files = [layer2, b"".join(_file(CASES[0], 1)), b"", b"no frames here" * 10, b"".join(_file(CASES[7], 2)), cut]
    errors = {}
    got = decode.decode_mp3_files(engine, files, nat.FMT_S16, errors=errors)
    assert sorted(errors) == [0, 2, 3] and "Layer 2" in errors[0]
    for i in (0, 2, 3):
        assert got[i][1] == 0 and got[i][0].size == 0
    _same([got[1], got[4], got[5]], _expect(engine, [files[1], files[4], files[5]], nat.FMT_S16), "good files beside bad ones")


def test_argument_errors_launch_nothing(engine):
    import symphonia_b200 as sb
    data = b"".join(_file(CASES[0], 9, n=4))
    _, packets = packetizer.mpa_index(data)
    jobs = np.zeros(4, dtype=nat.MP3_JOB_DTYPE)
    jobs["offset"], jobs["len"] = packets["offset"], packets["size"]
    engine.mp3_streams_alloc(4)
    cap = 2 * 4 * 1152
    ok = np.concatenate([_group(0, 2, 0, 2, 2, 0), _group(2, 2, 1, 2, 2, 2 * 2 * 1152)])
    engine.mp3_decode_host(data, jobs, ok, nat.FMT_S16, cap)
    outside = jobs.copy()
    outside["len"][3] = len(data)
    cases = {
        "overlapping groups": (jobs, np.concatenate([_group(0, 3, 0, 2, 2, 0), _group(2, 2, 1, 2, 2, 2 * 3 * 1152)]), cap, 6),
        "duplicate slot": (jobs, np.concatenate([_group(0, 2, 1, 2, 2, 0), _group(2, 2, 1, 2, 2, 2 * 2 * 1152)]), cap, 6),
        "three channels": (jobs, _group(0, 4, 0, 2, 3, 0), cap, 6),
        "odd offset for stereo": (jobs, _group(0, 1, 0, 2, 2, 1), cap, 6),
        "region beyond out": (jobs, _group(0, 4, 0, 2, 2, 2), cap, 3),
        "slot not allocated": (jobs, _group(0, 4, 4, 2, 2, 0), cap, 3),
        "job outside bytes": (outside, ok, cap, 6),
    }
    for what, (j, g, c, code) in cases.items():
        before = engine.launch_count
        with pytest.raises(sb.SymgpuError) as e:
            engine.mp3_decode_host(data, j, g, nat.FMT_S16, c)
        assert e.value.status == code, what
        assert engine.launch_count == before, what
    before = engine.launch_count
    _, r0, s0, n0 = engine.mp3_decode_host(b"", np.zeros(0, nat.MP3_JOB_DTYPE), _group(0, 0, 0, 2, 2, 0), nat.FMT_S16, 0)
    assert engine.launch_count == before and r0[0].tobytes() == bytes(24) and len(s0) == 0 and n0 == 0


def test_decode_mpeg_files_routes_every_layer(engine):
    rng = np.random.default_rng(81)
    l1 = b"".join(b12.gen_layer1_frame(rng, "1", 9, 0, 0, mode_ext=k % 4)[0] for k in range(6))
    l2 = b"".join(b12.gen_layer2_frame(rng, "1", 8, 0, 1, mode_ext=k % 4)[0] for k in range(6))
    files = [b"".join(_file(CASES[2], 82)), l2, b"junk" * 40, l1, _tagged(83), b"".join(_file(CASES[7], 84))]
    for device in (False, True):
        errors = {}
        got = decode.decode_mpeg_files(engine, files, nat.FMT_S16, device=device, errors=errors)
        assert sorted(errors) == [2] and got[2][1] == 0 and tuple(got[2][0].shape) == (0, 0)
        good = [0, 1, 3, 4, 5]
        _same([got[i] for i in good], _expect(engine, [files[i] for i in good], nat.FMT_S16), f"router, device={device}")
