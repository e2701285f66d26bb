"""MPEG Layer I / II decoded on the device, many files per call (symgpu_mpa12_decode_host / _dev, decode.decode_mpa12_files): every
file must come out exactly as decode.decode_mpeg_audio gives it -- the same bytes, shape and sample rate -- whose front-end runs on
the CPU.  Plus per-packet accept / refuse parity with the CPU front-end, trims, the device-resident variant, edge cases and argument
errors."""
import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import decode, frontend, packetizer
from tests import _mpa12_bitstream as bw

pytestmark = pytest.mark.gpu

FORMATS = (nat.FMT_F32, nat.FMT_S16, nat.FMT_S24, nat.FMT_S32, nat.FMT_U8)
# (layer, version, bitrate_idx, rate_idx, mode, protected): stereo / joint stereo (every bound, by mode_ext) / dual mono / mono, CRC,
# MPEG-1 / 2 / 2.5, and the five Layer II allocation tables (a, b, a at 48 kHz, c, d, d joint, MPEG-2 / 2.5 table)
CASES = [(1, "1", 9, 0, 0, False), (1, "1", 14, 1, 1, True), (1, "1", 2, 2, 3, False), (1, "2", 5, 0, 1, False), (1, "2.5", 3, 2, 3, True),
         (1, "1", 7, 0, 2, False),
         (2, "1", 8, 0, 0, False), (2, "1", 14, 0, 1, True), (2, "1", 12, 1, 0, False), (2, "1", 2, 0, 3, False), (2, "1", 1, 2, 3, False),
         (2, "1", 6, 2, 1, False), (2, "2", 10, 0, 1, False), (2, "2.5", 4, 1, 3, True), (2, "2", 14, 2, 2, False)]


@pytest.fixture(scope="module")
def engine():
    import symphonia_b200 as sb
    eng = sb.Engine(0)
    yield eng
    eng.close()


def _file(case, seed, n=8):
    layer, version, bitrate_idx, rate_idx, mode, protected = case
    rng = np.random.default_rng(seed)
    gen = bw.gen_layer1_frame if layer == 1 else bw.gen_layer2_frame
    return b"".join(gen(rng, version, bitrate_idx, rate_idx, mode, mode_ext=k % 4, protected=protected)[0] for k in range(n))


def _damaged_stream(seed):
    """Junk in front, a packet of another sample rate inside the stream (as in test_mpa12_frontend.test_refusals_and_streams)."""
    rng = np.random.default_rng(seed)
    frames = [bw.gen_layer2_frame(rng, "1", 8, 0, 0)[0] for _ in range(12)]
    alien = bw.gen_layer2_frame(rng, "1", 8, 1, 0)[0]
    noise = rng.integers(0, 255, 100, dtype=np.uint8).tobytes()
    return noise + b"".join(frames[:5]) + alien + b"".join(frames[5:])


def _corpus():
    return [_file(c, 100 + k) for k, c in enumerate(CASES)] + [_damaged_stream(7)]


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
    assert sum(len(w) for w, _ in want) > 0
    _same(decode.decode_mpa12_files(engine, files, fmt), want, f"format {fmt}")


def test_one_file_per_layer_against_the_oracle(engine, oracle):
    from tests.test_zz_file_to_pcm import _decode_expect
    for data in (_file(CASES[1], 11), _file(CASES[7], 12)):
        for fmt in (nat.FMT_S16, nat.FMT_F32):
            want, rate, channels, total = _decode_expect(oracle, data, fmt)
            (got, got_rate), = decode.decode_mpa12_files(engine, [data], fmt)
            assert got_rate == rate and got.shape == (total, channels) and got.tobytes() == want.tobytes()


def _mixed(n, seed):
    rng = np.random.default_rng(seed)
    return [_file(CASES[int(rng.integers(len(CASES)))], seed + k, n=int(rng.integers(3, 12))) for k in range(n)]


def test_many_files_in_one_call_with_a_constant_launch_count(engine):
    few, many = _mixed(8, 500), _mixed(64, 600)
    for files in (few, many):
        assert {packetizer.mpa_index(f)[0]["layer"] for f in files} == {1, 2}
        assert {packetizer.mpa_index(f)[0]["channels"] for f in files} == {1, 2}
    counts = []
    for files in (few, many):
        want = _expect(engine, files, nat.FMT_S16)
        before = engine.launch_count
        got = decode.decode_mpa12_files(engine, files, nat.FMT_S16)
        counts.append(engine.launch_count - before)
        _same(got, want, f"{len(files)} files")
    assert counts[0] == counts[1] > 0, counts


def _jobs_of(packets_list):
    """Raw packets -> (data, jobs) with one job per packet, back to back."""
    data = b"".join(packets_list)
    jobs = np.zeros(len(packets_list), dtype=nat.MPA12_JOB_DTYPE)
    jobs["offset"] = np.cumsum([0] + [len(p) for p in packets_list[:-1]]) if packets_list else []
    jobs["len"] = [len(p) for p in packets_list]
    return data, jobs


def _group(first, n, slot, layer, out_offset):
    g = np.zeros(1, dtype=nat.MPA12_GROUP_DTYPE)
    g[0] = (out_offset, first, n, slot, layer, (0, 0, 0))
    return g


def test_per_packet_status_equals_the_front_end(engine):
    rng = np.random.default_rng(31)
    f1 = [bw.gen_layer1_frame(rng, "1", 9, 0, 0, mode_ext=k % 4)[0] for k in range(6)]
    f2 = [bw.gen_layer2_frame(rng, "1", 8, 0, 1, mode_ext=k % 4)[0] for k in range(6)]
    bad = bytearray(f1[1])
    bad[4] |= 0xF0                                                    # Layer I allocation 15
    flip = bytearray(f2[2])
    flip[6] ^= 0xFF                                                   # allocation bits of Layer II
    p1 = [f1[0], bytes(bad), f1[2][:-1], f2[0], f1[3], b"\x00\x01", f1[4] + b"\0", f1[5]]
    p2 = [f2[0], f2[1], bytes(flip), f1[0], f2[3][:50], rng.integers(0, 256, 5, dtype=np.uint8).tobytes() + f2[4], f2[5]]
    junk = [rng.integers(0, 256, 200, dtype=np.uint8).tobytes() for _ in range(3)]
    data, jobs = _jobs_of(p1 + p2 + junk)
    n1, n2 = len(p1), len(p2)
    groups = np.concatenate([_group(0, n1, 0, 1, 0), _group(n1, n2, 1, 2, 2 * n1 * 384), _group(n1 + n2, 3, 2, 2, 2 * (n1 * 384 + n2 * 1152)),
                             _group(n1 + n2 + 3, 0, 3, 1, 0)])
    engine.mp3_streams_alloc(4)
    cap = 2 * (n1 * 384 + (n2 + 3) * 1152)
    out, results, status = engine.mpa12_decode_host(data, jobs, groups, nat.FMT_S16, cap)
    for (lo, n, layer) in ((0, n1, 1), (n1, n2, 2), (n1 + n2, 3, 2)):
        pk = np.zeros(n, dtype=nat.MPA_PACKET_DTYPE)
        pk["offset"], pk["size"] = jobs["offset"][lo:lo + n], jobs["len"][lo:lo + n]
        _, frame_of, _ = frontend.mpa12_decode_packets(data, pk, layer)
        want = np.full(n, nat.MPA12_JOB_REFUSED, np.uint8)
        want[frame_of] = nat.MPA12_JOB_DECODED
        assert status[lo:lo + n].tolist() == want.tolist(), layer
    assert 0 < results["packets"][0] < n1 and 0 < results["packets"][1] < n2
    assert results["packets"][2] == 0 and results["frames"][2] == 0 and results["sample_rate"][2] == 0 and results["channels"][2] == 0
    assert results[3].tobytes() == bytes(24)                          # a group with no jobs
    assert (results["frames"][:2] == results["packets"][:2] * np.array([384, 1152])).all()
    # a call without jobs launches nothing; a file that starts with a cut frame, through the file-level call
    before = engine.launch_count
    out0, res0, st0 = engine.mpa12_decode_host(b"", np.zeros(0, nat.MPA12_JOB_DTYPE), _group(0, 0, 0, 2, 0), nat.FMT_S16, 0)
    assert engine.launch_count == before and res0[0].tobytes() == bytes(24) and len(st0) == 0
    junk_file = bw.gen_layer2_frame(rng, "1", 8, 0, 0)[0][:-7] + bw.gen_layer2_frame(rng, "1", 8, 0, 0)[0]
    errors = {}
    got = decode.decode_mpa12_files(engine, [junk_file, _file(CASES[6], 3)], nat.FMT_S16, errors=errors)
    _same(got, _expect(engine, [junk_file, _file(CASES[6], 3)], nat.FMT_S16), "refused packets")


def test_trims_are_clamped_as_the_one_file_decoder_clamps_them(engine):
    """Packets of Layer I / II files rarely carry trims (their tags are Layer III only), so the jobs get them here: some beyond the
    frame, some summing past it; the expectation is the host front-end + synthesis + output stage with decode.mpeg_audio_plan's
    clamps."""
    rng = np.random.default_rng(41)
    for layer, case in ((1, CASES[1]), (2, CASES[7])):
        data = _file(case, 50 + layer, n=10)
        track, packets = packetizer.mpa_index(data)
        per = 384 if layer == 1 else 1152
        ts = rng.integers(0, per + 200, len(packets)).astype(np.uint32)
        te = rng.integers(0, per + 200, len(packets)).astype(np.uint64)
        ts[0], te[0], ts[-1], te[-1] = 100, 37, 0, per - 5
        packets["trim_start"], packets["trim_end"] = ts, te
        sub, frame_of, info = frontend.mpa12_decode_packets(data, packets, layer)
        runs = np.zeros(1, dtype=nat.MPA12_RUN_DTYPE)
        runs[0] = (0, 0, len(sub), int(info["channels"]), (0, 0, 0))
        engine.mp3_streams_alloc(1)
        pcm = engine.mpa12_synth_host(sub, runs)
        spans = np.zeros(len(sub), dtype=nat.PCM_SPAN_DTYPE)
        spans["src"] = np.arange(len(sub), dtype=np.uint64) * 2304
        spans["plane_stride"], spans["frames"] = 1152, per
        spans["trim_start"] = np.minimum(ts[frame_of], per)
        spans["trim_end"] = np.minimum(te[frame_of], per - spans["trim_start"])
        left = per - spans["trim_start"].astype(np.int64) - spans["trim_end"].astype(np.int64)
        spans["dst_frame"] = np.concatenate([[0], np.cumsum(left)[:-1]]).astype(np.uint64)
        ch = int(info["channels"])
        want = engine.pcm_pack_host(pcm, spans, ch, nat.FMT_S32, int(left.sum()))
        jobs = np.zeros(len(packets), dtype=nat.MPA12_JOB_DTYPE)
        jobs["offset"], jobs["len"], jobs["trim_start"], jobs["trim_end"] = packets["offset"], packets["size"], ts, te
        engine.mp3_streams_alloc(2)
        out, results, status = engine.mpa12_decode_host(data, jobs, _group(0, len(jobs), 1, layer, 0), nat.FMT_S32, 2 * len(jobs) * per)
        n = int(results["frames"][0])
        assert n == int(left.sum()) and int(results["channels"][0]) == ch
        assert out[:n * ch].tobytes() == want.tobytes(), layer


def test_device_resident_variant_equals_the_host_variant(engine):
    import torch
    files = _corpus() + [b"not an mpeg file", _mixed(1, 77)[0]]
    for fmt in (nat.FMT_S16, nat.FMT_F32):
        e_host, e_dev = {}, {}
        host = decode.decode_mpa12_files(engine, files, fmt, errors=e_host)
        dev = decode.decode_mpa12_files(engine, files, fmt, device=True, errors=e_dev)
        assert sorted(e_host) == sorted(e_dev) == [len(files) - 2]
        _same(dev, host, f"device variant, format {fmt}")
        ptrs = {t.untyped_storage().data_ptr() for t, _ in dev if t.numel()}
        assert len(ptrs) == 1 and all(isinstance(t, torch.Tensor) and t.is_cuda for t, _ in dev)


def test_layer3_and_unindexable_files_do_not_stop_the_others(engine):
    from tests import _mp3_bitstream as b3
    rng = np.random.default_rng(61)
    mp3 = b"".join(b3.gen_stream(rng, 6, version="1", mode=0, bitrate_idx=9)[0])
    files = [mp3, _file(CASES[0], 1), b"", _file(CASES[8], 2)]
    errors = {}
    got = decode.decode_mpa12_files(engine, files, nat.FMT_S16, errors=errors)
    assert sorted(errors) == [0, 2] and "Layer 3" in errors[0]
    assert got[0][1] == 0 and got[0][0].size == 0 and got[2][1] == 0
    _same([got[1], got[3]], _expect(engine, [files[1], files[3]], nat.FMT_S16), "good files beside bad ones")


def test_argument_errors_launch_nothing(engine):
    import symphonia_b200 as sb
    data = _file(CASES[6], 9, n=4)
    _, packets = packetizer.mpa_index(data)
    jobs = np.zeros(4, dtype=nat.MPA12_JOB_DTYPE)
    jobs["offset"], jobs["len"] = packets["offset"], packets["size"]
    engine.mp3_streams_alloc(4)
    cap = 2 * 4 * 1152 * 2
    ok = np.concatenate([_group(0, 2, 0, 2, 0), _group(2, 2, 1, 2, 2 * 2 * 1152)])
    engine.mpa12_decode_host(data, jobs, ok, nat.FMT_S16, cap)
    outside = jobs.copy()
    outside["len"][3] = len(data)
    cases = {
        "overlapping groups": (jobs, np.concatenate([_group(0, 3, 0, 2, 0), _group(2, 2, 1, 2, 2 * 3 * 1152)]), cap, 6),
        "duplicate slot": (jobs, np.concatenate([_group(0, 2, 1, 2, 0), _group(2, 2, 1, 2, 2 * 2 * 1152)]), cap, 6),
        "layer 3": (jobs, _group(0, 4, 0, 3, 0), cap, 6),
        "region beyond out": (jobs, _group(0, 4, 0, 2, cap - 2 * 4 * 1152 + 2), cap, 3),
        "slot not allocated": (jobs, _group(0, 4, 4, 2, 0), cap, 3),
        "job outside bytes": (outside, ok, cap, 6),
    }
    for what, (j, g, c, code) in cases.items():
        before = engine.launch_count
        with pytest.raises(sb.SymgpuError) as e:
            engine.mpa12_decode_host(data, j, g, nat.FMT_S16, c)
        assert e.value.status == code, what
        assert engine.launch_count == before, what
