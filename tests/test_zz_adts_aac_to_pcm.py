"""ADTS file bytes -> frames -> raw_data_blocks -> AAC-LC entropy front-end -> synthesis -> interleaved samples
(`symphonia_b200.decode.adts_aac_plan` / `decode_adts_aac`).  The CPU test runs everything up to the launch, renders the plan with
the synthesis and output-stage oracles and compares with an expectation built from the stream WRITER's ground truth; the GPU test
compares `decode_adts_aac` with the
rendered plan byte for byte."""
import os

import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import decode
from tests import _aac_bitstream as ab
from tests import _oracle
from tests import _streams as st

RATE_IDX = {96000: 0, 88200: 1, 64000: 2, 48000: 3, 44100: 4, 32000: 5, 24000: 6, 22050: 7, 16000: 8, 12000: 9, 11025: 10, 8000: 11}


@pytest.fixture(scope="module")
def oracle():
    return _oracle.load()


def _file(seed, rate=44100, channels=2, n=14):
    rng = np.random.default_rng(seed)
    s = ab.Stream(rng, rate=rate, channels=channels)
    frames, truth = [], []
    for k in range(n):
        pkt, t = s.packet()
        frames.append(st.adts_frame(rng, 0, rate_idx=RATE_IDX[rate], channels=channels, protected=bool(k % 3 == 1), payload=pkt))
        truth.append(t)
    return b"".join(frames), truth


def _render(oracle, plan, fmt):
    rc, pcm = _oracle.aac_batch(oracle, plan["units"], plan["tns"], plan["coeffs"], plan["runs"], 1)
    assert rc == 0
    return _oracle.pcm_pack(oracle, pcm, plan["spans"], plan["channels"], fmt, plan["total_frames"])


def test_plan_up_to_the_launch(oracle):
    for seed, (rate, channels) in enumerate([(44100, 2), (48000, 2), (22050, 1), (8000, 2), (96000, 1)]):
        data, truth = _file(500 + seed, rate, channels)
        plan = decode.adts_aac_plan(data)
        n = len(truth)
        assert plan["units"].shape == (n, 2) and plan["sample_rate"] == rate and plan["channels"] == channels and plan["total_frames"] == 1024 * n
        # the writer's values, frame by frame
        at = 0
        for k, t in enumerate(truth):
            for c in range(channels):
                u = plan["units"][k, c]
                assert (int(u["window_sequence"]), int(u["window_shape"]), int(u["prev_window_shape"])) == (t[c]["window_sequence"], t[c]["window_shape"], t[c]["prev_window_shape"])
                assert np.array_equal(plan["coeffs"][k, c].view(np.uint32), t[c]["coeffs"].view(np.uint32))
                assert int(u["n_tns"]) == len(t[c]["tns"]) and (int(u["tns_first"]) == at or not t[c]["tns"])
                for j, f in enumerate(t[c]["tns"]):
                    r = plan["tns"][at + j]
                    assert (int(r["start"]), int(r["end"]), int(r["order"]), int(r["direction"])) == tuple(f[:4])
                    assert np.array_equal(r["lpc"].view(np.uint32), np.array(f[4], dtype=np.float32).view(np.uint32))
                at += len(t[c]["tns"])
        assert at == len(plan["tns"])
        got = _render(oracle, plan, nat.FMT_F32)
        assert got.shape == (1024 * n, channels)
        assert np.abs(got[np.isfinite(got)]).max() > 0


def test_plan_drops_frames_the_front_end_refuses(oracle):
    data, truth = _file(600, n=10)
    # cut inside a frame's payload: the reader stops there (adts.rs: cut payload), the frames before it decode as before
    plan_all = decode.adts_aac_plan(data)
    assert len(plan_all["units"]) == 10
    plan = decode.adts_aac_plan(data[:len(data) * 6 // 10])
    assert 0 < len(plan["units"]) < 10
    k = len(plan["units"])
    assert np.array_equal(plan["coeffs"].view(np.uint32), plan_all["coeffs"][:k].view(np.uint32))


@pytest.mark.gpu
def test_adts_file_to_pcm_on_the_device(oracle):
    import symphonia_b200 as sb
    with sb.Engine(0) as eng:
        eng.aac_streams_alloc(2)
        for seed, (rate, channels) in enumerate([(44100, 2), (48000, 2), (22050, 1), (8000, 2), (96000, 1)]):
            data, _ = _file(500 + seed, rate, channels)
            for fmt in (nat.FMT_S16, nat.FMT_F32):
                want = _render(oracle, decode.adts_aac_plan(data), fmt)
                got, got_rate = decode.decode_adts_aac(eng, data, fmt, stream=1)
                assert got_rate == rate and got.shape == want.shape
                assert (got.view(np.uint8) == want.view(np.uint8)).all()


@pytest.mark.gpu
def test_cpp_aac_decoder_on_adts_files(tmp_path, oracle):
    """The C++ mirror of the plug-in interface: registry -> GpuAacDecoder, one decode() per raw_data_block."""
    import subprocess
    from tests.test_cpp_host import _build
    for seed, (rate, channels) in enumerate([(44100, 2), (22050, 1)]):
        data, _ = _file(500 + 2 * seed, rate, channels)
        want = _render(oracle, decode.adts_aac_plan(data), nat.FMT_F32)
        inp, outp = tmp_path / f"in{seed}.aac", tmp_path / f"out{seed}.bin"
        inp.write_bytes(data)
        res = subprocess.run([_build(), "file", "aac", str(inp), str(outp)], capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stdout + res.stderr
        got = np.frombuffer(outp.read_bytes(), dtype=np.float32).reshape(-1, channels, 1024).transpose(0, 2, 1).reshape(-1, channels)
        assert got.shape == want.shape and (got.view(np.uint32) == np.ascontiguousarray(want).view(np.uint32)).all()


def test_one_long_stream_as_jobs_gives_the_same_plan():
    data, _ = _file(520, 44100, 2, n=40)
    a, b = decode.adts_aac_plan(data), decode.adts_aac_plan(data, threads=4)
    for key in ("units", "tns", "coeffs", "runs", "spans"):
        assert a[key].tobytes() == b[key].tobytes(), key
    # a stream with a damaged block falls back to the serial path, with the same result as without threads
    hurt = bytearray(data)
    hurt[len(hurt) // 2] ^= 0x3C
    a, b = decode.adts_aac_plan(bytes(hurt)), decode.adts_aac_plan(bytes(hurt), threads=4)
    for key in ("units", "tns", "coeffs", "runs", "spans"):
        assert a[key].tobytes() == b[key].tobytes(), key
