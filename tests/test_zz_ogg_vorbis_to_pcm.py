"""Vorbis-in-Ogg file bytes -> pages -> packets -> headers -> entropy front-end -> synthesis -> trimmed interleaved samples
(`symphonia_b200.decode.ogg_vorbis_plan` / `decode_ogg_vorbis`).  The CPU test runs everything up to the launch, renders the plan
with the synthesis and output-stage oracles and compares with an expectation built from the stream WRITER's ground truth (which
never saw a bit reader); the GPU test
compares `decode_ogg_vorbis` with the rendered plan byte for byte."""
import os

import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import decode
from tests import _oracle
from tests import _streams as st
from tests import _vorbis_bitstream as vb


@pytest.fixture(scope="module")
def oracle():
    return _oracle.load()


def _file(seed, n_packets=20, pad=37, channels=2):
    """(ogg bytes, writer truth per packet, granule position of the end of the stream)."""
    rng = np.random.default_rng(seed)
    s = vb.Stream(rng, channels=channels, bs_exp=(8, 11), per_word=1)
    pk, truth = [], []
    for _ in range(n_packets):
        b, t = s.packet()
        pk.append(b), truth.append(t)
    bs = {False: 1 << 8, True: 1 << 11}
    g, gran = 0, []
    for k, t in enumerate(truth):
        if k:
            g += (bs[bool(t["prev_block_flag"])] + bs[bool(t["block_flag"])]) // 4
        gran.append(g)
    end = max(g - pad, gran[-2] if n_packets > 1 else 0)
    gran[-1] = end
    headers = [s.ident, b"\x03vorbis" + bytes(20), s.setup]
    pages = st.ogg_paginate(77, headers[:1], rng, eos=False) + st.ogg_paginate(77, headers[1:], rng, first_sequence=1, bos=False, eos=False)
    first = len(pages)
    pages += st.ogg_paginate(77, pk, rng, max_segments=int(rng.integers(3, 40)), first_sequence=first, bos=False, granule_of=gran)
    return b"".join(pages), s, truth, end


def _render(oracle, plan, fmt):
    wl = dict(streams=plan["stream"], floors=plan["floors"], units=plan["units"], floor_y=plan["floor_y"], residue=plan["residue"],
              runs=plan["runs"], slot=plan["slot"])
    rc, pcm = _oracle.vorbis_batch(oracle, wl)
    assert rc == 0
    return _oracle.pcm_pack(oracle, pcm, plan["spans"], plan["channels"], fmt, plan["total_frames"])


def _expect_from_truth(oracle, s, truth, end, plan):
    """The writer's floor / residue values through the synthesis oracle, packet outputs laid end to end from the second packet on,
    cut at the final granule position."""
    n = len(truth)
    units = np.zeros(n, dtype=nat.VORBIS_UNIT_DTYPE)
    for k, t in enumerate(truth):
        units[k]["block_flag"], units[k]["prev_block_flag"] = int(t["block_flag"]), int(t["prev_block_flag"])
        units[k]["do_not_decode"] = [int(x) for x in t["do_not_decode"]]
        units[k]["floor"] = [0xFFFF if f is None else f for f in t["floor"]]
    wl = dict(streams=plan["stream"], floors=plan["floors"], units=units, floor_y=np.stack([t["floor_y"] for t in truth]),
              residue=np.stack([t["residue"] for t in truth]), runs=plan["runs"], slot=plan["slot"])
    rc, pcm = _oracle.vorbis_batch(oracle, wl)
    assert rc == 0
    bs = {0: 1 << 8, 1: 1 << 11}
    rows = []
    for k in range(1, n):
        frames = (bs[int(units[k]["prev_block_flag"])] + bs[int(units[k]["block_flag"])]) // 4
        rows.append(pcm[k, :s.channels, :frames].T)
    return np.concatenate(rows)[:end]


def test_plan_up_to_the_launch(oracle):
    for seed in range(8):
        data, s, truth, end = _file(300 + seed, channels=1 if seed == 5 else 2, pad=[37, 0, 300, 1, 37, 37, 900, 5][seed])
        plan = decode.ogg_vorbis_plan(data)
        assert len(plan["units"]) == len(truth) and plan["channels"] == s.channels and plan["sample_rate"] == 44100
        assert plan["total_frames"] == end
        sp = plan["spans"]
        left = sp["frames"].astype(np.int64) - sp["trim_start"] - sp["trim_end"]
        assert left[0] == 0 and (left >= 0).all() and int(left.sum()) == end
        assert (sp["dst_frame"] == np.concatenate([[0], np.cumsum(left)[:-1]])).all()
        got = _render(oracle, plan, nat.FMT_F32)
        want = _expect_from_truth(oracle, s, truth, end, plan)
        assert got.shape == want.shape == (end, s.channels)
        assert (got.view(np.uint32) == np.ascontiguousarray(want).view(np.uint32)).all()
        assert np.isfinite(got).all() and np.abs(got).max() > 0


def test_plan_drops_packets_the_front_end_refuses(oracle):
    data, s, truth, end = _file(400, pad=0)
    # a stray non-decodable audio packet cannot be spliced into a checksummed page here; the front-end's refusal path is covered in
    # test_vorbis_frontend.py -- this checks the plan's behaviour on a stream cut in the middle of a page instead
    cut = data[:len(data) * 2 // 3]
    plan = decode.ogg_vorbis_plan(cut)
    assert 0 < len(plan["units"]) < len(truth)
    got = _render(oracle, plan, nat.FMT_S16)
    assert got.shape == (plan["total_frames"], 2)


@pytest.mark.gpu
def test_ogg_vorbis_file_to_pcm_on_the_device(oracle):
    import symphonia_b200 as sb
    with sb.Engine(0) as eng:
        for seed in range(8):
            data, s, truth, end = _file(300 + seed, channels=1 if seed == 5 else 2)
            for fmt in (nat.FMT_S16, nat.FMT_F32):
                want = _render(oracle, decode.ogg_vorbis_plan(data), fmt)
                got, rate = decode.decode_ogg_vorbis(eng, data, fmt)
                assert rate == 44100 and got.shape == want.shape
                assert (got.view(np.uint8) == want.view(np.uint8)).all()


@pytest.mark.gpu
def test_cpp_vorbis_decoder_on_ogg_files(tmp_path, oracle):
    """The C++ mirror of the plug-in interface: pages -> packets -> mapping -> registry -> GpuVorbisDecoder, one decode() per packet
    with the reader's trims."""
    import subprocess
    from tests.test_cpp_host import _build
    for seed in (300, 303, 305):
        data, s, _, end = _file(seed, channels=1 if seed == 305 else 2)
        plan = decode.ogg_vorbis_plan(data)
        want = _render(oracle, plan, nat.FMT_F32)
        inp, outp = tmp_path / f"in{seed}.ogg", tmp_path / f"out{seed}.bin"
        inp.write_bytes(data)
        res = subprocess.run([_build(), "file", "vorbis", str(inp), str(outp)], capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stdout + res.stderr
        flat = np.frombuffer(outp.read_bytes(), dtype=np.float32)
        sp = plan["spans"]
        left = sp["frames"].astype(np.int64) - sp["trim_start"] - sp["trim_end"]
        rows, at = [], 0
        for n in left:
            rows.append(flat[at:at + n * s.channels].reshape(s.channels, n).T)
            at += n * s.channels
        assert at == flat.size
        got = np.concatenate(rows)
        assert got.shape == want.shape and (np.ascontiguousarray(got).view(np.uint32) == np.ascontiguousarray(want).view(np.uint32)).all()


def test_one_long_stream_as_jobs_gives_the_same_plan():
    data, _, _, _ = _file(330, n_packets=48, pad=11)
    a, b = decode.ogg_vorbis_plan(data), decode.ogg_vorbis_plan(data, threads=4)
    assert len(a["units"]) == 48
    for key in ("units", "floor_y", "residue", "runs", "spans", "floors", "stream"):
        assert a[key].tobytes() == b[key].tobytes(), key
    assert a["total_frames"] == b["total_frames"]
