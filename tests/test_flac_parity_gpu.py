"""GPU parity of the FLAC integer restoration (SURVEY §8f N4): identical to the oracle, and -- the property the
format exists for -- identical to the PCM the residuals were computed from.  Covers every sub-frame type (CONSTANT,
VERBATIM, FIXED orders 0..4, LPC orders 1..32), all channel assignments and wasted bits."""
import os

import numpy as np
import pytest

from symphonia_b200 import workloads
from symphonia_b200._native import FLAC_LPC
from tests import test_oracle_kat_flac as kat

pytestmark = [pytest.mark.gpu]


@pytest.fixture(scope="module")
def engine():
    import symphonia_b200 as sb
    eng = sb.Engine(0)
    yield eng
    eng.close()


@pytest.mark.parametrize("bps,channels,block", [(16, 2, 512), (24, 2, 1152), (16, 1, 300), (8, 2, 64), (32, 2, 97), (16, 2, 4096)])
def test_restore_matches_oracle_and_source_pcm(engine, oracle, bps, channels, block):
    n_frames = 40 if block < 2000 else 10
    frames, subs, samples, expect = workloads.flac_batch(n_frames, block, seed=900 + bps + block, bps=bps, channels=channels,
                                                         return_pcm=True)
    rc, want = kat._restore(oracle, frames, subs, samples)
    assert rc == 0
    got = engine.flac_restore_host(frames, subs, samples.copy())
    assert (got == want).all(), f"{int((got != want).sum())} samples differ from the oracle, first at {np.argwhere(got != want)[0]}"
    for sf in subs:  # lossless: the encoder's PCM comes back
        a, n = int(sf["offset"]), int(sf["n"])
        assert (got[a:a + n] == expect[a:a + n]).all()
    assert (subs["type"] == FLAC_LPC).any() and np.abs(expect).max() > 0


def test_malformed_descriptors(engine):
    import symphonia_b200 as sb
    frames, subs, samples = workloads.flac_batch(2, 64, seed=7)
    for field, value, status in (("order", 40, 1), ("shift", 20, 2), ("type", 9, 1)):
        bad = subs.copy()
        bad[0]["type"] = FLAC_LPC if field != "type" else value
        bad[0]["order"], bad[0]["shift"] = 2, 3
        if field != "type":
            bad[0][field] = value
        with pytest.raises(sb.SymgpuError) as e:
            engine.flac_restore_host(frames, bad, samples.copy())
        assert e.value.status == status
    bad = subs.copy()
    bad[1]["offset"] = samples.size - 3
    with pytest.raises(sb.SymgpuError) as e:
        engine.flac_restore_host(frames, bad, samples.copy())
    assert e.value.status == 6
    good = engine.flac_restore_host(frames, subs, samples.copy())  # still healthy
    assert good.shape == samples.shape


def test_flac_file_bytes_to_pcm(engine):
    """.flac bytes -> container splitter -> front-end (both CPU) -> restoration kernel == the PCM the encoder started from."""
    from symphonia_b200 import _native as nat
    from symphonia_b200 import frontend, packetizer
    from tests import _flac_bitstream as fw
    rng = np.random.default_rng(61)
    bps, channels, block, n_frames = 16, 2, 1152, 40
    frames, subs, samples, expect = workloads.flac_batch(n_frames, block, seed=777, bps=bps, channels=channels, return_pcm=True)
    order = [f for f in range(n_frames) if f % 7] + [0]
    pk = []
    for number, f in enumerate(order):
        fr = frames[f]
        pk.append(fw.write_frame(rng, fr, subs[int(fr["first_subframe"]):int(fr["first_subframe"]) + channels], samples, number, stream_bps=bps))
    total = sum(int(subs[int(frames[f]["first_subframe"])]["n"]) for f in order)
    data = fw.native_file(pk, fw.stream_info_block(block, block, 44100, channels, bps, total))
    info, packets = packetizer.flac_index(data)
    assert len(packets) == len(pk)
    table = np.zeros(len(packets), dtype=nat.PIECE_DTYPE)
    table["offset"], table["len"] = packets["offset"], packets["size"]
    gf, gi, gof, gs, gsm = frontend.flac_decode_packets(data, table, bps, channels, block)
    got = engine.flac_restore_host(gf, gs, gsm.copy())
    for k, f in enumerate(order):
        for c in range(channels):
            a, b = subs[f * channels + c], gs[int(gf[k]["first_subframe"]) + c]
            n = int(a["n"])
            assert (got[int(b["offset"]):int(b["offset"]) + n] == expect[int(a["offset"]):int(a["offset"]) + n]).all(), (k, c)
