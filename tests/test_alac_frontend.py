"""ALAC packet decoding on the CPU: the oracle gives back the writer's PCM, and the front-end (alac_entropy.h, the code the device
decoder runs) decodes every packet, intact or damaged, exactly as the oracle does."""
import ctypes

import numpy as np
import pytest

import symphonia_b200._native as nat
from tests import _alac_cases as cases


@pytest.fixture(scope="module")
def orc():
    return cases.oracle_lib()


def fe_decode(packets, ck):
    """(status, frames, samples) of symgpu_alac_fe_decode_packets over a list of packets."""
    data = b"".join(packets)
    pieces = np.zeros(len(packets), dtype=nat.PIECE_DTYPE)
    at = 0
    for k, p in enumerate(packets):
        pieces[k]["offset"], pieces[k]["len"] = at, len(p)
        at += len(p)
    g = np.zeros(1, dtype=nat.ALAC_GROUP_DTYPE)
    for k in ("frame_length", "bit_depth", "pb", "mb", "kb", "channels"):
        g[k] = ck[k]
    status = np.zeros(len(packets), dtype=np.uint8)
    frames = np.zeros(len(packets), dtype=np.uint32)
    cap = len(packets) * ck["frame_length"] * ck["channels"]
    out = np.zeros(max(cap, 1), dtype=np.int32)
    n = ctypes.c_size_t(0)
    buf = np.frombuffer(data, dtype=np.uint8) if data else np.zeros(1, dtype=np.uint8)
    vp = ctypes.c_void_p
    rc = nat.lib().symgpu_alac_fe_decode_packets(vp(buf.ctypes.data), len(data), vp(pieces.ctypes.data), len(packets), vp(g.ctypes.data),
                                                 vp(status.ctypes.data), vp(frames.ctypes.data), vp(out.ctypes.data), cap, ctypes.byref(n))
    assert rc == 0
    return status, frames, out[:n.value]


ALL = cases.cases()


@pytest.mark.parametrize("name,ck,pcm,packet", ALL, ids=[c[0] for c in ALL])
def test_oracle_returns_the_encoded_pcm(orc, name, ck, pcm, packet):
    refused, got = cases.oracle_packet(orc, packet, ck)
    assert not refused
    want = (pcm.astype(np.int64) << (32 - ck["bit_depth"])).astype(np.uint32).view(np.int32)
    assert got.shape == want.shape and (got == want).all()


@pytest.mark.parametrize("name,ck,pcm,packet", ALL, ids=[c[0] for c in ALL])
def test_frontend_equals_oracle(orc, name, ck, pcm, packet):
    status, frames, samples = fe_decode([packet], ck)
    refused, want = cases.oracle_packet(orc, packet, ck)
    assert status[0] == (1 if refused else 0)
    assert frames[0] == len(want) and (samples.reshape(-1, ck["channels"]) == want).all()


def _damaged(rng, packet):
    b = bytearray(packet)
    kind = rng.integers(0, 3)
    if kind == 0 and b:
        for _ in range(int(rng.integers(1, 4))):
            k = int(rng.integers(0, len(b) * 8))
            b[k // 8] ^= 0x80 >> (k % 8)
    elif kind == 1:
        b = b[:int(rng.integers(0, len(b) + 1))]
    else:
        k = int(rng.integers(0, max(len(b), 1)))
        b[k:k + 1] = bytes([int(rng.integers(0, 256))])
    return bytes(b)


def _forced(packet, bit, width, value):
    """packet with `width` bits at `bit` set to value."""
    v = int.from_bytes(packet, "big")
    n = len(packet) * 8
    mask = ((1 << width) - 1) << (n - bit - width)
    v = (v & ~mask) | ((value << (n - bit - width)) & mask)
    return v.to_bytes(len(packet), "big")


def test_damaged_packets_get_the_oracles_decisions(orc):
    rng = np.random.default_rng(11)
    small = [c for c in ALL if c[1]["frame_length"] <= 4096]
    packets, cks = [], []
    for name, ck, pcm, packet in small:
        for _ in range(12):
            packets.append(_damaged(rng, packet))
            cks.append(ck)
        # reserved element tags, non-zero unused bits, bad shifts, modes 1..14: the first element's header fields
        for tag in (2, 5):
            packets.append(_forced(packet, 0, 3, tag)), cks.append(ck)
        packets.append(_forced(packet, 7, 12, 1)), cks.append(ck)
        packets.append(_forced(packet, 20, 2, 3)), cks.append(ck)
        if ck["bit_depth"] <= 16:
            packets.append(_forced(packet, 20, 2, 2)), cks.append(ck)
        for mode in (1, 7, 14):
            packets.append(_forced(packet, 3 + 4 + 12 + 4 + (32 if len(pcm) != ck["frame_length"] else 0) + 16, 4, mode)), cks.append(ck)
    refusals = 0
    for packet, ck in zip(packets, cks):
        status, frames, samples = fe_decode([packet], ck)
        refused, want = cases.oracle_packet(orc, packet, ck)
        refusals += refused
        assert status[0] == (1 if refused else 0), packet.hex()
        assert frames[0] == len(want) and (samples.reshape(-1, ck["channels"]) == want).all()
    assert refusals > len(packets) // 4


def test_many_packets_in_one_call(orc):
    rng = np.random.default_rng(3)
    from tests import _alac_bitstream as ab
    ck = cases.cookie(channels=2, frame_length=128)
    packets = [ab.encode_packet(ab.signal(rng, 128 if k % 5 else 50, 2, 16), ck) for k in range(20)]
    packets[7] = packets[7][:5]
    status, frames, samples = fe_decode(packets, ck)
    want = [cases.oracle_packet(orc, p, ck) for p in packets]
    assert list(status) == [1 if r else 0 for r, _ in want]
    assert (samples.reshape(-1, 2) == np.concatenate([w for _, w in want])).all()
