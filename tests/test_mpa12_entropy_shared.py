"""The Layer I / II packet rules shared by the CPU front-end and the device kernels (symphonia_b200/csrc/mpa12_entropy.h), on the CPU.

tests/cpp/mpa12_entropy_driver.cpp runs them twice over a packet corpus: as symgpu_mpa12_fe_decode_packets (the front-end loop), and
in the device's schedule -- the prologue of every packet, then the side read and the fit rule of every packet, then every sample
codeword decoded on its own at its closed-form bit position, in a shuffled order.  The driver is built with the device's bit window
(SYMGPU_MP3E_DEVICE_WINDOW) and once more with AddressSanitizer + UndefinedBehaviorSanitizer; the output and the accept / refuse
decisions of both parts must be those of the library's normal build.  This is the proof of the parallel decomposition."""
import os
import struct
import subprocess

import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import frontend
from tests import _mpa12_bitstream as bw
from tests import _streams as st

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "symphonia_b200", "csrc")


@pytest.fixture(scope="module")
def drivers(tmp_path_factory):
    d = tmp_path_factory.mktemp("mpa12_entropy")
    src = [os.path.join(ROOT, "tests", "cpp", "mpa12_entropy_driver.cpp"), os.path.join(CSRC, "mpa12_frontend.cpp")]
    common = ["g++", "-std=c++17", "-ffp-contract=off", "-DSYMGPU_MP3E_DEVICE_WINDOW", "-I/usr/local/cuda/include"]
    plain, sanitized = str(d / "driver_devwin"), str(d / "driver_sanitized")
    subprocess.check_call(common + ["-O2", "-o", plain] + src)
    subprocess.check_call(common + ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-o", sanitized] + src)
    return d, {"device window": plain, "sanitized": sanitized}


def _run(driver, tmp, packets, layer):
    blob = struct.pack("<2I", layer, len(packets)) + b"".join(struct.pack("<I", len(p)) + p for p in packets)
    src, dst = str(tmp / "in.bin"), str(tmp / "out.bin")
    with open(src, "wb") as f:
        f.write(blob)
    res = subprocess.run([driver, src, dst], capture_output=True, text=True, timeout=600,
                         env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=1"))
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    with open(dst, "rb") as f:
        return f.read()


def _check(drivers, packets, layer):
    """Both parts of every driver build against symgpu_mpa12_fe_decode_packets of the library; returns the accepted count."""
    tmp, exes = drivers
    data = b"".join(packets)
    table = np.zeros(len(packets), dtype=nat.MPA_PACKET_DTYPE)
    table["offset"] = np.cumsum([0] + [len(p) for p in packets[:-1]]) if packets else []
    table["size"] = [len(p) for p in packets]
    sub, frame_of, _ = frontend.mpa12_decode_packets(data, table, layer)
    part1 = struct.pack("<2Q", 0, len(frame_of)) + frame_of.astype(np.uint32).tobytes() + sub.tobytes()
    accepted = np.zeros(len(packets), dtype=np.uint8)
    accepted[frame_of] = 1
    for name, exe in exes.items():
        got = _run(exe, tmp, packets, layer)
        assert got[:len(part1)] == part1, f"{name}: the front-end loop differs from the library's"
        at = len(part1)
        assert got[at:at + len(packets)] == accepted.tobytes(), f"{name}: the device schedule accepts / refuses other packets"
        at += len(packets)
        rest = np.frombuffer(got[at:], dtype=np.float32)
        assert rest.size == sub.size and (rest.view(np.uint32) == sub.reshape(-1).view(np.uint32)).all(), \
            f"{name}: codewords decoded one by one differ from the front-end's samples"
    return len(frame_of)


def _frames(layer, seed, n, **kw):
    rng = np.random.default_rng(seed)
    gen = bw.gen_layer1_frame if layer == 1 else bw.gen_layer2_frame
    out, truths = [], []
    for k in range(n):
        f, t = gen(rng, mode_ext=k % 4, **kw)
        out.append(f), truths.append(t)
    return out, truths


STREAMS = [  # (layer, version, bitrate_idx, rate_idx, mode, protected): every Layer II allocation table, every mode, CRC, MPEG-1 / 2 / 2.5
    (1, "1", 9, 0, 0, False), (1, "1", 14, 1, 1, True), (1, "1", 2, 2, 3, False), (1, "2", 5, 0, 1, False), (1, "2.5", 3, 2, 3, True),
    (1, "1", 7, 0, 2, False),
    (2, "1", 8, 0, 0, False), (2, "1", 14, 0, 1, True), (2, "1", 12, 1, 0, False), (2, "1", 2, 0, 3, False), (2, "1", 1, 2, 3, False),
    (2, "1", 6, 2, 1, False), (2, "2", 10, 0, 1, False), (2, "2.5", 4, 1, 3, True), (2, "2", 14, 2, 2, False)]


@pytest.mark.parametrize("layer,version,bitrate_idx,rate_idx,mode,protected", STREAMS)
def test_writer_streams(drivers, layer, version, bitrate_idx, rate_idx, mode, protected):
    frames, _ = _frames(layer, 40 + bitrate_idx + 7 * mode, 12, version=version, bitrate_idx=bitrate_idx, rate_idx=rate_idx, mode=mode,
                        protected=protected, density=0.95)
    assert _check(drivers, frames, layer) == 12


def _field_ends(layer, t, protected):
    """Byte positions (in the packet) just past the fields the side read and the samples consume: allocation, scfsi, each scale
    factor, each granule."""
    n_ch, bound = t["n_ch"], t["bound"]
    head = 4 + (2 if protected else 0)
    ends, bits = [], 0
    if layer == 1:
        bits += 4 * sum(n_ch if sb < bound else 1 for sb in range(32))
        ends.append(bits)
        for sb in range(32):
            for ch in range(n_ch):
                if t["alloc"][ch][sb]:
                    bits += 6
                    ends.append(bits)
        g = sum(t["alloc"][ch][sb] + 1 for sb in range(32) for ch in range(n_ch if sb < bound else 1) if t["alloc"][ch][sb])
    else:
        table, sblimit = t["table"], t["sblimit"]
        bits += sum(table[sb][0] * (n_ch if sb < bound else 1) for sb in range(sblimit))
        ends.append(bits)
        bits += 2 * sum(1 for sb in range(sblimit) for ch in range(n_ch) if t["alloc"][ch][sb])
        ends.append(bits)
        for sb in range(sblimit):
            for ch in range(n_ch):
                if t["alloc"][ch][sb]:
                    bits += 6 * {0: 3, 1: 2, 2: 1, 3: 2}[t["scfsi"][ch][sb]]
                    ends.append(bits)

        def code_bits(levels):
            return {3: 5, 5: 7, 9: 10}.get(levels) or 3 * (levels + 1).bit_length() - 3
        g = sum(code_bits(table[sb][1][t["alloc"][ch][sb]]) for sb in range(sblimit) for ch in range(n_ch if sb < bound else 1) if t["alloc"][ch][sb])
    ends += [bits + g * k for k in range(1, 13)]
    return sorted({head + (b + 7) // 8 for b in ends})


def _relabel(frame, layer, version, rate_idx, mode, mode_ext, protected, bitrate_idx, padding):
    """The frame's first bytes under a header whose declared size is another bitrate's: the body is cut where that size ends, so the
    side read or the samples run out wherever the cut falls."""
    n = st.mpa_frame_len(version, layer, bitrate_idx, rate_idx, padding)
    word = st.mpa_word(version=version, layer=layer, bitrate_idx=bitrate_idx, rate_idx=rate_idx, mode=mode, mode_ext=mode_ext, padding=padding,
                       protected=protected)
    body = frame[4:n] + bytes(max(0, n - len(frame)))
    return word.to_bytes(4, "big") + body


@pytest.mark.parametrize("layer,version,bitrate_idx,rate_idx,mode,protected", [STREAMS[1], STREAMS[4], STREAMS[7], STREAMS[11], STREAMS[13]])
def test_damaged_packets(drivers, layer, version, bitrate_idx, rate_idx, mode, protected):
    rng = np.random.default_rng(900 + bitrate_idx)
    frames, truths = _frames(layer, 77 + bitrate_idx, 6, version=version, bitrate_idx=bitrate_idx, rate_idx=rate_idx, mode=mode,
                             protected=protected, density=0.95)
    hit = []
    for k, (f, t) in enumerate(zip(frames, truths)):
        head = 4 + (2 if protected else 0)
        ends = _field_ends(layer, t, protected)
        hit += [f[:e] for e in ends if e < len(f)]                                       # cut at a field boundary (the size check refuses it)
        for b in range(1, 15):                                                           # a header declaring a shorter frame
            for pad in (0, 1):
                hit.append(_relabel(f, layer, version, rate_idx, mode, k % 4, protected, b, pad))
        side_end = ends[min(len(ends) - 1, 3)]
        for _ in range(12):                                                              # bit flips in allocation / scfsi / scale factors
            b = bytearray(f)
            b[int(rng.integers(head, max(head + 1, side_end)))] ^= 1 << int(rng.integers(8))
            hit.append(bytes(b))
        hit.append(bytes(rng.integers(0, 256, int(rng.integers(1, 9)), dtype=np.uint8).tobytes()) + f)   # junk before the sync word
        hit.append(f + b"\0")                                                            # wrong size
        hit.append(f)
    other = bw.gen_layer2_frame(rng)[0] if layer == 1 else bw.gen_layer1_frame(rng)[0]
    hit.append(other)                                                                    # wrong layer
    n = _check(drivers, hit, layer)
    assert 6 <= n < len(hit)
    _check(drivers, [other] + frames, layer)                                              # a wrong-layer packet first fixes the specification


def test_layer1_allocation_15_and_edge_packets(drivers):
    rng = np.random.default_rng(5)
    f1, _ = bw.gen_layer1_frame(rng, "1", 9, 0, 0)
    f2, _ = bw.gen_layer2_frame(rng, "1", 8, 0, 0)
    bad = bytearray(f1)
    bad[4] |= 0xF0                                                                       # first allocation field = 15
    bad_late = bytearray(f1)
    bad_late[10] |= 0x0F                                                                 # a later allocation field = 15
    alien = bw.gen_layer1_frame(rng, "1", 9, 1, 0)[0]                                    # another sample rate
    mono = bw.gen_layer1_frame(rng, "1", 9, 0, 3)[0]                                     # another channel count
    seq = [b"", f1[:3], bytes(bad), f1, bytes(bad_late), f2, alien, mono, f1[:40], f1]
    assert _check(drivers, seq, 1) == 2
    assert _check(drivers, [f2, f1, f2[:100], f2], 2) == 2
    assert _check(drivers, [], 1) == 0
