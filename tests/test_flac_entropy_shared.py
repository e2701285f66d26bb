"""The FLAC frame decoder shared by the CPU front-end and the device kernel (symphonia_b200/csrc/flac_entropy.h), on the CPU.

tests/cpp/flac_entropy_driver.cpp runs it twice over a packet corpus: as symgpu_flac_fe_decode_packets (the front-end loop) and
packet by packet as flac_decode_kernel calls it (one packet's records and channels x slot samples, in buffers of exactly that
size).  The driver is built with the device's bit window (SYMGPU_MP3E_DEVICE_WINDOW: five byte loads instead of one 8-byte load)
and once more with AddressSanitizer + UndefinedBehaviorSanitizer; both must give what the library's normal build gives."""
import os
import struct
import subprocess

import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import frontend, workloads
from tests import _flac_bitstream as fw

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "symphonia_b200", "csrc")
DECODED, REFUSED, NO_ROOM = 0, 1, 2


@pytest.fixture(scope="module")
def drivers(tmp_path_factory):
    d = tmp_path_factory.mktemp("flac_entropy")
    src = [os.path.join(ROOT, "tests", "cpp", "flac_entropy_driver.cpp"), os.path.join(CSRC, "flac_frontend.cpp")]
    common = ["g++", "-std=c++17", "-ffp-contract=off", "-DSYMGPU_MP3E_DEVICE_WINDOW", "-I/usr/local/cuda/include"]
    plain, sanitized = str(d / "driver_devwin"), str(d / "driver_sanitized")
    subprocess.check_call(common + ["-O2", "-o", plain] + src)
    subprocess.check_call(common + ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-o", sanitized] + src)
    return d, {"device window": plain, "sanitized": sanitized}


def _stream(seed, n_frames, block, bps, channels):
    rng = np.random.default_rng(seed)
    frames, subs, samples = workloads.flac_batch(n_frames, block, seed=seed, bps=bps, channels=channels)
    return [fw.write_frame(rng, frames[f], subs[int(frames[f]["first_subframe"]):int(frames[f]["first_subframe"]) + channels], samples, f, stream_bps=bps)
            for f in range(n_frames)]


def _header_len(p):
    return next(e for e in range(5, 17) if fw.crc8(bytes(p[:e])) == p[e])


def _damaged(packets, seed):
    """Bit flips in the header and in the sub-frames, truncations, junk before the sync code, reserved header codes with a valid
    CRC-8."""
    rng = np.random.default_rng(seed)
    out = []
    for k, p in enumerate(packets):
        b = bytearray(p)
        kind = k % 7
        if kind == 1:
            b[int(rng.integers(2, 6))] ^= 1 << int(rng.integers(8))
        elif kind == 2:
            for _ in range(3):
                b[int(rng.integers(8, len(b)))] ^= 1 << int(rng.integers(8))
        elif kind == 3:
            b = b[:int(rng.integers(1, len(b)))]
        elif kind == 4:
            b = bytearray(rng.integers(0, 256, int(rng.integers(1, 9)), dtype=np.uint8).tobytes()) + b
        elif kind == 5:
            h = _header_len(p)
            i, value = [(2, b[2] & 0x0F), (2, b[2] | 0x0F), (3, (b[3] & 0x0F) | 0xB0), (3, (b[3] & 0xF1) | 0x06), (3, b[3] | 0x01), (4, 0xFF),
                        (4, 0x80)][int(rng.integers(7))]
            b[i] = value
            b[h] = fw.crc8(bytes(b[:h]))
        out.append(bytes(b))
    return out


def _run(driver, tmp, packets, bps, channels, max_block, slots):
    blob = struct.pack("<4I", bps, channels, max_block, len(packets)) + b"".join(struct.pack("<2I", s, len(p)) + p for s, p in zip(slots, packets))
    src, dst = str(tmp / "in.bin"), str(tmp / "out.bin")
    with open(src, "wb") as f:
        f.write(blob)
    res = subprocess.run([driver, src, dst], capture_output=True, text=True, timeout=600,
                         env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=1"))
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    with open(dst, "rb") as f:
        return f.read()


def _expected(packets, bps, channels, max_block, slots):
    """The same two parts from the library's normal build (front-end) and the format's rules (per packet)."""
    data = b"".join(packets)
    table = np.zeros(len(packets), dtype=nat.PIECE_DTYPE)
    table["offset"] = np.cumsum([0] + [len(p) for p in packets[:-1]])
    table["len"] = [len(p) for p in packets]
    frames, infos, frame_of, subs, samples = frontend.flac_decode_packets(data, table, bps, channels, max_block)
    head = struct.pack("<4Q", 0, len(frames), len(subs), len(samples))
    part1 = head + frames.tobytes() + infos.tobytes() + frame_of.astype(np.uint32).tobytes() + subs.tobytes() + samples.tobytes()
    return part1, (frames, infos, frame_of, subs, samples)


def _check(drivers, packets, bps, channels, max_block, slots=None):
    tmp, exes = drivers
    if slots is None:
        slots = [65536] * len(packets)
    part1, (frames, infos, frame_of, subs, samples) = _expected(packets, bps, channels, max_block, slots)
    accepted = {int(i): k for k, i in enumerate(frame_of)}
    for name, exe in exes.items():
        got = _run(exe, tmp, packets, bps, channels, max_block, slots)
        assert got[:len(part1)] == part1, f"{name}: front-end output differs from the library's"
        at = len(part1)
        for i in range(len(packets)):
            st = got[at]
            at += 1
            if i in accepted and slots[i] >= int(infos[accepted[i]]["block_size"]):
                assert st == DECODED, (name, i, st)
            elif i in accepted:
                assert st == NO_ROOM, (name, i, st)
            else:
                assert st in (REFUSED, NO_ROOM) if slots[i] < 65536 else st == REFUSED, (name, i, st)
            if st != DECODED:
                continue
            k = accepted[i]
            fr = np.frombuffer(got[at:at + 16], dtype=nat.FLAC_FRAME_DTYPE)[0]
            info = np.frombuffer(got[at + 16:at + 40], dtype=nat.FLAC_FRAME_INFO_DTYPE)[0]
            at += 40
            c, n = int(fr["channels"]), int(info["block_size"])
            assert got[at - 24:at] == infos[k].tobytes()
            want_fr = frames[k].copy()
            want_fr["first_subframe"] = 0
            assert fr.tobytes() == want_fr.tobytes()
            sf = np.frombuffer(got[at:at + 144 * c], dtype=nat.FLAC_SUBFRAME_DTYPE)
            at += 144 * c
            first = int(frames[k]["first_subframe"])
            ref = subs[first:first + c].copy()
            base = int(ref[0]["offset"])
            ref["offset"] -= base
            assert sf.tobytes() == ref.tobytes(), (name, i)
            smp = np.frombuffer(got[at:at + 4 * c * n], dtype=np.int32)
            at += 4 * c * n
            assert (smp == samples[base:base + c * n]).all(), (name, i)
        assert at == len(got)
    return len(accepted)


@pytest.mark.parametrize("bps,channels,block", [(16, 2, 576), (24, 2, 1152), (8, 1, 192), (20, 3, 300), (12, 2, 97), (32, 1, 256), (16, 8, 64)])
def test_device_window_and_sanitizers_match_the_front_end(drivers, bps, channels, block):
    packets = _stream(1000 + bps + block, 10, block, bps, channels)
    assert _check(drivers, packets, bps, channels, block) == 10
    assert _check(drivers, packets, 0, 0, 0) > 0                         # nothing known about the stream: frames carry their own bps


def test_damaged_packets(drivers):
    packets = _stream(1201, 42, 576, 16, 2)
    hit = _damaged(packets, 5)
    n = _check(drivers, hit, 16, 2, 576)
    assert 10 < n < 42
    _check(drivers, packets[:8], 16, 1, 576)                              # more channels than the stream
    _check(drivers, packets[:8], 16, 2, 100)                              # a larger block than the stream
    _check(drivers, packets[:8], 0, 2, 576)                               # bps neither in the frame nor in the stream for some


def test_slots_smaller_than_the_block(drivers):
    """A block larger than the slot is NO_ROOM, the case a device job of too small a slot meets; a refused header stays REFUSED."""
    packets = _stream(1301, 12, 576, 16, 2)
    slots = [575 if k % 2 else 576 for k in range(12)]
    hit = _damaged(packets, 9)
    _check(drivers, packets, 16, 2, 576, slots)
    _check(drivers, hit, 16, 2, 576, slots)
