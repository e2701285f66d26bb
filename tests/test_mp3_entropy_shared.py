"""The Layer III packet rules shared by the CPU front-end and the device kernels (symphonia_b200/csrc/mp3_entropy.h), on the CPU.

tests/cpp/mp3_entropy_driver.cpp runs them twice over a corpus of files: as symgpu_mp3_fe_decode_packets (the front-end loop), and
in the device's schedule -- the prologue of every packet, then the side read of every packet, then rounds of the per-file reservoir
walk, the main-data gather and every granule-channel decoded on its own in a shuffled order, until no file fails.  The driver is
built with the device's bit window (SYMGPU_MP3E_DEVICE_WINDOW) and once more with AddressSanitizer + UndefinedBehaviorSanitizer.
The front-end loop must give the library's output; the device schedule must give the library's frames with the joint-stereo window
mismatches left out, the same accept / refuse decisions, and the rounds of symgpu_mp3_entropy_decode_cpu."""
import os
import struct
import subprocess

import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import frontend
from tests import _mp3_bitstream as bw

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "symphonia_b200", "csrc")
DECODED, REFUSED, FAILED, LEFT_OUT = 0, 1, 2, 3
F_MIXED, F_MID_SIDE, F_INTENSITY, F_MUTE = 1 << 0, 1 << 4, 1 << 5, 1 << 7   # SYMGPU_MP3_F_*


@pytest.fixture(scope="module")
def drivers(tmp_path_factory):
    d = tmp_path_factory.mktemp("mp3_entropy")
    src = [os.path.join(ROOT, "tests", "cpp", "mp3_entropy_driver.cpp"), os.path.join(CSRC, "mp3_frontend.cpp"), os.path.join(CSRC, "tables.cpp")]
    common = ["g++", "-std=c++17", "-ffp-contract=off", "-DSYMGPU_MP3E_DEVICE_WINDOW", "-I/usr/local/cuda/include"]
    plain, sanitized = str(d / "driver_devwin"), str(d / "driver_sanitized")
    subprocess.check_call(common + ["-O2", "-o", plain] + src)
    subprocess.check_call(common + ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-o", sanitized] + src)
    return d, {"device window": plain, "sanitized": sanitized}


def _run(driver, tmp, files):
    blob = struct.pack("<I", len(files))
    for packets in files:
        blob += struct.pack("<I", len(packets)) + b"".join(struct.pack("<I", len(p)) + p for p in packets)
    src, dst = str(tmp / "in.bin"), str(tmp / "out.bin")
    with open(src, "wb") as f:
        f.write(blob)
    res = subprocess.run([driver, src, dst], capture_output=True, text=True, timeout=900,
                         env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=1"))
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    with open(dst, "rb") as f:
        return f.read()


def _table(packets):
    table = np.zeros(len(packets), dtype=nat.MPA_PACKET_DTYPE)
    table["offset"] = np.cumsum([0] + [len(p) for p in packets[:-1]]) if packets else []
    table["size"] = [len(p) for p in packets]
    return table


def mismatch(units):
    """Frames whose joint-stereo channels are on different window sequences (stereo.rs:503-505), from the front-end's units."""
    flags, bt = units["flags"].astype(np.int64), units["block_type"].astype(np.int64)
    joint = (flags[:, 0, 0] & (F_MID_SIDE | F_INTENSITY)) != 0
    out = np.zeros(len(units), dtype=bool)
    for gr in range(2):
        a, b = (slice(None), gr, 0), (slice(None), gr, 1)
        present = ((flags[a] & F_MUTE) == 0) & ((flags[b] & F_MUTE) == 0)
        mixed = ((flags[a] ^ flags[b]) & F_MIXED) != 0
        out |= joint & present & ((bt[a] != bt[b]) | ((bt[a] == nat.MP3_SHORT) & mixed))
    return out


def _check(drivers, files):
    """Both parts of every driver build against the library; returns (decoded, left out, failed) over all files."""
    tmp, exes = drivers
    part1, totals = b"", np.zeros(3, dtype=np.int64)
    for packets in files:
        data = b"".join(packets)
        units, quant, frame_of, _ = frontend.Mp3Frontend().decode_packets(data, _table(packets))
        part1 += struct.pack("<2Q", 0, len(frame_of)) + frame_of.astype(np.uint32).tobytes() + units.tobytes() + quant.tobytes()
        *_, rounds = frontend.entropy_decode_cpu(data, _table(packets))
        out = mismatch(units)
        totals += [int((~out).sum()), int(out.sum()), rounds - 1]
    for name, exe in exes.items():
        got = _run(exe, tmp, files)
        assert got[:len(part1)] == part1, f"{name}: the front-end loop differs from the library's"
        at = len(part1)
        for packets in files:
            data = b"".join(packets)
            units, quant, frame_of, _ = frontend.Mp3Frontend().decode_packets(data, _table(packets))
            *_, rounds = frontend.entropy_decode_cpu(data, _table(packets))
            out = mismatch(units)
            got_rounds = struct.unpack_from("<I", got, at)[0]
            at += 4
            status = np.frombuffer(got, dtype=np.uint8, count=len(packets), offset=at)
            at += len(packets)
            assert got_rounds == rounds, f"{name}: {got_rounds} rounds, symgpu_mp3_entropy_decode_cpu takes {rounds}"
            want = np.full(len(packets), REFUSED, dtype=np.uint8)
            want[frame_of] = np.where(out, LEFT_OUT, DECODED)
            refused = want == REFUSED
            assert (status[~refused] == want[~refused]).all(), f"{name}: the device schedule decides other packets"
            assert np.isin(status[refused], (REFUSED, FAILED)).all() and int((status == FAILED).sum()) == rounds - 1, \
                f"{name}: refused / failed packets disagree with the rounds"
            n = int((~out).sum())
            gu = got[at:at + n * 4 * nat.MP3_GC_DTYPE.itemsize]
            at += len(gu)
            gq = got[at:at + n * 4 * 576 * 2]
            at += len(gq)
            assert gu == units[~out].tobytes(), f"{name}: units differ from the front-end's"
            assert gq == quant[~out].tobytes(), f"{name}: spectra differ from the front-end's"
        assert at == len(got)
    return totals


STREAMS = [  # (version, mode, rate_idx, bitrate_idx, protected): MPEG-1 / 2 / 2.5, every channel mode, CRC
    ("1", 1, 0, 9, False), ("1", 0, 1, 14, True), ("1", 3, 2, 5, False), ("1", 2, 0, 11, False),
    ("2", 1, 0, 8, False), ("2", 3, 1, 4, True), ("2.5", 1, 2, 6, False), ("2.5", 0, 0, 3, True)]


@pytest.mark.parametrize("version,mode,rate_idx,bitrate_idx,protected", STREAMS)
def test_writer_streams(drivers, version, mode, rate_idx, bitrate_idx, protected):
    rng = np.random.default_rng(300 + bitrate_idx + 7 * mode)
    files = [bw.gen_stream(rng, 24, version=version, mode=mode, rate_idx=rate_idx, bitrate_idx=bitrate_idx, protected=protected, pair_blocks=True)[0]
             for _ in range(2)]
    decoded, left_out, failed = _check(drivers, files)
    assert decoded == 48 and left_out == 0 and failed == 0


def test_window_mismatches_are_left_out(drivers):
    rng = np.random.default_rng(41)
    files = [bw.gen_stream(rng, 40, version=v, mode=1, bitrate_idx=9, pair_blocks=False, force_mode_ext=lambda k: 3)[0] for v in ("1", "2")]
    decoded, left_out, _ = _check(drivers, files)
    assert left_out > 0 and decoded > 0


def _p23_at(version, n_ch):
    """Bit offset, in the side information, of the first part2_3_length."""
    return (18 if n_ch == 1 else 20) if version == "1" else (9 if n_ch == 1 else 10)


def _set_bits(b, at, width, value):
    for k in range(width):
        bit = (value >> (width - 1 - k)) & 1
        i, m = (at + k) // 8, 0x80 >> ((at + k) % 8)
        b[i] = (b[i] | m) if bit else (b[i] & ~m)


def _side_len(version, n_ch):
    return (17 if n_ch == 1 else 32) if version == "1" else (9 if n_ch == 1 else 17)


@pytest.mark.parametrize("version,mode", [("1", 1), ("1", 3), ("2", 0), ("2.5", 1)])
def test_damaged_files(drivers, version, mode):
    rng = np.random.default_rng(700 + 3 * mode)
    frames, truth = bw.gen_stream(rng, 48, version=version, mode=mode, bitrate_idx=9, pair_blocks=True)
    side = 4 + _side_len(version, 1 if mode == 3 else 2)
    hit = []
    for k, f in enumerate(frames):
        b = bytearray(f)
        r = k % 8
        if r == 1:
            hit.append(bytes(b[:side - 3]))                                   # cut inside the side information
            continue
        if r == 2:
            b[4 + int(rng.integers(0, side - 4))] ^= 1 << int(rng.integers(8))  # a flipped bit in the side information
        elif r == 3 and len(b) > side + 4:
            for _ in range(4):
                b[int(rng.integers(side, len(b)))] ^= 1 << int(rng.integers(8))  # flipped bits in main data
        elif r == 4:
            b[4] |= 0xFF                                                      # main_data_begin far beyond the reservoir
        elif r in (0, 7) and k:
            _set_bits(b, 8 * 4 + _p23_at(version, 1 if mode == 3 else 2), 12, 4095)  # the first part2_3_length beyond the main data
        hit.append(bytes(b))
    over = [bytearray(f) for f in frames]
    for k in range(5, len(over), 8):
        _set_bits(over[k], 8 * 4 + _p23_at(version, 1 if mode == 3 else 2), 12, 4095)     # main data over-reads only
    files = [hit, [bytes(b) for b in over], frames[20:] + frames[:20], frames[7:31] + frames[:5]]    # (and files joined mid-stream)
    decoded, _, failed = _check(drivers, files)
    assert decoded > 0 and (failed > 0 or mode == 3)   # (a mono frame's window may hold all 4095 bits)


def test_edge_files(drivers):
    rng = np.random.default_rng(5)
    f1, _ = bw.gen_stream(rng, 6, version="1", mode=1, bitrate_idx=9, pair_blocks=True)
    f2, _ = bw.gen_stream(rng, 6, version="2", mode=3, bitrate_idx=8, pair_blocks=True)
    alien = bw.gen_stream(rng, 2, version="1", mode=1, rate_idx=1, bitrate_idx=9, pair_blocks=True)[0]
    decoded, _, _ = _check(drivers, [[b"", f1[0][:3]], f1[:2] + f2[:2] + alien + f1[2:] + [f1[0] + b"\0"], f2 + f1[:1]])
    assert decoded > 0
