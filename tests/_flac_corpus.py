"""Seeded native FLAC files for the device FLAC index (symgpu_flac_index_dev) and its CPU schedule (tests/cpp/flac_index_driver.cpp).

The splitter only reads frame headers, CRC-8s and CRC-16s, so most frames here carry random bodies behind a valid header and a
valid CRC-16; decodable files come from tests/test_flac_decode_gpu.py.  Every case the splitter's rules can meet is pinned: both
blocking strategies, every depth and channel count, false sync words with valid headers inside frames, corrupted frames, repeated,
decreasing and zero sequence numbers, junk, cut frames, every way open() fails, sync-dense junk, long chains and a frame whose
CRC-valid end lies past the 16 MiB window."""
import numpy as np

from tests import _flac_bitstream as fw

_BPS_CODE = {8: 1, 12: 2, 16: 4, 20: 5, 24: 6, 32: 7}
_RATE_CODE = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10, 96000: 11}


def header(seq, block, channels, bps, rate=44100, by_sample=False, explicit=False):
    """A frame header with its CRC-8: the block size as a code when there is one (else 16-bit explicit), the rate and depth in
    the header or (explicit=False, half of the time by the caller's choice) left to STREAMINFO."""
    codes = {192: 1, **{576 << k: 2 + k for k in range(4)}, **{256 << k: 8 + k for k in range(8)}}
    if block in codes and not explicit:
        bs, tail = codes[block], b""
    elif block <= 256:
        bs, tail = 6, bytes([block - 1])
    else:
        bs, tail = 7, (block - 1).to_bytes(2, "big")
    sr = _RATE_CODE.get(rate, 0) if not explicit else 13
    sr_tail = rate.to_bytes(2, "big") if sr == 13 else b""
    ch = channels - 1
    head = bytes([0xFF, 0xF8 | int(by_sample), bs << 4 | sr, ch << 4 | _BPS_CODE[bps] << 1]) + fw.utf8_encode(seq) + tail + sr_tail
    return head + bytes([fw.crc8(head)])


def frame(rng, seq, block, channels, bps, body=None, **kw):
    """header + body (random, with no sync word, when not given) + CRC-16."""
    if body is None:
        body = rng.integers(0, 255, int(rng.integers(0, 200)), dtype=np.uint8).tobytes()   # no 0xff: no sync word inside
    f = header(seq, block, channels, bps, **kw) + body
    return f + fw.crc16(f).to_bytes(2, "big")


def stream(frames, block_min, block_max, channels, bps, rate=44100, extra_blocks=()):
    return fw.native_file(frames, fw.stream_info_block(block_min, block_max, rate, channels, bps, 0), extra_blocks)


def _plain(rng, n, block, channels, bps, by_sample=False, **kw):
    frames, at = [], 0
    for k in range(n):
        frames.append(frame(rng, at if by_sample else k, block, channels, bps, by_sample=by_sample, explicit=bool(rng.integers(2)), **kw))
        at += block
    return frames


def files(seed=70):
    """[(name, bytes)]."""
    rng = np.random.default_rng(seed)
    out = []
    # blocking strategies, depths, channel counts
    for k, (bps, ch) in enumerate([(8, 1), (12, 2), (16, 2), (20, 3), (24, 4), (32, 5), (16, 6), (24, 7), (16, 8)]):
        out.append((f"fixed {bps} bits {ch} ch", stream(_plain(rng, 20, 576, ch, bps), 576, 576, ch, bps)))
    for k, (bps, ch) in enumerate([(16, 2), (24, 1), (8, 8)]):
        blocks = [int(b) for b in rng.integers(16, 4000, 15)]
        frames, at = [], 0
        for b in blocks:
            frames.append(frame(rng, at, b, ch, bps, by_sample=True))
            at += b
        out.append((f"variable {bps} bits {ch} ch", stream(frames, 16, 4096, ch, bps)))
    # false sync words with valid, fitting headers inside frame bodies
    frames = []
    for k in range(30):
        fake = header(k + 1 + int(rng.integers(0, 3)), 576, 2, 16)
        body = rng.integers(0, 255, 40, dtype=np.uint8).tobytes() + fake + rng.integers(0, 255, 30, dtype=np.uint8).tobytes()
        frames.append(frame(rng, k, 576, 2, 16, body=body))
    out.append(("false syncs", stream(frames, 576, 576, 2, 16)))
    # a corrupted frame: its CRC-16 fails, the next frame is found by resync with the carried sequence threshold
    frames = _plain(rng, 12, 576, 2, 16)
    bad = bytearray(frames[5])
    bad[len(bad) // 2] ^= 0x5A
    frames[5] = bytes(bad)
    out.append(("corrupted frame", stream(frames, 576, 576, 2, 16)))
    # repeated, decreasing and zero sequence numbers
    for name, seqs in (("repeated", [0, 1, 2, 2, 3, 3, 3, 4]), ("decreasing", [5, 6, 7, 3, 4, 8, 2, 9]), ("zeros", [0, 0, 3, 0, 2, 0, 7, 7]),
                       ("wrap", [1, 2, 3, 0, 1, 2, 3, 1])):
        out.append((f"{name} sequence numbers", stream([frame(rng, s, 576, 1, 16) for s in seqs], 576, 576, 1, 16)))
    # junk between frames and after the last; a cut last frame; a frame ending exactly at the end
    frames = _plain(rng, 10, 1024, 2, 24)
    junk = [rng.integers(0, 256, int(rng.integers(1, 50)), dtype=np.uint8).tobytes() for _ in frames]
    out.append(("junk between frames", stream([f + j for f, j in zip(frames, junk)], 1024, 1024, 2, 24)))
    out.append(("junk after the last", stream(frames, 1024, 1024, 2, 24) + b"\xff\xf8\x00junk\xff"))
    out.append(("cut last frame", stream(frames, 1024, 1024, 2, 24)[:-7]))
    out.append(("ends at the end", stream(frames, 1024, 1024, 2, 24)))
    # open() failures and edges
    good = stream(_plain(rng, 3, 576, 2, 16), 576, 576, 2, 16)
    info = fw.stream_info_block(576, 576, 44100, 2, 16, 0)
    out.append(("no marker", b"fLaX" + good[4:]))
    out.append(("bad STREAMINFO", fw.native_file([], fw.stream_info_block(8, 576, 44100, 2, 16, 0))))
    out.append(("zero rate", fw.native_file([], fw.stream_info_block(576, 576, 0, 2, 16, 0))))
    out.append(("STREAMINFO not first", b"fLaC" + bytes([1, 0, 0, 4]) + bytes(4) + bytes([0x80, 0, 0, 34]) + info))
    out.append(("cut metadata", good[:30]))
    out.append(("cut block header", good[:40]))
    out.append(("long metadata chain", fw.native_file(_plain(rng, 6, 576, 2, 16), info,
                                                      [(1 + k % 5, rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8).tobytes())
                                                       for k in range(60)])))
    out.append(("metadata only", fw.native_file([], info)))
    for n in range(8):
        out.append((f"{n} bytes", b"fLaC\x80\x00\x00\x22"[:n]))
    # sync-dense junk after the metadata, and a stream whose frames sit inside it
    out.append(("sync-dense junk", fw.native_file([], info) + b"\xff\xf8" * 20000))
    dense = [frame(rng, k, 576, 2, 16, body=b"\xff\xf8\xc9\x18" * 30) for k in range(20)]
    out.append(("sync-dense frames", stream(dense, 576, 576, 2, 16)))
    # many plausible headers sharing one key: back-to-back 8-byte frames (every frame start of a stream has the frame's key) whose
    # numbers repeat, so most of them are rejected as ends by the sequence rule
    tiny = [tiny_frame(s) for s in [1] * 300 + [2] + [0] * 50 + list(range(3, 100)) + [5] * 200]
    out.append(("one key", stream(tiny, 192, 192, 2, 16)))
    return out


def tiny_frame(seq, channels=2):
    """The smallest frame: a 6-byte header (block 192, rate and depth from STREAMINFO) and the CRC-16: 8 bytes for seq < 128."""
    head = bytes([0xFF, 0xF8, 0x10, (channels - 1) << 4]) + fw.utf8_encode(seq)
    head += bytes([fw.crc8(head)])
    return head + fw.crc16(head).to_bytes(2, "big")


def long_chain(n_frames=(1 << 15) - 8):
    """n_frames 8-byte frames numbered 0 (which always follows): a chain of n_frames nodes that needs every doubling round."""
    return stream([tiny_frame(0)] * n_frames, 192, 192, 2, 16)


def past_window(seed=71):
    """A first frame of about 17 MiB whose CRC-valid end lies past the 16 MiB window, behind a sync word planted at 16.5 MiB (so
    the end search stops there), then ordinary frames.  The first frame is no frame; the rest are found by resync."""
    rng = np.random.default_rng(seed)
    body = bytearray(rng.integers(0, 255, 17 << 20, dtype=np.uint8).tobytes())
    body[(33 << 19) - 100:(33 << 19) - 98] = b"\xff\xf8"
    first = frame(rng, 0, 576, 2, 16, body=bytes(body))
    rest = [frame(rng, k, 576, 2, 16) for k in range(1, 6)]
    return stream([first] + rest, 576, 576, 2, 16)


def within_window(seed=72):
    """The same 17 MiB first frame without the planted sync word: the first sync past the window is the next frame, which the
    search examines, so the big frame is found."""
    rng = np.random.default_rng(seed)
    body = rng.integers(0, 255, 17 << 20, dtype=np.uint8).tobytes()
    return stream([frame(rng, 0, 576, 2, 16, body=body)] + [frame(rng, k, 576, 2, 16) for k in range(1, 4)], 576, 576, 2, 16)


def hundred_thousand(seed=73):
    """One stream of 100 000 small frames (random bodies), for measuring that no file is walked by one thread."""
    rng = np.random.default_rng(seed)
    return stream([frame(rng, k % 0x7FFFFFFF, 576, 2, 16, body=rng.integers(0, 255, 60, dtype=np.uint8).tobytes()) for k in range(100000)],
                  576, 576, 2, 16)


def pack(data, seed):
    """The files in one buffer in a shuffled order, with runs of 1 to 8 bytes of 0xff 0xf8 before each file and after the last, so
    that whatever reads past a file's end meets sync words.  Returns (buffer as a uint8 array, [(offset, len)] in the order of
    `data`)."""
    rng = np.random.default_rng(seed)
    parts, ranges, at = [], [None] * len(data), 0
    for i in rng.permutation(len(data)):
        gap = b"\xff\xf8" * int(rng.integers(1, 5))
        parts += [gap, data[i]]
        ranges[i] = (at + len(gap), len(data[i]))
        at += len(gap) + len(data[i])
    parts.append(b"\xff\xf8" * 4)
    return np.frombuffer(b"".join(parts), dtype=np.uint8).copy(), ranges
