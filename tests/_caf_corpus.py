"""Seeded CAF files holding ALAC packets of tests/_alac_bitstream.py, with what the index must find in each.

corpus() -> [(name, file bytes, expect)]: expect is None for a file that must not open, else dict(cookie, packets (the packet
bytes the index must find, in order), pcm (the frames those packets decode to, or None when some are refused)).
"""
import struct

import numpy as np

from tests import _alac_bitstream as ab
from tests import _alac_cases as cases


def varint(v):
    out = [v & 0x7F]
    v >>= 7
    while v:
        out.append(0x80 | (v & 0x7F))
        v >>= 7
    return bytes(reversed(out))


def chunk(tag, body, size=None):
    return tag + struct.pack(">q", len(body) if size is None else size) + body


def desc(ck, rate=44100.0, fmt=b"alac", fpp=None, bpp=0, channels=None):
    return chunk(b"desc", struct.pack(">d", rate) + fmt + struct.pack(">IIIII", 1, bpp, ck["frame_length"] if fpp is None else fpp,
                                                                       ck["channels"] if channels is None else channels, ck["bit_depth"]))


def pakt(sizes, ck, priming=0, remainder=0):
    return chunk(b"pakt", struct.pack(">qqii", len(sizes), len(sizes) * ck["frame_length"] - priming - remainder, priming, remainder)
                 + b"".join(varint(s) for s in sizes))


def caf(chunks):
    return b"caff" + struct.pack(">HH", 1, 0) + b"".join(chunks)


def stream(rng, ck, n_packets, last=None):
    """(packets, pcm) of a stream: full packets and a shorter last one."""
    pk, pcm = [], []
    for k in range(n_packets):
        n = ck["frame_length"] if k + 1 < n_packets else (last or ck["frame_length"])
        x = ab.signal(rng, n, ck["channels"], ck["bit_depth"])
        pk.append(ab.encode_packet(x, ck))
        pcm.append(x)
    return pk, np.concatenate(pcm)


def corpus(seed=5):
    rng = np.random.default_rng(seed)
    out = []
    ck2 = cases.cookie(channels=2, frame_length=256)
    for wrap in (None, "alac", "frma"):
        for layout in (False, True):
            pk, pcm = stream(rng, ck2, 5, last=100)
            body = caf([desc(ck2), chunk(b"kuki", ab.cookie_bytes(ck2, layout=layout, wrap=wrap)), pakt([len(p) for p in pk], ck2),
                        chunk(b"data", bytes(4) + b"".join(pk))])
            out.append((f"cookie_{wrap}_{'layout' if layout else 'bare'}", body, dict(cookie=ck2, packets=pk, pcm=pcm)))
    for ch in range(1, 9):
        ck = cases.cookie(channels=ch, frame_length=128, bit_depth=16 if ch % 2 else 24)
        pk, pcm = stream(rng, ck, 3, last=70)
        body = caf([desc(ck), chunk(b"chan", struct.pack(">III", 0, 0, 1) + bytes(20)), chunk(b"kuki", ab.cookie_bytes(ck, layout=ch > 2)),
                    chunk(b"data", bytes(4) + b"".join(pk)), pakt([len(p) for p in pk], ck, priming=10, remainder=5)])
        out.append((f"channels{ch}_chan_pakt_after_data", body, dict(cookie=ck, packets=pk, pcm=pcm)))
    ck = cases.cookie(channels=2, frame_length=4096)
    pk, pcm = stream(rng, ck, 2, last=3000)  # packets of more than 127 bytes: multi-byte integers
    body = caf([desc(ck), chunk(b"free", bytes(9)), chunk(b"kuki", ab.cookie_bytes(ck)), chunk(b"XYZW", b"junk"), pakt([len(p) for p in pk], ck),
                chunk(b"data", bytes(4) + b"".join(pk)), chunk(b"info", bytes(3))])
    out.append(("unknown_chunks_multibyte", body, dict(cookie=ck, packets=pk, pcm=pcm)))
    pk, pcm = stream(rng, ck2, 4)
    body = caf([desc(ck2), chunk(b"kuki", ab.cookie_bytes(ck2)), pakt([len(p) for p in pk], ck2), chunk(b"data", bytes(4) + b"".join(pk)[:-3])])
    out.append(("cut_last_packet", body, dict(cookie=ck2, packets=pk[:3], pcm=pcm[:3 * 256])))
    out.append(("data_size_minus_one_empty", caf([desc(ck2), chunk(b"kuki", ab.cookie_bytes(ck2)), pakt([len(p) for p in pk], ck2),
                                                   chunk(b"data", bytes(4), size=-1)]), dict(cookie=ck2, packets=[], pcm=pcm[:0])))
    out.append(("data_size_minus_one", caf([desc(ck2), chunk(b"kuki", ab.cookie_bytes(ck2)), pakt([len(p) for p in pk], ck2),
                                             chunk(b"data", bytes(4) + b"".join(pk), size=-1)]), None))
    out.append(("not_alac", caf([desc(ck2, fmt=b"lpcm"), chunk(b"data", bytes(8))]), None))
    out.append(("no_cookie", caf([desc(ck2), pakt([len(p) for p in pk], ck2), chunk(b"data", bytes(4) + b"".join(pk))]), None))
    out.append(("bad_cookie_version", caf([desc(ck2), chunk(b"kuki", ab.cookie_bytes(ck2)[:4] + b"\x01" + ab.cookie_bytes(ck2)[5:]),
                                            chunk(b"data", bytes(4))]), None))
    out.append(("frame_length_too_large", caf([desc(ck2), chunk(b"kuki", ab.cookie_bytes(dict(ck2, frame_length=65537))), chunk(b"data", bytes(4))]), None))
    out.append(("pakt_first", caf([pakt([1], ck2), desc(ck2)]), None))
    out.append(("unterminated_integer", caf([desc(ck2), chunk(b"kuki", ab.cookie_bytes(ck2)), chunk(b"pakt", struct.pack(">qqii", 1, 0, 0, 0) + b"\xff" * 10)]), None))
    out.append(("junk", rng.integers(0, 256, size=3000, dtype=np.uint8).tobytes(), None))
    out.append(("empty", b"", None))
    return out
