"""Seeded FLAC-in-Ogg files, each with its native twin: a native FLAC file holding the same STREAMINFO and exactly the frames the
FLAC decoder accepts from the Ogg file, in order (what decode_flac_files must give for both).

Decodable frames come from workloads.flac_batch through _flac_bitstream.write_frame, frames with random bodies (refused by the
decoder, but with valid headers and slots) from _flac_corpus.frame.  The corpus covers metadata packets (comment, picture,
padding, types 0x00 / 0x80), frames spanning pages, many frames per page, a lost page, a truncated last page, granule
positions that disagree with the frames, a corrupt CRC-8, a block above STREAMINFO's maximum, identification packets of 50 and
52 bytes, major version 2, a wrong "fLaC", a non-STREAMINFO first block, a refused STREAMINFO, a FLAC stream multiplexed with
another stream in both serial orders, an Ogg file without packets, 1 to 8 channels and 8 to 32 bits per sample."""
import numpy as np

from oracle import flac_frontend_oracle as ffo
from oracle import ogg_flac_oracle
from symphonia_b200 import workloads
from tests import _flac_bitstream as fw
from tests import _flac_corpus
from tests._streams import ogg_page, ogg_paginate


def frames(seed, bps, channels, block, n_frames):
    """Decodable frames in stream order (flac_batch's short blocks, every 7th, left out), numbered from 0."""
    rng = np.random.default_rng(seed)
    fr, subs, samples = workloads.flac_batch(n_frames, block, seed=seed, bps=bps, channels=channels)
    keep = [f for f in range(n_frames) if f % 7]
    return [fw.write_frame(rng, fr[f], subs[int(fr[f]["first_subframe"]):int(fr[f]["first_subframe"]) + channels], samples, k, stream_bps=bps)
            for k, f in enumerate(keep)]


def info_block(block, channels, bps, **kw):
    return fw.stream_info_block(kw.get("block_min", block), kw.get("block_max", block), 44100, channels, bps, 0)


def ident(info, major=1, marker=b"fLaC", block_type=0, block_len=34, extra=b""):
    """The identification packet: 0x7f "FLAC", version, header count, "fLaC", the STREAMINFO block header and the block."""
    return b"\x7fFLAC" + bytes([major, 0]) + (1).to_bytes(2, "big") + marker + bytes([block_type]) + block_len.to_bytes(3, "big") + info + extra


def metadata(kind, body, last=False):
    return bytes([(0x80 if last else 0) | kind]) + len(body).to_bytes(3, "big") + body


def comment():
    vendor = b"reference libFLAC 1.4.3"
    tags = [b"TITLE=ogg flac", b"ARTIST=corpus"]
    body = len(vendor).to_bytes(4, "little") + vendor + len(tags).to_bytes(4, "little") + b"".join(len(t).to_bytes(4, "little") + t for t in tags)
    return metadata(4, body)


def picture():
    mime, desc, data = b"image/png", b"cover", bytes(range(40))
    body = (3).to_bytes(4, "big") + len(mime).to_bytes(4, "big") + mime + len(desc).to_bytes(4, "big") + desc
    body += (1).to_bytes(4, "big") + (1).to_bytes(4, "big") + (24).to_bytes(4, "big") + (0).to_bytes(4, "big") + len(data).to_bytes(4, "big") + data
    return metadata(6, body)


def ogg(packets, seed, serial=0x0F1AC, **kw):
    return b"".join(ogg_paginate(serial, packets, np.random.default_rng(seed), **kw))


def twin(data):
    """The native FLAC file of the frames the decoder accepts from `data` (by the oracle), or None when the file fails."""
    got = ogg_flac_oracle.read(data)
    if got["status"] != "ok":
        return None
    i = got["info"]
    accepted = []
    for p, _ in got["audio"]:
        try:
            ffo.decode_packet(p, i["bits_per_sample"], i["channels"], i["block_max"])
            accepted.append(p)
        except Exception:  # noqa: BLE001 -- refused by the decoder: not in the twin
            pass
    block = fw.stream_info_block(i["block_min"], i["block_max"], i["sample_rate"], i["channels"], i["bits_per_sample"], i["n_samples"],
                                 i["frame_min"], i["frame_max"], i["md5"])
    return fw.native_file(accepted, block)


def files(seed=90):
    """[(name, ogg bytes, twin bytes or None)]."""
    rng = np.random.default_rng(seed)
    out = []

    def add(name, data):
        out.append((name, data, twin(data)))
    base = frames(seed, 16, 2, 576, 12)
    head = ident(info_block(576, 2, 16))
    add("plain stereo", ogg([head, comment()] + base, 1))
    add("metadata packets", ogg([head, comment(), picture(), metadata(1, bytes(100)), b"\x00\x01\x02", b"\x80" + bytes(10)] + base, 2))
    add("frames spanning pages", ogg([head] + base, 3, max_segments=2))
    add("many frames per page", ogg([ident(info_block(64, 1, 8))] + frames(seed + 1, 8, 1, 64, 40), 4, max_segments=255))
    pages = ogg_paginate(7, [head] + base, np.random.default_rng(5), max_segments=3)
    add("lost page", b"".join(pages[:4] + pages[5:]))
    whole = ogg([head] + base, 6, max_segments=6)
    add("truncated last page", whole[:len(whole) - 40])
    add("granule positions off", ogg([head] + base, 7, granule_of=[int(v) for v in rng.integers(0, 1 << 40, len(base) + 1)]))
    bad = bytearray(base[3])
    bad[ffo.read_frame_header(bytes(bad), 0)[1] - 1] ^= 0x55   # the header's CRC-8
    add("corrupt CRC-8", ogg([head] + base[:3] + [bytes(bad)] + base[4:], 8))
    big = frames(seed + 2, 16, 2, 1152, 3)[0]
    add("block above STREAMINFO maximum", ogg([head] + base[:2] + [big] + base[2:], 9))
    junk = [_flac_corpus.frame(rng, k, 576, 2, 16) for k in range(4)]
    add("frames the decoder refuses", ogg([head] + junk + base[:3], 10))
    info = info_block(576, 2, 16)
    add("identification packet of 50 bytes", ogg([head[:50]] + base, 11))
    add("identification packet of 52 bytes", ogg([head + b"\x00"] + base, 12))
    add("major version 2", ogg([ident(info, major=2)] + base, 13))
    add("wrong fLaC", ogg([ident(info, marker=b"fLaX")] + base, 14))
    add("first block not STREAMINFO", ogg([ident(info, block_type=4)] + base, 15))
    add("STREAMINFO refused", ogg([ident(info_block(576, 2, 16, block_min=8))] + base, 16))
    other = ogg_paginate(0x20, [b"\x01vorbis" + bytes(23), b"\x03vorbis" + bytes(8)], np.random.default_rng(17))
    mine = ogg_paginate(0x10, [head] + base, np.random.default_rng(18))
    mixed = [p for pair in zip(other + [b""] * len(mine), mine) for p in pair]
    add("FLAC with a second stream of higher serial", b"".join(mixed))
    mine = ogg_paginate(0x30, [head] + base, np.random.default_rng(19))
    mixed = [p for pair in zip(mine, other + [b""] * len(mine)) for p in pair]
    add("FLAC with a second stream of lower serial", b"".join(mixed))
    add("no packets", ogg_page(0x10, 0, 0, [255], bytes(255), first=True))
    for k, (bps, ch, block) in enumerate([(8, 1, 192), (12, 3, 256), (20, 4, 300), (24, 5, 128), (32, 1, 256), (16, 6, 64), (24, 7, 64), (16, 8, 64)]):
        add(f"{bps} bits {ch} channels", ogg([ident(info_block(block, ch, bps))] + frames(seed + 10 + k, bps, ch, block, 9), 20 + k))
    return out


def long_file(n_frames=2000, seed=95):
    """One long file: n_frames stereo frames of 576 samples."""
    base = frames(seed, 16, 2, 576, n_frames + n_frames // 6 + 2)[:n_frames]
    data = ogg([ident(info_block(576, 2, 16)), comment()] + base, seed)
    return data, twin(data)
