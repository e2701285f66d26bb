"""ORACLE (test infrastructure, NOT product code): a Python restatement of how the reference opens a CAF file holding ALAC and which
packets it reads, for comparison with the host and device CAF indexes.

  CafReader::check_file_header, read_chunks          symphonia-format-caf/src/demuxer.rs:362-560
  Chunk::read, AudioDescription::read, AudioData::read, ChannelLayout::read, PacketTable::read, read_variable_length_integer
                                                      chunks.rs:82-614
  MagicCookie::read                                   symphonia-common/src/apple/audio/alac.rs:34-171
  AlacDecoder::try_new's frame-length limit           symphonia-codec-alac/src/lib.rs:295-300
  next_packet for variable packets                    demuxer.rs:148-160

open_caf(data) -> (status, reason, fields or None, packets [(offset, size)]): status 0 ok, 1 a decode error (IoError included),
2 unsupported; reason one of the SYMGPU_CAF_* codes.  Only ALAC with variable bytes and constant frames per packet opens.
"""
import struct

OK, DECODE, UNSUPPORTED = 0, 1, 2
TRUNCATED, NOT_CAF, VERSION, BAD_CHUNK, NO_DESC, BAD_DESC, NOT_ALAC, LAYOUT, BAD_TABLE, NO_COOKIE, BAD_COOKIE = range(1, 12)
KNOWN_FORMATS = {b"lpcm", b"ima4", b"aac ", b"MAC3", b"MAC6", b"ulaw", b"alaw", b".mp1", b".mp2", b".mp3", b"alac", b"flac", b"opus"}
LAYOUT_TAGS = {1: 100, 2: 101, 3: 113, 4: 116, 5: 120, 6: 124, 7: 142, 8: 127}


class _Fail(Exception):
    def __init__(self, status, reason):
        super().__init__(reason)
        self.status, self.reason = status, reason


def _varint(d, at):
    v = 0
    for _ in range(9):
        if at >= len(d):
            raise _Fail(DECODE, TRUNCATED)
        b = d[at]
        at += 1
        v |= b & 0x7F
        if not b & 0x80:
            return v, at
        v <<= 7
    raise _Fail(DECODE, BAD_TABLE)


def _cookie(c):
    if len(c) < 24:
        raise _Fail(UNSUPPORTED, BAD_COOKIE)
    if c[4:8] == b"frma":
        c = c[12:]
    if c[4:8] == b"alac":
        c = c[12:]
    if len(c) not in (24, 48):
        raise _Fail(UNSUPPORTED, BAD_COOKIE)
    fl, ver, bd, pb, mb, kb, ch, max_run, mfb, abr, rate = struct.unpack(">IBBBBBBHIII", c[:24])
    if ver > 0:
        raise _Fail(UNSUPPORTED, BAD_COOKIE)
    if bd > 32 or not 1 <= ch <= 8:
        raise _Fail(DECODE, BAD_COOKIE)
    if len(c) == 48:
        size, tag4, version, tag, r0, r1 = struct.unpack(">I4sIIII", c[24:48])
        if size != 24 or tag4 != b"chan" or version != 0:
            raise _Fail(DECODE, BAD_COOKIE)
        count = tag & 0xFFFF
        if count not in LAYOUT_TAGS or tag >> 16 != LAYOUT_TAGS[count] or count != ch or r0 or r1:
            raise _Fail(DECODE, BAD_COOKIE)
    if fl > 65536:
        raise _Fail(UNSUPPORTED, BAD_COOKIE)
    return dict(frame_length=fl, compatible_version=ver, bit_depth=bd, pb=pb, mb=mb, kb=kb, channels=ch, max_run=max_run,
                max_frame_bytes=mfb, avg_bit_rate=abr, sample_rate=rate)


def _walk(d):
    n = len(d)
    if n < 4:
        raise _Fail(DECODE, TRUNCATED)
    if d[:4] != b"caff":
        raise _Fail(UNSUPPORTED, NOT_CAF)
    if n < 8:
        raise _Fail(DECODE, TRUNCATED)
    if struct.unpack(">H", d[4:6])[0] != 1:
        raise _Fail(UNSUPPORTED, VERSION)
    at, desc, cookie, table, data_start = 8, None, None, None, None
    while True:
        if n - at < 12:
            raise _Fail(DECODE, TRUNCATED)
        tag, size = d[at:at + 4], struct.unpack(">q", d[at + 4:at + 12])[0]
        body = at + 12
        left = n - body
        if tag == b"desc":
            if size != 32:
                raise _Fail(DECODE, BAD_CHUNK)
            if left < 32:
                raise _Fail(DECODE, TRUNCATED)
            rate, fmt, _flags, bpp, fpp, ch, _bits = struct.unpack(">d4sIIIII", d[body:body + 32])
            if rate == 0.0:
                raise _Fail(DECODE, BAD_DESC)
            if fmt not in KNOWN_FORMATS:
                raise _Fail(UNSUPPORTED, NOT_ALAC)
            if ch == 0:
                raise _Fail(DECODE, BAD_DESC)
            if fmt != b"alac":
                raise _Fail(UNSUPPORTED, NOT_ALAC)
            if desc is not None:
                raise _Fail(DECODE, BAD_CHUNK)
            if ch > 26:
                raise _Fail(UNSUPPORTED, BAD_DESC)
            if bpp != 0 or fpp == 0:
                raise _Fail(UNSUPPORTED, LAYOUT)
            desc = fpp
            at = body + 32
        elif tag == b"data":
            if size != -1 and size < 4:
                raise _Fail(DECODE, BAD_CHUNK)
            if left < 4:
                raise _Fail(DECODE, TRUNCATED)
            if size == -1:
                data_start, at = None, body + 4
            else:
                if size - 4 > n - body - 4:
                    raise _Fail(DECODE, TRUNCATED)
                data_start, at = body + 4, body + 4 + size - 4
        elif tag == b"chan":
            if size < 12:
                raise _Fail(DECODE, BAD_CHUNK)
            if left < 12 or struct.unpack(">I", d[body + 8:body + 12])[0] * 20 > left - 12:
                raise _Fail(DECODE, TRUNCATED)
            at = body + 12 + struct.unpack(">I", d[body + 8:body + 12])[0] * 20
        elif tag == b"pakt":
            if size < 24:
                raise _Fail(DECODE, BAD_CHUNK)
            if desc is None:
                raise _Fail(DECODE, NO_DESC)
            if left < 24:
                raise _Fail(DECODE, TRUNCATED)
            total, valid, priming, remainder = struct.unpack(">qqii", d[body:body + 24])
            if total < 0 or valid < 0:
                raise _Fail(DECODE, BAD_TABLE)
            at, sizes = body + 24, []
            for _ in range(total):
                v, at = _varint(d, at)
                sizes.append(v)
            table = dict(sizes=sizes, valid_frames=valid, priming_frames=priming, remainder_frames=remainder, table_at=body + 24,
                         table_bytes=at - body - 24, table_packets=total)
        else:
            if size < 0:
                raise _Fail(DECODE, BAD_CHUNK)
            if size > left:
                raise _Fail(DECODE, TRUNCATED)
            if tag == b"kuki":
                cookie = d[body:body + size]
            at = body + size
        if desc is None:
            raise _Fail(DECODE, NO_DESC)
        if at == n:
            break
    if cookie is None:
        raise _Fail(UNSUPPORTED, NO_COOKIE)
    fields = _cookie(cookie)
    fields.update(frames_per_packet=desc, data_start=n if data_start is None else data_start)
    if table is None:
        table = dict(sizes=[], valid_frames=0, priming_frames=0, remainder_frames=0, table_at=0, table_bytes=0, table_packets=0)
    fields.update({k: v for k, v in table.items() if k != "sizes"})
    packets, offset = [], 0
    for s in table["sizes"]:
        start = fields["data_start"] + offset
        if s > 0xFFFFFFFF or start + s > n:
            break
        packets.append((start, s))
        offset += s
    fields["n_packets"] = len(packets)
    return fields, packets


def open_caf(data):
    try:
        fields, packets = _walk(bytes(data))
    except _Fail as f:
        return f.status, f.reason, None, []
    return OK, 0, fields, packets
