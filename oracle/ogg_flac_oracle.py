"""FLAC-in-Ogg oracle: symphonia-format-ogg/src/mappings/flac.rs restated in Python on top of the Ogg oracle
(packetizer_oracle.ogg_index / OggLogical), with every audio packet's frame read by flac_frontend_oracle.decode_packet.
TEST INFRASTRUCTURE ONLY.

  detect()           flac.rs:43-125   the 51-byte identification packet; StreamInfo::read (symphonia-common/src/xiph/audio/flac/
                                      mod.rs) on its STREAMINFO block
  map_packet()       flac.rs:299-345  0xff: audio; 0x00 / 0x80: unknown; anything else: a metadata block (no audio)
  the decoder        symphonia-bundle-flac/src/decoder.rs:93-228: STREAMINFO as extra data, every audio packet decoded, no trim

The stream chosen is the one symgpu_ogg_index lists first: its packets are grouped by serial, in ascending order, so that is
the smallest serial whose logical stream holds a packet."""
from oracle import flac_frontend_oracle as ffo
from oracle import packetizer_oracle as po
from oracle.mp3_frontend_oracle import DecodeError

IDENT_LEN = 51


def read_stream_info(b):
    """StreamInfo::read on 34 bytes: dict, or raises DecodeError."""
    block_min, block_max = int.from_bytes(b[0:2], "big"), int.from_bytes(b[2:4], "big")
    if block_min < 16 or block_max < 16:
        raise DecodeError("minimum block length is 16 samples")
    if block_max < block_min:
        raise DecodeError("maximum block length is less than the minimum")
    frame_min, frame_max = int.from_bytes(b[4:7], "big"), int.from_bytes(b[7:10], "big")
    if frame_min and frame_max and frame_max < frame_min:
        raise DecodeError("maximum frame length is less than the minimum")
    bits = int.from_bytes(b[10:18], "big")
    rate = bits >> 44
    if rate < 1 or rate > 655350:
        raise DecodeError("sample rate out of bounds")
    channels, bps = ((bits >> 41) & 7) + 1, ((bits >> 36) & 31) + 1
    if bps < 4:
        raise DecodeError("bits per sample out of bounds")
    return dict(block_min=block_min, block_max=block_max, frame_min=frame_min, frame_max=frame_max, sample_rate=rate, channels=channels,
                bits_per_sample=bps, n_samples=bits & ((1 << 36) - 1), md5=bytes(b[18:34]))


def detect(packet):
    """flac.rs:43-125: None when the packet does not make the stream Ogg FLAC, else its STREAMINFO (DecodeError when that is
    refused)."""
    p = bytes(packet)
    if len(p) != IDENT_LEN or p[0] != 0x7F or p[1:5] != b"FLAC" or p[5] != 1 or p[9:13] != b"fLaC":
        return None
    if p[13] & 0x7F != 0 or int.from_bytes(p[14:17], "big") != 34:
        return None
    return read_stream_info(p[17:51])


def map_packet(packet):
    """flac.rs:299-345: 'audio' (first byte 0xff), 'unknown' (0x00 / 0x80) or 'metadata'; an empty packet is 'error'."""
    if not len(packet):
        return "error"
    if packet[0] == 0xFF:
        return "audio"
    return "unknown" if packet[0] in (0x00, 0x80) else "metadata"


def slot(packet):
    """The block size of the frame the decoder reads from the packet (its first sync code, then the header), 0 when it refuses
    the header."""
    at = 0
    while True:
        if at + 2 > len(packet):
            return 0
        if packet[at] == 0xFF and (packet[at + 1] & 0xFC) == 0xF8:
            break
        at += 1
    try:
        h, _ = ffo.read_frame_header(packet, at)
    except DecodeError:
        return 0
    return h["block"]


def chosen_stream(data):
    """[packet bytes] of the logical stream the readers choose, or None when the file has no packet."""
    _, streams = po.ogg_index(data)
    serials = sorted(s for s, pk in streams.items() if pk)
    if not serials:
        return None
    return [b"".join(bytes(data[a:a + n]) for a, n in pieces) for pieces, _, _, _ in streams[serials[0]]]


def read(data):
    """dict(status: 'ok' | 'no packets' | 'not flac' | 'bad streaminfo', info, audio: [(packet bytes, slot)], decoded: [(header,
    sub-frames) of every packet the decoder accepts, in order])."""
    packets = chosen_stream(data)
    if packets is None:
        return dict(status="no packets", info=None, audio=[], decoded=[])
    try:
        info = detect(packets[0])
    except DecodeError:
        return dict(status="bad streaminfo", info=None, audio=[], decoded=[])
    if info is None:
        return dict(status="not flac", info=None, audio=[], decoded=[])
    audio = [(p, slot(p)) for p in packets[1:] if map_packet(p) == "audio"]
    decoded = []
    for p, _ in audio:
        try:
            decoded.append(ffo.decode_packet(p, info["bits_per_sample"], info["channels"], info["block_max"]))
        except (DecodeError, ffo.Unsupported):
            pass
    return dict(status="ok", info=info, audio=audio, decoded=decoded)
