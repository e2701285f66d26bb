"""Host-side packetisers (SURVEY §8f N2): file bytes -> numpy packet tables through the C ABI of libsymgpu.so
(`symgpu_mpa_index`, `symgpu_adts_index`, `symgpu_ogg_index`, `symgpu_vorbis_*`; include/symgpu.h).  No device is
needed and nothing is copied: the tables reference the caller's buffer, which can then go to the GPU in one piece.
The reference interfaces these mirror: `MpaReader` (symphonia-bundle-mp3/src/demuxer.rs:160-218, :414-487),
`AdtsReader` (symphonia-codec-aac/src/adts.rs:278-309), `PageReader` + `LogicalStream`
(symphonia-format-ogg/src/page.rs:166-271, logical.rs:104-205) and the Vorbis mapper (mappings/vorbis.rs:45-405)."""
import ctypes

import numpy as np

from . import _native as nat
from .engine import SymgpuError

_vp = ctypes.c_void_p


def _buf(data):
    a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data, dtype=np.uint8)
    return a, _vp(a.ctypes.data) if a.size else _vp(0)


def _check(rc, what):
    if rc != 0:
        raise SymgpuError(rc, what)


def mpa_index(data, seekable=True):
    """(track record, packets) of an MPEG audio elementary stream.  SymgpuError(status 1) if it holds no frame."""
    L = nat.lib()
    a, p = _buf(data)
    track = np.zeros(1, dtype=nat.MPA_TRACK_DTYPE)
    n = ctypes.c_size_t(0)
    _check(L.symgpu_mpa_index(p, a.size, int(seekable), _vp(track.ctypes.data), None, 0, ctypes.byref(n)), "symgpu_mpa_index")
    packets = np.zeros(n.value, dtype=nat.MPA_PACKET_DTYPE)
    if n.value:
        _check(L.symgpu_mpa_index(p, a.size, int(seekable), _vp(track.ctypes.data), _vp(packets.ctypes.data), n.value, ctypes.byref(n)),
               "symgpu_mpa_index")
    return track[0], packets


def adts_index(data):
    """(packets, stop) with stop = the status the reference's reader ends on: 0 clean end, 3 cut payload, 1 / 2 bad header."""
    L = nat.lib()
    a, p = _buf(data)
    n, stop = ctypes.c_size_t(0), ctypes.c_int(0)
    _check(L.symgpu_adts_index(p, a.size, None, 0, ctypes.byref(n), ctypes.byref(stop)), "symgpu_adts_index")
    packets = np.zeros(n.value, dtype=nat.ADTS_PACKET_DTYPE)
    if n.value:
        _check(L.symgpu_adts_index(p, a.size, _vp(packets.ctypes.data), n.value, ctypes.byref(n), ctypes.byref(stop)), "symgpu_adts_index")
    return packets, stop.value


def ogg_index(data):
    """(packets, pieces): every packet of every announced logical stream as a gather list over `data`."""
    L = nat.lib()
    a, p = _buf(data)
    n, m = ctypes.c_size_t(0), ctypes.c_size_t(0)
    rc = L.symgpu_ogg_index(p, a.size, None, 0, ctypes.byref(n), None, 0, ctypes.byref(m))
    if rc not in (0, 1):
        _check(rc, "symgpu_ogg_index")
    packets, pieces = np.zeros(n.value, dtype=nat.OGG_PACKET_DTYPE), np.zeros(m.value, dtype=nat.PIECE_DTYPE)
    if n.value or m.value:
        L.symgpu_ogg_index(p, a.size, _vp(packets.ctypes.data), n.value, ctypes.byref(n), _vp(pieces.ctypes.data), m.value, ctypes.byref(m))
    return packets, pieces


def gather(data, packet, pieces):
    """The bytes of one Ogg packet (host copy; the device path gathers from the resident file instead)."""
    a, _ = _buf(data)
    pc = pieces[int(packet["first_piece"]):int(packet["first_piece"]) + int(packet["n_pieces"])]
    return b"".join(a[int(o):int(o) + int(n)].tobytes() for o, n in zip(pc["offset"], pc["len"]))


def vorbis_ident(packet):
    a, p = _buf(packet)
    out = np.zeros(1, dtype=nat.VORBIS_IDENT_DTYPE)
    _check(nat.lib().symgpu_vorbis_ident_parse(p, a.size, _vp(out.ctypes.data)), "symgpu_vorbis_ident_parse")
    return out[0]


def vorbis_setup_modes(packet, ident):
    """(number of modes, long-block bit mask) of a setup packet."""
    a, p = _buf(packet)
    idb = np.array([ident], dtype=nat.VORBIS_IDENT_DTYPE)
    n, mask = ctypes.c_uint32(0), ctypes.c_uint64(0)
    _check(nat.lib().symgpu_vorbis_setup_modes(p, a.size, _vp(idb.ctypes.data), ctypes.byref(n), ctypes.byref(mask)), "symgpu_vorbis_setup_modes")
    return n.value, mask.value


def vorbis_packet_durations(ident, n_modes, mask, packets, prev_exp=0, heads=None, lens=None):
    """(dur, discard, prev_exp) for a run of audio packets given as bytes objects -- or as `heads` (first two bytes, little-endian) and
    `lens` (min(length, 2)) arrays."""
    if heads is None:
        heads = np.array([int.from_bytes(bytes(pk[:2]).ljust(2, b"\0"), "little") for pk in packets], dtype=np.uint16)
        lens = np.array([min(len(pk), 2) for pk in packets], dtype=np.uint8)
    else:
        heads, lens = np.ascontiguousarray(heads, dtype=np.uint16), np.ascontiguousarray(lens, dtype=np.uint8)
        packets = heads
    dur, discard = np.zeros(len(packets), dtype=np.uint32), np.zeros(len(packets), dtype=np.uint32)
    idb = np.array([ident], dtype=nat.VORBIS_IDENT_DTYPE)
    prev = np.array([prev_exp], dtype=np.uint8)
    _check(nat.lib().symgpu_vorbis_packet_durations(_vp(idb.ctypes.data), n_modes, mask, _vp(heads.ctypes.data), _vp(lens.ctypes.data), len(packets),
                                                    _vp(prev.ctypes.data), _vp(dur.ctypes.data), _vp(discard.ctypes.data)),
           "symgpu_vorbis_packet_durations")
    return dur, discard, int(prev[0])


def flac_index(data):
    """(stream info record, packets) of a native FLAC file; SymgpuError status 2 without the "fLaC" marker, 1 for bad metadata."""
    L = nat.lib()
    a, p = _buf(data)
    info = np.zeros(1, dtype=nat.FLAC_STREAM_INFO_DTYPE)
    n = ctypes.c_size_t(0)
    _check(L.symgpu_flac_index(p, a.size, _vp(info.ctypes.data), None, 0, ctypes.byref(n)), "symgpu_flac_index")
    packets = np.zeros(n.value, dtype=nat.FLAC_PACKET_DTYPE)
    if n.value:
        _check(L.symgpu_flac_index(p, a.size, _vp(info.ctypes.data), _vp(packets.ctypes.data), n.value, ctypes.byref(n)), "symgpu_flac_index")
    return info[0], packets


def caf_index(data):
    """(info record, packets) of a CAF file holding ALAC: CAF_INFO_DTYPE and CAF_PACKET_DTYPE records.  SymgpuError status 2 for a
    file that is not CAF, not ALAC or not in the packet layout ALAC uses, 1 for a malformed one; its message names the reason."""
    L = nat.lib()
    a, p = _buf(data)
    info = np.zeros(1, dtype=nat.CAF_INFO_DTYPE)
    n = ctypes.c_size_t(0)
    rc = L.symgpu_caf_index(p, a.size, _vp(info.ctypes.data), None, 0, ctypes.byref(n))
    if rc != 0:
        raise SymgpuError(rc, f"symgpu_caf_index: {nat.CAF_REASONS.get(int(info['reason'][0]), 'refused')}")
    packets = np.zeros(n.value, dtype=nat.CAF_PACKET_DTYPE)
    if n.value:
        _check(L.symgpu_caf_index(p, a.size, _vp(info.ctypes.data), _vp(packets.ctypes.data), n.value, ctypes.byref(n)), "symgpu_caf_index")
    return info[0], packets


def vorbis_setup_parse(packet, ident):
    """(info record, floors [n_floors] VORBIS_FLOOR1_DTYPE): the decoder's reading of a setup packet; floors of type 1 are ready for
    Engine.vorbis_floors_set."""
    a, p = _buf(packet)
    idb = np.array([ident], dtype=nat.VORBIS_IDENT_DTYPE)
    info = np.zeros(1, dtype=nat.VORBIS_SETUP_INFO_DTYPE)
    floors = np.zeros(64, dtype=nat.VORBIS_FLOOR1_DTYPE)
    _check(nat.lib().symgpu_vorbis_setup_parse(p, a.size, _vp(idb.ctypes.data), _vp(info.ctypes.data), _vp(floors.ctypes.data)), "symgpu_vorbis_setup_parse")
    return info[0], floors[:int(info[0]["n_floors"])]


def ogg_page_end_trims(page_sequence, page_absgp, dur, discard):
    """End trims of one logical stream's packets against the granule positions of the pages they end on (logical.rs:164-302)."""
    seq = np.ascontiguousarray(page_sequence, dtype=np.uint32)
    gp = np.ascontiguousarray(page_absgp, dtype=np.uint64)
    d, c = np.ascontiguousarray(dur, dtype=np.uint32), np.ascontiguousarray(discard, dtype=np.uint32)
    out = np.zeros(len(seq), dtype=np.uint32)
    _check(nat.lib().symgpu_ogg_page_end_trims(_vp(seq.ctypes.data), _vp(gp.ctypes.data), _vp(d.ctypes.data), _vp(c.ctypes.data), len(seq),
                                               _vp(out.ctypes.data)), "symgpu_ogg_page_end_trims")
    return out


def ogg_gather(data, packets, pieces):
    """(blob, table): the packets copied back to back, table[i] (PIECE_DTYPE) = where packet i lies in `blob`."""
    a, p = _buf(data)
    packets = np.ascontiguousarray(packets, dtype=nat.OGG_PACKET_DTYPE)
    pieces = np.ascontiguousarray(pieces, dtype=nat.PIECE_DTYPE)
    blob = np.zeros(int(packets["len"].sum()), dtype=np.uint8)
    table = np.zeros(len(packets), dtype=nat.PIECE_DTYPE)
    used = ctypes.c_size_t(0)
    _check(nat.lib().symgpu_ogg_gather(p, a.size, _vp(packets.ctypes.data), len(packets), _vp(pieces.ctypes.data), len(pieces),
                                       _vp(blob.ctypes.data) if blob.size else None, blob.size, _vp(table.ctypes.data), ctypes.byref(used)), "symgpu_ogg_gather")
    return blob, table


def ogg_flac_packets(blob, table):
    """(STREAMINFO record, audio, slot) of one gathered logical stream (ogg_gather's blob and table) read as FLAC in Ogg
    (mappings/flac.rs): packet 0 must be the 51-byte identification packet -- SymgpuError status 2 when it is not Ogg FLAC, 1 when
    its STREAMINFO is refused.  audio[k]: packet k carries a frame (first byte 0xff); slot[k]: that frame's block size under the
    decoder's header rules, 0 where the decoder refuses the header (and for every other packet)."""
    a, p = _buf(blob)
    table = np.ascontiguousarray(table, dtype=nat.PIECE_DTYPE)
    info = np.zeros(1, dtype=nat.FLAC_STREAM_INFO_DTYPE)
    audio, slot = np.zeros(len(table), dtype=np.uint8), np.zeros(len(table), dtype=np.uint32)
    _check(nat.lib().symgpu_ogg_flac_packets(p, a.size, _vp(table.ctypes.data) if len(table) else None, len(table), _vp(info.ctypes.data),
                                             _vp(audio.ctypes.data) if len(table) else None, _vp(slot.ctypes.data) if len(table) else None),
           "symgpu_ogg_flac_packets")
    return info[0], audio.astype(bool), slot
