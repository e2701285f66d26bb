"""Ogg Vorbis streams for the device decoder's tests, on the writer of tests/_vorbis_bitstream.py: residue types 0, 1 and 2; mono,
coupled and uncoupled stereo; class words of 2-3 partitions with short blocks after long ones (a class word that spills into the
next channel's entries); residues that begin beyond the short block; block sizes up to 8192; and damaged packets -- truncations at
every byte, bit flips, empty and one-byte packets, mode numbers beyond the mode list, packets refused before their window flags
(a mode list of 40 entries) and packets refused mid-residue by a pass that names a codebook without VQ values.  The writer's
random codebooks are not libvorbis output."""
import inspect
import sys

import numpy as np

from tests import _streams as st
from tests import _vorbis_bitstream as vb


def writer(seed, n, **kw):
    """(stream, packets): `n` writer packets of a stream made with vb.Stream(**kw)."""
    s = vb.Stream(np.random.default_rng(seed), **kw)
    return s, [s.packet()[0] for _ in range(n)]


def _mode_beyond(s):
    """A packet whose mode number is beyond the mode list, or None when the list's bit width cannot name one."""
    n = len(s.modes)
    bits = vb._ilog(n - 1)
    v = (1 << bits) - 1
    if v < n:
        return None
    return bytes([(v << 1) & 0xff, 0x5a, 0xa5])


class _Recording(st.BitWriterRtl):
    """The writer's bit writer, logging (line, bit offset, width, value) of every put vb.Stream.__init__ makes."""
    log = None

    def put(self, value, width):
        f = sys._getframe(1)
        if _Recording.log is not None and f.f_code is vb.Stream.__init__.__code__:
            _Recording.log.append((f.f_lineno, self.n, width, value))
        super().put(value, width)


def _recorded(seed, **kw):
    """(stream, log): a writer stream and where its setup header's fields lie (bit offsets after the 7-byte packet header)."""
    _Recording.log, old = [], vb.BitWriterRtl
    vb.BitWriterRtl = _Recording
    try:
        s = vb.Stream(np.random.default_rng(seed), **kw)
    finally:
        vb.BitWriterRtl = old
    log, _Recording.log = _Recording.log, None
    return s, log


def _line(text):
    src, first = inspect.getsourcelines(vb.Stream.__init__)
    return first + next(i for i, line in enumerate(src) if text in line)


def non_vq(seed=1200, n=14, pick=2):
    """(stream, packets): a stereo stream whose setup names floor book 1 -- scalar, without VQ values -- for one pass >= 1 of a
    residue class (the `pick`-th such entry).  The packets are written for the unpatched setup; those that reach that class in that pass have read their
    class words and earlier passes, and are refused there (residue.rs: "not a vq codebook")."""
    s, log = _recorded(seed, channels=2, bs_exp=(7, 10), per_word=2, residue_type=1)
    fields = [at for line, at, _, _ in log if line == _line("w.put(vbooks[ci][j], 8)")]
    k, later = 0, []
    for r in s.residues:
        for u in r["used"]:
            for j in range(8):
                if u >> j & 1:
                    if j >= 1:
                        later.append(fields[k])
                    k += 1
    assert k == len(fields)
    target = later[pick]
    pk = [s.packet()[0] for _ in range(n)]
    v = (int.from_bytes(s.setup[7:], "little") & ~(0xff << target)) | (1 << target)   # book 1 (the reader refuses index 0 here)
    s.setup = s.setup[:7] + v.to_bytes(len(s.setup) - 7, "little")
    return s, pk


def many_modes(seed=1210, n=8, n_modes=40):
    """(stream, packets): a stereo stream whose setup has `n_modes` modes (6 mode bits), alternately long and short.  After its
    writer packets come one-byte packets of long modes, which end after the first window flag, and of short modes."""
    s, log = _recorded(seed, channels=2, bs_exp=(7, 10))
    at = next(a for line, a, _, _ in log if line == _line("w.put(n_modes - 1, 6)"))
    w = st.BitWriterRtl()
    w.v, w.n = int.from_bytes(s.setup[7:], "little") & ((1 << at) - 1), at
    modes = [(k % 2 == 0, k % len(s.mappings)) for k in range(n_modes)]
    w.put(n_modes - 1, 6)
    for flag, mp in modes:
        w.put(int(flag), 1), w.put(0, 16), w.put(0, 16), w.put(mp, 8)
    w.put(1, 1)
    s.setup, s.modes = b"\x05vorbis" + w.bytes(), modes
    pk = [s.packet()[0] for _ in range(n)]
    return s, pk[:4] + [bytes([(m << 1) & 0xff]) for m in (0, 2, 1, 38, 3)] + pk[4:]


def damaged(seed, n, **kw):
    """Writer packets with every byte-length truncation of two packets, bit flips, and refused packets in between."""
    s, pk = writer(seed, n, **kw)
    rng = np.random.default_rng(seed + 1)
    out = []
    for k, p in enumerate(pk):
        out.append(p)
        if k in (2, 5):
            out += [p[:m] for m in range(1, len(p))]
        if k % 3 == 1:
            b = bytearray(p)
            for _ in range(2):
                i = int(rng.integers(1, len(b) * 8))   # (bit 0 stays clear: the packet stays an audio packet)
                b[i // 8] ^= 1 << (i % 8)
            out.append(bytes(b))
    # an empty packet, a one-byte packet, and a mode number beyond the mode list
    out += [b"", bytes([0])]
    beyond = _mode_beyond(s)
    if beyond is not None:
        out.append(beyond)
    return s, out


def streams():
    """[(name, stream, packets)] -- the logical streams of the corpus."""
    out = []
    for rtype in (0, 1, 2):
        for ch, coupled in ((1, None), (2, True), (2, False)):
            s, pk = writer(900 + 10 * rtype + ch + (coupled is True), 10, channels=ch, bs_exp=(7, 10), residue_type=rtype, coupled=coupled,
                           per_word=2 + rtype % 2)
            out.append((f"type{rtype}-{ch}ch-{'coupled' if coupled else 'plain'}", s, pk))
    s, pk = writer(950, 12, channels=2, bs_exp=(6, 9), per_word=3, residue_begin=48)   # residue begins beyond the short block (32)
    out.append(("begin-beyond-short", s, pk))
    s, pk = writer(951, 8, channels=2, bs_exp=(8, 13))                                  # 8192-sample long blocks
    out.append(("long-8192", s, pk))
    s, pk = damaged(960, 9, channels=2, bs_exp=(7, 10), per_word=2)
    out.append(("damaged-stereo", s, pk))
    s, pk = damaged(961, 9, channels=1, bs_exp=(7, 9), per_word=3)
    out.append(("damaged-mono", s, pk))
    out.append(("non-vq-pass", *non_vq()))
    out.append(("forty-modes", *many_modes()))
    for seed in range(970, 1000):   # a stream whose mode list has 3 entries: a mode number of 3 is beyond it
        s, pk = writer(seed, 4, channels=2, bs_exp=(7, 9))
        if _mode_beyond(s) is not None:
            out.append(("mode-beyond", s, pk[:2] + [_mode_beyond(s)] + pk[2:]))
            break
    return out


def ogg(s, packets, seed, serial=77, pad=37):
    """The packets as an Ogg Vorbis file: header pages, then audio pages whose granule positions follow the writer's block sizes
    (the last one `pad` frames short of the end, so the page end trim cuts the last packet)."""
    rng = np.random.default_rng(seed)
    bs0, bs1 = 1 << s.bs_exp[0], 1 << s.bs_exp[1]
    flags = []
    for p in packets:   # the block flag the packet's mode names, where it names one
        n = len(s.modes)
        b = vb._ilog(n - 1)
        m = (int.from_bytes(p[:4].ljust(4, b"\0"), "little") >> 1) & ((1 << b) - 1)
        flags.append(bool(s.modes[m][0]) if m < n else False)
    g, gran, prev = 0, [], None
    for f in flags:
        if prev is not None:
            g += ((bs1 if prev else bs0) + (bs1 if f else bs0)) // 4
        gran.append(g)
        prev = f
    gran[-1] = max(gran[-1] - pad, gran[-2] if len(gran) > 1 else 0)
    headers = [s.ident, b"\x03vorbis" + bytes(20), s.setup]
    pages = st.ogg_paginate(serial, headers[:1], rng, eos=False) + st.ogg_paginate(serial, headers[1:], rng, first_sequence=1, bos=False, eos=False)
    pages += st.ogg_paginate(serial, packets, rng, max_segments=int(rng.integers(3, 40)), first_sequence=len(pages), bos=False, granule_of=gran)
    return b"".join(pages)


def files():
    """[(name, ogg bytes)]: every corpus stream as a file (without its empty packets, which the reader skips); two files that
    share one stream's headers; and a file cut mid-page."""
    out = []
    for k, (name, s, pk) in enumerate(streams()):
        out.append((name, ogg(s, [p for p in pk if p], 1000 + k)))
    s, pk = writer(990, 14, channels=2, bs_exp=(8, 11))
    out.append(("shared-a", ogg(s, pk[:7], 1100)))
    out.append(("shared-b", ogg(s, pk[7:], 1101)))
    whole = ogg(*writer(991, 16, channels=2, bs_exp=(8, 11)), 1102)
    out.append(("cut-mid-page", whole[:len(whole) * 2 // 3]))
    return out
