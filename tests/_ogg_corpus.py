"""Ogg files for the device page index and its CPU restatement: the streams tests/test_packetizer.py indexes, rebuilt from
tests/_streams.py (lacing edges 0 / 254 / 255 / 256 / 510 / 65 025 bytes and packets longer than a page; multiplexed serials
with junk, false capture patterns and an unannounced serial; lost, swapped, repeated and corrupted pages, refused headers;
truncations), single-bit hits on a clean stream, the Vorbis corpus and a few degenerate files."""
import numpy as np

from tests import _streams as st
from tests import _vorbis_corpus


def _packets(rng, n, sizes):
    return [rng.integers(0, 256, int(sizes[int(rng.integers(len(sizes)))]), dtype=np.uint8).tobytes() for _ in range(n)]


def many_serials(n, seed):
    """n minimal pages, each announcing its own serial (shuffled), every fourth followed by a page that continues it, a few of
    them before their announcement (orphans): the worst case for a walk that visits the file once per logical stream."""
    rng = np.random.default_rng(seed)
    serials = rng.permutation(np.arange(n, dtype=np.uint64) * 2654435761 % 2**32)
    pages = []
    for k, s in enumerate(serials):
        if k % 97 == 5:
            pages.append(st.ogg_page(int(s), 9, 0, [3], b"abc"))   # before its first page: an orphan
        pages.append(st.ogg_page(int(s), 0, 0, [255], bytes(255), first=True) if k % 4 == 0 else st.ogg_page(int(s), 0, 0, [1], b"x", first=True))
        if k % 4 == 0:
            pages.append(st.ogg_page(int(s), 1, 64, [2], b"yz", continuation=True))
    return b"".join(pages)


def files():
    """[(name, bytes)]."""
    out = []
    rng = np.random.default_rng(31)
    sizes = [0, 1, 30, 254, 255, 256, 509, 510, 511, 4000, 65025, 70000, 140000]
    for trial in range(6):
        pages = st.ogg_paginate(0x1234ABCD, _packets(rng, 40, sizes), rng, max_segments=[255, 255, 40, 7, 3, 1][trial])
        out.append((f"lacing-{trial}", b"".join(pages)))
    rng = np.random.default_rng(32)
    a = st.ogg_paginate(7, _packets(rng, 60, [20, 300, 900, 3000]), rng, max_segments=20)
    b = st.ogg_paginate(0xFFFFFFFE, _packets(rng, 50, [100, 255, 5000]), rng, max_segments=30)
    c = st.ogg_paginate(9, _packets(rng, 10, [50]), rng, max_segments=4, bos=False)
    pools = {"a": a, "b": b, "c": c}
    for hostile in (False, True):
        idx = {"a": 1, "b": 1, "c": 0}
        mux = [a[0], b[0]]
        while any(idx[k] < len(pools[k]) for k in pools):
            k = ["a", "b", "c"][int(rng.integers(3))]
            if idx[k] >= len(pools[k]):
                continue
            mux.append(pools[k][idx[k]])
            idx[k] += 1
            if rng.integers(6) == 0:   # a capture pattern that fails its checksum: resume 4 bytes on
                mux.append(b"OggS\x00\x00" + rng.integers(0, 256, int(rng.integers(21, 90)), dtype=np.uint8).tobytes())
            if hostile and rng.integers(6) == 0:   # a refused header: resume 27 bytes on
                mux.append(b"OgOggOggSOg")
        data = b"".join(mux) + (bytes(66000) if not hostile else b"")
        out.append((f"mux-{int(hostile)}", data))
    out.append(("mux-cut", data[:len(data) * 2 // 3]))
    rng = np.random.default_rng(33)
    pages = st.ogg_paginate(5, _packets(rng, 80, [10, 200, 700, 2000, 20000]), rng, max_segments=12)
    for trial in range(25):
        dmg = list(pages)
        kind, at = trial % 5, int(rng.integers(1, len(pages) - 1))
        if kind == 0:
            del dmg[at]
        elif kind == 1:
            p = bytearray(dmg[at])
            p[len(p) // 2 + 13] ^= 0x10
            dmg[at] = bytes(p)
        elif kind == 2:
            p = bytearray(dmg[at])
            p[4 + int(rng.integers(2))] |= 0x08 if rng.integers(2) else 0x80
            dmg[at] = bytes(p)
        elif kind == 3:
            dmg[at], dmg[at + 1] = dmg[at + 1], dmg[at]
        else:
            dmg.insert(at, dmg[at])
        out.append((f"damage-{trial}", b"".join(dmg)))
    cont = [p for p in pages if p[5] & 1]
    k = pages.index(cont[0])
    out.append(("continued-head-lost", pages[0] + b"".join(pages[k + 1:])))
    clean = b"".join(pages[:12])
    for hit in range(40):   # single-bit hits anywhere: header fields, lacing, body
        d = bytearray(clean)
        bit = int(rng.integers(len(d) * 8))
        d[bit // 8] ^= 1 << (bit % 8)
        out.append((f"bit-{hit}", bytes(d)))
    for cut in (1, 4, 26, 27, 28, 100, len(clean) - 1):
        out.append((f"cut-{cut}", clean[:cut]))
    out.append(("one-page", st.ogg_page(1, 0, 0, [0], b"", first=True)))
    out.append(("many-serials", many_serials(3000, seed=35)))
    out.append(("empty", b""))
    out.append(("no-capture", bytes(range(256)) * 8))
    out.append(("junk", np.random.default_rng(34).integers(0, 256, 5000, dtype=np.uint8).tobytes()))
    out += [(f"vorbis-{name}", data) for name, data in _vorbis_corpus.files()]
    return out
