"""Seeded MP3 synthesis batches whose two channels take their block decisions independently.

`workloads.mp3_batch` draws one block-type chain per stream, so both channels of a granule always share block type and
mixed flag.  Outside joint stereo (stereo and dual-channel frames, and joint-stereo frames with mode_ext 0) the format lets
each channel switch windows on its own, and the synthesis kernels then make every per-channel decision twice in one lane:
block kind, IMDCT window, sub-band category and antialias bound.  `pair_batch` starts from `workloads.mp3_batch` (whose
output is not changed) and re-draws both channels of a chosen share of frames, with mid-side and intensity stereo off.  The
other frames keep their joint-stereo draws, so both regimes alternate within one stream.

`lane_categories` restates the kernels' per-lane choices (mp3_kernel_v2.cu, phases A6 and B) in numpy, so that the tests can
assert which paths a batch reaches instead of hoping for it.
"""
import numpy as np

from symphonia_b200 import _native as nat
from symphonia_b200 import workloads
from symphonia_b200._native import (F_INTENSITY, F_MID_SIDE, F_MIXED, F_MPEG1, F_MUTE, F_PREFLAG, F_SCALEFAC_SCALE, F_SFC_LSB,
                                    MP3_END, MP3_LONG, MP3_SHORT, MP3_START)

# per-channel kinds: (block_type, mixed flag)
KINDS = ((MP3_LONG, False), (MP3_START, False), (MP3_END, False), (MP3_SHORT, False), (MP3_SHORT, True))
KIND_NAMES = ("long", "start", "end", "short", "mixed")
# rzero of one channel while the other is full: nothing coded, one pair, ends inside sub-band 0 / 1 / 2, sub-band edges, all
EDGE_RZERO = (0, 2, 10, 16, 18, 20, 30, 36, 38, 50, 576)

# The three kernel shapes the launch plan picks (symgpu.cpp build_plan, launch_plan): (n_streams, frames per stream).
#   long  -- 80 granules per run: first generation, one tile per CTA (single-tile groups)
#   short -- 300 one-frame runs: second generation, compact instantiation (many run segments per share)
#   few   -- 14 granules per run on average: second generation, default instantiation
SHAPES = {"long": (4, 40), "short": (300, 1), "few": (6, 7)}
SEEDS = {"long": 8101, "short": 8102, "few": 8103}


def pair_batch(n_streams, frames_per_stream, seed, sample_rate_idx=0, differ=0.6, edge=0.25, joint=True):
    """(units, spectra, runs) like workloads.mp3_batch(channels=2): a share `differ` of the frames have mid-side and intensity
    stereo off and both channels re-drawn per granule with independent kinds.  The ordered kind pairs of the re-drawn granules
    run through random permutations of all 25, so every pair occurs once per 25 re-drawn granules, with transitions no strict
    encoder emits (LONG straight to SHORT, ...).  On a share `edge` of them one channel's rzero is an edge value and the other
    channel's is 576, cycling through every (channel, edge value) the same way.  joint=False: no frame uses mid-side or intensity stereo."""
    units, spectra, runs = workloads.mp3_batch(n_streams, frames_per_stream, seed=seed, sample_rate_idx=sample_rate_idx,
                                               joint=joint)
    rng = np.random.Generator(np.random.PCG64([seed, 0x9A125]))
    gpf = 2 if sample_rate_idx < 3 else 1
    n = len(units)
    sel = np.nonzero(rng.random(n) < differ)[0]
    units["flags"][sel] &= np.uint8(~(F_MID_SIDE | F_INTENSITY) & 0xff)
    fr = np.repeat(sel, gpf)
    gr = np.tile(np.arange(gpf), len(sel))
    m = len(fr)
    pair = np.concatenate([rng.permutation(25) for _ in range((m + 24) // 25)])[:m] if m else np.zeros(0, np.int64)
    kinds = np.stack([pair // 5, pair % 5], axis=1)                                   # [m, ch]
    rz = 2 * rng.integers(144, 289, size=(m, 2))
    on_edge = np.nonzero(rng.random(m) < edge)[0]
    n_combo = 2 * len(EDGE_RZERO)  # (channel, edge value), cycled like the kind pairs
    combo = np.concatenate([rng.permutation(n_combo) for _ in range(len(on_edge) // n_combo + 1)])[:len(on_edge)]
    rz[on_edge] = 576
    rz[on_edge, combo % 2] = np.array(EDGE_RZERO)[combo // 2]
    pow43 = nat.mp3_pow43()
    lam = np.linspace(40.0, 0.5, 576)
    for ch in range(2):
        bt = np.array([KINDS[k][0] for k in range(5)], np.uint8)[kinds[:, ch]]
        mixed = np.array([KINDS[k][1] for k in range(5)])[kinds[:, ch]]
        u = units[fr, gr, ch]
        u["block_type"] = bt
        flags = np.where(mixed, F_MIXED, 0).astype(np.uint8)
        flags |= np.where(rng.random(m) < 0.2, F_SCALEFAC_SCALE, 0).astype(np.uint8)
        flags |= np.where((rng.random(m) < 0.3) & (bt != MP3_SHORT), F_PREFLAG, 0).astype(np.uint8)
        flags |= np.where(rng.random(m) < 0.5, F_SFC_LSB, 0).astype(np.uint8)
        flags |= np.uint8(F_MPEG1 if gpf == 2 else 0)
        u["flags"] = flags
        u["global_gain"] = rng.integers(120, 201, size=m)
        u["subblock_gain"] = rng.integers(0, 8, size=(m, 3))
        sf = rng.integers(0, 16, size=(m, 39)).astype(np.uint8)
        idx = np.arange(39)[None, :]
        long_like = (bt != MP3_SHORT)[:, None]
        sf = np.where(long_like & (idx >= 21), 0, sf)
        sf = np.where(~long_like & (idx >= 36), 0, sf)
        u["scalefacs"] = sf
        u["rzero"] = rz[:, ch]
        units[fr, gr, ch] = u
        q = np.minimum(8206, np.floor(rng.exponential(lam[None, :], size=(m, 576)))).astype(np.int64)
        sign = np.where(rng.random((m, 576)) < 0.5, -1.0, 1.0).astype(np.float32)
        val = sign * pow43[q]
        val = np.where(np.arange(576)[None, :] < rz[:, ch:ch + 1], val, np.float32(0.0))
        val = np.where(q == 0, np.float32(0.0), val)
        spectra[fr, gr, ch] = val.astype(np.float32)
    return units, spectra, runs


def shape_batch(shape, **kw):
    s, f = SHAPES[shape]
    return pair_batch(s, f, SEEDS[shape], **kw)


def quantized(spectra):
    """The int16 Huffman values sign * q behind spectra built from POW43 (the inverse of the device's lookup)."""
    pow43 = nat.mp3_pow43()
    mag = np.abs(spectra)
    q = np.searchsorted(pow43, mag).astype(np.int64)
    assert (pow43[np.minimum(q, len(pow43) - 1)] == mag).all(), "a spectrum value is not a POW43 entry"
    assert not (np.signbit(spectra) & (spectra == 0)).any(), "no -0.0 in the spectra"
    return np.where(spectra < 0, -q, q).astype(np.int16)


def split_channel(units, spectra, runs, ch):
    """The mono batch made of channel `ch` of a stereo batch: its units and spectra in slot 0, slot 1 muted."""
    u, s = units.copy(), np.zeros_like(spectra)
    u[:, :, 0] = units[:, :, ch]
    u[:, :, 1] = np.zeros(1, dtype=u.dtype)
    u["flags"][:, :, 1] = F_MUTE
    s[:, :, 0] = spectra[:, :, ch]
    r = runs.copy()
    r["channels"] = 1
    return u, s, r


def swap_channels(units, spectra):
    return np.ascontiguousarray(units[:, :, ::-1]), np.ascontiguousarray(spectra[:, :, ::-1])


# ---- the kernels' per-lane decisions, restated ------------------------------------------------------------------------
# ISO/IEC 11172-3 Table B.8 / 13818-3 Table B.2: width of one window of each of the 13 short bands (layer3/common.rs:60-107)
_SHORT_WIDTHS = (
    (4, 4, 4, 4, 6, 8, 10, 12, 14, 18, 22, 30, 56), (4, 4, 4, 4, 6, 6, 10, 12, 14, 16, 20, 26, 66),
    (4, 4, 4, 4, 6, 8, 12, 16, 20, 26, 34, 42, 12), (4, 4, 4, 6, 6, 8, 10, 14, 18, 26, 32, 42, 18),
    (4, 4, 4, 6, 8, 10, 12, 14, 18, 24, 32, 44, 12), (4, 4, 4, 6, 8, 10, 12, 14, 18, 24, 30, 40, 18),
    (4, 4, 4, 6, 8, 10, 12, 14, 18, 24, 30, 40, 18), (4, 4, 4, 6, 8, 10, 12, 14, 18, 24, 30, 40, 18),
    (8, 8, 8, 12, 16, 20, 24, 28, 36, 2, 2, 2, 26))


def _short_quad_edges(sr, mixed):
    """Line at which each reordered window triple (quad) of a short or mixed block starts, and the end of the last one."""
    w = _SHORT_WIDTHS[sr]
    if not mixed:
        widths, start = list(w), 0
    elif sr == 8:  # the reference's own guess (layer3/common.rs:159-167): windows of 4 lines from line 36, then band 2 on
        widths, start = [4] + list(w[2:]), 36
    else:          # the short part of a mixed block starts at line 36 with short band 3 (layer3/common.rs:109-172)
        widths, start = list(w[3:]), 36
    return np.concatenate([[start], start + 3 * np.cumsum(widths)])


def reordered_rzero(rz, kind, sr):
    """rzero after the short-block reorder (hybrid_synthesis.rs:153-215): the end of the last window triple it reaches."""
    if KINDS[kind][0] != MP3_SHORT:
        return rz
    e = _short_quad_edges(sr, KINDS[kind][1])
    n_done = int((e[:-1] < rz).sum())
    return max(rz, int(e[n_done]))


def lane_categories(units, runs):
    """Per granule of every run: (cat [32, 2], wsel [2], kinds [2], joint) with cat 36 (IMDCT-36), 12 (3 x IMDCT-12) or 0
    (beyond the coded lines), as phases A6 and B of mp3_kernel_v2.cu choose them per sub-band and channel."""
    out = []
    lanes = np.arange(32)
    for r in runs:
        gpf = int(r["granules_per_frame"] or 2)
        for f in range(int(r["first_frame"]), int(r["first_frame"]) + int(r["n_frames"])):
            for g in range(gpf):
                u0, u1 = units[f, g, 0], units[f, g, 1]
                joint = bool(u0["flags"] & (F_MID_SIDE | F_INTENSITY))
                sr = int(u0["sample_rate_idx"])
                rz = [int(u0["rzero"]), int(u1["rzero"])]
                if joint:
                    rz = [max(rz)] * 2
                cats, wsel, kinds = np.zeros((32, 2), np.int64), [0, 0], [0, 0]
                for c, u in enumerate((u0, u1)):
                    bt, mixed = int(u["block_type"]), bool(u["flags"] & F_MIXED) and int(u["block_type"]) == MP3_SHORT
                    kind = KINDS.index((bt, mixed))
                    kinds[c] = kind
                    rzr = reordered_rzero(rz[c], kind, sr)
                    if bt == MP3_SHORT and not mixed:
                        cats[:, c] = np.where(lanes < (rzr + 17) // 18, 12, 0)
                    else:
                        sb_limit = min(2 if mixed else 32, rzr // 18 + 2)   # antialias bound = hybrid synthesis' sub-band limit
                        long_end = 2 if mixed else 32
                        cats[:, c] = np.where(lanes < min(long_end, sb_limit), 36, np.where(lanes < sb_limit, 12, 0))
                    wsel[c] = 1 if bt == MP3_START else 3 if bt == MP3_END else 0
                out.append((cats, wsel, kinds, joint))
    return out


def coverage(units, runs):
    """What a batch reaches: the ordered (cat0, cat1) lane pairs, the (wsel0, wsel1) pairs on lanes where both channels are
    long, and the ordered kind pairs -- each counted over the granules without joint stereo."""
    cat_pairs, wsel_pairs, kind_pairs = {}, {}, {}
    for cats, wsel, kinds, joint in lane_categories(units, runs):
        if joint:
            continue
        for a, b in set(map(tuple, cats.tolist())):
            cat_pairs[(a, b)] = cat_pairs.get((a, b), 0) + 1
        if ((cats[:, 0] == 36) & (cats[:, 1] == 36)).any():
            wsel_pairs[tuple(wsel)] = wsel_pairs.get(tuple(wsel), 0) + 1
        kind_pairs[tuple(kinds)] = kind_pairs.get(tuple(kinds), 0) + 1
    return cat_pairs, wsel_pairs, kind_pairs
