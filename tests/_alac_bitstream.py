"""An ALAC packet writer for tests, written from the decoder's definition (symphonia-codec-alac/src/lib.rs) and independent of
the decoders under test: it runs the decoder's predictor and its `mb` adaptation forward to choose each residual and each Golomb
code, so that decoding a packet gives back the PCM it was made from, bit for bit.

encode_packet(pcm, cookie, elements) -> bytes.  pcm: int array [frames, channels] of bit_depth-bit samples in output-channel
order.  cookie: dict(frame_length, bit_depth, pb, mb, kb, channels).  elements: one dict per element in stream order --
kind 'sce' / 'lfe' / 'cpe' / 'dse' / 'fil' / 'end', and for the channel elements any of shift (0 / 8 / 16 tail bits),
uncompressed, partial (write the frame count), order, mode (0 / 15), pbf (3-bit factor code), lpc_shift, coeffs, ms_weight,
ms_shift; for 'dse' count / align, for 'fil' count.
"""
import numpy as np

CHANNEL_MAPS = {1: [0], 2: [0, 1], 3: [2, 0, 1], 4: [2, 0, 1, 3], 5: [2, 0, 1, 3, 4], 6: [2, 0, 1, 4, 5, 3], 7: [2, 0, 1, 5, 6, 4, 3],
                8: [2, 4, 5, 0, 1, 6, 7, 3]}
# the element sequence an encoder writes for each channel count
LAYOUTS = {1: ["sce"], 2: ["cpe"], 3: ["sce", "cpe"], 4: ["sce", "cpe", "sce"], 5: ["sce", "cpe", "cpe"], 6: ["sce", "cpe", "cpe", "lfe"],
           7: ["sce", "cpe", "cpe", "sce", "lfe"], 8: ["sce", "cpe", "cpe", "cpe", "lfe"]}


class BitWriter:
    def __init__(self):
        self.bits = []

    def put(self, value, width):
        value &= (1 << width) - 1 if width else 0
        self.bits += [(value >> (width - 1 - k)) & 1 for k in range(width)]

    def align(self):
        while len(self.bits) % 8:
            self.bits.append(0)

    def bytes(self):
        self.align()
        b = np.packbits(np.array(self.bits, dtype=np.uint8)) if self.bits else np.zeros(0, dtype=np.uint8)
        return b.tobytes()


def _wrap(v, bits):
    """v as a signed bits-bit integer (the decoder's clip_msbs)."""
    m = 1 << bits
    v &= m - 1
    return v - m if v >= m >> 1 else v


def _i32(v):
    return _wrap(v, 32)


def _clz(v):
    return 32 - int(v).bit_length()


def _lg3a(mb):
    return 31 - _clz((mb >> 9) + 3)


def _rice(w, v, k, bps):
    """Writes v so that read_rice_code(k, bps) returns it."""
    m = (1 << k) - 1
    if k > 1:
        q, rem = divmod(v, m)
    elif k == 1:
        q, rem = v, 0
    else:
        q, rem = (0, 0) if v == 0 else (9, 0)
    if q > 8:
        assert v < (1 << bps), "escape value does not fit"
        w.put(0x1FF, 9)
        w.put(v, bps)
        return
    w.put((1 << q) - 1, q)
    w.put(0, 1)
    if k > 1:
        if rem == 0:
            w.put(0, k - 1)
        else:
            w.put((rem + 1) >> 1, k - 1)
            w.put((rem + 1) & 1, 1)


def _residuals(w, e, mb0, kb, bps, pb_factor):
    """Writes the residuals e as read_residuals reads them, with zero runs where the decoder expects one."""
    n, mb, sign, i = len(e), mb0, 0, 0
    while i < n:
        r = int(e[i])
        val = (r << 1) if r >= 0 else (-r << 1) - 1
        assert val - sign >= 0, "a residual of 0 right after a short zero run"
        _rice(w, val - sign, min(_lg3a(mb), kb), bps)
        mb = 0xFFFF if val > 0xFFFF else (mb + pb_factor * val - ((pb_factor * mb) >> 9)) & 0xFFFFFFFF
        sign = 0
        if mb < 128 and i + 1 < n:
            z = 0
            while i + 1 + z < n and e[i + 1 + z] == 0 and z < 0xFFFF:
                z += 1
            k = min(_clz(mb) - 24 + ((mb + 16) >> 6), kb)
            _rice(w, z, k, 16)
            if z < 0xFFFF:
                sign = 1
            mb = 0
            i += z
        i += 1


def _encode_predicted(x, bps, order, mode, lpc_shift, coeffs):
    """Residuals e for which ElementChannel::predict turns e into x (all values bps-bit signed)."""
    n = len(x)
    x = [int(v) for v in x]
    if order == 0 or n == 0:
        return list(x)
    clip = lambda v: _wrap(v, bps)  # noqa: E731
    e = [0] * n
    e[0] = x[0]
    for i in range(1, min(1 + order, n)):
        e[i] = clip(x[i] - x[i - 1])
    w = [int(coeffs[order - 1 - j]) for j in range(order)]  # w[j] multiplies x[i - order + j]
    for i in range(1 + order, n):
        past0 = x[i - order - 1]
        s = 0
        for j in range(order):
            s = _i32(s + _i32(w[j] * _i32(x[i - order + j] - past0)))
        val = _i32(s + ((1 << lpc_shift) >> 1)) >> lpc_shift
        r = clip(x[i] - past0 - val)
        e[i] = r
        if r != 0:
            pos = r > 0
            for j in range(order):
                d = _i32(past0 - x[i - order + j])
                sg = (d > 0) - (d < 0)
                sg = sg if pos else -sg
                w[j] = _i32(w[j] - sg)
                r = _i32(r - _i32((j + 1) * (_i32(sg * d) >> lpc_shift)))
                if (pos and r <= 0) or (not pos and r >= 0):
                    break
    if order == 31 or mode == 15:
        e = [e[0]] + [clip(e[i] - e[i - 1]) for i in range(1, n)]
    return e


def _channel_header(w, el, order, coeffs):
    w.put(el.get("mode", 0), 4)
    w.put(el.get("lpc_shift", 0), 4)
    w.put(el.get("pbf", 4), 3)
    w.put(order, 5)
    for c in coeffs[:order]:
        w.put(int(c), 16)


def _element(w, cookie, el, cols):
    """An SCE / LFE (cols: one column) or a CPE (two) of the output samples."""
    cpe = len(cols) == 2
    bd, fl = cookie["bit_depth"], cookie["frame_length"]
    n = len(cols[0])
    w.put(el.get("instance", 0), 4)
    w.put(0, 12)
    partial = el.get("partial", n != fl)
    shift = el.get("shift", 0)
    w.put(1 if partial else 0, 1)
    w.put(shift // 8, 2)
    w.put(1 if el.get("uncompressed") else 0, 1)
    if partial:
        w.put(n, 32)
    if el.get("uncompressed"):
        for t in range(n):
            for c in cols:
                w.put(int(c[t]), bd)
        return
    bps = bd - shift + (1 if cpe else 0)
    ms_weight, ms_shift = (el.get("ms_weight", 0), el.get("ms_shift", 0)) if cpe else (0, 0)
    w.put(ms_shift, 8)
    w.put(ms_weight, 8)
    hi = [[int(v) >> shift for v in c] for c in cols]
    tails = [[int(v) & ((1 << shift) - 1) for v in c] for c in cols]
    if cpe and ms_weight:  # decorrelate_mid_side inverted: s1 = L - R, s0 = R + ((s1 * w) >> shift)
        s1 = [_wrap(a - b, bps) for a, b in zip(*hi)]
        s0 = [_wrap(b + (_i32(d * ms_weight) >> ms_shift), bps) for b, d in zip(hi[1], s1)]
        hi = [s0, s1]
    orders = el.get("orders", [el.get("order", 0)] * len(cols))
    coeff_sets = el.get("coeff_sets", [el.get("coeffs", [0] * 32)] * len(cols))
    for o, cs in zip(orders, coeff_sets):
        _channel_header(w, el, o, list(cs) + [0] * 32)
    if shift:
        for t in range(n):
            for tl in tails:
                w.put(tl[t], shift)
    pb_factor = (el.get("pbf", 4) * cookie["pb"]) >> 2
    for h, o, cs in zip(hi, orders, coeff_sets):
        e = _encode_predicted(h, bps, o, el.get("mode", 0), el.get("lpc_shift", 0), list(cs) + [0] * 32)
        _residuals(w, e, cookie["mb"], cookie["kb"], bps, pb_factor)


def encode_packet(pcm, cookie, elements=None):
    pcm = np.asarray(pcm, dtype=np.int64).reshape(len(pcm), -1)
    ch = cookie["channels"]
    cmap = CHANNEL_MAPS[ch]
    if elements is None:
        elements = [dict(kind=k) for k in LAYOUTS[ch]]
    w, nxt = BitWriter(), 0
    tags = dict(sce=0, cpe=1, lfe=3, dse=4, fil=6, end=7)
    for el in elements:
        kind = el["kind"]
        w.put(tags[kind], 3)
        if kind in ("sce", "lfe"):
            _element(w, cookie, el, [pcm[:, cmap[nxt]]])
            nxt += 1
        elif kind == "cpe":
            _element(w, cookie, el, [pcm[:, cmap[nxt]], pcm[:, cmap[nxt + 1]]])
            nxt += 2
        elif kind == "dse":
            count = el.get("count", 3)
            w.put(0, 4)
            w.put(1 if el.get("align") else 0, 1)
            w.put(min(count, 255), 8)
            if count >= 255:
                w.put(count - 255, 8)
            if el.get("align"):
                w.align()
            w.put(0, 8 * count)
        elif kind == "fil":
            count = el.get("count", 2)
            w.put(min(count, 15), 4)
            if count >= 15:
                w.put(count - 14, 8)
            w.put(0, 8 * count)
        elif kind == "end":
            pass
    return w.bytes()


def cookie_bytes(cookie, sample_rate=44100, layout=False, wrap=None):
    """The 24-byte ALAC magic cookie (with the 24-byte channel layout part when layout=True), optionally behind the 'frma' and
    'alac' atoms (wrap='alac' or 'frma')."""
    c = cookie
    b = (c["frame_length"].to_bytes(4, "big") + bytes([0, c["bit_depth"], c["pb"], c["mb"], c["kb"], c["channels"]]) + (255).to_bytes(2, "big")
         + (0).to_bytes(4, "big") + (0).to_bytes(4, "big") + int(sample_rate).to_bytes(4, "big"))
    if layout:
        tag = ([100, 101, 113, 116, 120, 124, 142, 127][c["channels"] - 1] << 16) | c["channels"]
        b += (24).to_bytes(4, "big") + b"chan" + bytes(4) + tag.to_bytes(4, "big") + bytes(8)
    if wrap in ("alac", "frma"):
        b = (12 + len(b)).to_bytes(4, "big") + b"alac" + bytes(4) + b
    if wrap == "frma":
        b = (12).to_bytes(4, "big") + b"frma" + b"alac" + b
    return b


def signal(rng, n, channels, bit_depth, amp=0.3):
    """Smooth test PCM [n, channels]: a few sinusoids and a little noise, at amp of full scale."""
    t = np.arange(n)[:, None]
    f = rng.uniform(0.001, 0.05, size=(3, channels))
    x = sum(np.sin(2 * np.pi * f[k] * t + rng.uniform(0, 6)) for k in range(3)) / 3
    x = x * amp + rng.normal(0, 0.01, size=(n, channels))
    full = (1 << (bit_depth - 1)) - 1
    return np.clip(np.round(x * full), -full, full).astype(np.int64)
