"""ADTS AAC-LC files for the device decoder's tests: writer streams (noise, pulses, TNS, every window sequence) at several rate
classes, mono and stereo, and the files whose packets change the state that carries between raw_data_blocks -- refused packets
between noise packets, a layout fixed by a lone single-channel element, a layout that changes mid-file, and pulses in bands no
section coded, which read the scale factors an earlier packet left behind."""
import numpy as np

from tests import _aac_bitstream as ab
from tests import _streams as st
from tests.test_aac_frontend import QUAD_ZERO, _sce

RATE_IDX = {96000: 0, 88200: 1, 64000: 2, 48000: 3, 44100: 4, 32000: 5, 24000: 6, 22050: 7, 16000: 8, 12000: 9, 11025: 10, 8000: 11}


def adts(packets, rate, channels, seed=0):
    """The raw_data_blocks as one ADTS file; every third frame carries a CRC."""
    rng = np.random.default_rng(seed)
    return b"".join(st.adts_frame(rng, 0, rate_idx=RATE_IDX[rate], channels=channels, protected=k % 3 == 1, payload=p) for k, p in enumerate(packets))


def _writer(seed, rate, channels, n, layout=None):
    s = ab.Stream(np.random.default_rng(seed), rate=rate, channels=channels, layout=layout)
    return [s.packet()[0] for _ in range(n)]


def _damaged(seed, rate, channels, n):
    """Writer packets with truncated and bit-flipped ones in between."""
    rng = np.random.default_rng(seed + 7)
    pk = _writer(seed, rate, channels, n)
    for k in range(2, n, 3):
        p = bytearray(pk[k])
        if k % 2:
            p = p[:max(1, int(len(p) * rng.uniform(0.2, 0.9)))]
        else:
            for _ in range(3):
                i = int(rng.integers(len(p) * 8))
                p[i // 8] ^= 0x80 >> (i % 8)
        pk[k] = bytes(p)
    return pk


def _pulse_above(pulse_start=10):
    """A mono single-channel element with two coded bands and a pulse at `pulse_start`: its line reads scales[0][band] of a band
    this packet does not code."""
    return _sce(150, 2, [(1, 2)], scf=[("d", 0), ("d", 0)], pulse=(pulse_start, [(0, 5), (2, 3)]), spectral=[QUAD_ZERO, QUAD_ZERO])


def quiet(n=6):
    """Hand-built mono packets without noise bands."""
    return [_sce(150, 2, [(1, 2)], scf=[("d", 0), ("d", 1)], spectral=[QUAD_ZERO, QUAD_ZERO]) for _ in range(n)]


def corpus():
    """[(name, packets, rate, channels)]."""
    files = []
    for i, (rate, ch) in enumerate([(44100, 2), (48000, 2), (22050, 1), (8000, 2), (96000, 1), (32000, 2), (16000, 1), (24000, 2)]):
        files.append((f"writer-{rate}-{ch}", _writer(700 + i, rate, ch, 12), rate, ch))
    files.append(("two-sce", _writer(720, 44100, 2, 10, layout=["sce", "sce"]), 44100, 2))
    files.append(("damaged-stereo", _damaged(730, 44100, 2, 16), 44100, 2))
    files.append(("damaged-mono", _damaged(731, 22050, 1, 16), 22050, 1))
    # a stereo file whose first packet is a lone single-channel element: it fixes a layout that refuses the pairs behind it
    files.append(("lone-sce", _writer(740, 44100, 1, 1) + _writer(741, 44100, 2, 6), 44100, 2))
    # the layout changes mid-file: two single-channel elements, then pairs
    files.append(("layout-change", _writer(750, 44100, 2, 5, layout=["sce", "sce"]) + _writer(751, 44100, 2, 5), 44100, 2))
    # pulses above the coded bands: after decoded writer packets, after a refused one, and with no packet before
    mono = _writer(760, 44100, 1, 5)
    files.append(("pulse-after-decoded", mono + [_pulse_above(), _pulse_above(20)], 44100, 1))
    cut = _writer(761, 44100, 1, 4)
    cut[3] = cut[3][:len(cut[3]) * 2 // 3]
    files.append(("pulse-after-refused", cut + [_pulse_above(), _pulse_above(30)], 44100, 1))
    files.append(("pulse-first", [_pulse_above(), _pulse_above(5)] + _writer(762, 44100, 1, 3), 44100, 1))
    return files
