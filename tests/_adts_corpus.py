"""ADTS byte streams for the device ADTS index and the device-resident AAC decode: the random streams of
test_packetizer.py::test_adts_streams, the bad headers that stop an index, clean / cut-payload / cut-header ends, files with no
frame, a file with a sync candidate every 2 bytes, the _aac_corpus files and one long file; all seeded.  `pack` lays files out in
one buffer the way a caller's buffer may hold them."""
import numpy as np

from tests import _aac_corpus
from tests import _streams as st


def random_streams():
    """The 30 streams of test_adts_streams: every rate, channel configuration, profile and CRC setting, junk between frames,
    every third stream cut in its tail."""
    rng = np.random.default_rng(21)
    out = []
    for trial in range(30):
        parts = []
        for _ in range(int(rng.integers(1, 40))):
            parts.append(st.adts_frame(rng, int(rng.integers(0, 700)), rate_idx=int(rng.integers(13)), channels=int(rng.integers(8)),
                                       profile=int(rng.integers(4)), protected=bool(rng.integers(3) == 0), mpeg2=bool(rng.integers(2))))
            if rng.integers(6) == 0:
                parts.append(st.mpa_junk(rng, int(rng.integers(1, 60))))
        data = b"".join(parts)
        if trial % 3 == 0:
            data = data[:len(data) - int(rng.integers(1, 200))]
        out.append((f"random-{trial}", data))
    return out


def bad_headers():
    """Three good frames, a bad header, three good frames: reserved rates 13 and 15, two raw data blocks, a frame length below the
    header's, with and without a CRC."""
    rng = np.random.default_rng(22)
    good = b"".join(st.adts_frame(rng, 200) for _ in range(3))
    bad = [st.adts_frame(rng, 100, rate_idx=13), st.adts_frame(rng, 100, rate_idx=15), st.adts_frame(rng, 100, blocks=1),
           st.adts_frame(rng, 0, frame_len=5), st.adts_frame(rng, 0, frame_len=8, protected=True)]
    return [(f"bad-{k}", good + b + good) for k, b in enumerate(bad)]


def ends():
    rng = np.random.default_rng(23)
    clean = b"".join(st.adts_frame(rng, 300) for _ in range(10))
    return [("clean", clean), ("cut-payload", clean[:-5]), ("cut-header", clean + clean[:4])]


def frameless():
    return [("empty", b""), ("one-ff", b"\xff"), ("zeros", bytes(300)),
            ("noise", np.random.default_rng(24).integers(0, 256, 5000, dtype=np.uint8).tobytes())]


def dense_sync():
    """A sync candidate every 2 bytes; the first is a bad header (rate index 15)."""
    return b"\xff\xf1" * 4000


def aac_files():
    return [(name, _aac_corpus.adts(pk, rate, ch, seed=k)) for k, (name, pk, rate, ch) in enumerate(_aac_corpus.corpus())]


def long_file(n_frames=30000, seed=25):
    """n_frames short frames (random payloads of 0 to 40 bytes, so sync candidates also lie inside payloads)."""
    rng = np.random.default_rng(seed)
    payloads = rng.integers(0, 256, (n_frames, 40), dtype=np.uint8)
    lens = rng.integers(0, 41, n_frames)
    return b"".join(st.adts_frame(rng, 0, payload=payloads[k, :lens[k]].tobytes()) for k in range(n_frames))


def files():
    """[(name, bytes)]: every file above but the long one."""
    return random_streams() + bad_headers() + ends() + frameless() + [("dense-sync", dense_sync())] + aac_files()


def pack(data, seed):
    """The files in one buffer in a shuffled order, with gaps of b"\\xff\\xf1" repeated 1 to 8 times before each file and after the
    last, so that whatever reads past a file's end meets a sync word.  Returns (buffer as a uint8 array, [(offset, len)] in
    the order of `data`)."""
    rng = np.random.default_rng(seed)
    parts, ranges, at = [], [None] * len(data), 0
    for i in rng.permutation(len(data)):
        gap = b"\xff\xf1" * int(rng.integers(1, 9))
        parts += [gap, data[i]]
        ranges[i] = (at + len(gap), len(data[i]))
        at += len(gap) + len(data[i])
    parts.append(b"\xff\xf1" * 4)
    return np.frombuffer(b"".join(parts), dtype=np.uint8).copy(), ranges
