"""MPEG audio byte streams for the device MPEG index and the device-resident MPEG decode, all seeded: every version and layer,
junk and false syncs, free-format words (a refused header costs 4 bytes), rejected first frames (the hunt restarts one byte on),
Xing / Info / LAME (good, bad and zero CRC; cut extensions) and VBRI tags first and mid-stream, a tag as the only frame, a frame cut
at the end, frameless files, a dense run of refused words, a long first-frame hunt and a 30 000-frame file.  `decodable` gives
files whose frames carry real Layer I / II / III bitstreams.  `pack` lays files out in one buffer the way a caller's buffer may
hold them."""
import numpy as np

from tests import _mp3_bitstream as bw
from tests import _mpa12_bitstream as b12
from tests import _streams as st


def clean_streams():
    """25 frames of random body for every version, layer and a few modes."""
    rng = np.random.default_rng(41)
    out = []
    for version in ("1", "2", "2.5"):
        for layer in (1, 2, 3):
            for mode in (0, 3):
                params = st.mpa_random_params(rng, version, layer, mode)
                out.append((f"clean-{version}-{layer}-{mode}", b"".join(st.mpa_frame(rng, params) for _ in range(25))))
    return out


def junk_streams():
    """Junk in front of and between frames, mid-stream parameter changes, every third stream cut in its tail (a Stop)."""
    rng = np.random.default_rng(42)
    out = []
    for trial in range(24):
        params = st.mpa_random_params(rng)
        parts = [st.mpa_junk(rng, int(rng.integers(0, 300)))] if trial % 2 else []
        for k in range(int(rng.integers(1, 40))):
            if k and rng.integers(8) == 0:
                params = st.mpa_random_params(rng)
            parts.append(st.mpa_frame(rng, params))
            if rng.integers(5) == 0:
                parts.append(st.mpa_junk(rng, int(rng.integers(1, 200))))
        data = b"".join(parts)
        if trial % 3 == 0:
            data = data[:len(data) - int(rng.integers(1, 200))]
        out.append((f"junk-{trial}", data))
    return out


def refused_words():
    """A free-format or forbidden word in front of and inside a stream: it costs 4 bytes, so the frame starting in it is lost."""
    rng = np.random.default_rng(43)
    params = dict(version="1", layer=3, bitrate_idx=9, rate_idx=0, mode=0)
    frames = [st.mpa_frame(rng, params, protected=False) for _ in range(8)]
    out = []
    for k, lead in enumerate((b"\xff\xfb\x00", b"\xff\xfb\x02", b"\x11\xff\xfb\x00", b"\xff\xfd\xb0")):
        out.append((f"refused-{k}", lead + b"".join(frames)))
        out.append((f"refused-mid-{k}", b"".join(frames[:4]) + lead + b"".join(frames[4:])))
    return out


def rejected_first():
    """First-frame candidates the word behind them rejects: the hunt restarts one byte on."""
    rng = np.random.default_rng(44)
    params = dict(version="1", layer=3, bitrate_idx=9, rate_idx=0, mode=0)
    frames = [st.mpa_frame(rng, params, protected=False) for _ in range(6)]
    decoy = st.mpa_frame(rng, st.mpa_random_params(rng, "2", 1, 3))
    return [("rejected-ff", b"\xff\xff\x90" + b"".join(frames)), ("rejected-decoy", decoy + b"".join(frames)),
            ("decoy-mid", b"".join(frames) + decoy + b"".join(frames)), ("lone-last", st.mpa_junk(rng, 50) + frames[0])]


def tagged():
    """The tag cases of test_mpa_tags, each first, mid-stream and twice in front; a tag as the only frame."""
    rng = np.random.default_rng(45)
    out = []
    for version, mode in (("1", 0), ("1", 3), ("2", 1), ("2.5", 3)):
        params = dict(version=version, layer=3, bitrate_idx=9 if version == "1" else 8, rate_idx=0, mode=mode)
        audio = [st.mpa_frame(rng, params, protected=False) for _ in range(20)]
        cases = [dict(), dict(kind="Info", flags=0x1), dict(flags=0x0, lame_ext=0), dict(flags=0xF, crc="bad"), dict(flags=0xF, crc="zero"),
                 dict(flags=0xF, lame=b"Lavf58.20", protected=True), dict(flags=0xF, lame=b"Lavc58.54", crc="bad"),
                 dict(flags=0xF, lame=b"GOGO3.13 ", delay=700), dict(flags=0x7, lame_ext=30), dict(flags=0x3, lame_ext=20),
                 dict(flags=0xF, side_info_noise=True), dict(kind="VBRI", num_frames=321), dict(kind="VBRI", vbri_version=2),
                 dict(kind="VBRI", protected=True), dict(flags=0xF, delay=0, padding=0, num_frames=21),
                 dict(flags=0x1, num_frames=3, lame_ext=36, delay=1105, padding=2000)]
        for k, case in enumerate(cases):
            tag = st.mpa_tag_frame(rng, params, **case)
            out += [(f"tag-{version}-{mode}-{k}-first", tag + b"".join(audio)),
                    (f"tag-{version}-{mode}-{k}-mid", b"".join(audio[:7]) + tag + b"".join(audio[7:])),
                    (f"tag-{version}-{mode}-{k}-twice", tag + tag + b"".join(audio))]
        out.append((f"tag-only-{version}-{mode}", st.mpa_tag_frame(rng, params, num_frames=20)))
    # tag fields and LAME extensions cut by a short frame
    short = dict(version="2.5", layer=3, bitrate_idx=1, rate_idx=1, mode=0)
    audio = [st.mpa_frame(rng, short, protected=False, padding=0) for _ in range(20)]
    for flags in (0x0, 0x1, 0x3, 0x4, 0x7, 0xB, 0xF):
        out.append((f"tag-cut-{flags}", st.mpa_tag_frame(rng, short, flags=flags, lame_ext=0) + b"".join(audio)))
    mono = dict(short, mode=3)
    out.append(("lame-cut", st.mpa_tag_frame(rng, mono, flags=0x0, lame_ext=36, delay=700, padding=900) + b"".join(audio)))
    return out


def estimates():
    """Untagged streams around the estimate's 17 frames, and VBR streams the estimate gets wrong."""
    rng = np.random.default_rng(46)
    params = st.mpa_random_params(rng, "1", 3, 0)
    out = [(f"estimate-{n}", b"".join(st.mpa_frame(rng, params) for _ in range(n))) for n in (5, 16, 17, 18, 60)]
    lo, hi = dict(params, bitrate_idx=2), dict(params, bitrate_idx=14)
    out.append(("vbr-up", b"".join(st.mpa_frame(rng, lo) for _ in range(20)) + b"".join(st.mpa_frame(rng, hi) for _ in range(40))))
    out.append(("vbr-down", b"".join(st.mpa_frame(rng, hi) for _ in range(20)) + b"".join(st.mpa_frame(rng, lo) for _ in range(40))))
    return out


def frameless():
    rng = np.random.default_rng(47)
    params = dict(version="1", layer=3, bitrate_idx=9, rate_idx=0, mode=0)
    return [("empty", b""), ("one-ff", b"\xff"), ("three", b"\xff\xfb\x90"), ("zeros", bytes(300)),
            ("noise", rng.integers(0, 255, 5000, dtype=np.uint8).tobytes()),
            ("cut-only", st.mpa_frame(rng, params)[:-1])]


def dense_skip(n=1 << 20):
    """A refused (free-format) header word every 4 bytes: every candidate is a Skip."""
    return b"\xff\xfb\x00\x00" * (n // 4)


def long_hunt(n_frames=10000):
    """n_frames 32-byte Layer I frames, each followed by four zero bytes, so open() rejects each in turn and its hunt walks them
    all; then three back-to-back frames, the first of which is accepted."""
    w = st.mpa_word(version="1", layer=1, bitrate_idx=1, rate_idx=1, mode=3).to_bytes(4, "big")
    frame = w + bytes(28)
    assert st.mpa_frame_len("1", 1, 1, 1, 0) == 32
    return (frame + bytes(4)) * n_frames + frame * 3


def long_file(n_frames=30000, seed=48):
    """n_frames 32-byte Layer I frames with random bodies, so candidates also lie inside frames."""
    rng = np.random.default_rng(seed)
    params = dict(version="1", layer=1, bitrate_idx=1, rate_idx=1, mode=3)
    bodies = rng.integers(0, 256, (n_frames, 28), dtype=np.uint8)
    w = st.mpa_word(padding=0, **params).to_bytes(4, "big")
    return b"".join(w + bodies[k].tobytes() for k in range(n_frames))


def files():
    """[(name, bytes)]: every file above but the three long ones."""
    return clean_streams() + junk_streams() + refused_words() + rejected_first() + tagged() + estimates() + frameless()


def _mp3(rng, n, version="1", mode=1, rate_idx=0, bitrate_idx=9):
    frames, _ = bw.gen_stream(rng, n, version=version, mode=mode, rate_idx=rate_idx, bitrate_idx=bitrate_idx, pair_blocks=True)
    return frames


def decodable(seed=49):
    """[(name, bytes)] of real Layer I / II / III bitstreams: every version, mono and stereo, a LAME-tagged (gapless) file with junk,
    an Info tag as the only frame, a file whose first frames reach into missing reservoir bytes, and one whose main data over-reads."""
    rng = np.random.default_rng(seed)
    out = []
    for k, (version, mode, rate_idx, bitrate_idx) in enumerate((("1", 1, 0, 9), ("1", 3, 1, 5), ("2", 1, 0, 8), ("2", 3, 1, 6),
                                                                 ("2.5", 0, 2, 6), ("1", 0, 2, 14))):
        out.append((f"mp3-{k}", b"".join(_mp3(rng, 12 + k, version, mode, rate_idx, bitrate_idx))))
    for k, (version, mode) in enumerate((("1", 0), ("1", 3), ("2", 1))):
        out.append((f"layer1-{k}", b"".join(b12.gen_layer1_frame(rng, version, 9, 0, mode, mode_ext=j % 4)[0] for j in range(6))))
        out.append((f"layer2-{k}", b"".join(b12.gen_layer2_frame(rng, version, 8, 0, mode, mode_ext=j % 4)[0] for j in range(6))))
    frames = _mp3(rng, 20)
    tag = st.mpa_tag_frame(rng, dict(version="1", layer=3, bitrate_idx=9, rate_idx=0, mode=1), num_frames=20)
    noise = rng.integers(0, 255, 120, dtype=np.uint8).tobytes()
    out.append(("gapless", noise + tag + b"".join(frames[:9]) + noise[:29] + b"".join(frames[9:])))
    out.append(("tag-only", tag))
    out.append(("cut-front", b"".join(_mp3(rng, 30)[9:])))
    over = [bytearray(f) for f in _mp3(rng, 24, mode=0)]
    for k in (4, 11, 17):   # part2_3_length of granule 0, channel 0 set to 4095 bits: the main data over-reads
        at = 32 + 9 + 3 + 8   # behind the header word, main_data_begin, the private bits and scfsi of MPEG-1 stereo side information
        for b in range(12):
            byte, bit = divmod(at + b, 8)
            over[k][byte] |= 0x80 >> bit
    out.append(("over-read", b"".join(bytes(b) for b in over)))
    return out


def pack(data, seed):
    """The files in one buffer in a shuffled order, with runs of 1 to 8 0xff bytes before each file and after the last, so that
    whatever reads past a file's end meets sync bits.  Returns (buffer as a uint8 array, [(offset, len)] in the order of `data`)."""
    rng = np.random.default_rng(seed)
    parts, ranges, at = [], [None] * len(data), 0
    for i in rng.permutation(len(data)):
        gap = b"\xff" * int(rng.integers(1, 9))
        parts += [gap, data[i]]
        ranges[i] = (at + len(gap), len(data[i]))
        at += len(gap) + len(data[i])
    parts.append(b"\xff" * 4)
    return np.frombuffer(b"".join(parts), dtype=np.uint8).copy(), ranges
