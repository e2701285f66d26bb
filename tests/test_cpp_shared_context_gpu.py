"""Many decoders of every codec on ONE context (include/symgpu/decoder.hpp), driven from C++: `shared_context_host files` opens one
decoder thread per file through the registry, all on one GpuContext, and decodes packet by packet; the context batches whatever the
threads have in flight, per codec, and runs the batches of different codecs one at a time.  Every file's PCM must equal what the
single-decoder `decoder_host file` mode writes for it -- which the oracle pins (test_zz_*: the same expectations are built here) --
and every codec's launches must carry the packets of several decoders."""
import os
import re
import subprocess

import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import decode, frontend, packetizer
from tests import _oracle
from tests import _streams as st
from tests import _vorbis_bitstream as vb
from tests.test_cpp_host import _build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build_shared():
    """tests/cpp/shared_context_host, rebuilt when its source, the library or the headers are newer."""
    exe = os.path.join(ROOT, "tests", "cpp", "shared_context_host")
    src = os.path.join(ROOT, "tests", "cpp", "shared_context_host.cpp")
    lib = os.path.join(ROOT, "symphonia_b200", "libsymgpu.so")
    deps = [src, lib] + [os.path.join(ROOT, "include", "symgpu", h) for h in ("decoder.hpp", "packetizer.hpp")]
    if not os.path.exists(exe) or os.path.getmtime(exe) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-pthread", "-o", exe, src, "-L" + os.path.dirname(lib), "-lsymgpu",
                               "-Wl,-rpath," + os.path.dirname(lib)])
    return exe


# ------------------------------------------------------------------------------------------- files and what `file` mode writes

def _adts(oracle, seed):
    from tests import test_zz_adts_aac_to_pcm as t
    rate, channels = [(44100, 2), (48000, 2), (22050, 1), (32000, 2)][seed % 4]
    data, _ = t._file(seed, rate, channels)
    want = t._render(oracle, decode.adts_aac_plan(data), nat.FMT_F32)  # [frames, ch] interleaved
    return "aac", data, np.ascontiguousarray(want.reshape(-1, 1024, channels).transpose(0, 2, 1)).tobytes()


def _ogg_vorbis_file(seed, bs_exp, channels, n_packets=16, pad=29):
    """As test_zz_ogg_vorbis_to_pcm._file, with the block sizes as a parameter."""
    rng = np.random.default_rng(seed)
    s = vb.Stream(rng, channels=channels, bs_exp=bs_exp, per_word=1)
    pk, truth = [], []
    for _ in range(n_packets):
        b, t = s.packet()
        pk.append(b), truth.append(t)
    bs = {False: 1 << bs_exp[0], True: 1 << bs_exp[1]}
    g, gran = 0, []
    for k, t in enumerate(truth):
        if k:
            g += (bs[bool(t["prev_block_flag"])] + bs[bool(t["block_flag"])]) // 4
        gran.append(g)
    gran[-1] = max(g - pad, gran[-2])
    headers = [s.ident, b"\x03vorbis" + bytes(20), s.setup]
    pages = st.ogg_paginate(77, headers[:1], rng, eos=False) + st.ogg_paginate(77, headers[1:], rng, first_sequence=1, bos=False, eos=False)
    first = len(pages)
    pages += st.ogg_paginate(77, pk, rng, max_segments=int(rng.integers(3, 40)), first_sequence=first, bos=False, granule_of=gran)
    return b"".join(pages)


def _vorbis(oracle, seed):
    from tests import test_zz_ogg_vorbis_to_pcm as t
    bs_exp = [(8, 11), (7, 9)][seed % 2]  # two block-size pairs: the batch rows are longer than half the packets' slots
    channels = 1 if seed % 5 == 3 else 2
    data = _ogg_vorbis_file(seed, bs_exp, channels)
    plan = decode.ogg_vorbis_plan(data)
    want = t._render(oracle, plan, nat.FMT_F32)
    sp = plan["spans"]
    left = sp["frames"].astype(np.int64) - sp["trim_start"] - sp["trim_end"]
    out, at = [], 0
    for n in left:
        out.append(np.ascontiguousarray(want[at:at + n].T).tobytes())
        at += n
    return "vorbis", data, b"".join(out)


def _mpa12(oracle, seed, layer):
    from tests import _mpa12_bitstream as b12
    rng = np.random.default_rng(seed)
    if layer == 2:
        frames = [b12.gen_layer2_frame(rng, "1", 12, 0, 1, mode_ext=k % 4)[0] for k in range(12)] if seed % 3 else \
            [b12.gen_layer2_frame(rng, "2", 6, 1, 3)[0] for _ in range(12)]
    else:
        frames = [b12.gen_layer1_frame(rng, "1", 9, 1, 0 if seed % 2 else 3)[0] for _ in range(14)]
    data = b"".join(frames)
    track, pk = packetizer.mpa_index(data)
    sub, frame_of, info = frontend.mpa12_decode_packets(data, pk, layer)
    assert len(frame_of) == len(pk)
    runs = np.zeros(1, dtype=nat.MPA12_RUN_DTYPE)
    runs[0] = (0, 0, len(sub), int(info["channels"]), (0, 0, 0))
    rc, want, _ = _oracle.mpa12_batch(oracle, sub, runs, 1)
    assert rc == 0
    ch, n = int(info["channels"]), 32 * sub.shape[-1]
    cut = [(int(p["trim_start"]), n - min(int(p["trim_end"]), n - int(p["trim_start"]))) for p in pk]
    return str(layer), data, b"".join(want[k, c, a:b].tobytes() for k, (a, b) in enumerate(cut) for c in range(ch))


def _mp3(oracle, seed):
    from tests import _mp3_bitstream as bw
    from tests.test_zz_file_to_pcm import _batch, _spectra
    rng = np.random.default_rng(seed)
    frames, _ = bw.gen_stream(rng, 12, version="1", mode=1, bitrate_idx=9, pair_blocks=True)
    data = b"".join(frames)
    units, quant, runs, spans = _batch([data])
    rc, want, _ = _oracle.mp3_batch(oracle, units.reshape(-1), _spectra(quant), runs, 1)
    assert rc == 0
    dur, t0, t1 = spans[0]
    return "3", data, b"".join(want[k, ch, int(t0[k]):int(dur[k] - t1[k])].tobytes() for k in range(len(want)) for ch in range(2))


def _run_files(tmp_path, files, min_codecs):
    """files: [(kind, bytes, expected PCM bytes)] -> the harness's stdout after checking every file bit for bit."""
    args = []
    for i, (kind, data, _) in enumerate(files):
        p = tmp_path / f"f{i:03d}.{kind}"
        p.write_bytes(data)
        args.append(f"{kind}:{p}")
    res = subprocess.run([_build_shared(), "files"] + args, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout + res.stderr
    for i, (kind, _, want) in enumerate(files):
        got = (tmp_path / f"f{i:03d}.{kind}.pcm").read_bytes()
        assert len(got) == len(want) and got == want, (i, kind, len(got), len(want))
    stats = {m.group(1): (int(m.group(2)), int(m.group(3))) for m in re.finditer(r"codec (\w+) batches (\d+) frames (\d+)", res.stdout)}
    assert set(min_codecs) <= set(stats), res.stdout
    for codec, (batches, frames) in stats.items():
        assert batches < frames, f"{codec}: no launch carried the packets of several decoders: " + res.stdout
    print(res.stdout.strip())
    return res.stdout


@pytest.mark.gpu
def test_sixty_four_adts_decoders_share_one_context(tmp_path, oracle):
    _run_files(tmp_path, [_adts(oracle, 7000 + k) for k in range(64)], ["aac"])


@pytest.mark.gpu
def test_sixty_four_ogg_vorbis_decoders_share_one_context(tmp_path, oracle):
    _run_files(tmp_path, [_vorbis(oracle, 7100 + k) for k in range(64)], ["vorbis"])


@pytest.mark.gpu
def test_layer_one_and_two_decoders_share_one_context(tmp_path, oracle):
    files = [_mpa12(oracle, 7200 + k, 2) for k in range(32)] + [_mpa12(oracle, 7300 + k, 1) for k in range(16)]
    _run_files(tmp_path, files, ["mp1", "mp2"])


@pytest.mark.gpu
def test_every_codec_on_one_context(tmp_path, oracle):
    """MP3, Layer II, AAC and Vorbis decoders at once: their batches take turns on the context's launch lock.  One file of each
    codec is also decoded by the single-decoder `decoder_host file` mode, which must write the same bytes."""
    files = []
    for k in range(8):
        files += [_mp3(oracle, 7400 + k), _mpa12(oracle, 7500 + k, 2), _adts(oracle, 7600 + k), _vorbis(oracle, 7700 + k)]
    _run_files(tmp_path, files, ["mp3", "mp2", "aac", "vorbis"])
    for i in range(4):
        kind = files[i][0]
        src, out = tmp_path / f"f{i:03d}.{kind}", tmp_path / f"single{i}.bin"
        res = subprocess.run([_build(), "file", kind, str(src), str(out)], capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stdout + res.stderr
        assert out.read_bytes() == (tmp_path / f"f{i:03d}.{kind}.pcm").read_bytes(), kind


@pytest.mark.gpu
def test_vorbis_decoders_fill_the_context(tmp_path):
    """A Vorbis decoder takes one of the context's stream slots: 256 open on a context of 256, the 257th is a LimitError."""
    p = tmp_path / "a.ogg"
    p.write_bytes(_ogg_vorbis_file(7800, (8, 11), 2))
    res = subprocess.run([_build_shared(), "open", "vorbis", "256", str(p)], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "opened 256 refused LimitError" in res.stdout and "decode failures 0" in res.stdout, res.stdout
