"""The device front-end (SURVEY §8f N1 on the GPU): `symgpu_mp3_decode_files_host` -- side-information pass on the CPU,
Huffman decode of every granule-channel by one thread each, then the synthesis kernel -- against the oracle's synthesis
of what the CPU front-end decodes from the same bytes.  The kernel runs the same decode
functions the CPU tests cover (symphonia_b200/csrc/mp3_entropy.h)."""
import os

import numpy as np
import pytest

from symphonia_b200 import frontend, packetizer
from tests import _oracle
from tests import test_zz_file_to_pcm as chain

pytestmark = [pytest.mark.gpu]


def test_files_to_pcm_with_the_entropy_kernel(oracle):
    import symphonia_b200 as sb
    files = chain._corpus()
    units, quant, runs, _ = chain._batch(files)   # CPU front-end
    rc, want, _ = _oracle.mp3_batch(oracle, units.reshape(-1), chain._spectra(quant), runs, len(files))
    assert rc == 0
    tables = [packetizer.mpa_index(d)[1] for d in files]
    with sb.Engine(0) as eng:
        eng.mp3_streams_alloc(len(files))
        got, good, frame_of, rounds = eng.mp3_decode_files_host([(d, t, s) for s, (d, t) in enumerate(zip(files, tables))])
    assert good.tolist() == [len(t) for t in tables] and rounds == 1
    same = got.view(np.uint32) == want.view(np.uint32)
    assert same.all(), f"{int((~same).sum())} PCM words differ, first at {np.argwhere(~same)[0]}"


def test_damaged_file_replans_like_the_cpu_path(oracle):
    import symphonia_b200 as sb
    from tests import _mp3_bitstream as bw
    rng = np.random.default_rng(91)
    frames, _ = bw.gen_stream(rng, 80, version="1", mode=0, bitrate_idx=9)
    hit = []
    for f in frames:
        b = bytearray(f)
        if rng.integers(6) == 0:
            b[4 + int(rng.integers(1, 9))] |= 0xF0
        hit.append(bytes(b))
    data = b"".join(hit)
    _, packets = packetizer.mpa_index(data)
    cu, cq, cf, info, crounds = frontend.entropy_decode_cpu(data, packets)
    runs = np.zeros(1, dtype=chain.nat.MP3_RUN_DTYPE)
    runs[0] = (0, 0, len(cf), 2, 2, 0)
    rc, want, _ = _oracle.mp3_batch(oracle, cu.reshape(-1), chain._spectra(cq), runs, 1)
    assert rc == 0
    with sb.Engine(0) as eng:
        eng.mp3_streams_alloc(1)
        got, good, frame_of, rounds = eng.mp3_decode_files_host([(data, packets, 0)])
    assert frame_of.tolist() == cf.tolist() and rounds == crounds
    assert (got.view(np.uint32) == want.view(np.uint32)).all()
