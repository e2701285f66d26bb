"""The host CAF index (packetizer.hpp caf_open / caf_varint, symgpu_caf_index): the packets of every corpus file, the files that
must not open, and the reference's own variable-length-integer known answers."""
import ctypes

import numpy as np
import pytest

from symphonia_b200 import packetizer
from symphonia_b200.engine import SymgpuError
from oracle import caf_alac_oracle as cao
from tests import _caf_corpus

CORPUS = _caf_corpus.corpus()


def _mutants(seed=3):
    """The corpus files with bytes changed in their headers and packet tables, cut short, and with chunks swapped."""
    rng = np.random.default_rng(seed)
    out = []
    for _, data, _ in CORPUS:
        if len(data) < 16:
            continue
        for k in range(25):
            b = bytearray(data)
            head = min(len(b), 400)
            if k % 5 == 4:
                b = b[:int(rng.integers(0, len(b)))]
            else:
                for _ in range(int(rng.integers(1, 4))):
                    i = int(rng.integers(0, head))
                    b[i] = int(rng.integers(0, 256)) if k % 2 else b[i] ^ (1 << int(rng.integers(8)))
            out.append(bytes(b))
    return out


def host_vs_oracle(data):
    """None when the host index and the Python oracle agree on the file's open status, reason, fields and packets."""
    st, reason, fields, packets = cao.open_caf(data)
    try:
        info, got = packetizer.caf_index(data)
        rc = 0
    except SymgpuError as e:
        rc, info, got = e.status, None, []
    if rc != {cao.OK: 0, cao.DECODE: 1, cao.UNSUPPORTED: 2}[st]:
        return f"status {rc} != {st} (reason {reason})"
    if st != cao.OK:
        return None
    for k, v in fields.items():
        if int(info[k]) != v:
            return f"{k}: {int(info[k])} != {v}"
    if [(int(p["offset"]), int(p["size"])) for p in got] != packets:
        return "packets differ"
    return None


def test_host_index_equals_the_python_oracle():
    files = [c[1] for c in CORPUS] + _mutants()
    bad = [(i, m) for i, m in ((i, host_vs_oracle(f)) for i, f in enumerate(files)) if m]
    assert not bad, bad[:5]
    reasons = {cao.open_caf(f)[1] for f in files}
    assert len(reasons) >= 8, reasons


@pytest.mark.parametrize("name,data,expect", CORPUS, ids=[c[0] for c in CORPUS])
def test_index_finds_the_written_packets(name, data, expect):
    if expect is None:
        with pytest.raises(SymgpuError):
            packetizer.caf_index(data)
        return
    info, packets = packetizer.caf_index(data)
    ck = expect["cookie"]
    for k in ("frame_length", "bit_depth", "pb", "mb", "kb", "channels"):
        assert int(info[k]) == ck[k], k
    assert int(info["n_packets"]) == len(expect["packets"]) == len(packets)
    for p, want in zip(packets, expect["packets"]):
        assert data[int(p["offset"]):int(p["offset"]) + int(p["size"])] == want
        assert int(p["frames"]) == ck["frame_length"]


def test_variable_length_integer_known_answers():
    # chunks.rs:633-651
    for b, v in (([0x01], 1), ([0x11], 17), ([0x7F], 127), ([0x81, 0x00], 128), ([0x81, 0x02], 130), ([0x82, 0x01], 257), ([0xFF, 0x7F], 16383),
                 ([0x81, 0x80, 0x00], 16384)):
        assert _caf_corpus.varint(v) == bytes(b)
        ck = dict(frame_length=16, channels=1, bit_depth=16, pb=40, mb=10, kb=14)
        from tests import _alac_bitstream as ab
        data = _caf_corpus.caf([_caf_corpus.desc(ck), _caf_corpus.chunk(b"kuki", ab.cookie_bytes(ck)),
                                _caf_corpus.chunk(b"pakt", bytes(7) + b"\x01" + bytes(16) + bytes(b)), _caf_corpus.chunk(b"data", bytes(4) + bytes(v))])
        info, packets = packetizer.caf_index(data)
        assert len(packets) == 1 and int(packets[0]["size"]) == v
    bad = _caf_corpus.caf([_caf_corpus.chunk(b"desc", bytes(8)), ])
    with pytest.raises(SymgpuError):
        packetizer.caf_index(bad)


def test_non_alac_message_names_the_reason():
    data = dict((c[0], c[1]) for c in CORPUS)["not_alac"]
    with pytest.raises(SymgpuError, match="not ALAC"):
        packetizer.caf_index(data)
