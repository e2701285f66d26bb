"""A codeword longer than ten bits is matched by the trie walk against the bit cache padded with zeros, and must then fit in
what the cache really holds (codebook.rs:366-369, bit.rs:1211-1250): a packet that ends one bit short of such a codeword
ends there -- nothing is consumed, the floor is unused or the residue stops.  Writer packets are cut exactly one bit short of
every codeword of more than ten bits that ends one bit past a byte boundary, and the front-end must equal the oracle on each."""
import numpy as np

from oracle import vorbis_frontend_oracle as vo
from symphonia_b200 import frontend
from tests import _vorbis_bitstream as vb
from tests.test_vorbis_frontend import _both


def test_long_codeword_one_bit_short_of_the_packet_end(monkeypatch):
    spans = []
    put = vb.Book.put

    def recording_put(self, w, entry):
        spans.append((w.n, 1 if self.entries == 1 else int(self.lens[entry])))
        put(self, w, entry)
    monkeypatch.setattr(vb.Book, "put", recording_put)
    cuts = 0
    for seed in range(80):
        s = vb.Stream(np.random.default_rng(8100 + seed))
        fe, o = frontend.VorbisFrontend(s.ident, s.setup), vo.VorbisFrontend(s.ident, s.setup)
        for k in range(25):
            spans.clear()
            pkt, _ = s.packet()
            for start, length in list(spans):
                end = start + length
                if length > 10 and end % 8 == 1:
                    _both(fe, o, pkt[:end // 8], fe.slot, (seed, k, end))
                    cuts += 1
        fe.close()
    assert cuts >= 20
