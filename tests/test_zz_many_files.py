"""Many files at once (`symphonia_b200.decode.plan_files` / `decode_files`): MPEG audio (Layers I-III), ADTS AAC-LC and Ogg Vorbis files
planned on host threads and merged into ONE synthesis batch per codec, every file a stream of its own.  CPU test: the merged
batches rendered by the synthesis and output oracles equal every file rendered alone (index re-basing of TNS records, floor tables,
runs, spans; residues re-padded to a common slot).  GPU test:
`decode_files` equals the same rendering byte for byte."""
import os

import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import decode
from tests import _oracle
from tests import test_zz_adts_aac_to_pcm as ta
from tests import test_zz_file_to_pcm as tm
from tests import test_zz_ogg_vorbis_to_pcm as tv


@pytest.fixture(scope="module")
def oracle():
    return _oracle.load()


def _files():
    files = list(tm._corpus()) + [blob for _, blob in tm._mpa12_corpus()]
    files += [ta._file(500, 44100, 2)[0], ta._file(502, 22050, 1)[0], ta._file(503, 8000, 2, n=5)[0]]
    hurt = bytearray(ta._file(504, 44100, 2, n=9)[0])          # an ADTS file with damaged payloads: frames the front-end may refuse
    for at in (len(hurt) // 3, len(hurt) // 2, 2 * len(hurt) // 3):
        hurt[at] ^= 0x5A
    files.append(bytes(hurt))
    files += [tv._file(300)[0], tv._file(305, channels=1)[0], tv._file(302, n_packets=9)[0]]
    # a second Vorbis block-size pair: slots differ inside one batch
    rng = np.random.default_rng(12)
    s = tv.vb.Stream(rng, bs_exp=(7, 10), per_word=1)
    pk = [s.packet()[0] for _ in range(8)]
    pages = tv.st.ogg_paginate(5, [s.ident], rng, eos=False) + tv.st.ogg_paginate(5, [b"\x03vorbis" + bytes(9), s.setup], rng, first_sequence=1, bos=False, eos=False)
    pages += tv.st.ogg_paginate(5, pk, rng, first_sequence=len(pages), bos=False, granule_of=[10 ** 9] * len(pk))
    files.append(b"".join(pages))
    # a Vorbis stream with three modes and, in the middle, an audio packet that names mode 3: valid pages, a packet the decoder refuses
    seed = 0
    while True:
        rng = np.random.default_rng(4000 + seed)
        s = tv.vb.Stream(rng, bs_exp=(8, 11), per_word=1)
        if len(s.modes) == 3:
            break
        seed += 1
    pk, gran, g = [], [], 0
    for k in range(10):
        b, t = s.packet()
        if k:
            g += ((1 << (11 if t["prev_block_flag"] else 8)) + (1 << (11 if t["block_flag"] else 8))) // 4
        pk.append(b), gran.append(g)
        if k == 4:
            pk.append(bytes([3 << 1]) + bytes(12)), gran.append(g)
    pages = tv.st.ogg_paginate(6, [s.ident], rng, eos=False) + tv.st.ogg_paginate(6, [b"\x03vorbis" + bytes(9), s.setup], rng, first_sequence=1, bos=False, eos=False)
    pages += tv.st.ogg_paginate(6, pk, rng, max_segments=7, first_sequence=len(pages), bos=False, granule_of=gran)
    files.append(b"".join(pages))
    order = np.random.default_rng(3).permutation(len(files))
    return [files[i] for i in order]


def _render_batches(oracle, batches):
    pcm = {}
    for kind, b in batches.items():
        n = len(b["members"])
        if kind == "mp3":
            rc, out, _ = _oracle.mp3_batch(oracle, b["units"], tm._spectra(b["quant"]), b["runs"], n)
        elif kind in ("mpa1", "mpa2"):
            rc, out, _ = _oracle.mpa12_batch(oracle, b["subbands"], b["runs"], n)
        elif kind == "aac":
            rc, out = _oracle.aac_batch(oracle, b["units"], b["tns"], b["coeffs"], b["runs"], n)
        else:
            rc, out = _oracle.vorbis_batch(oracle, dict(streams=b["streams"], floors=b["floors"], units=b["units"], floor_y=b["floor_y"],
                                                        residue=b["residue"], runs=b["runs"], slot=b["slot"]))
        assert rc == 0, kind
        pcm[kind] = out
    return pcm


def _alone(oracle, data, fmt):
    kind = decode.sniff(data)
    if kind == "vorbis":
        return tv._render(oracle, decode.ogg_vorbis_plan(data), fmt)
    if kind == "aac":
        return ta._render(oracle, decode.adts_aac_plan(data), fmt)
    return tm._decode_expect(oracle, data, fmt)[0]


def test_merged_batches_equal_files_alone(oracle):
    files = _files()
    assert {decode.sniff(f) for f in files} == {"mpa", "aac", "vorbis"}
    plans, batches = decode.plan_files(files, threads=4)
    assert set(batches) == {"mp3", "mpa1", "mpa2", "aac", "vorbis"}
    assert sorted(i for b in batches.values() for i in b["members"]) == list(range(len(files)))
    pcm = _render_batches(oracle, batches)
    for fmt in (nat.FMT_S16, nat.FMT_F32):
        got = decode.pack_files(plans, batches, pcm, lambda p, sp, ch, f, total: _oracle.pcm_pack(oracle, p, sp, ch, f, total), fmt)
        for i, data in enumerate(files):
            want = _alone(oracle, data, fmt)
            assert got[i][0].shape == want.shape, (i, plans[i]["kind"])
            assert (got[i][0].view(np.uint8) == want.view(np.uint8)).all(), (i, plans[i]["kind"])
            assert got[i][1] == plans[i]["sample_rate"]


def test_arena_reuse_leaves_nothing_behind(oracle):
    """The same staging memory for two different batches: the second plan equals a plan made in fresh memory."""
    files = _files()
    arena = decode.Arena()
    decode.plan_files(files, threads=4, arena=arena)
    other = [f for f in files[::-1] if decode.sniff(f) == "aac"][:3] + files[:4]
    _, a = decode.plan_files(other, threads=4, arena=arena)
    _, b = decode.plan_files(other, threads=4)
    assert set(a) == set(b)
    holes = 0
    for kind in a:
        for key, v in a[kind].items():
            w = b[kind][key]
            if key in ("coeffs", "residue", "floor_y"):      # payload of unused slots is never read: compare what the runs name
                f0, cnt = ("first_packet", "n_packets") if kind == "vorbis" else ("first_frame", "n_frames")
                for r in a[kind]["runs"]:
                    lo, hi = int(r[f0]), int(r[f0]) + int(r[cnt])
                    assert v[lo:hi].tobytes() == w[lo:hi].tobytes()
                if kind == "aac":
                    holes = len(v) - int(a[kind]["runs"][cnt].sum())
                continue
            assert (np.asarray(v).tobytes() == np.asarray(w).tobytes()) if isinstance(v, np.ndarray) else v == w, (kind, key)
    assert holes > 0                                     # the damaged file lost frames: its slice has an unused tail
    assert len(a["vorbis"]["units"]) > int(a["vorbis"]["runs"]["n_packets"].sum()) or not any(len(f) and f[:4] == b"OggS" for f in other)
    # and the host entry point's descriptor check accepts the whole extent, unused tails included
    import symphonia_b200 as sb
    u, t = a["aac"]["units"], a["aac"]["tns"]
    assert sb.lib().symgpu_aac_units_check(u.ctypes.data, t.ctypes.data if len(t) else None, len(t), len(u)) == 0


def test_thread_count_does_not_change_the_plan():
    files = _files()
    _, a = decode.plan_files(files, threads=1)
    _, b = decode.plan_files(files, threads=8)
    for kind in a:
        for key, v in a[kind].items():
            w = b[kind][key]
            assert (np.asarray(v).tobytes() == np.asarray(w).tobytes()) if isinstance(v, np.ndarray) else v == w, (kind, key)


@pytest.mark.gpu
def test_many_files_on_the_device(oracle):
    import symphonia_b200 as sb
    files = _files()
    with sb.Engine(0) as eng:
        for fmt in (nat.FMT_S16, nat.FMT_F32):
            got = decode.decode_files(eng, files, fmt, threads=4)
            for i, data in enumerate(files):
                want = _alone(oracle, data, fmt)
                assert got[i][0].shape == want.shape and (got[i][0].view(np.uint8) == want.view(np.uint8)).all(), i


def test_one_bad_file_does_not_take_the_batch_down(oracle):
    """Files that cannot be indexed or planned at all -- an Ogg stream that is not Vorbis, a native FLAC file, an ADTS stream with a
    channel configuration the front-end does not take -- become error plans; every other file of the request renders as it does alone."""
    good = _files()
    rng = np.random.default_rng(99)
    not_vorbis = b"".join(tv.st.ogg_paginate(9, [b"\x7fOpusHead" + bytes(11)], rng, eos=True))
    flac = b"fLaC" + bytes(200)
    aac6 = bytearray(ta._file(510, 44100, 2, n=3)[0])
    for at in range(0, len(aac6) - 7):                      # every ADTS header: channel_configuration 2 -> 6
        if aac6[at] == 0xFF and (aac6[at + 1] & 0xF6) == 0xF0 and ((aac6[at + 2] & 1) << 2 | aac6[at + 3] >> 6) == 2:
            aac6[at + 2] = (aac6[at + 2] & 0xFE) | 1
            aac6[at + 3] = (aac6[at + 3] & 0x3F) | (2 << 6)
    files = [not_vorbis] + good[:5] + [flac] + good[5:] + [bytes(aac6)]
    bad = {0, 6, len(files) - 1}
    plans, batches = decode.plan_files(files, threads=4)
    for i in bad:
        assert plans[i]["kind"] == "error" and plans[i]["error"], i
    assert sorted(i for b in batches.values() for i in b["members"]) == [i for i in range(len(files)) if i not in bad]
    pcm = _render_batches(oracle, batches)
    got = decode.pack_files(plans, batches, pcm, lambda p, sp, ch, f, total: _oracle.pcm_pack(oracle, p, sp, ch, f, total), nat.FMT_S16)
    for i, data in enumerate(files):
        if i in bad:
            assert got[i][0].shape[0] == 0
            continue
        want = _alone(oracle, data, nat.FMT_S16)
        assert got[i][0].shape == want.shape and (got[i][0].view(np.uint8) == want.view(np.uint8)).all(), (i, plans[i]["kind"])
