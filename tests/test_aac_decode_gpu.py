"""ADTS AAC-LC files decoded on the device, many per call (`decode.decode_aac_files`, symgpu_aac_decode_host / _dev): the same
samples as `decode_adts_aac` file by file, the host front-end's per-packet decisions, a launch count that does not grow with the
number of files, and argument errors that launch nothing."""
import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import decode, frontend
from symphonia_b200.engine import SymgpuError
from tests import _aac_corpus as corpus
from tests import _oracle

FORMATS = (nat.FMT_F32, nat.FMT_S16, nat.FMT_S24, nat.FMT_S32, nat.FMT_U8)


def _files():
    return [(name, corpus.adts(pk, rate, ch, seed=i), pk, rate, ch) for i, (name, pk, rate, ch) in enumerate(corpus.corpus())]


def _host_status(pk, rate, ch):
    """symgpu_aac_fe_decode packet by packet, in order: 0 decoded, 1 refused, 2 unsupported."""
    fe, out = frontend.AacFrontend(rate, ch), []
    for p in pk:
        try:
            fe.decode(p)
            out.append(nat.AAC_JOB_DECODED)
        except SymgpuError as e:
            out.append(nat.AAC_JOB_UNSUPPORTED if e.status == 2 else nat.AAC_JOB_REFUSED)
    fe.close()
    return out


@pytest.mark.gpu
def test_files_equal_the_one_file_decoder_in_every_format():
    import symphonia_b200 as sb
    files = _files()
    data = [f[1] for f in files]
    with sb.Engine(0) as eng:
        for fmt in FORMATS:
            want = []
            for d in data:
                eng.aac_streams_alloc(1)
                want.append(decode.decode_adts_aac(eng, d, fmt))
            stats = {}
            got = decode.decode_aac_files(eng, data, fmt, stats=stats)
            for (name, *_), (w, wr), (g, gr) in zip(files, want, got):
                assert gr == wr and g.shape == w.shape and g.dtype == w.dtype, (name, fmt)
                assert g.tobytes() == w.tobytes(), (name, fmt)
            assert stats["n_redecoded"] > 0
            at = 0
            for name, _, pk, rate, ch in files:
                assert list(stats["status"][at:at + len(pk)]) == _host_status(pk, rate, ch), name
                at += len(pk)


@pytest.mark.gpu
def test_one_file_against_the_oracle():
    import symphonia_b200 as sb
    oracle = _oracle.load()
    name, data, pk, rate, ch = _files()[0]
    plan = decode.adts_aac_plan(data)
    rc, pcm = _oracle.aac_batch(oracle, plan["units"], plan["tns"], plan["coeffs"], plan["runs"], 1)
    assert rc == 0
    want = _oracle.pcm_pack(oracle, pcm, plan["spans"], plan["channels"], nat.FMT_S16, plan["total_frames"])
    with sb.Engine(0) as eng:
        (got, got_rate), = decode.decode_aac_files(eng, [data], nat.FMT_S16)
    assert got_rate == rate and got.tobytes() == want.tobytes()


@pytest.mark.gpu
def test_no_noise_decodes_once_and_launches_do_not_grow_with_files():
    import symphonia_b200 as sb
    quiet = corpus.adts(corpus.quiet(), 44100, 1)
    noisy = [f[1] for f in _files()]
    with sb.Engine(0) as eng:
        stats = {}
        decode.decode_aac_files(eng, [quiet] * 5, stats=stats)
        assert stats["n_redecoded"] == 0 and (stats["status"] == nat.AAC_JOB_DECODED).all()
        counts = []
        for n in (8, 64):
            files = [noisy[i % len(noisy)] for i in range(n)]
            before = eng.launch_count
            decode.decode_aac_files(eng, files)
            counts.append(eng.launch_count - before)
        assert counts[0] == counts[1]


@pytest.mark.gpu
def test_device_variant_returns_views_equal_to_the_host_variant():
    import symphonia_b200 as sb
    import torch
    data = [f[1] for f in _files()]
    with sb.Engine(0) as eng:
        host = decode.decode_aac_files(eng, data, nat.FMT_S32)
        dev = decode.decode_aac_files(eng, data, nat.FMT_S32, device=True)
    base = None
    for (h, hr), (d, dr) in zip(host, dev):
        assert isinstance(d, torch.Tensor) and d.is_cuda and dr == hr
        if d.numel():
            base = base or d.untyped_storage().data_ptr()
            assert d.untyped_storage().data_ptr() == base
        assert d.cpu().numpy().tobytes() == h.tobytes()


@pytest.mark.gpu
def test_a_bad_file_does_not_stop_the_others():
    import symphonia_b200 as sb
    files = _files()
    good = files[0][1]
    six = corpus.adts(corpus.quiet(2), 44100, 1)
    six = bytearray(six)
    six[3] = (six[3] & 0x3F) | (2 << 6)          # channel configuration 6 (three bits across bytes 2 / 3)
    six[2] = (six[2] & 0xFE) | 1
    inputs = [b"not audio at all", good, bytes(six), good]
    with sb.Engine(0) as eng:
        errors = {}
        got = decode.decode_aac_files(eng, inputs, errors=errors)
        want = decode.decode_adts_aac(eng, good)
    assert set(errors) == {0, 2}
    for i in (0, 2):
        assert got[i][0].shape == (0, 0) and got[i][1] == 0
    for i in (1, 3):
        assert got[i][1] == want[1] and got[i][0].tobytes() == want[0].tobytes()


@pytest.mark.gpu
def test_argument_errors_launch_nothing():
    import symphonia_b200 as sb
    plan = decode.aac_files_plan([_files()[0][1]])
    with sb.Engine(0) as eng:
        eng.aac_streams_alloc(1)
        before = eng.launch_count
        jobs = plan["jobs"].copy()
        jobs["len"][0] = len(plan["data"]) + 1
        with pytest.raises(SymgpuError):
            eng.aac_decode_host(plan["data"], jobs, plan["groups"], nat.FMT_S16, plan["out_samples"])
        bad = plan["groups"].copy()
        bad["channels"] = 3
        with pytest.raises(SymgpuError):
            eng.aac_decode_host(plan["data"], plan["jobs"], bad, nat.FMT_S16, plan["out_samples"])
        with pytest.raises(SymgpuError):
            eng.aac_decode_host(plan["data"], plan["jobs"], plan["groups"], nat.FMT_S16, plan["out_samples"] - 1)
        slot = plan["groups"].copy()
        slot["slot"] = 5
        with pytest.raises(SymgpuError):
            eng.aac_decode_host(plan["data"], plan["jobs"], slot, nat.FMT_S16, plan["out_samples"])
        with pytest.raises(SymgpuError):
            eng.aac_decode_host(plan["data"], plan["jobs"], plan["groups"], 9, plan["out_samples"], out=np.zeros(plan["out_samples"], np.int16))
        assert eng.launch_count == before
