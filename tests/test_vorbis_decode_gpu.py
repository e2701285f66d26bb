"""Ogg Vorbis files decoded on the device, many per call (decode.decode_vorbis_files, symgpu_vorbis_decode_host / _dev): every
file equal to decode_ogg_vorbis byte for byte in every sample format, per-packet statuses equal to the host front-end's accept
list, one file against the synthesis and output-stage oracles, launch counts that do not grow with the number of files, the
device-resident variant, bad files next to good ones and argument errors that launch nothing.  The corpus is
tests/_vorbis_corpus.py."""
import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import decode
from tests import _oracle
from tests import _vorbis_corpus as corpus

pytestmark = pytest.mark.gpu

FORMATS = (nat.FMT_S16, nat.FMT_F32, nat.FMT_S24, nat.FMT_S32, nat.FMT_U8)


@pytest.fixture(scope="module")
def engine():
    import symphonia_b200 as sb
    with sb.Engine(0) as eng:
        yield eng


@pytest.fixture(scope="module")
def files():
    return [d for _, d in corpus.files()]


def _accepted(data):
    """The host front-end's accept list over the file's audio packets."""
    ix = decode.ogg_vorbis_index(data)
    _, _, _, keep = ix["fe"].decode_packets(ix["blob"], ix["table"])
    ix["fe"].close()
    ok = np.zeros(len(ix["table"]), dtype=bool)
    ok[keep] = True
    return ok


@pytest.mark.parametrize("fmt", FORMATS)
def test_every_file_equals_decode_ogg_vorbis(engine, files, fmt):
    stats = {}
    got = decode.decode_vorbis_files(engine, files, fmt, stats=stats)
    assert stats["n_setups"] == len(files) - 1      # two files share their headers
    for k, data in enumerate(files):
        want, rate = decode.decode_ogg_vorbis(engine, data, fmt)
        assert got[k][1] == rate and got[k][0].shape == want.shape, k
        assert got[k][0].dtype == want.dtype
        assert (got[k][0].view(np.uint8) == want.view(np.uint8)).all(), k
    status = stats["status"]
    want_status = np.concatenate([np.where(_accepted(d), nat.VORBIS_JOB_DECODED, nat.VORBIS_JOB_REFUSED) for d in files])
    assert (status == want_status).all()
    assert (status == nat.VORBIS_JOB_REFUSED).sum() >= 1 and (status == nat.VORBIS_JOB_DECODED).sum() > 200


def test_one_file_against_the_oracles(engine, files):
    orc = _oracle.load()
    data = files[2]
    plan = decode.ogg_vorbis_plan(data)
    wl = dict(streams=plan["stream"], floors=plan["floors"], units=plan["units"], floor_y=plan["floor_y"], residue=plan["residue"],
              runs=plan["runs"], slot=plan["slot"])
    rc, pcm = _oracle.vorbis_batch(orc, wl)
    assert rc == 0
    for fmt in (nat.FMT_F32, nat.FMT_S16):
        want = _oracle.pcm_pack(orc, pcm, plan["spans"], plan["channels"], fmt, plan["total_frames"])
        got, rate = decode.decode_vorbis_files(engine, [data], fmt)[0]
        assert rate == plan["sample_rate"] and got.shape == want.shape
        assert (got.view(np.uint8) == want.view(np.uint8)).all()


def test_launch_count_does_not_grow_with_files(engine, files):
    counts = []
    for n in (8, 64):
        batch = [files[k % len(files)] for k in range(n)]
        before = engine.launch_count
        decode.decode_vorbis_files(engine, batch, nat.FMT_S16)
        counts.append(engine.launch_count - before)
    assert counts[0] == counts[1] and counts[0] > 0


def test_device_variant_views_equal_the_host_variant(engine, files):
    import torch
    host = decode.decode_vorbis_files(engine, files, nat.FMT_S16)
    dev = decode.decode_vorbis_files(engine, files, nat.FMT_S16, device=True)
    base = None
    for (h, hr), (d, dr) in zip(host, dev):
        assert d.is_cuda and hr == dr
        assert (d.cpu().numpy() == h).all()
        if d.numel():
            storage = d.untyped_storage().data_ptr()
            assert base is None or storage == base
            base = storage
    assert isinstance(dev[0][0], torch.Tensor)


def test_a_bad_file_does_not_stop_the_others(engine, files):
    bad = [b"not an ogg file", files[0][:60], b"OggS" + bytes(40)]
    batch = [bad[0], files[0], bad[1], files[1], bad[2]]
    errors = {}
    got = decode.decode_vorbis_files(engine, batch, nat.FMT_S16, errors=errors)
    assert set(errors) == {0, 2, 4}
    for k in (0, 2, 4):
        assert got[k][1] == 0 and got[k][0].size == 0
    for k, i in ((1, 0), (3, 1)):
        want, rate = decode.decode_ogg_vorbis(engine, files[i], nat.FMT_S16)
        assert got[k][1] == rate and (got[k][0] == want).all()
    assert decode.decode_vorbis_files(engine, [bad[0]], nat.FMT_S16, errors={})[0][1] == 0


def test_argument_errors_launch_nothing(engine, files):
    plan = decode.vorbis_files_plan(files[:3])
    args = (plan["headers"], plan["setups"], plan["data"], plan["jobs"], plan["groups"], nat.FMT_S16, plan["out_samples"])

    def refused(*a, **kw):
        before = engine.launch_count
        with pytest.raises(Exception):
            engine.vorbis_decode_host(*a, **kw)
        assert engine.launch_count == before

    jobs = plan["jobs"].copy()
    jobs["offset"][1] = len(plan["data"])           # a job outside the bytes
    refused(*args[:3], jobs, *args[4:])
    groups = plan["groups"].copy()
    groups["setup"][0] = 7                            # no such setup
    refused(*args[:4], groups, *args[5:])
    groups = plan["groups"].copy()
    groups["n_jobs"][0] += 1                          # overlaps the next group
    refused(*args[:4], groups, *args[5:])
    refused(*args[:6], plan["out_samples"] - 1)       # the output does not fit
    setups = plan["setups"].copy()
    setups["setup_len"][0] -= 20                      # a setup the front-end refuses
    refused(args[0], setups, *args[2:])
    setups = plan["setups"].copy()
    setups["setup_offset"][0] = len(plan["headers"])  # a header outside the blob
    refused(args[0], setups, *args[2:])
    refused(*args[:5], 99, args[6])                   # unknown format


def test_a_job_outside_the_bytes_is_invalid_on_the_device(engine, files):
    import torch
    plan = decode.vorbis_files_plan(files[:3])
    groups, cap = plan["groups"], plan["out_samples"]
    out_h, res_h, status_h = engine.vorbis_decode_host(plan["headers"], plan["setups"], plan["data"], plan["jobs"], groups, nat.FMT_S16, cap)
    jobs = plan["jobs"].copy()
    k = int(groups[1]["first_job"]) + 1
    jobs["offset"][k] = len(plan["data"]) + 5
    dev = torch.device("cuda", engine.device)
    as_t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to(dev)  # noqa: E731
    data_t, jobs_t = as_t(plan["data"]), as_t(jobs)
    out = torch.zeros(cap, dtype=torch.int16, device=dev)
    results_t = torch.zeros(len(groups) * nat.VORBIS_RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    status_t = torch.empty(len(jobs), dtype=torch.uint8, device=dev)
    torch.cuda.current_stream(dev).synchronize()
    engine.vorbis_decode_dev(plan["headers"], plan["setups"], data_t, jobs_t, groups, nat.FMT_S16, out, results_t, status_t)
    engine.sync()
    status = status_t.cpu().numpy()
    results = results_t.cpu().numpy().view(nat.VORBIS_RESULT_DTYPE)
    assert status[k] == nat.VORBIS_JOB_INVALID
    assert (np.delete(status, k) == np.delete(status_h, k)).all()
    out = out.cpu().numpy()
    for g in (0, 2):   # the other files are untouched by it
        at, n = int(groups[g]["out_offset"]), int(res_h[g]["frames"]) * int(res_h[g]["channels"])
        assert results[g] == res_h[g] and (out[at:at + n] == out_h[at:at + n]).all()
    assert int(results[1]["packets"]) == int(res_h[1]["packets"]) - (status_h[k] == nat.VORBIS_JOB_DECODED)


def test_unnamed_jobs_and_empty_packets_are_refused(engine, files):
    plan = decode.vorbis_files_plan(files[:2])
    groups, cap = plan["groups"], plan["out_samples"]
    args = (plan["headers"], plan["setups"], plan["data"])
    out0, res0, status0 = engine.vorbis_decode_host(*args, plan["jobs"], groups, nat.FMT_S16, cap)
    # two jobs that no group names (an empty one and one with bytes): refused, and the groups' results do not move
    extra = np.zeros(2, dtype=nat.VORBIS_JOB_DTYPE)
    extra["len"][1] = 8
    out, res, status = engine.vorbis_decode_host(*args, np.concatenate([plan["jobs"], extra]), groups, nat.FMT_S16, cap)
    assert (status[-2:] == nat.VORBIS_JOB_REFUSED).all() and (status[:-2] == status0).all()
    assert (res == res0).all() and (out == out0).all()
    # an empty packet inside a file: refused before its packet-type bit, the file decodes one packet less
    k = int(groups[0]["first_job"]) + 2
    assert status0[k] == nat.VORBIS_JOB_DECODED
    jobs = plan["jobs"].copy()
    jobs["len"][k] = 0
    _, res, status = engine.vorbis_decode_host(*args, jobs, groups, nat.FMT_S16, cap)
    assert status[k] == nat.VORBIS_JOB_REFUSED and (np.delete(status, k) == np.delete(status0, k)).all()
    assert int(res[0]["packets"]) == int(res0[0]["packets"]) - 1
