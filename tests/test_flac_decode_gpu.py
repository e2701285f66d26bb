"""FLAC decoded on the device (symgpu_flac_decode_*, decode.decode_flac_files): frame headers and Rice residuals in device code,
many files per call.  Every file must come out equal to decode.decode_flac (host front-end + restoration on the device) and to the
PCM the encoder started from (workloads.flac_batch, scaled to 32 bits as decode_flac scales it); damaged packets fed straight in
as jobs must be accepted or refused packet for packet as the host front-end decides."""
import numpy as np
import pytest

import symphonia_b200 as sb
from symphonia_b200 import _native as nat
from symphonia_b200 import decode, frontend, workloads
from tests import _flac_bitstream as fw
from tests.test_flac_entropy_shared import _damaged

pytestmark = pytest.mark.gpu


# ---- corpus ------------------------------------------------------------------------------------------------------------------

def _header(p):
    """(fields, header length) of a writer frame."""
    lead = p[4]
    ulen = 1 if lead < 0x80 else 2 if lead < 0xE0 else 3 if lead < 0xF0 else 4 if lead < 0xF8 else 5 if lead < 0xFC else 6 if lead < 0xFE else 7
    bs, sr = p[2] >> 4, p[2] & 15
    at = 4 + ulen
    bs_tail = p[at:at + {6: 1, 7: 2}.get(bs, 0)]
    at += len(bs_tail)
    sr_tail = p[at:at + {12: 1, 13: 2, 14: 2}.get(sr, 0)]
    at += len(sr_tail)
    assert fw.crc8(p[:at]) == p[at]
    return dict(bs=bs, bs_tail=bytes(bs_tail), sr=sr, sr_tail=bytes(sr_tail), ch=p[3] >> 4, bps=(p[3] >> 1) & 7), at + 1


def _reheader(p, number, by_sample=False, bs=None, bps_code=None):
    """The frame with a new header (blocking strategy, frame / sample number, block-size code, bps code) and both CRCs recomputed."""
    h, end = _header(p)
    if bs is not None:
        h["bs"], h["bs_tail"] = bs
    if bps_code is not None:
        h["bps"] = bps_code
    head = bytes([0xFF, 0xF8 | int(by_sample), h["bs"] << 4 | h["sr"], h["ch"] << 4 | h["bps"] << 1]) + fw.utf8_encode(number) + h["bs_tail"] + h["sr_tail"]
    body = head + bytes([fw.crc8(head)]) + p[end:-2]
    return body + fw.crc16(body).to_bytes(2, "big")


def _frames(seed, bps, channels, block, n_frames, force_po=None):
    """Writer frames in stream order (the short blocks flac_batch makes at every 7th frame moved to the end: the one place a
    fixed-blocksize stream may have one), and each frame's PCM [n, channels]."""
    rng = np.random.default_rng(seed)
    frames, subs, samples, expect = workloads.flac_batch(n_frames, block, seed=seed, bps=bps, channels=channels, return_pcm=True)
    order = [f for f in range(n_frames) if f % 7] + [f for f in range(n_frames) if f % 7 == 0][:1]
    pk, pcm = [], []
    for k, f in enumerate(order):
        ss = subs[int(frames[f]["first_subframe"]):int(frames[f]["first_subframe"]) + channels]
        pk.append(fw.write_frame(rng, frames[f], ss, samples, k, stream_bps=bps, force_po=force_po))
        n = int(ss[0]["n"])
        pcm.append(np.stack([expect[int(s["offset"]):int(s["offset"]) + n] for s in ss], axis=1))
    return pk, pcm


def _file(pk, pcm, bps, channels, block_min=None, block_max=None):
    sizes = [len(x) for x in pcm]
    info = fw.stream_info_block(block_min or max(sizes), block_max or max(sizes), 44100, channels, bps, sum(sizes), min(map(len, pk)), max(map(len, pk)))
    return fw.native_file(pk, info), np.concatenate(pcm) if pcm else np.zeros((0, channels), dtype=np.int32)


def _corpus():
    files = []
    # bit depths (with channel counts from 1 to 8 spread over them), sub-frame types, wasted bits, Rice / Rice2 / escapes
    for k, (bps, ch, block, n) in enumerate([(8, 1, 192, 8), (12, 2, 256, 15), (16, 2, 576, 15), (20, 3, 300, 6), (24, 2, 1152, 8), (32, 1, 256, 8),
                                              (16, 4, 64, 8), (16, 5, 64, 8), (24, 6, 128, 8), (16, 7, 64, 8), (16, 8, 64, 8)]):
        pk, pcm = _frames(100 + k, bps, ch, block, n)
        files.append(("bps %d, %d ch, block %d" % (bps, ch, block),) + _file(pk, pcm, bps, ch, block, block))
    # bits per sample from STREAMINFO only (bps code 0 in every frame header)
    for k, (bps, ch, block) in enumerate([(16, 2, 512), (24, 6, 128), (12, 1, 200)]):
        pk, pcm = _frames(200 + k, bps, ch, block, 8)
        pk = [_reheader(p, i, bps_code=0) for i, p in enumerate(pk)]
        files.append(("bps from STREAMINFO, %d bits" % bps,) + _file(pk, pcm, bps, ch, block, block))
    # partition orders up to the writer's limit and beyond it (LPC orders above block >> order are refused by both paths)
    for k, po in enumerate((8, 12)):
        pk, pcm = _frames(300 + k, 16, 1, 4096, 3, force_po=po)
        files.append(("partition order %d" % po,) + _file(pk, pcm, 16, 1, 4096, 4096))
    # every block-size code: 192, 576 << 0..3, 256 << 0..7, and the 8- and 16-bit explicit sizes
    codes = [(1, 192)] + [(2 + k, 576 << k) for k in range(4)] + [(8 + k, 256 << k) for k in range(8)] + [(6, 100), (7, 5000)]
    for code, block in codes:
        pk, pcm = _frames(400 + code, 16, 1, block, 2)
        p = pk[0]
        tail = bytes([block - 1]) if code == 6 else (block - 1).to_bytes(2, "big") if code == 7 else b""
        files.append(("block-size code %d" % code,) + _file([_reheader(p, 0, bs=(code, tail))], pcm[:1], 16, 1, block, block))
    # a variable-blocksize stream: blocking-strategy bit set, headers numbered by sample
    pk, pcm, at = [], [], 0
    for k, (block, ch_seed) in enumerate([(300, 1), (1000, 2), (64, 3), (4096, 4), (192, 5), (77, 6)]):
        p1, s1 = _frames(500 + ch_seed, 16, 2, block, 2)
        pk.append(_reheader(p1[0], at, by_sample=True))
        pcm.append(s1[0])
        at += len(s1[0])
    files.append(("variable block size",) + _file(pk, pcm, 16, 2, 64, 4096))
    return files


@pytest.fixture(scope="module")
def corpus():
    return _corpus()


@pytest.fixture(scope="module")
def eng():
    with sb.Engine(0) as e:
        yield e


# ---- 1. parity with the host path and with the encoder ------------------------------------------------------------------------

def test_parity_with_decode_flac_and_the_encoder(eng, corpus):
    got = decode.decode_flac_files(eng, [d for _, d, _ in corpus])
    assert len(got) == len(corpus)
    for (name, data, want), (pcm, rate) in zip(corpus, got):
        host, host_rate = decode.decode_flac(eng, data)
        assert rate == host_rate == 44100, name
        assert pcm.dtype == np.int32 and pcm.shape == host.shape and (pcm == host).all(), name
        if not name.startswith("partition order"):   # (LPC orders above block >> order are refused there by design)
            assert pcm.shape == want.shape and (pcm == want).all(), name
    # the corpus reaches what it claims to
    assignments, types = set(), set()
    for name, data, _ in corpus:
        plan = decode.flac_plan(data)
        assignments |= {int(a) for a in plan["frames"]["assignment"]}
        types |= {(int(s["type"]), int(s["order"]) if int(s["type"]) == nat.FLAC_FIXED else 0) for s in plan["subframes"]}
        assert len(plan["frames"]) > 0 or name == "partition order 12", name
    assert assignments == {0, 1, 2, 3}
    assert {(nat.FLAC_FIXED, o) for o in range(5)} <= types and (nat.FLAC_CONSTANT, 0) in types and (nat.FLAC_VERBATIM, 0) in types


# ---- 2. many files, one call --------------------------------------------------------------------------------------------------

def test_many_files_one_call(eng, corpus):
    files = [corpus[k % len(corpus)][1] for k in range(64)]
    before = eng.launch_count
    got = decode.decode_flac_files(eng, files, threads=4)
    launches_64 = eng.launch_count - before
    before = eng.launch_count
    decode.decode_flac_files(eng, files[:2])
    assert launches_64 == eng.launch_count - before                    # launches do not grow with the number of files
    for f, (pcm, rate) in zip(files, got):
        alone, _ = decode.decode_flac_files(eng, [f])[0]
        assert pcm.shape == alone.shape and (pcm == alone).all()


# ---- 3. damaged packets as jobs -----------------------------------------------------------------------------------------------

def _jobs_of(packets, slot, group=0):
    jobs = np.zeros(len(packets), dtype=nat.FLAC_JOB_DTYPE)
    jobs["offset"] = np.cumsum([0] + [len(p) for p in packets[:-1]])
    jobs["len"], jobs["group"], jobs["slot"] = [len(p) for p in packets], group, slot
    return b"".join(packets), jobs


def _same_as_front_end(eng, packets, bps, channels, max_block, slot=None):
    slot = slot or max(max_block, 1)
    data, jobs = _jobs_of(packets, slot)
    groups = np.zeros(1, dtype=nat.FLAC_GROUP_DTYPE)
    groups[0]["max_block"], groups[0]["bits_per_sample"], groups[0]["channels"] = max_block, bps, channels
    out, gf, status = eng.flac_decode_host(data, jobs, groups, channels * slot * len(packets))
    table = np.zeros(len(packets), dtype=nat.PIECE_DTYPE)
    table["offset"], table["len"] = jobs["offset"], jobs["len"]
    frames, infos, frame_of, subs, samples = frontend.flac_decode_packets(data, table, bps, channels, max_block)
    want_status = np.full(len(packets), nat.FLAC_JOB_REFUSED, dtype=np.uint8)
    want_status[frame_of] = nat.FLAC_JOB_DECODED
    assert status.tolist() == want_status.tolist()
    total = int(sum(int(subs[int(f["first_subframe"])]["n"]) for f in frames))
    assert int(gf[0]) == total
    if len(frames):
        restored = eng.flac_restore_host(frames, subs, samples.copy())
        want = decode.flac_interleave(dict(frames=frames, subframes=subs, total_frames=total, channels=channels), restored)
        assert (out[:total * channels].reshape(total, channels) == want).all()
    return len(frames)


def test_damaged_packets_match_the_front_end(eng):
    pk, _ = _frames(601, 16, 2, 576, 36)
    hit = _damaged(pk, 3)
    assert 8 < _same_as_front_end(eng, hit, 16, 2, 576) < 36                 # cut, flipped bits, moved sync, reserved codes
    assert _same_as_front_end(eng, pk, 16, 1, 576) == 0                       # more channels than the stream
    assert _same_as_front_end(eng, pk, 16, 2, 300) == 1                       # larger blocks than the stream (the short last one stays)
    no_bps = [_reheader(p, k, bps_code=0) if k % 2 else p for k, p in enumerate(pk)]
    assert 0 < _same_as_front_end(eng, no_bps, 0, 2, 576) <= len(pk) // 2 + 1     # bps neither in the frame nor in the stream
    assert _same_as_front_end(eng, pk[:6], 16, 8, 576) == 6                   # fewer channels than the stream: the other columns 0
    # a slot smaller than the block is its own status
    data, jobs = _jobs_of(pk[:4], 576)
    jobs["slot"][1] = 575
    groups = np.zeros(1, dtype=nat.FLAC_GROUP_DTYPE)
    groups[0]["max_block"], groups[0]["bits_per_sample"], groups[0]["channels"] = 576, 16, 2
    out, gf, status = eng.flac_decode_host(data, jobs, groups, 2 * 576 * 4)
    assert status.tolist() == [0, nat.FLAC_JOB_NO_ROOM, 0, 0] and int(gf[0]) == 3 * 576


# ---- 4. device-resident variant -----------------------------------------------------------------------------------------------

def test_device_resident_equals_host(eng, corpus):
    import torch
    files = [d for _, d, _ in corpus[:12]]
    host = decode.decode_flac_files(eng, files)
    dev = decode.decode_flac_files(eng, files, device=True)
    for (a, ra), (b, rb) in zip(host, dev):
        assert b.is_cuda and b.dtype == torch.int32 and ra == rb
        assert (b.cpu().numpy() == a).all()
    # a job outside the buffers it is given is INVALID on the device, the others decode
    pk, _ = _frames(701, 16, 2, 576, 3)
    data, jobs = _jobs_of(pk, 576)
    jobs = np.concatenate([jobs, jobs[:1]])
    jobs[-1]["offset"] = len(data) + 10
    jobs[1]["group"] = 5
    groups = np.zeros(1, dtype=nat.FLAC_GROUP_DTYPE)
    groups[0]["max_block"], groups[0]["bits_per_sample"], groups[0]["channels"] = 576, 16, 2
    d = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to(d)  # noqa: E731
    out, gf, st = torch.zeros(2 * 576 * 4, dtype=torch.int32, device=d), torch.zeros(1, dtype=torch.int64, device=d), torch.zeros(4, dtype=torch.uint8, device=d)
    data_t, jobs_t, groups_t = t(np.frombuffer(data, dtype=np.uint8).copy()), t(jobs), t(groups)
    torch.cuda.synchronize()
    eng.flac_decode_dev(data_t, jobs_t, groups_t, out, gf, st)
    eng.sync()
    assert st.cpu().tolist() == [0, nat.FLAC_JOB_INVALID, 0, nat.FLAC_JOB_INVALID]


# ---- 5. edge cases ------------------------------------------------------------------------------------------------------------

def test_edge_cases_and_argument_errors(eng, corpus):
    assert decode.decode_flac_files(eng, []) == []
    name, good, want = corpus[2]
    empty = fw.native_file([], fw.stream_info_block(576, 576, 44100, 2, 16, 0))
    pk, _ = _frames(801, 16, 2, 576, 4)
    refused = fw.native_file(pk, fw.stream_info_block(576, 576, 44100, 1, 16, 0))   # stereo frames in a mono stream: every frame refused
    errors = {}
    got = decode.decode_flac_files(eng, [good, empty, b"fLaC" + bytes(5), refused, b"OggS" + bytes(60), good], errors=errors)
    assert (got[0][0] == want).all() and (got[5][0] == want).all()
    assert got[1][0].shape == (0, 2) and got[1][1] == 44100
    assert got[3][0].shape == (0, 1) and got[3][1] == 44100
    assert got[2][0].shape == (0, 0) and got[2][1] == 0 and got[4][1] == 0 and sorted(errors) == [2, 4]
    assert decode.decode_flac(eng, refused)[0].shape == (0, 1) and decode.decode_flac(eng, empty)[0].shape == (0, 2)
    # the host variant checks everything before any launch
    data, jobs = _jobs_of(pk, 576)
    groups = np.zeros(2, dtype=nat.FLAC_GROUP_DTYPE)
    groups["max_block"], groups["bits_per_sample"], groups["channels"] = 576, 16, 2
    groups[1]["out_offset"] = 2 * 576 * 4
    cap = 2 * 576 * 8

    def case(cap=cap, status=6, **edit):
        j, g = jobs.copy(), groups.copy()
        for (table, row, field), value in edit.get("set", {}).items():
            (j if table == "job" else g)[row][field] = value
        if "job_groups" in edit:
            j["group"] = edit["job_groups"]
        return j, g, cap, status
    cases = [case(set={("job", 2, "offset"): len(data)}),                   # a job past the bytes
             case(set={("job", 3, "len"): int(jobs[3]["len"]) + 1}),        # one byte too long
             case(set={("job", 0, "group"): 2}),                            # a group that does not exist
             case(job_groups=[0, 1, 0, 1]),                                 # a group's jobs not consecutive
             case(set={("group", 1, "out_offset"): cap + 1}),               # a region that starts outside `out`
             case(set={("group", 0, "channels"): 9}),
             case(cap=2 * 576 * 4 - 1, status=3,                            # out_cap too small for group 0's four slots
                  set={("group", 1, "out_offset"): 0}),
             case(cap=2 * 576 * 4, status=3, job_groups=[0, 0, 1, 1],       # group 1's region ends past out_cap
                  set={("group", 1, "out_offset"): 2 * 576 * 3})]
    before = eng.launch_count
    for j, g, c, status in cases:
        with pytest.raises(sb.SymgpuError) as e:
            eng.flac_decode_host(data, j, g, c)
        assert e.value.status == status
    assert eng.launch_count == before
    got = decode.decode_flac_files(eng, [good])
    assert (got[0][0] == want).all()
