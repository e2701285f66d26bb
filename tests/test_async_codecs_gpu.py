"""Thread-safe submission for AAC, Layer I / II and Vorbis (symgpu_{aac,mpa12,vorbis}_submit / _wait) through the Engine
wrappers: one Python thread per stream submits its frames in order and waits for each one's PCM, all threads on ONE context, so
the context gathers the frames of different streams into shared launches.  Every frame is compared with the oracle bit for bit."""
import threading

import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import workloads
from tests import _oracle

ERR_DECODE, ERR_LIMIT, ERR_ARG = 1, 3, 6


def _per_stream_threads(n_streams, body):
    """Runs body(s, start_gate) on one thread per stream; start_gate() is a barrier every thread passes once, after submitting
    its first frame and before waiting for it, so that the first batch holds a frame of every stream."""
    gate = threading.Barrier(n_streams)
    errors = []

    def run(s):
        try:
            body(s, gate.wait)
        except BaseException as e:  # noqa: BLE001 - reported below
            gate.abort()
            errors.append((s, e))

    threads = [threading.Thread(target=run, args=(s,)) for s in range(n_streams)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors[:3]


def _aac_frame(units, tns, f):
    """Frame f's two units and the TNS filters they name, tns_first counted from the start of that list."""
    u = units[f].copy()
    parts, at = [], 0
    for c in range(2):
        n = int(u[c]["n_tns"])
        if n:
            first = int(u[c]["tns_first"])
            parts.append(tns[first:first + n])
            u[c]["tns_first"] = at
            at += n
    return u, (np.concatenate(parts) if parts else np.zeros(0, dtype=nat.AAC_TNS_DTYPE))


def _same(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


@pytest.mark.gpu
def test_aac_threads_share_launches(oracle):
    import symphonia_b200 as sb
    F = 6
    sets = [workloads.aac_batch(12, F, seed=9101, tns_prob=0.5), workloads.aac_batch(6, F, seed=9102, channels=1, tns_prob=0.5)]
    want = [_oracle.aac_batch(oracle, u, t, c, r, len(r))[1] for (u, t, c, r) in sets]
    streams = [(k, s) for k, (_, _, _, r) in enumerate(sets) for s in range(len(r))]  # context stream i = streams[i]
    got = {}
    with sb.Engine(0) as eng:
        eng.aac_streams_alloc(len(streams))

        def body(i, gate):
            k, s = streams[i]
            units, tns, coeffs, runs = sets[k]
            ch = int(runs[s]["channels"])
            for f in range(F):
                row = s * F + f
                u, t = _aac_frame(units, tns, row)
                if i == 3 and f == 2:  # a malformed unit is refused at submission and never reaches a batch
                    bad = u.copy()
                    bad[0]["window_sequence"] = 7
                    with pytest.raises(sb.SymgpuError) as e:
                        eng.aac_submit(i, bad, t, coeffs[row], ch)
                    assert e.value.status == ERR_DECODE
                ticket = eng.aac_submit(i, u, t, coeffs[row], ch)
                if f == 0:
                    gate()
                got[(i, f)] = eng.aac_wait(ticket)

        _per_stream_threads(len(streams), body)
        batches, frames = eng.async_stats(nat.CODEC_AAC)
        assert frames == len(streams) * F and batches < frames, (batches, frames)
        # a ticket is redeemed once; a second wait, or a wait of another codec, is an argument error
        u, t = _aac_frame(sets[0][0], sets[0][1], 0)
        ticket = eng.aac_submit(0, u, t, sets[0][2][0])
        with pytest.raises(sb.SymgpuError) as e:
            eng.vorbis_wait(ticket, 1024)
        assert e.value.status == ERR_ARG
        eng.aac_wait(ticket)
        with pytest.raises(sb.SymgpuError) as e:
            eng.aac_wait(ticket)
        assert e.value.status == ERR_ARG
    for i, (k, s) in enumerate(streams):
        ch = int(sets[k][3][s]["channels"])
        for f in range(F):
            assert _same(got[(i, f)][:ch], want[k][s * F + f, :ch]), (k, s, f)


@pytest.mark.gpu
def test_mpa12_threads_both_layers(oracle):
    import symphonia_b200 as sb
    F = 5
    sets = [workloads.mpa12_batch(6, F, layer=1, seed=9201), workloads.mpa12_batch(6, F, layer=2, seed=9202, channels=1)]
    want = [_oracle.mpa12_batch(oracle, sub, runs, len(runs))[1] for sub, runs in sets]
    streams = [(k, s) for k, (_, r) in enumerate(sets) for s in range(len(r))]
    got = {}
    with sb.Engine(0) as eng:
        eng.mp3_streams_alloc(len(streams))

        def body(i, gate):
            k, s = streams[i]
            sub, runs = sets[k]
            for f in range(F):
                ticket = eng.mpa12_submit(i, sub[s * F + f], int(runs[s]["channels"]))
                if f == 0:
                    gate()
                got[(i, f)] = eng.mpa12_wait(ticket)

        _per_stream_threads(len(streams), body)
        for codec in (nat.CODEC_MP1, nat.CODEC_MP2):
            batches, frames = eng.async_stats(codec)
            assert frames == 6 * F and batches < frames, (codec, batches, frames)
    for i, (k, s) in enumerate(streams):
        sub, runs = sets[k]
        n, ch = 32 * sub.shape[-1], int(runs[s]["channels"])
        for f in range(F):
            pcm = got[(i, f)]
            assert _same(pcm[:ch, :n], want[k][s * F + f, :ch, :n]), (k, s, f)
            assert not pcm[:, n:].any()


@pytest.mark.gpu
def test_vorbis_slots_of_two_block_size_pairs(oracle):
    """Streams with block sizes (256, 2048) and (128, 512), each in a slot configured with its own floor setups: the batch rows
    are 1024 floats, the packets' own slots 1024 and 256, and every unit's floor index is counted from its slot's floor_base."""
    import symphonia_b200 as sb
    F = 6
    sets = [workloads.vorbis_batch(6, F, seed=9301, bs_exp=(8, 11)), workloads.vorbis_batch(6, F, seed=9302, bs_exp=(7, 9), channels=1)]
    want = [_oracle.vorbis_batch(oracle, wl)[1] for wl in sets]
    streams = [(k, s) for k, wl in enumerate(sets) for s in range(len(wl["streams"]))]
    got = {}
    with sb.Engine(0) as eng:
        eng.vorbis_streams_alloc(len(streams))
        bases = [eng.vorbis_stream_configure(i, sets[k]["streams"][s], sets[k]["floors"]) for i, (k, s) in enumerate(streams)]
        assert bases == [nat.VORBIS_SLOT_FLOORS * i for i in range(len(streams))]

        def body(i, gate):
            k, s = streams[i]
            wl = sets[k]
            for f in range(F):
                row = s * F + f
                unit = wl["units"][row:row + 1].copy()
                floor = unit["floor"][0]
                unit["floor"][0] = np.where(floor == 0xFFFF, floor, floor + bases[i])
                if i == 2 and f == 3:  # a floor outside the slot's setups is refused at submission
                    bad = unit.copy()
                    bad["floor"][0, 0] = bases[i] + len(wl["floors"])
                    with pytest.raises(sb.SymgpuError) as e:
                        eng.vorbis_submit(i, bad, wl["floor_y"][row], wl["residue"][row])
                    assert e.value.status == ERR_DECODE
                ticket = eng.vorbis_submit(i, unit, wl["floor_y"][row], wl["residue"][row])
                if f == 0:
                    gate()
                got[(i, f)] = eng.vorbis_wait(ticket, wl["slot"])

        _per_stream_threads(len(streams), body)
        batches, frames = eng.async_stats(nat.CODEC_VORBIS)
        assert frames == len(streams) * F and batches < frames, (batches, frames)
        with pytest.raises(sb.SymgpuError) as e:  # slots beyond the reservation
            eng.vorbis_stream_configure(len(streams), sets[0]["streams"][0], sets[0]["floors"])
        assert e.value.status == ERR_LIMIT
    for i, (k, s) in enumerate(streams):
        wl = sets[k]
        ch = int(wl["streams"][s]["channels"])
        for f in range(F):
            row = s * F + f
            n = int(wl["out_len"][row])
            pcm = got[(i, f)]
            assert pcm.shape == (2, wl["slot"])
            assert _same(pcm[:ch, :n], want[k][row, :ch, :n]), (k, s, f)
            assert not pcm[:, n:].any()


@pytest.mark.gpu
def test_vorbis_slots_fill_the_reservation():
    """256 slots on one context take 256 configurations; the 257th slot does not exist."""
    import symphonia_b200 as sb
    wl = workloads.vorbis_batch(1, 1, seed=9401)
    with sb.Engine(0) as eng:
        eng.vorbis_streams_alloc(256)
        for i in range(256):
            assert eng.vorbis_stream_configure(i, wl["streams"][0], wl["floors"]) == 64 * i
        with pytest.raises(sb.SymgpuError) as e:
            eng.vorbis_stream_configure(256, wl["streams"][0], wl["floors"])
        assert e.value.status == ERR_LIMIT
