"""File bytes in, gapless interleaved samples out: the public call for MPEG audio files (what a user of the reference does with
`MpaReader` + `MpaDecoder` + `copy_to_slice_interleaved`).  Packetiser and entropy front-end on the CPU (SURVEY §8f N2 / N1),
synthesis and the output stage (N3) on the GPU.  Every device entry point used here is part of the round-1 GPU parity suite."""
import numpy as np

from . import _native as nat
from . import frontend, packetizer


def mpeg_audio_plan(data):
    """CPU half: (kind, payload, runs, spans, sample_rate, channels, total_frames).  kind 3: payload = (units, quant); kind 1 / 2:
    payload = sub-band samples.  spans carry the packetiser's trims (encoder delay / padding from a LAME tag, or the end trim of
    an extrapolated length) and where every packet's surviving frames go in the output."""
    track, packets = packetizer.mpa_index(data)
    layer = int(track["layer"])
    if layer == 3:
        units, quant, frame_of, info = frontend.Mp3Frontend().decode_packets(data, packets)
        payload = (units.reshape(-1), quant)
        n, per = len(units), 1152 if int(info["granules"]) == 2 else 576
        runs = np.zeros(1, dtype=nat.MP3_RUN_DTYPE)
        runs[0] = (0, 0, n, int(info["granules"]), int(info["channels"]), 0)
    else:
        sub, frame_of, info = frontend.mpa12_decode_packets(data, packets, layer)
        payload = sub
        n, per = len(sub), 32 * sub.shape[-1]
        runs = np.zeros(1, dtype=nat.MPA12_RUN_DTYPE)
        runs[0] = (0, 0, n, int(info["channels"]), (0, 0, 0))
    kept = packets[frame_of]
    spans = np.zeros(n, dtype=nat.PCM_SPAN_DTYPE)
    spans["src"] = np.arange(n, dtype=np.uint64) * 2304          # every frame slot holds 2 planes of 1152 floats
    spans["plane_stride"], spans["frames"] = 1152, per
    spans["trim_start"] = np.minimum(kept["trim_start"], per)
    spans["trim_end"] = np.minimum(kept["trim_end"], per - spans["trim_start"])
    left = per - spans["trim_start"].astype(np.int64) - spans["trim_end"].astype(np.int64)
    spans["dst_frame"] = np.concatenate([[0], np.cumsum(left)[:-1]]).astype(np.uint64) if n else 0
    return layer, payload, runs, spans, int(info["sample_rate"]) if n else int(track["sample_rate"]), int(info["channels"]) if n else int(track["channels"]), int(left.sum())


def decode_mpeg_audio(engine, data, fmt=nat.FMT_S16, stream=0):
    """(samples [frames, channels] of `fmt`, sample_rate).  Layers I-III; one stream slot of `engine` is used and reset first."""
    layer, payload, runs, spans, rate, channels, total = mpeg_audio_plan(data)
    runs["stream"] = stream
    if len(spans) == 0:
        return np.zeros((0, channels), dtype=nat.FMT_NUMPY[fmt]), rate
    engine.mp3_stream_reset(stream)
    pcm = engine.mp3_synth_host_quantized(payload[0], payload[1], runs) if layer == 3 else engine.mpa12_synth_host(payload, runs)
    return engine.pcm_pack_host(pcm, spans, channels, fmt, total), rate


def ogg_logical_stream(data, serial=None):
    """(packets, blob, table) of one logical stream of an Ogg file: pages -> packets (symgpu_ogg_index), those of `serial` (by
    default the first packet's) and their bytes gathered back to back (table[k]: where packet k lies in blob).  ValueError for a
    file without packets.  Both Ogg mappings, Vorbis and FLAC, start from it."""
    packets, pieces = packetizer.ogg_index(data)
    if len(packets) == 0:
        raise ValueError("no Ogg packets")
    serial = int(packets["serial"][0]) if serial is None else serial
    mine = packets[packets["serial"] == serial]
    blob, table = packetizer.ogg_gather(data, mine, pieces)
    return mine, blob, table


def _stream_of(data, streams, i):
    """ogg_logical_stream(data) for file i of a many-file call, unless decode_any_files has already indexed it: then streams[i]
    is what that gave, or the exception it raised, raised again here."""
    stream = None if streams is None else streams[i]
    if isinstance(stream, Exception):
        raise stream
    return ogg_logical_stream(data) if stream is None else stream


def ogg_vorbis_index(data, serial=None):
    """Everything about a Vorbis-in-Ogg file short of decoding its audio packets: pages -> packets (symgpu_ogg_index), the logical
    stream gathered back to back, identification / setup headers, the front-end object (codebooks, floors, ...), per audio packet its
    place, duration, leading discard (mappings/vorbis.rs:45-107) and end trim against the page granule positions
    (symphonia-format-ogg/src/logical.rs:164-302)."""
    return _vorbis_index_of(ogg_logical_stream(data, serial))


def _vorbis_index_of(stream):
    """ogg_vorbis_index of a stream ogg_logical_stream has gathered."""
    mine, blob, table = stream
    off, ln = table["offset"].astype(np.int64), table["len"].astype(np.int64)
    padded = np.concatenate([blob, np.zeros(8, dtype=np.uint8)])
    b0, b1 = padded[off], padded[off + 1]                           # (bytes beyond a short packet are masked by `ln` below)
    ident_b = blob[off[0]:off[0] + ln[0]].tobytes()
    is_setup = (ln >= 7) & (b0 == 5)
    for k, c in enumerate(b"vorbis"):
        is_setup &= padded[off + 1 + k] == c
    is_setup[0] = False
    at = int(np.argmax(is_setup)) if is_setup.any() else None
    setup_b = blob[off[at]:off[at] + ln[at]].tobytes() if at is not None else None
    ident, n_modes, mask, fe = vorbis_open_headers(ident_b, setup_b)
    audio = np.nonzero((np.arange(len(mine)) > at) & (ln > 0) & ((b0 & 1) == 0))[0]
    heads = b0[audio].astype(np.uint16) | (np.where(ln[audio] > 1, b1[audio], 0).astype(np.uint16) << 8)
    dur, discard, _ = packetizer.vorbis_packet_durations(ident, n_modes, mask, None, heads=heads, lens=np.minimum(ln[audio], 2))
    dur, discard = dur.astype(np.int64), discard.astype(np.int64)
    trim_end = packetizer.ogg_page_end_trims(mine["page_sequence"][audio], mine["page_absgp"][audio], dur, discard).astype(np.int64)
    return dict(blob=blob, table=table[audio], ident=ident, fe=fe, discard=discard, trim_end=trim_end, headers=(ident_b, setup_b))


def vorbis_open_headers(ident_b, setup_b):
    """The checks ogg_vorbis_index makes of a stream's identification and setup packets (setup_b None: the stream has none),
    in its order and with its exceptions: (ident record, number of modes, long-block mask, VorbisFrontend on the two)."""
    ident = packetizer.vorbis_ident(ident_b)
    if setup_b is None:
        raise ValueError("no Vorbis setup header")
    n_modes, mask = packetizer.vorbis_setup_modes(setup_b, ident)
    return ident, n_modes, mask, frontend.VorbisFrontend(ident_b, setup_b)


def ogg_vorbis_plan(data, serial=None, index=None, out=None, slot=None, floor_base=0, threads=1):
    """CPU half for a Vorbis-in-Ogg file: ogg_vorbis_index, then the entropy front-end (symgpu_vorbis_fe_*) over the audio packets
    -> the synthesis stage's batch and the output spans with the reader's trims.  Returns dict(stream, floors, units, floor_y, residue,
    runs, slot, spans, channels, sample_rate, total_frames).  Packets the front-end refuses are dropped, as a caller of the reference
    drops a DecodeError.  index / out / slot / floor_base: for `plan_files` (decode into slices of a batch whose residue rows are
    `slot` long and whose floor tables start at `floor_base`)."""
    ix = ogg_vorbis_index(data, serial) if index is None else index
    fe, ident, discard, trim_end = ix["fe"], ix["ident"], ix["discard"], ix["trim_end"]
    slot = fe.slot if slot is None else slot
    if threads > 1 and out is None and len(ix["table"]) >= 32:   # one long stream: its packets as independent jobs (identical output, DESIGN 10.9)
        ju, jf, jr, keep = frontend.vorbis_decode_packets_jobs(ix["headers"][0], ix["headers"][1], ix["blob"], ix["table"], slot, floor_base, threads)
        units, fy, res = ju[keep], jf[keep], jr[keep]
    else:
        units, fy, res, keep = fe.decode_packets(ix["blob"], ix["table"], slot=slot, floor_base=floor_base, out=out)
    n = len(units)
    stream, floors = np.array([fe.stream], dtype=nat.VORBIS_STREAM_DTYPE), fe.floors.copy()
    fe.close()
    bs0, bs1 = 1 << int(ident["bs0_exp"]), 1 << int(ident["bs1_exp"])
    frames = (np.where(units["prev_block_flag"] != 0, bs1, bs0) + np.where(units["block_flag"] != 0, bs1, bs0)).astype(np.int64) // 4
    ts = np.minimum(discard[keep], frames)
    te = np.minimum(trim_end[keep], frames - ts)
    if n:
        ts[0], te[0] = frames[0], 0   # the first packet after a reset is silenced in gapless mode (codec-vorbis lib.rs:318-322)
    left = frames - ts - te
    spans = np.zeros(n, dtype=nat.PCM_SPAN_DTYPE)
    spans["src"] = np.arange(n, dtype=np.uint64) * (2 * slot)
    spans["plane_stride"], spans["frames"], spans["trim_start"], spans["trim_end"] = slot, frames, ts, te
    spans["dst_frame"] = np.concatenate([[0], np.cumsum(left)[:-1]]).astype(np.uint64) if n else 0
    total = int(left.sum())
    runs = np.zeros(1, dtype=nat.VORBIS_RUN_DTYPE)
    runs["n_packets"] = n
    return dict(stream=stream, floors=floors, units=units, floor_y=fy, residue=res, runs=runs, slot=slot, spans=spans,
                channels=int(ident["channels"]), sample_rate=int(ident["sample_rate"]), total_frames=total)


def decode_ogg_vorbis(engine, data, fmt=nat.FMT_S16, serial=None, threads=1):
    """(samples [frames, channels] of `fmt`, sample_rate) of one Vorbis logical stream (mono / stereo, floor 1: what the synthesis
    kernel takes).  Registers the stream as slot 0 of `engine` with its floors from index 0."""
    plan = ogg_vorbis_plan(data, serial, threads=threads)
    if len(plan["units"]) == 0:
        return np.zeros((0, plan["channels"]), dtype=nat.FMT_NUMPY[fmt]), plan["sample_rate"]
    engine.vorbis_streams_set(plan["stream"])
    engine.vorbis_floors_set(plan["floors"])
    pcm = engine.vorbis_synth_host(plan["units"], plan["floor_y"], plan["residue"], plan["runs"], plan["slot"])
    return engine.pcm_pack_host(pcm, plan["spans"], plan["channels"], fmt, plan["total_frames"]), plan["sample_rate"]


def _aac_refusal(n_frames, channels):
    """Why an ADTS stream of n_frames frames whose first frame has `channels` cannot be decoded, or None when it can."""
    if n_frames == 0:
        return "no ADTS frames"
    if channels not in (1, 2):
        return "channel configuration outside AAC-LC mono / stereo"


def adts_aac_index(data):
    """(packets, sample_rate, channels): the ADTS frame index and the stream's parameters (the first frame's, AdtsReader::try_new)."""
    packets, _ = packetizer.adts_index(data)
    rate, channels = (int(packets[0]["sample_rate"]), int(packets[0]["channels"])) if len(packets) else (0, 0)
    refusal = _aac_refusal(len(packets), channels)
    if refusal:
        raise ValueError(refusal)
    return packets, rate, channels


def adts_aac_plan(data, index=None, out=None, threads=1):
    """CPU half for an ADTS file: frames (symgpu_adts_index: header rules of adts.rs:130-309) -> raw_data_block payloads -> AAC-LC
    entropy front-end (symgpu_aac_fe_*) -> the synthesis stage's batch.  The reader gives every frame 1024 samples and trims
    nothing.  Returns dict(units [n,2], tns, coeffs [n,2,1024], runs, spans, channels, sample_rate, total_frames).  Packets the
    front-end refuses are dropped, as a caller of the reference drops a DecodeError.  index: the result of adts_aac_index (else
    computed here); out: (units, coeffs) staging slices with room for every packet; threads > 1: a stream of 32 blocks or more is
    decoded as independent jobs when it allows that."""
    packets, rate, channels = adts_aac_index(data) if index is None else index
    table = np.zeros(len(packets), dtype=nat.PIECE_DTYPE)
    table["offset"], table["len"] = packets["offset"], packets["size"]
    jobs = frontend.aac_decode_packets_jobs(rate, channels, data, table, threads=threads) if (threads > 1 and out is None and len(packets) >= 32) else None
    if jobs is not None:            # one long stream: its blocks as independent jobs on host threads (identical output, DESIGN 10.9)
        units, tns, coeffs = jobs
    else:                           # (or the stream needs the serial path: a refused block, a changed layout, ...)
        fe = frontend.AacFrontend(rate, channels)
        units, tns, coeffs, _ = fe.decode_packets(data, table, out=out)
        fe.close()
    n = len(units)
    runs = np.zeros(1, dtype=nat.AAC_RUN_DTYPE)
    runs[0]["n_frames"], runs[0]["channels"] = n, channels
    spans = np.zeros(n, dtype=nat.PCM_SPAN_DTYPE)
    spans["src"] = np.arange(n, dtype=np.uint64) * 2048
    spans["plane_stride"], spans["frames"] = 1024, 1024
    spans["dst_frame"] = np.arange(n, dtype=np.uint64) * 1024
    return dict(units=units, tns=tns, coeffs=coeffs, runs=runs, spans=spans, channels=channels, sample_rate=rate,
                total_frames=1024 * n)


class Arena:
    """Reusable staging memory for `plan_files`: take(name, shape, dtype) hands out a view of a buffer that persists across calls (and
    grows when too small), so that a serving loop's front-ends write into pages that are already mapped instead of paying the first
    touch of fresh allocations on every batch (DESIGN 5g).  Contents are whatever the last user left."""

    def __init__(self):
        self._buf = {}

    def take(self, name, shape, dtype):
        need = int(np.prod(shape, dtype=np.int64)) * np.dtype(dtype).itemsize
        b = self._buf.get(name)
        if b is None or b.size < need:
            b = np.zeros(max(need + need // 4, 1), dtype=np.uint8)
            b[::4096] = 0          # touch every page once, here
            self._buf[name] = b
        return b[:need].view(dtype).reshape(shape)


def decode_adts_aac(engine, data, fmt=nat.FMT_S16, stream=0, threads=1):
    """(samples [frames, channels] of `fmt`, sample_rate) of an ADTS AAC-LC file; stream slot `stream` of `engine` is reset first."""
    plan = adts_aac_plan(data, threads=threads)
    if len(plan["units"]) == 0:
        return np.zeros((0, plan["channels"]), dtype=nat.FMT_NUMPY[fmt]), plan["sample_rate"]
    plan["runs"]["stream"] = stream
    engine.aac_stream_reset(stream)
    pcm = engine.aac_synth_host(plan["units"], plan["tns"], plan["coeffs"], plan["runs"])
    return engine.pcm_pack_host(pcm, plan["spans"], plan["channels"], fmt, plan["total_frames"]), plan["sample_rate"]


# ---- many files at once: one synthesis launch per codec --------------------------------------------------------------------

def sniff(data):
    """'vorbis' (Ogg capture pattern), 'flac' (native FLAC marker), 'alac' (CAF marker), 'aac' (ADTS: 12 sync bits, layer field 00)
    or 'mpa' (anything else: the MPEG audio indexer looks for a frame, skipping tags and junk)."""
    head = bytes(data[:4])
    if head == b"OggS":
        return "vorbis"
    if head == b"fLaC":
        return "flac"  # the integer path has its own entry point (decode_flac); plan_files reports it as an error for that file
    if head == b"caff":
        return "alac"
    if len(head) >= 2 and head[0] == 0xFF and (head[1] & 0xF6) == 0xF0:
        return "aac"
    return "mpa"


def plan_file(data):
    """CPU half of one file: dict(kind, ...) -- kind 'mp3' / 'mpa1' / 'mpa2' / 'aac' / 'vorbis'."""
    kind = sniff(data)
    if kind == "vorbis":
        return dict(ogg_vorbis_plan(data), kind="vorbis")
    if kind == "aac":
        return dict(adts_aac_plan(data), kind="aac")
    if kind in ("flac", "alac"):
        raise ValueError(f"{'native FLAC' if kind == 'flac' else 'ALAC in CAF'} goes through the integer decoders (decode_flac_files, "
                         "decode_alac_files), not through the f32 synthesis batches")
    layer, payload, runs, spans, rate, channels, total = mpeg_audio_plan(data)
    return dict(kind={1: "mpa1", 2: "mpa2", 3: "mp3"}[layer], payload=payload, runs=runs, spans=spans, sample_rate=rate, channels=channels, total_frames=total)


def plan_files(files, threads=None, arena=None):
    """Plans every file (front-ends on `threads` host threads: the native calls release the interpreter lock) and merges the plans
    into one batch per codec, every file a stream of its own.  Returns (plans, batches): batches[kind] = dict(members = indices into
    `files`, first = each member's first unit in the batch, + the arrays of that codec's synthesis entry point).  AAC files are indexed
    first and then decoded straight into their slices of the batch arrays (taken from `arena` when given: reusable staging memory);
    a file whose front-end refuses packets leaves the tail of its slice unused -- runs name what is valid.
    A file that cannot be indexed or planned at all (an Ogg stream that is not Vorbis, more than two channels, floor 0, an ADTS channel
    configuration outside 1 / 2, a native FLAC file, ...) does not take the others down: its plan is dict(kind="error", error=<message>)
    with no spans, it is in no batch, and pack_files returns an empty result for it."""
    import concurrent.futures
    import os
    kinds = [sniff(f) for f in files]
    errors = {}

    def guarded(fn):
        def run(i):
            try:
                return fn(i)
            except Exception as e:  # noqa: BLE001 -- one bad file must not abort the batch; the message is kept in its plan
                errors[i] = f"{type(e).__name__}: {e}"
                return None
        return run

    def error_plan(i):
        return dict(kind="error", error=errors[i], spans=np.zeros(0, dtype=nat.PCM_SPAN_DTYPE), channels=0, sample_rate=0, total_frames=0)
    aac = [i for i, k in enumerate(kinds) if k == "aac"]
    with concurrent.futures.ThreadPoolExecutor(max_workers=threads or os.cpu_count()) as pool:
        index = dict(zip(aac, pool.map(guarded(lambda i: adts_aac_index(files[i])), aac)))
        aac = [i for i in aac if i not in errors]
        starts, total = {}, 0
        for i in aac:
            starts[i] = total
            total += len(index[i][0])
        take = arena.take if arena is not None else (lambda name, shape, dtype: np.zeros(shape, dtype=dtype))
        aac_units, aac_coeffs = take("aac_units", (total, 2), nat.AAC_UNIT_DTYPE), take("aac_coeffs", (total, 2, 1024), np.float32)
        vor = [i for i, k in enumerate(kinds) if k == "vorbis"]
        vindex = dict(zip(vor, pool.map(guarded(lambda i: ogg_vorbis_index(files[i])), vor)))
        vor = [i for i in vor if i not in errors]
        vstarts, vfloor, vtotal, nfl = {}, {}, 0, 0
        for i in vor:
            vstarts[i], vfloor[i] = vtotal, nfl
            vtotal += len(vindex[i]["table"])
            nfl += len(vindex[i]["fe"].floors)
        vslot = max([vindex[i]["fe"].slot for i in vor], default=0)
        v_units, v_fy = take("vorbis_units", (vtotal,), nat.VORBIS_UNIT_DTYPE), take("vorbis_floor_y", (vtotal, 2, 65), np.uint16)
        v_res = take("vorbis_residue", (vtotal, 2, vslot), np.float32)

        def plan(i):
            if i in errors:
                return error_plan(i)
            if kinds[i] == "vorbis":
                a, n = vstarts[i], len(vindex[i]["table"])
                p = ogg_vorbis_plan(files[i], index=vindex[i], out=(v_units[a:a + n], v_fy[a:a + n], v_res[a:a + n]), slot=vslot, floor_base=vfloor[i])
                tail = v_units[a + len(p["units"]):a + n].view(np.uint8)
                tail[...] = 0
                return dict(p, kind="vorbis", slice_start=a)
            if kinds[i] != "aac":
                return plan_file(files[i])
            a, n = starts[i], len(index[i][0])
            p = adts_aac_plan(files[i], index[i], out=(aac_units[a:a + n], aac_coeffs[a:a + n]))
            aac_units[a + len(p["units"]):a + n].view(np.uint8)[...] = 0   # refused packets: the unused tail holds valid (empty) records
            return dict(p, kind="aac", slice_start=a)
        plans = list(pool.map(guarded(plan), range(len(files))))
    for i, p in enumerate(plans):
        if p is None:  # failed in the plan stage: its slice of the batch arrays stays empty records, its front-end is released now
            plans[i] = error_plan(i)
            if kinds[i] == "vorbis" and i in vindex and vindex[i] is not None and hasattr(vindex[i].get("fe"), "close"):
                vindex[i]["fe"].close()
            if kinds[i] == "vorbis" and i in vstarts:
                a, n = vstarts[i], len(vindex[i]["table"])
                v_units[a:a + n].view(np.uint8)[...] = 0
            if kinds[i] == "aac" and i in starts:
                a, n = starts[i], len(index[i][0])
                aac_units[a:a + n].view(np.uint8)[...] = 0
    batches = {}
    for kind in ("mp3", "mpa1", "mpa2", "aac", "vorbis"):
        members = [i for i, p in enumerate(plans) if p["kind"] == kind and len(p["spans"])]
        if not members:
            continue
        first, at = [], 0
        for i in members:
            first.append(at)
            at += len(plans[i]["spans"])
        b = dict(members=members, first=first)
        if kind == "mp3":
            b["units"] = np.concatenate([plans[i]["payload"][0] for i in members])
            b["quant"] = np.concatenate([plans[i]["payload"][1] for i in members])
            runs = np.concatenate([plans[i]["runs"] for i in members])
        elif kind in ("mpa1", "mpa2"):
            b["subbands"] = np.concatenate([plans[i]["payload"] for i in members])
            runs = np.concatenate([plans[i]["runs"] for i in members])
        elif kind == "aac":
            base = 0
            for i in members:                                  # the units already lie in the batch array: re-base their TNS references
                u = plans[i]["units"]
                u["tns_first"] = np.where(u["n_tns"] > 0, u["tns_first"] + base, 0)
                base += len(plans[i]["tns"])
            b["first"] = first = [plans[i]["slice_start"] for i in members]
            b["units"], b["coeffs"] = aac_units, aac_coeffs
            b["tns"] = np.concatenate([plans[i]["tns"] for i in members])
            runs = np.concatenate([plans[i]["runs"] for i in members])
        else:
            b["first"] = first = [plans[i]["slice_start"] for i in members]
            b["streams"] = np.concatenate([plans[i]["stream"] for i in members])
            b["floors"] = np.concatenate([vindex[i]["fe"].floors for i in vor])      # every Vorbis file's tables, in file order (floor_base)
            b["units"], b["floor_y"], b["residue"], b["slot"] = v_units, v_fy, v_res, vslot
            runs = np.concatenate([plans[i]["runs"] for i in members])
        runs = runs.copy()
        runs["stream"] = np.arange(len(members))
        runs["first_packet" if kind == "vorbis" else "first_frame"] = first
        b["runs"] = runs
        batches[kind] = b
    return plans, batches


def _file_spans(plan, batch, k, unit_floats, plane_stride=None):
    """The file's spans, re-based onto its slice of the batch's PCM (unit_floats per unit)."""
    sp = plan["spans"].copy()
    sp["src"] = np.arange(len(sp), dtype=np.uint64) * unit_floats
    if plane_stride is not None:
        sp["plane_stride"] = plane_stride
    return sp


def pack_files(plans, batches, pcm, pack, fmt):
    """Output stage per file: pcm[kind] = the batch's planar output, pack(pcm_slice, spans, channels, fmt, total_frames) the packer."""
    out = [None] * len(plans)
    for i, p in enumerate(plans):
        if not len(p["spans"]):
            out[i] = (np.zeros((0, p["channels"]), dtype=nat.FMT_NUMPY[fmt]), p["sample_rate"])
    for kind, b in batches.items():
        flat = np.ascontiguousarray(pcm[kind]).reshape(-1)
        per = flat.size // len(pcm[kind])          # floats per unit: two planes
        for k, i in enumerate(b["members"]):
            p = plans[i]
            n = len(p["spans"])
            sl = flat[b["first"][k] * per:(b["first"][k] + n) * per]
            sp = _file_spans(p, b, k, per, per // 2)
            out[i] = (pack(sl, sp, p["channels"], fmt, p["total_frames"]), p["sample_rate"])
    return out


def decode_files(engine, files, fmt=nat.FMT_S16, threads=None):
    """[(samples [frames, channels], sample_rate)] for a list of MPEG audio / ADTS AAC-LC / Ogg Vorbis files: front-ends on host threads,
    ONE synthesis launch per codec over all files (every file a stream), output stage per file.  (Re)allocates the engine's stream
    slots."""
    plans, batches = plan_files(files, threads)
    pcm = {}
    for kind, b in batches.items():
        n_streams = len(b["members"])
        if kind == "mp3":
            engine.mp3_streams_alloc(n_streams)
            pcm[kind] = engine.mp3_synth_host_quantized(b["units"], b["quant"], b["runs"])
        elif kind in ("mpa1", "mpa2"):
            engine.mp3_streams_alloc(n_streams)
            pcm[kind] = engine.mpa12_synth_host(b["subbands"], b["runs"])
        elif kind == "aac":
            engine.aac_streams_alloc(n_streams)
            pcm[kind] = engine.aac_synth_host(b["units"], b["tns"], b["coeffs"], b["runs"])
        else:
            engine.vorbis_streams_set(b["streams"])
            engine.vorbis_floors_set(b["floors"])
            pcm[kind] = engine.vorbis_synth_host(b["units"], b["floor_y"], b["residue"], b["runs"], b["slot"])
    return pack_files(plans, batches, pcm, engine.pcm_pack_host, fmt)


# ---- FLAC (integer path: restoration on the GPU, samples int32 as in the reference's AudioBuffer<i32> until the output stage) -----

def flac_plan(data):
    """CPU half for a native FLAC file: marker + STREAMINFO + checksum-validated frame split (symgpu_flac_index), frame / sub-frame / Rice
    reader (symgpu_flac_fe_decode_packets) -> dict(frames, subframes, samples (int32: warm-up samples + residuals), info, channels,
    sample_rate, bits_per_sample, total_frames): the input of Engine.flac_restore_host."""
    info, packets = packetizer.flac_index(data)
    table = np.zeros(len(packets), dtype=nat.PIECE_DTYPE)
    table["offset"], table["len"] = packets["offset"], packets["size"]
    frames, infos, frame_of, subs, samples = frontend.flac_decode_packets(data, table, int(info["bits_per_sample"]), int(info["channels"]), int(info["block_max"]))
    total = int(sum(int(subs[int(f["first_subframe"])]["n"]) for f in frames))
    return dict(frames=frames, subframes=subs, samples=samples, info=info, channels=int(info["channels"]), sample_rate=int(info["sample_rate"]),
                bits_per_sample=int(info["bits_per_sample"]), total_frames=total)


def flac_interleave(plan, restored):
    """[total_frames, channels] int32 from the restored planes (each sub-frame's n samples at its offset), frames in stream order."""
    out = np.zeros((plan["total_frames"], plan["channels"]), dtype=np.int32)
    at = 0
    for f in plan["frames"]:
        first = int(f["first_subframe"])
        n = int(plan["subframes"][first]["n"])
        for c in range(int(f["channels"])):
            sf = plan["subframes"][first + c]
            out[at:at + n, c] = restored[int(sf["offset"]):int(sf["offset"]) + n]
        at += n
    return out


def flac_convert(samples, fmt):
    """The decoder's int32 samples (scaled to 32 bits) as `fmt`, as the reference's FromSample<i32> converts them
    (symphonia-core/src/audio/conv.rs:516-531) -- every case exact:  s32: s;  s24: s >> 8 (in an int32, as the f32 output stage
    stores s24);  s16: (s >> 16) as i16;  u8: ((s as u32).wrapping_add(0x8000_0000) >> 24) as u8;  f32: (s as f64 / 2^31) as f32."""
    s = np.asarray(samples, dtype=np.int32)
    if fmt == nat.FMT_S32:
        return s
    if fmt == nat.FMT_S24:
        return s >> 8
    if fmt == nat.FMT_S16:
        return (s >> 16).astype(np.int16)
    if fmt == nat.FMT_U8:
        return ((s.view(np.uint32) + np.uint32(0x80000000)) >> np.uint32(24)).astype(np.uint8)
    if fmt == nat.FMT_F32:
        return (s.astype(np.float64) / 2147483648.0).astype(np.float32)
    raise ValueError(f"unknown sample format {fmt}")


def decode_flac(engine, data, fmt=nat.FMT_S32):
    """(samples [frames, channels] of `fmt`, sample_rate): int32 scaled to 32 bits as the reference's FLAC decoder leaves them by
    default, any other format by flac_convert."""
    plan = flac_plan(data)
    if len(plan["frames"]) == 0:
        return np.zeros((0, plan["channels"]), dtype=nat.FMT_NUMPY[fmt]), plan["sample_rate"]
    restored = engine.flac_restore_host(plan["frames"], plan["subframes"], plan["samples"].copy())
    return flac_convert(flac_interleave(plan, restored), fmt), plan["sample_rate"]


# ---- many files per device call: the steps every codec's files path shares ---------------------------------------------------

_TORCH_DTYPES = {nat.FMT_F32: "float32", nat.FMT_S16: "int16", nat.FMT_S24: "int32", nat.FMT_S32: "int32", nat.FMT_U8: "uint8"}


def _index_files(files, index_fn, threads):
    """index_fn(file) of every file on `threads` host threads: ([index | None], {i: message}).  A file whose index_fn raises
    gets None and its message; the others are still indexed."""
    import concurrent.futures
    import os
    messages = {}

    def index(i):
        try:
            return index_fn(files[i])
        except Exception as e:  # noqa: BLE001 -- one bad file must not abort the batch; its message is kept
            messages[i] = f"{type(e).__name__}: {e}"
            return None
    with concurrent.futures.ThreadPoolExecutor(max_workers=threads or os.cpu_count()) as pool:
        ix = list(pool.map(index, range(len(files))))
    return ix, messages


def _packed(n_groups, good, sizes):
    """Every group's start when the good groups' sizes lie back to back in their order and a failed group starts at their end."""
    sizes = np.array(sizes, dtype=np.int64)
    starts = np.full(n_groups, sizes.sum(), dtype=np.int64)
    starts[good] = np.cumsum(sizes) - sizes
    return starts


def _place(groups, parts, first_job):
    """Lays out one call's groups.  parts: (i, n_jobs, fields, out samples) of every good file in order, which gets `fields`;
    out_offset is _packed (a failed file's group, in no part, gets the end of the output).  Where the record has them, a good
    group gets n_jobs and every group first_job[i], its start in the job table.  Returns (output total, failed files)."""
    good = [p[0] for p in parts]
    groups["out_offset"] = _packed(len(groups), good, [p[3] for p in parts])
    for k in parts[0][2] if parts else ():
        groups[k][good] = [p[2][k] for p in parts]
    if "first_job" in groups.dtype.names:
        groups["first_job"], groups["n_jobs"][good] = first_job, [p[1] for p in parts]
    placed = set(good)
    return sum(p[3] for p in parts), [i for i in range(len(groups)) if i not in placed]


def _batch(groups, parts, job_dtype):
    """One call's bytes, jobs and groups.  groups: one record per file, already holding what a failed file's group keeps;
    parts: (i, bytes, jobs, fields, out samples) of every good file in order, its jobs' offsets relative to its bytes; their
    bytes and jobs go back to back.  Returns (data, jobs, output total, failed files)."""
    srcs, byte_at = [], 0
    for _, src, j, _, _ in parts:
        src = np.frombuffer(src, dtype=np.uint8) if not isinstance(src, np.ndarray) else np.ascontiguousarray(src, dtype=np.uint8)
        j["offset"] += np.uint64(byte_at)
        srcs.append(src)
        byte_at += src.size
    out_at, failed = _place(groups, [(i, len(j), fields, n_out) for i, _, j, fields, n_out in parts],
                            _packed(len(groups), [p[0] for p in parts], [len(p[2]) for p in parts]))
    data = np.concatenate(srcs) if srcs else np.zeros(0, dtype=np.uint8)
    jobs = np.concatenate([p[2] for p in parts]) if parts else np.zeros(0, dtype=job_dtype)
    return data, jobs, out_at, failed


def _u8(device, count):
    import torch
    return torch.empty(int(count), dtype=torch.uint8, device=device)


def _decode_dev(engine, device, fmt, cap, n_groups, result_dtype, n_jobs, decode, read_status=True):
    """decode(out_t, results_t, status_t) -> extra queued on new tensors (`cap` samples of `fmt`, n_groups result_dtype records,
    n_jobs status bytes), a wait for the engine's stream, and the results (and with read_status the status) read back.  Returns
    (out_t, results, status or None, extra, bytes read back)."""
    import torch
    out = torch.empty(cap, dtype=getattr(torch, _TORCH_DTYPES[fmt]), device=device)
    results_t, status_t = _u8(device, n_groups * result_dtype.itemsize), _u8(device, n_jobs)
    extra = decode(out, results_t, status_t)
    engine.sync()
    results = results_t.cpu().numpy().view(result_dtype)
    status = status_t.cpu().numpy() if read_status else None
    return out, results, status, extra, results.nbytes + (status.nbytes if read_status else 0)


def _decode_batch(engine, device, inputs, cap, fmt, n_groups, result_dtype, host, dev):
    """One device call: host() -> (out, results, status, extra) on numpy arrays, or with device=True the `inputs` copied to the
    device and _decode_dev of dev(*inputs_t, out_t, results_t, status_t) -> extra, with a status byte per job of inputs[1].
    Returns (out, results, status, extra)."""
    if not device:
        return host()
    import torch
    d = torch.device("cuda", engine.device)
    staged = [torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to(d) for a in inputs]
    torch.cuda.current_stream(d).synchronize()  # the copies above are on torch's stream, the decode on the engine's
    return _decode_dev(engine, d, fmt, cap, n_groups, result_dtype, len(inputs[1]), lambda *outputs: dev(*staged, *outputs))[:4]


def _resident_files(data_t, ranges, name, limit):
    """The FILE_RANGE_DTYPE records of `ranges`, after the checks a call on device-resident files makes before any launch: at
    most `limit` files, data_t a contiguous uint8 CUDA tensor, every range inside it.  name: the call, for the messages."""
    import torch

    from .engine import file_ranges
    r = file_ranges(ranges)
    if len(r) > limit:
        raise ValueError(f"{name} takes at most {limit} files per call, not {len(r)}")
    if not (data_t.is_cuda and data_t.dtype == torch.uint8 and data_t.is_contiguous()):
        raise ValueError(f"{name} takes a contiguous uint8 CUDA tensor")
    size = data_t.numel()
    if ((r["offset"] > size) | (r["len"] > size - np.minimum(r["offset"], size))).any():
        raise ValueError(f"a file range lies outside the {size} bytes of data_t")
    return r


def _good_status(status, groups, failed):
    """The per-packet status of every group not in `failed`, in group order: what the host-indexed path's status holds."""
    failed = set(failed)
    runs = [status[int(g["first_job"]):int(g["first_job"]) + int(g["n_jobs"])] for k, g in enumerate(groups) if k not in failed]
    return np.concatenate(runs) if runs else np.zeros(0, dtype=np.uint8)


# each codec's group rule: from what the index says about one good file, (its group fields, its output samples)

def _aac_group(sample_rate, channels, n_packets):
    return dict(sample_rate=sample_rate, channels=channels), n_packets * 1024 * channels


def _mp3_group(track, n_packets):
    granules, channels = 2 if int(track["version"]) == 0 else 1, int(track["channels"])
    return dict(granules=granules, channels=channels), n_packets * granules * 576 * channels


def _mpa12_group(track, n_packets):
    layer = int(track["layer"])
    return dict(layer=layer), 2 * n_packets * (384 if layer == 1 else 1152)


def _vorbis_group(ident, n_packets, setup):
    return dict(setup=setup), n_packets * ((1 << int(ident["bs1_exp"])) >> 1) * int(ident["channels"])


def _aac_groups(n):
    """n AAC groups, group i on state slot i, each holding what a failed file's group keeps (mono, 44.1 kHz)."""
    groups = np.zeros(n, dtype=nat.AAC_GROUP_DTYPE)
    groups["slot"] = np.arange(n)
    groups["channels"], groups["sample_rate"] = 1, 44100
    return groups


def _vorbis_setups(pairs):
    """One setup per distinct (identification, setup) header pair of `pairs`: ([each pair's setup index],
    VORBIS_SETUP_REF_DTYPE records, the header bytes they point into)."""
    index, refs, headers, at = {}, [], [], 0
    for ident_b, setup_b in pairs:
        if (ident_b, setup_b) not in index:
            index[(ident_b, setup_b)] = len(refs)
            refs.append((at, at + len(ident_b), len(ident_b), len(setup_b)))
            headers += [ident_b, setup_b]
            at += len(ident_b) + len(setup_b)
    return [index[p] for p in pairs], np.array(refs, dtype=nat.VORBIS_SETUP_REF_DTYPE), b"".join(headers)


def _per_file(out, groups, failed, shape):
    """[(samples [frames, channels], sample_rate)] cut from `out` at each group's out_offset; shape(g) -> (frames, channels,
    sample_rate).  A failed file gives (out[:0].reshape(0, 0), 0)."""
    failed = set(failed)
    result = []
    for g in range(len(groups)):
        if g in failed:
            result.append((out[:0].reshape(0, 0), 0))
            continue
        n, ch, rate = shape(g)
        at = int(groups[g]["out_offset"])
        result.append((out[at:at + n * ch].reshape(n, ch), rate))
    return result


# ---- native FLAC, many files decoded on the device (frame headers and Rice residuals in device code) --------------------------

def flac_files_plan(files, threads=None, errors=None):
    """Host half of decode_flac_files: every file indexed (symgpu_flac_index, on `threads` host threads), their bytes concatenated
    once, one job per packet and one group per file.  Returns dict(data, jobs, groups, rates, out_cap, failed).  A file that cannot
    be indexed (listed in `failed`) gets a group without jobs; its message goes to errors[i] when `errors` is a dict."""
    ix, messages = _index_files(files, packetizer.flac_index, threads)
    if errors is not None:
        errors.update(messages)
    groups = np.zeros(len(files), dtype=nat.FLAC_GROUP_DTYPE)
    groups["channels"] = 1
    rates = np.zeros(len(files), dtype=np.int64)
    parts = []
    for i, x in enumerate(ix):
        if x is None:
            continue
        info, packets = x
        rates[i] = int(info["sample_rate"])
        j = np.zeros(len(packets), dtype=nat.FLAC_JOB_DTYPE)
        j["offset"], j["len"], j["group"], j["slot"] = packets["offset"], packets["size"], i, packets["dur"]
        fields = dict(max_block=int(info["block_max"]), bits_per_sample=int(info["bits_per_sample"]), channels=int(info["channels"]))
        parts.append((i, files[i], j, fields, int(packets["dur"].astype(np.int64).sum()) * int(info["channels"])))
    data, jobs, cap, failed = _batch(groups, parts, nat.FLAC_JOB_DTYPE)
    return dict(data=data, jobs=jobs, groups=groups, rates=rates, out_cap=cap, failed=failed)


def decode_flac_files(engine, files, threads=None, device=False, errors=None, fmt=nat.FMT_S32):
    """[(samples [frames, channels] of `fmt`, sample_rate)] for a list of native FLAC files, each equal to decode_flac(engine, file,
    fmt): the files are indexed on host threads, and ONE device call decodes every packet of every file -- frame headers and Rice
    residuals in device code (one thread per packet), restoration, and interleaving with the conversion to `fmt` (int32 scaled to
    32 bits by default) on the GPU.  device=True: the bytes go to the device once and the samples are CUDA tensors, views of one
    output tensor.  A file that cannot be indexed yields an empty result with sample rate 0 (its message in errors[i] when
    `errors` is a dict)."""
    plan = flac_files_plan(files, threads, errors)
    groups, rates, cap = plan["groups"], plan["rates"], plan["out_cap"]
    def dev(data_t, jobs_t, groups_t, out_t, frames_t, status_t):
        import torch
        engine.flac_decode_dev(data_t, jobs_t, groups_t, out_t, frames_t.view(torch.int64), status_t, fmt)
    out, group_frames, _, _ = _decode_batch(engine, device, (plan["data"], plan["jobs"], groups), cap, fmt, len(groups), np.dtype(np.int64),
                                            lambda: (*engine.flac_decode_host(plan["data"], plan["jobs"], groups, cap, fmt=fmt), None), dev)
    return _per_file(out, groups, plan["failed"], lambda g: (int(group_frames[g]), int(groups[g]["channels"]), int(rates[g])))


def decode_flac_files_dev(engine, data_t, ranges, fmt=nat.FMT_S32, errors=None, stats=None):
    """decode_flac_files(engine, files, device=True, fmt=fmt) for native FLAC files already in device memory: file i is
    data_t[offset : offset + len] of ranges[i] ((offset, len) pairs or FILE_RANGE_DTYPE records) in a uint8 CUDA tensor, and its
    result and its message in errors[i] are what decode_flac_files gives for those bytes.  The frames are found on the device
    (symgpu_flac_index_dev) into a job table the decode reads in place; only the per-file index records and stream infos, the
    frames written per file and the per-packet status come back to the host.  stats: a dict that receives `read_back_bytes`, every
    byte the call copies from the device.  At most 65 536 files."""
    import torch

    from .engine import SymgpuError
    r = _resident_files(data_t, ranges, "decode_flac_files_dev", nat.FLAC_MAX_FILES)
    n = len(r)
    if n == 0:
        return []
    dev = data_t.device
    # 1. every file's frames as jobs, the table sized by the bound (a frame is at least 8 bytes)
    _, jobs_t, ix, infos = engine._index_dev(engine.flac_index_dev_queue, data_t, r, None, nat.FLAC_MIN_FRAME, (None, nat.FLAC_JOB_DTYPE),
                                             (nat.FLAC_FILE_INDEX_DTYPE, nat.FLAC_STREAM_INFO_DTYPE))
    messages = {i: f"SymgpuError: {SymgpuError(int(ix['open'][i]), 'symgpu_flac_index')}" for i in range(n) if ix["open"][i]}
    if errors is not None:
        errors.update(messages)
    # 2. the groups, as flac_files_plan lays them out
    groups = np.zeros(n, dtype=nat.FLAC_GROUP_DTYPE)
    groups["channels"] = 1
    parts = []
    for i in range(n):
        if i not in messages:
            info = infos[i]
            fields = dict(max_block=int(info["block_max"]), bits_per_sample=int(info["bits_per_sample"]), channels=int(info["channels"]))
            parts.append((i, int(ix["n_packets"][i]), fields, int(ix["samples"][i]) * int(info["channels"])))
    out_at, failed = _place(groups, parts, None)
    # 3. the decode, on the job table in place
    n_jobs = int(ix["first_packet"][-1]) + int(ix["n_packets"][-1])
    groups_t = torch.from_numpy(groups.view(np.uint8).copy()).to(dev)
    torch.cuda.current_stream(dev).synchronize()   # the copy is on torch's stream, the decode on the engine's
    out, frames, _, _, read = _decode_dev(
        engine, dev, fmt, out_at, n, np.dtype(np.int64), n_jobs,
        lambda out_t, results_t, status_t: engine.flac_decode_dev(data_t, jobs_t[:n_jobs * nat.FLAC_JOB_DTYPE.itemsize], groups_t, out_t,
                                                                   results_t.view(torch.int64), status_t, fmt))
    if stats is not None:
        stats["read_back_bytes"] = ix.nbytes + infos.nbytes + read
    return _per_file(out, groups, failed, lambda g: (int(frames[g]), int(groups[g]["channels"]), int(infos["sample_rate"][g])))


# ---- ALAC in CAF, many files decoded on the device (elements, residuals and the adaptive predictor in device code) -------------

def alac_files_plan(files, threads=None, errors=None):
    """Host half of decode_alac_files: every CAF file indexed (packetizer.caf_index, on `threads` host threads), their bytes
    concatenated once, one job per packet (slot: the cookie's frame length) and one group per file.  Returns dict(data, jobs,
    groups, rates, infos, out_cap, failed).  A file that cannot be opened (listed in `failed`) gets a group without jobs; its
    message goes to errors[i] when `errors` is a dict."""
    ix, messages = _index_files(files, packetizer.caf_index, threads)
    if errors is not None:
        errors.update(messages)
    groups = np.zeros(len(files), dtype=nat.ALAC_GROUP_DTYPE)
    groups["channels"] = 1
    infos = np.zeros(len(files), dtype=nat.CAF_INFO_DTYPE)
    parts = []
    for i, x in enumerate(ix):
        if x is None:
            continue
        info, packets = x
        infos[i] = info
        j = np.zeros(len(packets), dtype=nat.FLAC_JOB_DTYPE)
        j["offset"], j["len"], j["group"], j["slot"] = packets["offset"], packets["size"], i, int(info["frame_length"])
        fields = {k: int(info[k]) for k in ("frame_length", "bit_depth", "pb", "mb", "kb", "channels")}
        parts.append((i, files[i], j, fields, len(packets) * int(info["frame_length"]) * int(info["channels"])))
    data, jobs, cap, failed = _batch(groups, parts, nat.FLAC_JOB_DTYPE)
    return dict(data=data, jobs=jobs, groups=groups, rates=infos["sample_rate"].astype(np.int64), infos=infos, out_cap=cap, failed=failed)


def decode_alac_files(engine, files, fmt=nat.FMT_S32, threads=None, device=False, errors=None, stats=None):
    """[(samples [frames, channels] of `fmt`, sample_rate)] for a list of CAF files holding ALAC: the files are indexed on host
    threads, and ONE device call decodes every packet of every file -- elements and adaptive Golomb residuals (one thread per
    packet), the adaptive predictor (one thread per channel of a packet), mid/side, tail bits and the conversion to `fmt` (int32
    scaled to 32 bits by default) on the GPU.  device=True: the bytes go to the device once and the samples are CUDA tensors,
    views of one output tensor.  A file that cannot be opened yields an empty result with sample rate 0 (its message in errors[i]
    when `errors` is a dict); a refused packet adds no frames, as a caller of the reference drops it.  No priming or remainder
    trim is applied: the reference's CAF reader applies none.  stats: a dict that receives `status`, the per-packet
    FLAC_JOB_* values in job order."""
    plan = alac_files_plan(files, threads, errors)
    groups, rates, cap = plan["groups"], plan["rates"], plan["out_cap"]

    def dev(data_t, jobs_t, groups_t, out_t, frames_t, status_t):
        import torch
        engine.alac_decode_dev(data_t, jobs_t, groups_t, out_t, frames_t.view(torch.int64), status_t, fmt)
    out, group_frames, status, _ = _decode_batch(engine, device, (plan["data"], plan["jobs"], groups), cap, fmt, len(groups), np.dtype(np.int64),
                                                 lambda: (*engine.alac_decode_host(plan["data"], plan["jobs"], groups, cap, fmt=fmt), None), dev)
    if stats is not None:
        stats["status"] = np.asarray(status)
    return _per_file(out, groups, plan["failed"], lambda g: (int(group_frames[g]), int(groups[g]["channels"]), int(rates[g])))


def _caf_message(info):
    """The message decode_alac_files gives for a file whose index record did not open."""
    from .engine import SymgpuError
    e = SymgpuError(int(info["open"]), f"symgpu_caf_index: {nat.CAF_REASONS.get(int(info['reason']), 'refused')}")
    return f"{type(e).__name__}: {e}"


def decode_alac_files_dev(engine, data_t, ranges, fmt=nat.FMT_S32, errors=None, stats=None):
    """decode_alac_files(engine, files, fmt, device=True) for CAF files already in device memory: file i is data_t[offset :
    offset + len] of ranges[i] ((offset, len) pairs or FILE_RANGE_DTYPE records) in a uint8 CUDA tensor, and its result, its
    message in errors[i] and its packets' status are what decode_alac_files gives for those bytes.  The chunks and packet tables
    are read on the device (Engine.caf_index_dev) into a job table the decode reads in place; only the per-file records, the
    frames written per file and the per-packet status come back.  stats: a dict that receives `status` and `read_back_bytes`,
    every byte the call copies from the device.  At most 65 536 files."""
    import torch
    r = _resident_files(data_t, ranges, "decode_alac_files_dev", nat.CAF_MAX_FILES)
    n = len(r)
    if n == 0:
        return []
    dev = data_t.device
    infos, first, _, jobs_t, read = engine.caf_index_dev(data_t, r)
    messages = {i: _caf_message(infos[i]) for i in range(n) if infos["open"][i]}
    if errors is not None:
        errors.update(messages)
    groups = np.zeros(n, dtype=nat.ALAC_GROUP_DTYPE)
    groups["channels"] = 1
    parts = []
    for i in range(n):
        if i not in messages:
            info = infos[i]
            fields = {k: int(info[k]) for k in ("frame_length", "bit_depth", "pb", "mb", "kb", "channels")}
            parts.append((i, int(info["n_packets"]), fields, int(info["n_packets"]) * int(info["frame_length"]) * int(info["channels"])))
    out_at, failed = _place(groups, parts, None)
    n_jobs = int(first[-1]) + int(infos["n_packets"][-1])
    groups_t = torch.from_numpy(groups.view(np.uint8).copy()).to(dev)
    torch.cuda.current_stream(dev).synchronize()   # the copy is on torch's stream, the decode on the engine's
    out, frames, status, _, read2 = _decode_dev(
        engine, dev, fmt, out_at, n, np.dtype(np.int64), n_jobs,
        lambda out_t, results_t, status_t: engine.alac_decode_dev(data_t, jobs_t[:n_jobs * nat.FLAC_JOB_DTYPE.itemsize], groups_t, out_t,
                                                                   results_t.view(torch.int64), status_t, fmt))
    if stats is not None:
        stats.update(status=status, read_back_bytes=read + read2)
    return _per_file(out, groups, failed, lambda g: (int(frames[g]), int(groups[g]["channels"]), int(infos["sample_rate"][g])))


# ---- FLAC in Ogg, many files decoded on the device (the native FLAC decoder on jobs made from the Ogg packets) ----------------

def _is_ogg_flac_ident(packet):
    """Whether a stream whose first packet is `packet` is FLAC in Ogg (mappings/flac.rs detect(): the 51-byte identification
    packet), whatever its STREAMINFO holds -- a refused STREAMINFO fails the file as Ogg FLAC, as the reference's reader fails.
    A packet of another length or lead-in (every Vorbis identification header) is decided without a library call."""
    from .engine import SymgpuError
    if len(packet) != nat.OGG_FLAC_IDENT_LEN or bytes(packet[:5]) != b"\x7fFLAC":
        return False
    table = np.zeros(1, dtype=nat.PIECE_DTYPE)
    table["len"] = len(packet)
    try:
        packetizer.ogg_flac_packets(packet, table)
    except SymgpuError as e:
        if e.status == 2:      # SYMGPU_ERR_UNSUPPORTED: not Ogg FLAC
            return False
        if e.status != 1:      # (SYMGPU_ERR_DECODE: Ogg FLAC whose STREAMINFO is refused)
            raise
    return True


def ogg_flac_index(data):
    """Everything about a FLAC-in-Ogg file short of decoding its frames (symphonia-format-ogg/src/mappings/flac.rs): the logical
    stream of the first packet's serial gathered back to back (ogg_logical_stream), its identification packet's STREAMINFO, and
    its audio packets -- dict(info, blob, table (where each audio packet lies in blob), slot (each one's block size from its
    frame header, 0 where the decoder refuses the header)).  Metadata packets carry no audio, and no Ogg granule trim applies:
    the reference's FLAC decoder has none.  ValueError without packets; SymgpuError status 2 when the stream is not Ogg FLAC, 1
    when its STREAMINFO is refused."""
    return _ogg_flac_index_of(ogg_logical_stream(data))


def _ogg_flac_index_of(stream):
    """ogg_flac_index of a stream ogg_logical_stream has gathered."""
    _, blob, table = stream
    info, audio, slot = packetizer.ogg_flac_packets(blob, table)
    return dict(info=info, blob=blob, table=table[audio], slot=slot[audio])


def _flac_fields(info):
    """A FLAC group's fields from STREAMINFO."""
    return dict(max_block=int(info["block_max"]), bits_per_sample=int(info["bits_per_sample"]), channels=int(info["channels"]))


def ogg_flac_files_plan(files, threads=None, errors=None):
    """Host half of decode_ogg_flac_files: every file indexed (ogg_flac_index, on `threads` host threads), the gathered logical
    streams concatenated once, one job per audio packet (slot: its block size) and one group per file, in decode_flac_files'
    layout.  Returns dict(data, jobs, groups, rates, out_cap, failed).  A file that cannot be indexed (listed in `failed`) gets a
    group without jobs; its message goes to errors[i] when `errors` is a dict."""
    return _ogg_flac_files_plan(files, threads, errors, None)


def _ogg_flac_files_plan(files, threads, errors, streams):
    """ogg_flac_files_plan; streams: as _stream_of takes them."""
    ix, messages = _index_files(range(len(files)), lambda i: _ogg_flac_index_of(_stream_of(files[i], streams, i)), threads)
    if errors is not None:
        errors.update(messages)
    groups = np.zeros(len(files), dtype=nat.FLAC_GROUP_DTYPE)
    groups["channels"] = 1
    rates = np.zeros(len(files), dtype=np.int64)
    parts = []
    for i, x in enumerate(ix):
        if x is None:
            continue
        info = x["info"]
        rates[i] = int(info["sample_rate"])
        j = np.zeros(len(x["table"]), dtype=nat.FLAC_JOB_DTYPE)
        j["offset"], j["len"], j["group"], j["slot"] = x["table"]["offset"], x["table"]["len"], i, x["slot"]
        parts.append((i, x["blob"], j, _flac_fields(info), int(x["slot"].astype(np.int64).sum()) * int(info["channels"])))
    data, jobs, cap, failed = _batch(groups, parts, nat.FLAC_JOB_DTYPE)
    return dict(data=data, jobs=jobs, groups=groups, rates=rates, out_cap=cap, failed=failed)


def decode_ogg_flac_files(engine, files, threads=None, device=False, errors=None, fmt=nat.FMT_S32, stats=None):
    """[(samples [frames, channels] of `fmt`, sample_rate)] for a list of FLAC-in-Ogg files (.oga, flac --ogg), each what
    decode_flac_files gives for a native FLAC file holding the same STREAMINFO and frames: the files are indexed on host threads,
    and ONE device call decodes every audio packet of every file with the native FLAC decoder (frame headers and Rice residuals
    in device code, restoration and interleaving with the conversion to `fmt` on the GPU).  Every frame the decoder accepts is
    output, back to back; no Ogg granule trim applies.  device=True: the bytes go to the device once and the samples are CUDA
    tensors, views of one output tensor.  A file that cannot be indexed -- no packets, not Ogg FLAC, a refused STREAMINFO --
    yields an empty result with sample rate 0 (its message in errors[i] when `errors` is a dict), and the others still decode.
    stats: a dict that receives the per-packet `status` (SYMGPU_FLAC_JOB_*).  At most 65 536 files per call."""
    return _decode_ogg_flac_files(engine, files, threads, device, errors, fmt, stats, None)


def _decode_ogg_flac_files(engine, files, threads, device, errors, fmt, stats, streams):
    """decode_ogg_flac_files; streams: as _stream_of takes them."""
    if len(files) > nat.FLAC_MAX_FILES:
        raise ValueError(f"decode_ogg_flac_files takes at most {nat.FLAC_MAX_FILES} files per call, not {len(files)}")
    plan = _ogg_flac_files_plan(files, threads, errors, streams)
    groups, rates, cap = plan["groups"], plan["rates"], plan["out_cap"]

    def dev(data_t, jobs_t, groups_t, out_t, frames_t, status_t):
        import torch
        engine.flac_decode_dev(data_t, jobs_t, groups_t, out_t, frames_t.view(torch.int64), status_t, fmt)
    out, group_frames, status, _ = _decode_batch(engine, device, (plan["data"], plan["jobs"], groups), cap, fmt, len(groups), np.dtype(np.int64),
                                                 lambda: (*engine.flac_decode_host(plan["data"], plan["jobs"], groups, cap, fmt=fmt), None), dev)
    if stats is not None:
        stats["status"] = status
    return _per_file(out, groups, plan["failed"], lambda g: (int(group_frames[g]), int(groups[g]["channels"]), int(rates[g])))


def _ogg_flac_refusal(status):
    """The message ogg_flac_index gives for a file whose device record has this status."""
    from .engine import SymgpuError
    if status == nat.OGG_FLAC_NO_PACKETS:
        return "ValueError: no Ogg packets"
    return f"SymgpuError: {SymgpuError(2 if status == nat.OGG_FLAC_NOT_FLAC else 1, 'symgpu_ogg_flac_packets')}"


def decode_ogg_flac_files_dev(engine, data_t, ranges, fmt=nat.FMT_S32, errors=None, stats=None):
    """decode_ogg_flac_files(engine, files, device=True, fmt=fmt) for FLAC-in-Ogg files already in device memory: file i is
    data_t[offset : offset + len] of ranges[i] ((offset, len) pairs or FILE_RANGE_DTYPE records) in a uint8 CUDA tensor, and its
    result, its message in errors[i] and `stats["status"]` are what decode_ogg_flac_files gives for those bytes.  The pages are
    indexed, the identification packets checked and every audio packet's job built on the device (symgpu_ogg_index_dev,
    symgpu_ogg_flac_heads_dev, symgpu_ogg_flac_jobs_dev), and the FLAC decode reads that job table in place; only the per-file
    records, the frames written per file and the per-packet status come back to the host.  stats also receives
    `read_back_bytes`, every byte the call copies from the device.  A constant number of launches and host waits per call.  At
    most 65 536 files."""
    import torch
    r = _resident_files(data_t, ranges, "decode_ogg_flac_files_dev", nat.FLAC_MAX_FILES)
    n = len(r)
    if n == 0:
        return []
    dev = data_t.device
    torch.cuda.current_stream(dev).synchronize()   # data_t is torch's: written on its stream
    index_t = _u8(dev, n * nat.OGG_FILE_INDEX_DTYPE.itemsize)
    engine.ogg_index_dev_queue(data_t, r, _u8(dev, 0), _u8(dev, 0), index_t)
    engine.sync()
    ix = index_t.cpu().numpy().view(nat.OGG_FILE_INDEX_DTYPE)
    n_packets, n_pieces = int(ix["first_packet"][-1]) + int(ix["n_packets"][-1]), int(ix["first_piece"][-1]) + int(ix["n_pieces"][-1])
    packets_t, pieces_t = _u8(dev, n_packets * nat.OGG_PACKET_DTYPE.itemsize), _u8(dev, n_pieces * nat.PIECE_DTYPE.itemsize)
    engine.ogg_index_dev_queue(data_t, r, packets_t, pieces_t, index_t)
    messages, kind_stats = {}, {}
    out = _ogg_flac_dev(engine, data_t, r, (packets_t, pieces_t, index_t), list(range(n)), fmt, messages, kind_stats)
    kind_stats["read_back_bytes"] += ix.nbytes
    if errors is not None:
        errors.update(messages)
    if stats is not None:
        stats.update(kind_stats)
    return out


def _ogg_flac_dev(engine, data_t, r, tables, mine, fmt, messages, stats):
    """The files r[mine] (indices rising) decoded as FLAC in Ogg from the page index tables (packets_t, pieces_t, index_t) that
    symgpu_ogg_index_dev wrote for all of r: one group per file of `mine`, the jobs built on the device and decoded in place.
    Returns the results in the order of `mine`; messages[k] and stats (`status`, `read_back_bytes`: the records, frames and
    status this reads back) as decode_ogg_flac_files_dev gives them."""
    import torch
    packets_t, pieces_t, index_t = tables
    dev, n = data_t.device, len(mine)
    group_of = np.full(len(r), nat.OGG_FLAC_NO_GROUP, dtype=np.uint32)
    group_of[mine] = np.arange(n)
    # 1. each file's identification packet and audio packets, the slots read from their frame headers
    heads_t = _u8(dev, n * nat.OGG_FLAC_FILE_DTYPE.itemsize)
    ranks_t = _u8(dev, packets_t.numel() // nat.OGG_PACKET_DTYPE.itemsize * nat.OGG_FLAC_PACKET_RANK_DTYPE.itemsize)
    engine.ogg_flac_heads_dev(data_t, r, packets_t, pieces_t, index_t, group_of, heads_t, ranks_t)
    engine.sync()
    heads = heads_t.cpu().numpy().view(nat.OGG_FLAC_FILE_DTYPE)
    messages.update({g: _ogg_flac_refusal(int(h["status"])) for g, h in enumerate(heads) if h["status"]})
    # 2. the groups, as ogg_flac_files_plan lays them out, and every audio packet's bytes and job
    groups = np.zeros(n, dtype=nat.FLAC_GROUP_DTYPE)
    groups["channels"] = 1
    parts = [(g, int(h["n_audio"]), _flac_fields(h["info"]), int(h["samples"]) * int(h["info"]["channels"])) for g, h in enumerate(heads) if not h["status"]]
    out_at, failed = _place(groups, parts, None)
    n_jobs, n_bytes = int(heads["n_audio"].astype(np.int64).sum()), int(heads["audio_bytes"].astype(np.int64).sum())
    audio_t, jobs_t = _u8(dev, n_bytes), _u8(dev, n_jobs * nat.FLAC_JOB_DTYPE.itemsize)
    engine.ogg_flac_jobs_dev(data_t, r, packets_t, pieces_t, index_t, group_of, ranks_t, audio_t, jobs_t)
    # 3. the decode, on the job table in place
    groups_t = torch.from_numpy(groups.view(np.uint8).copy()).to(dev)
    torch.cuda.current_stream(dev).synchronize()   # the copy is on torch's stream, the decode on the engine's
    out, frames, status, _, read = _decode_dev(
        engine, dev, fmt, out_at, n, np.dtype(np.int64), n_jobs,
        lambda out_t, results_t, status_t: engine.flac_decode_dev(audio_t, jobs_t, groups_t, out_t, results_t.view(torch.int64), status_t, fmt))
    stats.update(status=status, read_back_bytes=heads.nbytes + read)
    return _per_file(out, groups, failed, lambda g: (int(frames[g]), int(groups[g]["channels"]), int(heads["info"]["sample_rate"][g])))


# ---- MPEG Layer I / II, many files decoded on the device (header, side information and samples in device code) ----------------

def mpa_index_files(files, threads=None):
    """symgpu_mpa_index of every file on `threads` host threads: [(track, packets) | None], {i: message} for the files that cannot be
    indexed."""
    return _index_files(files, packetizer.mpa_index, threads)


def _keep_layers(ix, messages, layers, what):
    """The index with the files of other layers dropped (and their message added)."""
    ix = list(ix)
    for i, t in enumerate(ix):
        if t is not None and int(t[0]["layer"]) not in layers:
            messages[i] = f"ValueError: MPEG Layer {int(t[0]['layer'])}: {what}"
            ix[i] = None
    return ix


def _mpa_jobs(packets, job_dtype):
    """One job per indexed MPEG packet, its offset within the file and its trims (the end trim saturated to 32 bits)."""
    j = np.zeros(len(packets), dtype=job_dtype)
    j["offset"], j["len"] = packets["offset"], packets["size"]
    j["trim_start"] = packets["trim_start"]
    j["trim_end"] = np.minimum(packets["trim_end"].astype(np.uint64), np.uint64(0xFFFFFFFF))
    return j


def _mpa_shape(r, track):
    """(frames, channels, sample_rate) of an MPEG file's group result."""
    if int(r["packets"]) == 0:   # no frame survived: the track's parameters, as decode_mpeg_audio reports them
        return 0, int(track["channels"]), int(track["sample_rate"])
    return int(r["frames"]), int(r["channels"]), int(r["sample_rate"])


def _mpa_files_plan(files, threads, errors, index, layers, what, group_dtype, job_dtype, group_rule, **failed_fields):
    """mpa12_files_plan / mp3_files_plan: the files of `layers` (the others refused with `what`) get their group from
    group_rule, group i uses state slot i, and a failed file's group holds failed_fields."""
    ix, messages = mpa_index_files(files, threads) if index is None else (index[0], dict(index[1]))
    ix = _keep_layers(ix, messages, layers, what)
    if errors is not None:
        errors.update(messages)
    groups = np.zeros(len(files), dtype=group_dtype)
    groups["slot"] = np.arange(len(files))
    for k, v in failed_fields.items():
        groups[k] = v
    parts = []
    for i, x in enumerate(ix):
        if x is not None:
            track, packets = x
            parts.append((i, files[i], _mpa_jobs(packets, job_dtype), *group_rule(track, len(packets))))
    data, jobs, cap, failed = _batch(groups, parts, job_dtype)
    tracks = [None if t is None else t[0] for t in ix]
    return dict(data=data, jobs=jobs, groups=groups, tracks=tracks, out_samples=cap, failed=failed)


def mpa12_files_plan(files, threads=None, errors=None, index=None):
    """Host half of decode_mpa12_files: every file indexed (symgpu_mpa_index, on `threads` host threads), their bytes concatenated
    once, one job per packet and one group per file (group i uses state slot i).  Returns dict(data, jobs, groups, tracks, out_samples,
    failed).  A file that cannot be indexed or is not Layer I / II (listed in `failed`) gets a group without jobs; its message goes to
    errors[i] when `errors` is a dict.  index: the result of mpa_index_files (else computed here)."""
    return _mpa_files_plan(files, threads, errors, index, (1, 2), "decode_mpa12_files takes Layer I / II files", nat.MPA12_GROUP_DTYPE,
                           nat.MPA12_JOB_DTYPE, _mpa12_group, layer=1)


def decode_mpa12_files(engine, files, fmt=nat.FMT_S16, threads=None, device=False, errors=None, index=None):
    """[(samples [frames, channels] of `fmt`, sample_rate)] for a list of MPEG Layer I / II files, each equal to
    decode_mpeg_audio(engine, file, fmt): the files are indexed on host threads, and ONE device call decodes every packet of every
    file -- headers, bit allocation, scale factors and samples in device code, synthesis and the output stage on the GPU.
    device=True: the bytes go to the device once and the samples are CUDA tensors, views of one output tensor.  A Layer III file or
    one that cannot be indexed yields an empty result with sample rate 0 (its message in errors[i] when `errors` is a dict).
    (Re)allocates the engine's MP3 state slots, one per file.  index: the result of mpa_index_files (else computed here)."""
    plan = mpa12_files_plan(files, threads, errors, index)
    groups, cap = plan["groups"], plan["out_samples"]
    engine.mp3_streams_alloc(max(len(files), 1))
    out, results, _, _ = _decode_batch(
        engine, device, (plan["data"], plan["jobs"]), cap, fmt, len(groups), nat.MPA12_RESULT_DTYPE,
        lambda: (*engine.mpa12_decode_host(plan["data"], plan["jobs"], groups, fmt, cap), None),
        lambda data_t, jobs_t, out_t, results_t, status_t: engine.mpa12_decode_dev(data_t, jobs_t, groups, fmt, out_t, results_t, status_t))
    return _per_file(out, groups, plan["failed"], lambda g: _mpa_shape(results[g], plan["tracks"][g]))


# ---- MPEG Layer III, many files decoded on the device (side information, bit reservoir and Huffman data in device code) ---------

def mp3_files_plan(files, threads=None, errors=None, index=None):
    """Host half of decode_mp3_files: every file indexed (symgpu_mpa_index, on `threads` host threads), their bytes concatenated once,
    one job per packet and one group per file (group i uses state slot i; granules and channels from the file's track).  Returns
    dict(data, jobs, groups, tracks, out_samples, failed).  A file that cannot be indexed or is not Layer III (listed in `failed`) gets
    a group without jobs; its message goes to errors[i] when `errors` is a dict.  index: the result of mpa_index_files."""
    return _mpa_files_plan(files, threads, errors, index, (3,), "decode_mp3_files takes Layer III files", nat.MP3_GROUP_DTYPE,
                           nat.MP3_JOB_DTYPE, _mp3_group, granules=2, channels=2)


def decode_mp3_files(engine, files, fmt=nat.FMT_S16, threads=None, device=False, errors=None, index=None, stats=None):
    """[(samples [frames, channels] of `fmt`, sample_rate)] for a list of MP3 (MPEG Layer III) files, each equal to
    decode_mpeg_audio(engine, file, fmt): the files are indexed on host threads, and ONE device call decodes every packet of every
    file -- headers, side information, the bit reservoir, scale factors and Huffman data in device code, synthesis and the output
    stage on the GPU.  device=True: the bytes go to the device once and the samples are CUDA tensors, views of one output tensor.
    A Layer I / II file or one that cannot be indexed yields an empty result with sample rate 0 (its message in errors[i] when
    `errors` is a dict).  One deviation from decode_mpeg_audio: a joint-stereo frame whose channels are on different window
    sequences (which the reference refuses after reading it) is left out whole.  stats: a dict that receives `rounds` and the
    per-packet `status`.  (Re)allocates the engine's MP3 state slots, one per file.  index: the result of mpa_index_files."""
    plan = mp3_files_plan(files, threads, errors, index)
    groups, cap = plan["groups"], plan["out_samples"]
    engine.mp3_streams_alloc(max(len(files), 1))
    out, results, status, rounds = _decode_batch(
        engine, device, (plan["data"], plan["jobs"]), cap, fmt, len(groups), nat.MP3_RESULT_DTYPE,
        lambda: engine.mp3_decode_host(plan["data"], plan["jobs"], groups, fmt, cap),
        lambda data_t, jobs_t, out_t, results_t, status_t: engine.mp3_decode_dev(data_t, jobs_t, groups, fmt, out_t, results_t, status_t))
    if stats is not None:
        stats.update(rounds=rounds, status=status)
    return _per_file(out, groups, plan["failed"], lambda g: _mpa_shape(results[g], plan["tracks"][g]))


# ---- ADTS AAC-LC, many files decoded on the device (elements, scale factors, Huffman spectra and noise in device code) ----------

def aac_files_plan(files, threads=None, errors=None):
    """Host half of decode_aac_files: every file indexed (adts_aac_index, on `threads` host threads), their bytes concatenated once,
    one job per raw_data_block and one group per file (group i uses state slot i).  Returns dict(data, jobs, groups, out_samples,
    failed).  A file that cannot be indexed or whose channel configuration is outside 1 / 2 (listed in `failed`) gets a group
    without jobs; its message goes to errors[i] when `errors` is a dict."""
    ix, messages = _index_files(files, adts_aac_index, threads)
    if errors is not None:
        errors.update(messages)
    groups = _aac_groups(len(files))
    parts = []
    for i, x in enumerate(ix):
        if x is not None:
            packets, rate, channels = x
            j = np.zeros(len(packets), dtype=nat.PIECE_DTYPE)
            j["offset"], j["len"] = packets["offset"], packets["size"]
            parts.append((i, files[i], j, *_aac_group(rate, channels, len(packets))))
    data, jobs, cap, failed = _batch(groups, parts, nat.PIECE_DTYPE)
    return dict(data=data, jobs=jobs, groups=groups, out_samples=cap, failed=failed)


def decode_aac_files(engine, files, fmt=nat.FMT_S16, threads=None, device=False, errors=None, stats=None):
    """[(samples [frames, channels] of `fmt`, sample_rate)] for a list of ADTS AAC-LC files, each equal to decode_adts_aac(engine, file,
    fmt): the files are indexed on host threads, and ONE device call decodes every raw_data_block of every file -- elements, scale
    factors, Huffman spectra, noise and TNS filters in device code, synthesis and the output stage on the GPU (pulses' new line
    values on the host).  device=True: the bytes go to the device once and the samples are CUDA tensors, views of one output tensor.
    A file that cannot be indexed, or whose channel configuration is outside 1 / 2, yields an empty result with sample rate 0 (its
    message in errors[i] when `errors` is a dict).  stats: a dict that receives the per-packet `status` and `n_redecoded` (packets
    decoded twice because they drew noise).  (Re)allocates the engine's AAC state slots, one per file, as decode_files does: a
    streaming AAC decoder on the same engine loses its state.  At most 65 536 files per call (the state slot is 16 bits)."""
    if len(files) > 1 << 16:
        raise ValueError(f"decode_aac_files takes at most 65536 files per call, not {len(files)}")
    plan = aac_files_plan(files, threads, errors)
    groups, cap = plan["groups"], plan["out_samples"]
    engine.aac_streams_alloc(max(len(files), 1))
    out, results, status, redone = _decode_batch(
        engine, device, (plan["data"], plan["jobs"]), cap, fmt, len(groups), nat.AAC_RESULT_DTYPE,
        lambda: engine.aac_decode_host(plan["data"], plan["jobs"], groups, fmt, cap),
        lambda data_t, jobs_t, out_t, results_t, status_t: engine.aac_decode_dev(data_t, jobs_t, groups, fmt, out_t, results_t, status_t))
    if stats is not None:
        stats.update(status=status, n_redecoded=redone)
    return _per_file(out, groups, plan["failed"],
                     lambda g: (int(results[g]["frames"]), int(groups[g]["channels"]), int(groups[g]["sample_rate"])))


def decode_aac_files_dev(engine, data_t, ranges, fmt=nat.FMT_S16, errors=None, stats=None):
    """decode_aac_files(engine, files, fmt, device=True) for ADTS AAC-LC files already in device memory: file i is
    data_t[offset : offset + len] of ranges[i] ((offset, len) pairs or FILE_RANGE_DTYPE records) in a uint8 CUDA tensor, and its
    result, its message in errors[i] and `stats` (`status`, `n_redecoded`) are what decode_aac_files gives for those bytes.
    The frames are indexed on the device (symgpu_adts_index_dev) into a job table the decode reads in place; only the per-file
    index records, the decode's results and its per-packet status come back to the host.  stats also receives
    `read_back_bytes`, every byte the call copies from the device.  A failed file's packets stay in the job table, named by no
    group.  At most 65 536 files; (re)allocates the engine's AAC state slots, one per file, as decode_aac_files does."""
    r = _resident_files(data_t, ranges, "decode_aac_files_dev", nat.ADTS_MAX_FILES)
    n = len(r)
    if n == 0:
        return []
    # 1. every file's frames as jobs, the table sized by the bound (a frame is at least 7 bytes)
    _, jobs_t, ix = engine._index_dev(engine.adts_index_dev_queue, data_t, r, None, 7, (None, nat.PIECE_DTYPE), (nat.ADTS_FILE_INDEX_DTYPE,))
    # 2. the groups, as aac_files_plan lays them out (a failed file's group starts at its own packets), with adts_aac_index's messages
    messages, parts = {}, []
    for i in range(n):
        n_jobs, channels = int(ix["n_packets"][i]), int(ix["channels"][i])
        refusal = _aac_refusal(n_jobs, channels)
        if refusal:
            messages[i] = f"ValueError: {refusal}"
        else:
            parts.append((i, n_jobs, *_aac_group(int(ix["sample_rate"][i]), channels, n_jobs)))
    groups = _aac_groups(n)
    out_at, failed = _place(groups, parts, ix["first_packet"])
    if errors is not None:
        errors.update(messages)
    # 3. the decode, on the job table in place
    n_jobs = int(ix["first_packet"][-1]) + int(ix["n_packets"][-1])
    engine.aac_streams_alloc(n)
    out, results, status, redone, read = _decode_dev(
        engine, data_t.device, fmt, out_at, n, nat.AAC_RESULT_DTYPE, n_jobs,
        lambda out_t, results_t, status_t: engine.aac_decode_dev(data_t, jobs_t[:n_jobs * nat.PIECE_DTYPE.itemsize], groups, fmt, out_t,
                                                                 results_t, status_t))
    if stats is not None:
        stats.update(status=_good_status(status, groups, failed), n_redecoded=redone, read_back_bytes=ix.nbytes + read)
    return _per_file(out, groups, failed, lambda g: (int(results[g]["frames"]), int(groups[g]["channels"]), int(groups[g]["sample_rate"])))


def decode_mpeg_files(engine, files, fmt=nat.FMT_S16, threads=None, device=False, errors=None, stats=None):
    """[(samples [frames, channels] of `fmt`, sample_rate)] for a list of MPEG audio files of any layer, each what
    decode_mpeg_audio(engine, file, fmt) returns: every file is indexed once, Layer III files go to decode_mp3_files and Layer I / II
    files to decode_mpa12_files (one device call each).  A file that cannot be indexed yields an empty result with sample rate 0 (its
    message in errors[i] when `errors` is a dict).  stats: a dict that receives what decode_mp3_files' `stats` does, when there is a
    Layer III file."""
    ix, messages = mpa_index_files(files, threads)
    if errors is not None:
        errors.update(messages)
    result = [None] * len(files)
    for layers, decode, more in (((3,), decode_mp3_files, dict(stats=stats)), ((1, 2), decode_mpa12_files, {})):
        mine = [i for i, t in enumerate(ix) if t is not None and int(t[0]["layer"]) in layers]
        if mine:
            got = decode(engine, [files[i] for i in mine], fmt, threads, device, None, ([ix[i] for i in mine], {}), **more)
            for i, r in zip(mine, got):
                result[i] = r
    for i in messages:
        empty = np.zeros((0, 0), dtype=nat.FMT_NUMPY[fmt])
        if device:
            import torch
            empty = torch.empty((0, 0), dtype=getattr(torch, _TORCH_DTYPES[fmt]), device=torch.device("cuda", engine.device))
        result[i] = (empty, 0)
    return result


def decode_mpeg_files_dev(engine, data_t, ranges, fmt=nat.FMT_S16, errors=None, stats=None):
    """decode_mpeg_files(engine, files, fmt, device=True) for MPEG audio files already in device memory: file i is
    data_t[offset : offset + len] of ranges[i] ((offset, len) pairs or FILE_RANGE_DTYPE records) in a uint8 CUDA tensor, and its
    result, its message in errors[i] and `stats` (`rounds` and the Layer III per-packet `status`, when there is a Layer III file)
    are what decode_mpeg_files gives for those bytes.  The frames, tags and trims are found on the device (symgpu_mpa_index_dev)
    into one job table that the Layer III and the Layer I / II decoders read in place, each over the span of the table between its
    first and last file; only the per-file index records and tracks, the decodes' results and the Layer III per-packet status come
    back to the host.  stats also receives `read_back_bytes`, every byte the call copies from the device.  At most 65 536 files;
    (re)allocates the engine's MP3 state slots, one per file."""
    import torch

    from .engine import SymgpuError
    r = _resident_files(data_t, ranges, "decode_mpeg_files_dev", nat.MPA_MAX_FILES)
    n = len(r)
    if n == 0:
        return []
    dev = data_t.device
    # 1. every file's frames as jobs, the table sized by the bound (a frame is at least MPA_MIN_FRAME bytes)
    _, jobs_t, ix, tracks = engine._index_dev(engine.mpa_index_dev_queue, data_t, r, None, nat.MPA_MIN_FRAME, (None, nat.MP3_JOB_DTYPE),
                                              (nat.MPA_FILE_INDEX_DTYPE, nat.MPA_TRACK_DTYPE))
    read = ix.nbytes + tracks.nbytes
    messages = {i: f"SymgpuError: {SymgpuError(1, 'symgpu_mpa_index')}" for i in range(n) if ix["status"][i] & nat.MPA_NO_FRAME}
    if errors is not None:
        errors.update(messages)
    # 2. one decode per layer family, on the job table in place, with the groups decode_mp3_files / decode_mpa12_files make
    engine.mp3_streams_alloc(n)
    result = [(torch.empty((0, 0), dtype=getattr(torch, _TORCH_DTYPES[fmt]), device=dev), 0)] * n
    families = (((3,), nat.MP3_GROUP_DTYPE, nat.MP3_RESULT_DTYPE, engine.mp3_decode_dev, _mp3_group),
                ((1, 2), nat.MPA12_GROUP_DTYPE, nat.MPA12_RESULT_DTYPE, engine.mpa12_decode_dev, _mpa12_group))
    for layers, group_dtype, result_dtype, decode, group_rule in families:
        mine = [i for i in range(n) if i not in messages and int(tracks["layer"][i]) in layers]
        if not mine:
            continue
        lo = int(ix["first_packet"][mine[0]])
        hi = int(ix["first_packet"][mine[-1]]) + int(ix["n_packets"][mine[-1]])
        groups = np.zeros(len(mine), dtype=group_dtype)
        groups["slot"] = mine
        parts = [(g, int(ix["n_packets"][i]), *group_rule(tracks[i], int(ix["n_packets"][i]))) for g, i in enumerate(mine)]
        out_at, _ = _place(groups, parts, ix["first_packet"][mine] - lo)
        out, results, status, rounds, nread = _decode_dev(
            engine, dev, fmt, out_at, len(mine), result_dtype, hi - lo,
            lambda out_t, results_t, status_t: decode(data_t, jobs_t[lo * nat.MP3_JOB_DTYPE.itemsize:hi * nat.MP3_JOB_DTYPE.itemsize], groups,
                                                      fmt, out_t, results_t, status_t),
            read_status=layers == (3,))
        read += nread
        if status is not None and stats is not None:
            stats.update(rounds=rounds, status=_good_status(status, groups, []))
        for i, got in zip(mine, _per_file(out, groups, [], lambda g: _mpa_shape(results[g], tracks[mine[g]]))):
            result[i] = got
    if stats is not None:
        stats["read_back_bytes"] = read
    return result


# ---- Ogg Vorbis, many files decoded on the device (codebooks, floors, residues in device code) --------------------------------

def vorbis_files_plan(files, threads=None, errors=None):
    """Host half of decode_vorbis_files: every file indexed (ogg_vorbis_index, on `threads` host threads), the gathered logical
    streams concatenated once, one job per audio packet with the reader's leading discard and page end trim, files with
    byte-identical identification and setup headers sharing one setup, and one group per file.  Returns dict(data, headers,
    setups, jobs, groups, out_samples, failed).  A file that cannot be indexed or opened -- not Ogg, more than two channels, floor
    type 0, ... (listed in `failed`) -- gets a group without jobs; its message goes to errors[i] when `errors` is a dict."""
    return _vorbis_files_plan(files, threads, errors, None)


def _vorbis_files_plan(files, threads, errors, streams):
    """vorbis_files_plan; streams: as _stream_of takes them."""
    def index(i):
        ix = _vorbis_index_of(_stream_of(files[i], streams, i))
        ix["fe"].close()   # (it checked the setup; the device call builds its own)
        return ix
    ix, messages = _index_files(range(len(files)), index, threads)
    if errors is not None:
        errors.update(messages)
    groups = np.zeros(len(files), dtype=nat.VORBIS_GROUP_DTYPE)
    good = [i for i, x in enumerate(ix) if x is not None]
    setup_of, setups, headers = _vorbis_setups([ix[i]["headers"] for i in good])
    parts = []
    for i, setup in zip(good, setup_of):
        x = ix[i]
        j = np.zeros(len(x["table"]), dtype=nat.VORBIS_JOB_DTYPE)
        j["offset"], j["len"] = x["table"]["offset"], x["table"]["len"]
        j["discard"] = np.clip(x["discard"], 0, 0xffffffff)
        j["trim_end"] = np.clip(x["trim_end"], 0, 0xffffffff)
        parts.append((i, x["blob"], j, *_vorbis_group(x["ident"], len(j), setup)))
    data, jobs, cap, failed = _batch(groups, parts, nat.VORBIS_JOB_DTYPE)
    return dict(data=data, headers=headers, setups=setups, jobs=jobs, groups=groups, out_samples=cap, failed=failed)


def decode_vorbis_files(engine, files, fmt=nat.FMT_S16, threads=None, device=False, errors=None, stats=None):
    """[(samples [frames, channels] of `fmt`, sample_rate)] for a list of Ogg Vorbis files (mono / stereo, floor 1), each equal to
    decode_ogg_vorbis(engine, file, fmt): the files are indexed on host threads, and ONE device call decodes every audio packet of
    every file -- codebooks, floors and residues in device code, synthesis and the output stage on the GPU.  device=True: the
    bytes go to the device once and the samples are CUDA tensors, views of one output tensor.  A file that cannot be indexed or
    opened yields an empty result with sample rate 0 (its message in errors[i] when `errors` is a dict), and the others still
    decode.  stats: a dict that receives the per-packet `status` and `n_setups`, the number of distinct setups.  Replaces the
    engine's Vorbis stream and floor registration, as decode_ogg_vorbis does.  At most 65 536 files per call."""
    return _decode_vorbis_files(engine, files, fmt, threads, device, errors, stats, None)


def _decode_vorbis_files(engine, files, fmt, threads, device, errors, stats, streams):
    """decode_vorbis_files; streams: as _stream_of takes them."""
    if len(files) > nat.VORBIS_MAX_FILES:
        raise ValueError(f"decode_vorbis_files takes at most {nat.VORBIS_MAX_FILES} files per call, not {len(files)}")
    plan = _vorbis_files_plan(files, threads, errors, streams)
    groups, cap, setups = plan["groups"], plan["out_samples"], plan["setups"]

    def host():
        if not len(setups):   # no file could be opened: nothing to decode
            return np.zeros(0, dtype=nat.FMT_NUMPY[fmt]), np.zeros(len(groups), dtype=nat.VORBIS_RESULT_DTYPE), np.zeros(0, dtype=np.uint8), None
        return (*engine.vorbis_decode_host(plan["headers"], setups, plan["data"], plan["jobs"], groups, fmt, cap), None)

    def dev(data_t, jobs_t, out_t, results_t, status_t):
        if len(setups):       # (else every file failed: no result is read)
            engine.vorbis_decode_dev(plan["headers"], setups, data_t, jobs_t, groups, fmt, out_t, results_t, status_t)
    out, results, status, _ = _decode_batch(engine, device, (plan["data"], plan["jobs"]), cap, fmt, len(groups),
                                            nat.VORBIS_RESULT_DTYPE, host, dev)
    if stats is not None:
        stats.update(status=status, n_setups=len(setups))
    return _per_file(out, groups, plan["failed"],
                     lambda g: (int(results[g]["frames"]), int(results[g]["channels"]), int(results[g]["sample_rate"])))


def decode_vorbis_files_dev(engine, data_t, ranges, fmt=nat.FMT_S16, errors=None, stats=None):
    """decode_vorbis_files(engine, files, fmt, device=True) for Ogg Vorbis files already in device memory: file i is
    data_t[offset : offset + len] of ranges[i] ((offset, len) pairs or FILE_RANGE_DTYPE records) in a uint8 CUDA tensor, and
    its result, its message in errors[i] and `stats` (`status`, `n_setups`) are what decode_vorbis_files gives for those bytes.
    The pages are indexed, the headers chosen and every audio packet's job built on the device; only per-file records and the
    identification and setup packets come back to the host, which builds the setups from them.  stats also receives
    `read_back_bytes`, every byte the call copies from the device.  A constant number of launches and host waits per call
    (DESIGN §5f).  At most 65 536 files, mono / stereo, floor 1; replaces the engine's Vorbis stream and floor registration."""
    return _vorbis_files_dev(engine, data_t, ranges, fmt, errors, stats)


def _vorbis_files_dev(engine, data_t, ranges, fmt, errors, stats, mark=None):
    """decode_vorbis_files_dev; mark(phase, state), when given, is called as each phase has been queued: 'start', 'index',
    'heads', 'setup' (the host's work on the headers), 'jobs' (state: the gathered audio bytes, the job table and the groups,
    on the device), 'decode'; state is {} for the others."""
    r = _resident_files(data_t, ranges, "decode_vorbis_files_dev", nat.VORBIS_MAX_FILES)
    out, parts = _ogg_files_dev(engine, data_t, r, fmt, mark, route_flac=False)
    _, _, messages, kind_stats = parts[0]
    if errors is not None:
        errors.update(messages)
    if stats is not None:
        stats.update(kind_stats)
    return out


def _ogg_files_dev(engine, data_t, r, fmt, mark, route_flac):
    """The Ogg files r (FILE_RANGE_DTYPE records, checked) of data_t decoded on the device, their pages indexed once.  With
    route_flac, a file whose chosen stream's first packet is an Ogg FLAC identification packet goes to the FLAC decoder (the
    device has already gathered that packet for the Vorbis header checks, so classifying costs no read), every other file to
    the Vorbis decoder; without, every file goes to Vorbis.  Returns (results, parts): parts lists ('vorbis', ...) and then
    ('oggflac', ...) for each kind with a file, as (kind, members (indices into r), {k: message} (k an index into members),
    stats).  Each kind's stats `read_back_bytes` holds its own files' share of the shared reads -- their page-index and Vorbis
    head records and their gathered header packets -- plus what its decode reads back, so that the kinds' counts sum to every
    byte read."""
    import torch
    n = len(r)
    mark = mark or (lambda phase, state: None)
    dev = data_t.device
    torch.cuda.current_stream(dev).synchronize()   # data_t is torch's: written on its stream
    mark("start", {})
    # 1. the page index, as Engine.ogg_index_dev builds it: sizes first, then the tables; the index stays on the device
    index_t = _u8(dev, n * nat.OGG_FILE_INDEX_DTYPE.itemsize)
    engine.ogg_index_dev_queue(data_t, r, _u8(dev, 0), _u8(dev, 0), index_t)
    engine.sync()
    ix = index_t.cpu().numpy().view(nat.OGG_FILE_INDEX_DTYPE)
    n_packets = int(ix["first_packet"][-1]) + int(ix["n_packets"][-1]) if n else 0
    n_pieces = int(ix["first_piece"][-1]) + int(ix["n_pieces"][-1]) if n else 0
    packets_t, pieces_t = _u8(dev, n_packets * nat.OGG_PACKET_DTYPE.itemsize), _u8(dev, n_pieces * nat.PIECE_DTYPE.itemsize)
    engine.ogg_index_dev_queue(data_t, r, packets_t, pieces_t, index_t)
    mark("index", {})
    # 2. each file's headers and audio packets
    heads_t, ranks_t = _u8(dev, n * nat.VORBIS_FILE_HEADS_DTYPE.itemsize), _u8(dev, n_packets * nat.VORBIS_PACKET_RANK_DTYPE.itemsize)
    engine.vorbis_heads_dev(data_t, r, packets_t, pieces_t, index_t, heads_t, ranks_t)
    mark("heads", {})
    engine.sync()
    heads = heads_t.cpu().numpy().view(nat.VORBIS_FILE_HEADS_DTYPE)
    per_file = np.full(n, nat.OGG_FILE_INDEX_DTYPE.itemsize + nat.VORBIS_FILE_HEADS_DTYPE.itemsize, dtype=np.int64)   # each file's share of the reads
    # 3. the header packets gathered into one buffer, read back, and checked on the host as ogg_vorbis_index checks them
    refs, spans, at = [], {}, 0
    for i in range(n):
        h = heads[i]
        if h["status"] == nat.VORBIS_NO_PACKETS:
            continue
        refs.append((at, i, 0))
        spans[i] = [(at, int(h["ident_len"]))]
        at += int(h["ident_len"])
        if h["status"] == 0:
            refs.append((at, i, int(h["setup"])))
            spans[i].append((at, int(h["setup_len"])))
            at += int(h["setup_len"])
        per_file[i] += sum(ln for _, ln in spans[i])
    head_t = _u8(dev, at)
    engine.ogg_gather_dev(data_t, r, packets_t, pieces_t, index_t, np.array(refs, dtype=nat.OGG_PACKET_REF_DTYPE), head_t)
    engine.sync()
    head_bytes = head_t.cpu().numpy().tobytes()
    flac = [i for i in spans if route_flac and _is_ogg_flac_ident(head_bytes[spans[i][0][0]:spans[i][0][0] + spans[i][0][1]])]
    flac_set = set(flac)
    vor = [i for i in range(n) if i not in flac_set]
    messages, opened = {}, {}

    def check(ident_b, setup_b):
        try:
            ident, n_modes, mask, fe = vorbis_open_headers(ident_b, setup_b)
            fe.close()   # (it checked the setup; the device call builds its own)
            return ident, n_modes, mask
        except Exception as e:  # noqa: BLE001 -- one bad file must not abort the batch; its message is kept
            return f"{type(e).__name__}: {e}"
    keys = {}
    for g, i in enumerate(vor):
        if i not in spans:
            messages[g] = "ValueError: no Ogg packets"
            continue
        parts = [head_bytes[a:a + ln] for a, ln in spans[i]]
        key = (parts[0], parts[1] if len(parts) > 1 else None)
        if key not in opened:    # identical headers are checked once: the checks depend on nothing else
            opened[key] = check(*key)
        if isinstance(opened[key], str):
            messages[g] = opened[key]
        else:
            keys[g] = key
    # setups shared by identical headers, groups (one per Vorbis file) and each file's share of the jobs, as vorbis_files_plan
    # lays them out
    setup_of, setups, headers = _vorbis_setups(list(keys.values()))
    file_jobs = np.zeros(n, dtype=nat.VORBIS_FILE_JOBS_DTYPE)
    placed, job_at, byte_at = [], 0, 0
    for (g, key), setup in zip(keys.items(), setup_of):
        i = vor[g]
        ident, n_modes, mask = opened[key]
        n_audio, n_bytes = int(heads[i]["n_audio"]), int(heads[i]["audio_bytes"])
        placed.append((g, n_audio, *_vorbis_group(ident, n_audio, setup)))
        file_jobs[i] = (mask, byte_at, n_bytes, job_at, n_audio, n_modes, ident["bs0_exp"], ident["bs1_exp"], 0)
        job_at, byte_at = job_at + n_audio, byte_at + n_bytes
    groups = np.zeros(len(vor), dtype=nat.VORBIS_GROUP_DTYPE)
    out_at, failed = _place(groups, placed, _packed(len(vor), list(keys), [p[1] for p in placed]))
    mark("setup", {})
    # 4. every audio packet's bytes and job
    result, parts = [None] * n, []
    if vor or not route_flac:
        audio_t, jobs_t = _u8(dev, byte_at), _u8(dev, job_at * nat.VORBIS_JOB_DTYPE.itemsize)
        engine.vorbis_jobs_dev(data_t, r, packets_t, pieces_t, index_t, ranks_t, file_jobs, audio_t, jobs_t)
        mark("jobs", dict(audio=audio_t, jobs=jobs_t, groups=groups))
        # 5. the decode (when every file failed, nothing is decoded and no result is read)
        out, results, status = torch.empty(0, dtype=getattr(torch, _TORCH_DTYPES[fmt]), device=dev), None, np.zeros(0, dtype=np.uint8)
        read = int(per_file[vor].sum())
        if len(setups):
            def decode(out_t, results_t, status_t):
                engine.vorbis_decode_dev(headers, setups, audio_t, jobs_t, groups, fmt, out_t, results_t, status_t)
                mark("decode", {})
            out, results, status, _, nread = _decode_dev(engine, dev, fmt, out_at, len(vor), nat.VORBIS_RESULT_DTYPE, job_at, decode)
            read += nread
        got = _per_file(out, groups, failed, lambda g: (int(results[g]["frames"]), int(results[g]["channels"]), int(results[g]["sample_rate"])))
        for i, res in zip(vor, got):
            result[i] = res
        parts.append(("vorbis", vor, messages, dict(status=status, n_setups=len(setups), read_back_bytes=read)))
    if flac:
        flac_messages, flac_stats = {}, {}
        got = _ogg_flac_dev(engine, data_t, r, (packets_t, pieces_t, index_t), flac, fmt, flac_messages, flac_stats)
        flac_stats["read_back_bytes"] += int(per_file[flac].sum())
        for i, res in zip(flac, got):
            result[i] = res
        parts.append(("oggflac", flac, flac_messages, flac_stats))
    return result, parts


# ---- a mixed list: every file to the device decoder of its kind ----------------------------------------------------------------

def _stream_or_error(data):
    """ogg_logical_stream(data), or the exception it raises."""
    try:
        return ogg_logical_stream(data)
    except Exception as e:  # noqa: BLE001 -- kept, and raised again where the file is decoded
        return e


def decode_any_files(engine, files, fmt=nat.FMT_S16, threads=None, device=False, errors=None, stats=None):
    """[(samples [frames, channels] of `fmt`, sample_rate)], one per file in input order, for a list of native FLAC, ADTS AAC-LC,
    Ogg Vorbis, FLAC-in-Ogg, MPEG audio (Layers I-III) and ALAC-in-CAF files in any mix: every file is sniffed, and the files of
    each kind go, at most once per kind, to decode_flac_files, decode_aac_files, decode_vorbis_files, decode_ogg_flac_files,
    decode_mpeg_files and decode_alac_files; a kind without a file makes no call.  An Ogg file's pages are indexed once: it is FLAC in Ogg when its
    chosen stream's first packet is an Ogg FLAC identification packet (mappings/flac.rs detect()), else Vorbis.  Every result is
    what that decoder returns for the file alone with the same `fmt` and `device`.  device=True: the samples are CUDA tensors,
    views of their kind's output tensor.  A file its decoder cannot index or open yields an empty [0, 0] result with sample rate
    0, and its message goes to errors[i], i its place in `files`, when `errors` is a dict.  stats: a dict that receives `calls`,
    the kinds that ran ('flac', 'aac', 'vorbis', 'oggflac', 'mpa', 'alac'), and under each such kind a dict of what that decoder's
    `stats` gives (`status`, `n_redecoded`, `n_setups`, `rounds`).  The decoders' limits hold per kind: more than 65 536 AAC,
    Vorbis or Ogg FLAC files is their ValueError.  As those decoders do, the call (re)allocates the engine's MP3 and AAC state
    slots and replaces its Vorbis stream and floor registration: streaming decoders on the same engine lose their state."""
    import concurrent.futures
    import os
    kinds = [sniff(f) for f in files]
    ogg = [i for i, k in enumerate(kinds) if k == "vorbis"]
    streams = {}
    if ogg:
        with concurrent.futures.ThreadPoolExecutor(max_workers=threads or os.cpu_count()) as pool:
            streams = dict(zip(ogg, pool.map(lambda i: _stream_or_error(files[i]), ogg)))
    for i, st in streams.items():
        if not isinstance(st, Exception) and len(st[2]) and _is_ogg_flac_ident(st[1][int(st[2]["offset"][0]):][:int(st[2]["len"][0])]):
            kinds[i] = "oggflac"

    def pick(mine):
        return [files[i] for i in mine]
    decoders = (("flac", lambda mine, e, st: decode_flac_files(engine, pick(mine), threads, device, e, fmt)),
                ("aac", lambda mine, e, st: decode_aac_files(engine, pick(mine), fmt, threads, device, e, st)),
                ("vorbis", lambda mine, e, st: _decode_vorbis_files(engine, pick(mine), fmt, threads, device, e, st, [streams[i] for i in mine])),
                ("oggflac", lambda mine, e, st: _decode_ogg_flac_files(engine, pick(mine), threads, device, e, fmt, st, [streams[i] for i in mine])),
                ("mpa", lambda mine, e, st: decode_mpeg_files(engine, pick(mine), fmt, threads, device, e, st)),
                ("alac", lambda mine, e, st: decode_alac_files(engine, pick(mine), fmt, threads, device, e, st)))
    result, calls = [None] * len(files), []
    for kind, decode in decoders:
        mine = [i for i, k in enumerate(kinds) if k == kind]
        if not mine:
            continue
        messages, kind_stats = {}, {}
        got = decode(mine, messages, kind_stats)
        for i, r in zip(mine, got):
            result[i] = r
        if errors is not None:
            errors.update({mine[k]: m for k, m in messages.items()})
        calls.append(kind)
        if stats is not None:
            stats[kind] = kind_stats
    if stats is not None:
        stats["calls"] = calls
    return result


def decode_any_files_dev(engine, data_t, ranges, fmt=nat.FMT_S16, errors=None, stats=None):
    """decode_any_files(engine, files, fmt, device=True) for files already in device memory: file i is data_t[offset : offset + len]
    of ranges[i] ((offset, len) pairs or FILE_RANGE_DTYPE records) in a uint8 CUDA tensor.  Each file is sniffed from its first 4
    bytes (sniff's rules; the heads come back in one gather), and the files of each kind go, at most once per kind and in
    decode_any_files' order, to decode_flac_files_dev, decode_aac_files_dev, decode_vorbis_files_dev, decode_ogg_flac_files_dev
    and decode_mpeg_files_dev, then CAF files to decode_alac_files_dev, over their ranges on the same data_t: nothing is copied.  The Ogg files' pages are indexed once, on
    the device, and the identification packets the Vorbis header step gathers anyway tell FLAC in Ogg from Vorbis (the rule of
    decode_any_files); the Ogg FLAC files' jobs are then built from the same index.  Results and messages (errors[i], i its place
    in `ranges`) are what decode_any_files gives for those bytes.  stats: a dict that receives `calls`, under each kind that ran
    that decoder's `stats`, and `read_back_bytes`, every byte the call copies from the device: the 4-byte heads of every file
    plus each kind's `read_back_bytes`, where the reads the Ogg kinds share (page-index and Vorbis head records, gathered header
    packets) count under the kind of the file they belong to.  The per-kind limits and the effects on the engine's state slots
    and Vorbis registration are decode_any_files', with one difference: the Ogg files are indexed in one device call before they
    are told apart, so Ogg Vorbis and Ogg FLAC files share one limit of 65 536 files (SYMGPU_OGG_MAX_FILES), counted together."""
    import torch

    from .engine import file_ranges
    r = _resident_files(data_t, ranges, "decode_any_files_dev", len(file_ranges(ranges)))
    n = len(r)
    lens = np.minimum(r["len"], 4).astype(np.int64)
    heads = np.zeros((n, 4), dtype=np.uint8)
    if n and data_t.numel():
        at = r["offset"].astype(np.int64)[:, None] + np.minimum(np.arange(4)[None, :], np.maximum(lens[:, None] - 1, 0))
        heads = data_t[torch.from_numpy(np.minimum(at, data_t.numel() - 1)).to(data_t.device)].cpu().numpy()
    read = heads.nbytes
    kinds = [sniff(heads[i, :lens[i]].tobytes()) for i in range(n)]

    def ogg(data_t, rr, fmt):
        if len(rr) > nat.OGG_MAX_FILES:
            raise ValueError(f"decode_any_files_dev takes at most {nat.OGG_MAX_FILES} Ogg files (Vorbis and FLAC in Ogg together) per call, "
                             f"not {len(rr)}")
        return _ogg_files_dev(engine, data_t, rr, fmt, None, route_flac=True)

    def one(decode):
        def run(data_t, rr, fmt):
            messages, kind_stats = {}, {}
            got = decode(engine, data_t, rr, fmt, messages, kind_stats)
            return got, [(None, list(range(len(rr))), messages, kind_stats)]
        return run
    decoders = (("flac", one(decode_flac_files_dev)), ("aac", one(decode_aac_files_dev)), ("vorbis", ogg), ("mpa", one(decode_mpeg_files_dev)),
                ("alac", one(decode_alac_files_dev)))
    result, calls = [None] * n, []
    for kind, decode in decoders:
        mine = [i for i, k in enumerate(kinds) if k == kind]
        if not mine:
            continue
        got, parts = decode(data_t, r[mine], fmt)
        for i, res in zip(mine, got):
            result[i] = res
        for part_kind, members, messages, kind_stats in parts:
            if errors is not None:
                errors.update({mine[members[k]]: m for k, m in messages.items()})
            calls.append(part_kind or kind)
            read += kind_stats.get("read_back_bytes", 0)
            if stats is not None:
                stats[part_kind or kind] = kind_stats
    if stats is not None:
        stats.update(calls=calls, read_back_bytes=read)
    return result
