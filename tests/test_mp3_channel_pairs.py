"""Both MP3 synthesis kernels against the oracle on stereo granules whose channels switch windows independently.

Outside joint stereo each channel of a granule has its own block type, mixed flag and rzero, and the kernels, which carry both
channels in one warp, make every per-channel decision twice per lane: a sub-band can be long in one channel and short in the
other (the second-generation kernel's `hybrid_mixed`), the two IMDCT windows can differ, one channel can end its coded lines
where the other goes on.  Batches come from tests/_mp3_pairs.py.  Bar: every PCM word bit-identical to the oracle (uint32
view, sign of zero included).

CPU part: the generator keeps the rules of the units, the batches reach the per-lane cases they are meant to (restated from
the kernel in numpy), the oracle itself treats the channels independently, and the launch plans of the GPU cases have the
shapes the cases name.  GPU part (`gpu` marker): every kernel shape and every built second-generation instantiation, state
carried across calls, the other entry points, thread-safe submission, oracle-free properties at the bench size, and files.
"""
import ctypes
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

from symphonia_b200 import _native as nat
from tests import _mp3_bitstream as bw
from tests import _mp3_pairs as mp
from tests import _oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# The launch plans depend on the grid.  The cases below are sized for an H100 SXM: 132 SMs, one 16-warp CTA of the first
# generation per SM, 12 warps (shares) of the second generation per SM.
H100_SMS, V1_CTAS_PER_SM, V2_WARPS_PER_SM = 132, 1, 12
LOAD, STORE, CARRY_IN, CARRY_OUT, GROUP_END = 1, 2, 4, 8, 16
TILE_DTYPE = np.dtype([("first_frame", "<u4"), ("stream", "<u4"), ("first_gr", "<u2"), ("n_granules", "<u2"),
                       ("gpf", "u1"), ("n_ch", "u1"), ("flags", "u1"), ("pad", "u1")])
# kV2Variants (mp3_kernel_v2.cu): (warps per CTA, variant bits) of every built second-generation instantiation
V2_VARIANTS = ((12, 33), (12, 0), (12, 1), (12, 5), (12, 17), (12, 81), (12, 64), (14, 33), (14, 97), (10, 33), (12, 129),
               (12, 193))
# Layer III files of one call: (version, mode, rate_idx, bitrate_idx, mode_ext); mode 1 with mode_ext 0 is joint stereo
# without mid-side or intensity coding, whose channels may differ too
FILE_KINDS = [(v, mode, rate, br, ext) for v, rate, br in (("1", 0, 10), ("2", 1, 8))
              for mode, ext in ((0, None), (2, None), (1, 0))]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _compare(got, want, what):
    g, w = _bits(got), _bits(want)
    bad = np.nonzero(g != w)
    if len(bad[0]):
        f, c, i = bad[0][0], bad[1][0], bad[2][0]
        raise AssertionError(f"{what}: {len(bad[0])} of {g.size} PCM words differ; first at frame {f} ch {c} sample {i}: "
                             f"gpu {got[f, c, i]!r} oracle {want[f, c, i]!r}")


def _units_check(units, runs):
    return nat.lib().symgpu_mp3_units_check(units.ctypes.data, runs.ctypes.data, len(runs), len(units))


def _auto_picks_v2(runs):
    """symgpu.cpp build_plan: the second generation takes a call whose runs average fewer than 16 granules."""
    live = runs[runs["n_frames"] > 0]
    gran = int((live["n_frames"].astype(np.int64) * np.where(live["granules_per_frame"] == 1, 1, 2)).sum())
    return len(live) > 0 and gran < 16 * len(live)


def _plan(fn_name, size, runs, n_frames):
    fn = getattr(nat.lib(), fn_name)
    fn.restype = ctypes.c_size_t
    fn.argtypes = [ctypes.c_int, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p,
                   ctypes.c_size_t] + [ctypes.POINTER(ctypes.c_int)] * 3
    runs = np.ascontiguousarray(runs)
    n_groups, n_tiles, hdr = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    n = fn(size, len(runs), runs.ctypes.data, len(runs), n_frames, None, 0, n_groups, n_tiles, hdr)
    assert n > 0
    buf = np.zeros(n, dtype=TILE_DTYPE)
    fn(size, len(runs), runs.ctypes.data, len(runs), n_frames, buf.ctypes.data, n, n_groups, n_tiles, hdr)
    first = buf[:hdr.value].view(np.uint32)[:n_groups.value + 1]
    return first, buf[hdr.value:hdr.value + n_tiles.value]


def _v1_plan(runs, n_frames):
    return _plan("symgpu_debug_mp3_plan", H100_SMS * V1_CTAS_PER_SM, runs, n_frames)


def _v2_plan(runs, n_frames):
    return _plan("symgpu_debug_mp3_plan_v2", H100_SMS * V2_WARPS_PER_SM, runs, n_frames)


def _sr_cases():
    """Every sample rate with mixed blocks: a long-run and a short-run batch each (MPEG-2 and 2.5: one granule per frame)."""
    for sr in range(9):
        yield sr, "long", mp.pair_batch(2, 24 if sr < 3 else 40, 8200 + sr, sample_rate_idx=sr)
        yield sr, "short", mp.pair_batch(48, 1 if sr < 3 else 2, 8300 + sr, sample_rate_idx=sr)


# ================================================================================================ CPU part

@pytest.mark.parametrize("shape", sorted(mp.SHAPES))
def test_generator_keeps_the_rules_of_the_units(shape):
    units, spectra, runs = mp.shape_batch(shape)
    assert _units_check(units, runs) == 0
    bt, flags, rz = units["block_type"], units["flags"].astype(np.int64), units["rzero"].astype(np.int64)
    assert (bt <= nat.MP3_END).all()
    assert not ((flags & nat.F_MIXED) & (bt != nat.MP3_SHORT)).any(), "the mixed flag comes with SHORT only"
    assert not ((flags & nat.F_PREFLAG) & (bt == nat.MP3_SHORT)).any(), "preflag on non-short granules only"
    idx = np.arange(39)
    sf = units["scalefacs"]
    assert not sf[(bt != nat.MP3_SHORT)][:, idx >= 21].any() and not sf[(bt == nat.MP3_SHORT)][:, idx >= 36].any()
    assert (units["subblock_gain"] <= 7).all()
    assert (rz % 2 == 0).all() and (rz <= 576).all()
    beyond = np.arange(576)[None, None, None, :] >= rz[..., None]
    assert (_bits(np.where(beyond, spectra, 0)) == 0).all(), "lines at or beyond rzero are +0.0"
    assert (units["sample_rate_idx"][:, :, 0] == units["sample_rate_idx"][:, :, 1]).all()
    # frames whose channels differ have mid-side and intensity stereo off; joint frames with equal kinds remain in the runs
    joint = (flags[:, 0, 0] & (nat.F_MID_SIDE | nat.F_INTENSITY)) != 0
    differ = ((bt[:, :, 0] != bt[:, :, 1]) | ((flags[:, :, 0] ^ flags[:, :, 1]) & nat.F_MIXED != 0)).any(axis=1)
    assert not (joint & differ).any() and joint.any() and differ.any()
    if shape != "short":
        per_run = joint.reshape(len(runs), -1)
        assert (per_run.any(axis=1) & (~per_run).any(axis=1)).all(), "joint and independent frames alternate within a stream"
    # the default workload is untouched: the joint frames are workloads.mp3_batch's own draws
    from symphonia_b200 import workloads
    wu, ws, _ = workloads.mp3_batch(*mp.SHAPES[shape], seed=mp.SEEDS[shape])
    assert (wu[joint].tobytes() == units[joint].tobytes()) and (_bits(ws[joint]) == _bits(spectra[joint])).all()


def test_sample_rate_cases_keep_the_rules_and_carry_mixed_blocks():
    for sr, what, (units, spectra, runs) in _sr_cases():
        assert _units_check(units, runs) == 0, (sr, what)
        _, _, kinds = mp.coverage(units, runs)
        mixed = mp.KIND_NAMES.index("mixed")
        assert any(mixed in k and k[0] != k[1] for k in kinds), (sr, what)
        assert _auto_picks_v2(runs) == (what == "short"), (sr, what)


def test_encoder_illegal_transitions_occur():
    """A strict encoder goes LONG -> START -> SHORT -> END -> LONG; the decoder takes any order, and so must the kernels."""
    units, _, runs = mp.shape_batch("long")
    seen = set()
    for r in runs:
        f0, n = int(r["first_frame"]), int(r["n_frames"])
        bt = units["block_type"][f0:f0 + n].reshape(-1, 2)   # granule order per channel
        for c in range(2):
            seen |= set(zip(bt[:-1, c].tolist(), bt[1:, c].tolist()))
    for a, b in ((nat.MP3_LONG, nat.MP3_SHORT), (nat.MP3_SHORT, nat.MP3_LONG), (nat.MP3_START, nat.MP3_LONG),
                 (nat.MP3_END, nat.MP3_SHORT), (nat.MP3_LONG, nat.MP3_END)):
        assert (a, b) in seen, (a, b)


@pytest.mark.parametrize("shape", sorted(mp.SHAPES))
def test_each_kernel_shape_reaches_every_per_channel_case(shape):
    cat_pairs, wsel_pairs, kind_pairs = mp.coverage(*mp.shape_batch(shape)[::2])
    for pair in ((36, 12), (12, 36), (36, 0), (0, 36), (12, 0), (0, 12)):
        assert cat_pairs.get(pair, 0) >= 1, (shape, pair, cat_pairs)
    for pair in ((a, b) for a in (0, 1, 3) for b in (0, 1, 3)):
        assert wsel_pairs.get(pair, 0) >= 1, (shape, pair, wsel_pairs)
    assert len(kind_pairs) == 25, (shape, sorted(kind_pairs))


def test_edge_rzero_values_occur_next_to_a_full_channel():
    for shape in ("long", "short"):
        units, _, _ = mp.shape_batch(shape)
        rz = units["rzero"].astype(np.int64).reshape(-1, 2)
        bt = units["block_type"].reshape(-1, 2)
        for v in mp.EDGE_RZERO[:-1]:
            for c in range(2):
                assert ((rz[:, c] == v) & (rz[:, 1 - c] == 576)).any(), (shape, v, c)
        assert ((rz[:, 0] == 576) & (rz[:, 1] == 576) & (bt[:, 0] != bt[:, 1])).any()


def test_restated_window_triples_tile_the_granule():
    """The numpy restatement's window triples (13 short bands; 10 above the mixed switch, 12 with the 8 kHz guess) end at 576."""
    for sr in range(9):
        for mixed in (False, True):
            e = mp._short_quad_edges(sr, mixed)
            assert e[-1] == 576 and (np.diff(e) > 0).all() and len(e) == (14 if not mixed else 11 if sr < 8 else 13), (sr, mixed)


def test_the_oracle_treats_the_channels_independently(oracle):
    """Without mid-side or intensity stereo, the stereo oracle's channel c is the oracle on the mono stream of channel c's units
    and spectra, with its state carried over the whole run; swapping the channels swaps the output.  No kernel involved."""
    units, spectra, runs = mp.pair_batch(4, 16, 8401, joint=False, differ=0.8)
    rc, want, _ = _oracle.mp3_batch(oracle, units, spectra, runs, len(runs))
    assert rc == 0 and np.abs(want).max() > 1e-3
    for c in range(2):
        rc, mono, _ = _oracle.mp3_batch(oracle, *mp.split_channel(units, spectra, runs, c), len(runs))
        assert rc == 0
        assert (_bits(mono[:, 0]) == _bits(want[:, c])).all(), c
    rc, swapped, _ = _oracle.mp3_batch(oracle, *mp.swap_channels(units, spectra), runs, len(runs))
    assert rc == 0 and (_bits(swapped[:, ::-1]) == _bits(want)).all()


def test_the_launch_plans_of_the_cases_have_the_shapes_they_name():
    """Through the debug hooks, on the H100 SXM grid: the first generation with single-tile groups (long runs) and with groups
    of several tiles (forced onto short runs); the second generation compact (many short runs), default (few short runs) and
    with halos (forced onto long runs)."""
    def multi(first, tiles):   # some group of a chain holds more than one tile
        return not ((tiles["flags"] & GROUP_END) != 0).all()
    u, _, r = mp.shape_batch("long")
    assert not _auto_picks_v2(r)
    first, tiles = _v1_plan(r, len(u))
    assert not multi(first, tiles) and ((tiles["flags"] & (LOAD | STORE)) != 0).any()
    first, tiles = _v2_plan(r, len(u))   # SYMGPU_MP3_KERNEL=v2
    assert len(tiles) < 2 * (len(first) - 1) and ((tiles["flags"] & (LOAD | CARRY_IN)) == 0).sum() >= 8
    u, _, r = mp.shape_batch("short")
    assert _auto_picks_v2(r)
    first, tiles = _v2_plan(r, len(u))
    assert len(tiles) >= 2 * (len(first) - 1), "compact instantiation"
    first, tiles = _v1_plan(r, len(u))   # SYMGPU_MP3_KERNEL=v1
    assert multi(first, tiles), "MULTI=true: some group holds several tiles"
    u, _, r = mp.shape_batch("few")
    assert _auto_picks_v2(r)
    first, tiles = _v2_plan(r, len(u))
    assert len(tiles) < 2 * (len(first) - 1), "default instantiation"


def _carry_case():
    """3 streams x 24 frames cut into calls where, in at least two of the streams, the last granule before the cut and the first
    after it both have channels of different kinds.  Returns (S, F, units, spectra, runs, call bounds in frames)."""
    S, F = 3, 24
    units, spectra, runs = mp.pair_batch(S, F, 8602, differ=0.8)
    u4 = units.reshape(S, F, 2, 2)
    kinds = u4["block_type"].astype(np.int64) * 2 + ((u4["flags"] & nat.F_MIXED) != 0)
    differ = kinds[..., 0] != kinds[..., 1]                      # [S, F, granule]
    at = differ[:, :-1, 1] & differ[:, 1:, 0]                    # [S, F - 1]: a cut before frame f + 1 falls between two
    cuts = [f + 1 for f in range(F - 1) if at[:, f].sum() >= 2]
    assert len(cuts) >= 4 and all(at[s, [c - 1 for c in cuts]].any() for s in range(S)), cuts
    return S, F, units, spectra, runs, [0] + cuts + [F]


def test_state_carry_case_cuts_between_differing_granules():
    S, F, units, spectra, runs, bounds = _carry_case()
    assert _units_check(units, runs) == 0 and len(bounds) >= 6


def _file_corpus(n_short=4, long_frames=32, seed=8500):
    """(short files, long files): per kind of FILE_KINDS, `n_short` files of 1-6 frames and one of `long_frames` frames, each
    channel on its own window sequence (pair_blocks=False)."""
    rng = np.random.default_rng(seed)
    short, long_ = [], []
    for k, (version, mode, rate, br, ext) in enumerate(FILE_KINDS):
        kw = dict(version=version, mode=mode, rate_idx=rate, bitrate_idx=br, pair_blocks=False,
                  force_mode_ext=None if ext is None else (lambda i, e=ext: e))
        for _ in range(n_short):
            short.append(b"".join(bw.gen_stream(rng, int(rng.integers(1, 7)), **kw)[0]))
        long_.append(b"".join(bw.gen_stream(rng, long_frames, **kw)[0]))
    return short, long_


def _file_units(data):
    from symphonia_b200 import frontend, packetizer
    track, packets = packetizer.mpa_index(data)
    units, quant, frame_of, info = frontend.Mp3Frontend().decode_packets(data, packets)
    return units, frame_of, packets, info


def test_the_file_corpus_has_channels_on_different_windows():
    short, long_ = _file_corpus()
    n_differ = 0
    for data in short + long_:
        units, frame_of, packets, info = _file_units(data)
        assert len(frame_of) == len(packets) and int(info["channels"]) == 2
        assert not (units["flags"] & (nat.F_MID_SIDE | nat.F_INTENSITY)).any()
        bt, fl = units["block_type"].astype(np.int64), units["flags"].astype(np.int64)
        n_differ += int(((bt[:, :, 0] != bt[:, :, 1]) | (((fl[:, :, 0] ^ fl[:, :, 1]) & nat.F_MIXED) != 0)).sum())
    assert n_differ >= 40
    # the short files make a second-generation call, the long ones a first-generation one
    def runs_of(files):
        r = np.zeros(len(files), dtype=nat.MP3_RUN_DTYPE)
        for i, data in enumerate(files):
            units, _, _, info = _file_units(data)
            r[i] = (i, 0, len(units), int(info["granules"]), 2, 0)
        return r
    assert _auto_picks_v2(runs_of(short)) and not _auto_picks_v2(runs_of(long_))


# ================================================================================================ GPU part

def _check_card():
    import torch
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    assert n_sm == H100_SMS, (f"the device has {n_sm} SMs; the cases of this file are sized for the {H100_SMS} of an H100 SXM, so "
                              f"on this card they may not reach the kernel shapes they name (see "
                              f"test_the_launch_plans_of_the_cases_have_the_shapes_they_name)")


@pytest.fixture(scope="module")
def engine():
    import symphonia_b200 as sb
    _check_card()
    eng = sb.Engine(0)
    yield eng
    eng.close()


def _want(oracle, units, spectra, runs):
    rc, want, _ = _oracle.mp3_batch(oracle, units, spectra, runs, len(runs))
    assert rc == 0 and np.abs(want).max() > 1e-3
    return want


def _run(engine, units, spectra, runs, want, what):
    engine.mp3_streams_alloc(len(runs))
    got = engine.mp3_synth_host(units, spectra, runs)
    per = 1152 if int(units["sample_rate_idx"][0, 0, 0]) < 3 else 576
    _compare(got[:, :, :per], want[:, :, :per], what)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(mp.SHAPES))
def test_product_paths_match_the_oracle(engine, oracle, shape):
    units, spectra, runs = mp.shape_batch(shape)
    _run(engine, units, spectra, runs, _want(oracle, units, spectra, runs), f"auto, {shape} runs")


@pytest.mark.gpu
def test_every_sample_rate_with_mixed_blocks(engine, oracle):
    for sr, what, (units, spectra, runs) in _sr_cases():
        _run(engine, units, spectra, runs, _want(oracle, units, spectra, runs), f"sample_rate_idx {sr}, {what} runs")


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,shape", [("v1", "short"), ("v2", "long"), ("v1", "few"), ("v2", "short")])
def test_forced_kernels_match_the_oracle(oracle, monkeypatch, kernel, shape):
    """v1 on short runs: groups of several tiles (MULTI=true); v2 on long runs: pieces that recompute a halo."""
    import symphonia_b200 as sb
    _check_card()
    monkeypatch.setenv("SYMGPU_MP3_KERNEL", kernel)
    units, spectra, runs = mp.shape_batch(shape)
    want = _want(oracle, units, spectra, runs)
    with sb.Engine(0) as eng:
        _run(eng, units, spectra, runs, want, f"SYMGPU_MP3_KERNEL={kernel}, {shape} runs")


def _variants_child():
    """Runs in a child process: selects every built second-generation instantiation in turn (process-wide) and runs the
    short-run and long-run cases on each, on a new context.  Prints one line per instantiation."""
    import symphonia_b200 as sb
    assert os.environ.get("SYMGPU_MP3_KERNEL") == "v2"
    orc = _oracle.load()
    cases = []
    for shape in ("short", "long"):
        units, spectra, runs = mp.shape_batch(shape)
        cases.append((shape, units, spectra, runs, _want(orc, units, spectra, runs)))
    select = sb.lib().symgpu_debug_mp3_v2_variant
    select.restype, select.argtypes = ctypes.c_int, [ctypes.c_int, ctypes.c_int]
    for nw, mode in V2_VARIANTS:
        assert select(nw, mode) == 1, f"{nw}:{mode} is not a built instantiation"
        with sb.Engine(0) as eng:
            for shape, units, spectra, runs, want in cases:
                _run(eng, units, spectra, runs, want, f"instantiation {nw}:{mode}, {shape} runs")
        print(f"instantiation {nw}:{mode} matches", flush=True)
    assert select(99, 0) == 0


@pytest.mark.gpu
def test_every_built_v2_instantiation_matches_the_oracle():
    """Selecting an instantiation is process-wide and outlives the context, so the sweep runs in a child process."""
    _check_card()
    env = dict(os.environ, SYMGPU_MP3_KERNEL="v2")
    env.pop("SYMGPU_MP3_V2_VARIANT", None)
    r = subprocess.run([sys.executable, "-c", "from tests import test_mp3_channel_pairs as t; t._variants_child()"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count(" matches") == len(V2_VARIANTS), r.stdout


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["v1", "v2"])
def test_state_carries_across_calls_between_differing_granules(oracle, monkeypatch, kernel):
    """The stream state (overlap and polyphase history of both channels) crosses call boundaries that fall between granules
    whose channels are on different kinds."""
    import symphonia_b200 as sb
    _check_card()
    monkeypatch.setenv("SYMGPU_MP3_KERNEL", kernel)
    S, F, units, spectra, runs, bounds = _carry_case()
    want = _want(oracle, units, spectra, runs)
    u4, s4 = units.reshape(S, F, 2, 2), spectra.reshape(S, F, 2, 2, 576)
    got = np.zeros((S, F, 2, 1152), dtype=np.float32)
    with sb.Engine(0) as eng:
        eng.mp3_streams_alloc(S)
        for lo, hi in zip(bounds[:-1], bounds[1:]):
            r = runs.copy()
            r["first_frame"] = np.arange(S) * (hi - lo)
            r["n_frames"] = hi - lo
            out = eng.mp3_synth_host(np.ascontiguousarray(u4[:, lo:hi]).reshape(-1, 2, 2),
                                     np.ascontiguousarray(s4[:, lo:hi]).reshape(-1, 2, 2, 576), r)
            got[:, lo:hi] = out.reshape(S, hi - lo, 2, 1152)
    _compare(got.reshape(S * F, 2, 1152), want, f"state carried across calls at frames {bounds[1:-1]}, {kernel}")


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["long", "short"])
def test_quantized_and_packed_entry_points(engine, oracle, shape):
    units, spectra, runs = mp.shape_batch(shape)
    want = _want(oracle, units, spectra, runs)
    quant = mp.quantized(spectra)
    n = len(units)
    engine.mp3_streams_alloc(len(runs))
    _compare(engine.mp3_synth_host_quantized(units, quant, runs), want, f"quantized, planar f32, {shape} runs")
    for fmt in (nat.FMT_S16, nat.FMT_F32):
        expect = _oracle.pcm_pack(oracle, want, None, 2, fmt, n * 1152, plane_stride=1152, frames=1152, n_spans=n)
        engine.mp3_streams_alloc(len(runs))
        got = engine.mp3_synth_host_quantized(units, quant, runs, fmt)
        assert got.tobytes() == expect.tobytes(), (shape, "quantized", fmt)
        engine.mp3_streams_alloc(len(runs))
        got = engine.mp3_synth_host_packed(units, spectra, runs, fmt)
        assert got.tobytes() == expect.tobytes(), (shape, "packed", fmt)


@pytest.mark.gpu
def test_one_packet_per_call_on_a_dual_channel_stream(engine, oracle):
    F = 30
    units, spectra, runs = mp.pair_batch(1, F, 8701, joint=False, differ=0.8)
    want = _want(oracle, units, spectra, runs)
    one = runs.copy()
    one["n_frames"] = 1
    engine.mp3_streams_alloc(1)
    got = np.zeros((F, 2, 1152), dtype=np.float32)
    for f in range(F):
        got[f] = engine.mp3_synth_host(units[f:f + 1], spectra[f:f + 1], one)[0]
    _compare(got, want, "one packet per call")


@pytest.mark.gpu
def test_submit_and_wait_from_many_threads(oracle):
    """symgpu_mp3_submit / _wait: one Python thread per stream, one frame per call, all on one context.  How the queue groups
    the frames into launches is its own business; every frame's bits must be the oracle's."""
    import symphonia_b200 as sb
    _check_card()
    S, F = 32, 6
    units, spectra, runs = mp.pair_batch(S, F, 8801)
    want = _want(oracle, units, spectra, runs)
    got = np.zeros_like(want)
    gate = threading.Barrier(S)
    errors = []
    with sb.Engine(0) as eng:
        eng.mp3_streams_alloc(S)

        def body(s):
            try:
                for f in range(F):
                    row = s * F + f
                    ticket = eng.mp3_submit(s, units[row], spectra[row], 2, 2)
                    if f == 0:
                        gate.wait()
                    got[row] = eng.mp3_wait(ticket)
            except BaseException as e:  # noqa: BLE001 - reported below
                gate.abort()
                errors.append((s, e))

        threads = [threading.Thread(target=body, args=(s,)) for s in range(S)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors[:3]
        batches, frames = eng.async_stats(nat.CODEC_MP3)
        assert frames == S * F
    _compare(got, want, "submit / wait")


@pytest.mark.gpu
def test_channel_properties_at_the_bench_size(engine, oracle):
    """64 streams x 128 frames, no joint stereo, 60 % of the frames on independent kinds: swapping the channels swaps the output,
    and channel c of the stereo run is the mono run of channel c -- both exactly; then every word against the oracle."""
    S, F = 64, 128
    units, spectra, runs = mp.pair_batch(S, F, 8901, joint=False)
    engine.mp3_streams_alloc(S)
    stereo = engine.mp3_synth_host(units, spectra, runs)
    engine.mp3_streams_alloc(S)
    swapped = engine.mp3_synth_host(*mp.swap_channels(units, spectra), runs)
    _compare(swapped[:, ::-1], stereo, "swapped channels")
    for c in range(2):
        engine.mp3_streams_alloc(S)
        mono = engine.mp3_synth_host(*mp.split_channel(units, spectra, runs, c))
        _compare(mono[:, :1], stereo[:, c:c + 1], f"mono run of channel {c}")
    states = (_oracle.Mp3State * S)()
    want = np.zeros((S * F, 2, 1152), dtype=np.float32)
    rc = oracle.oracle_mp3_batch_mt(ctypes.byref(states), _oracle.ptr(units), _oracle.ptr(spectra), _oracle.ptr(runs),
                                    ctypes.c_uint32(S), _oracle.ptr(want), ctypes.c_int(min(os.cpu_count() or 1, S)))
    assert rc == 0
    _compare(stereo, want, "all 64 streams of the bench-size batch")


@pytest.mark.gpu
@pytest.mark.parametrize("call", ["short", "long"])
def test_files_decode_like_the_oracle(engine, oracle, call):
    """Layer III files whose channels switch windows on their own (stereo, dual channel, joint stereo with mode_ext 0; MPEG-1
    and MPEG-2) through the three many-file decoders: many files of 1-6 frames (a second-generation call) or a few of 32
    frames (first generation).  Every file equals the oracle's decode byte for byte, and no packet is left out."""
    import torch
    from symphonia_b200 import decode
    from tests.test_zz_file_to_pcm import _decode_expect
    short, long_ = _file_corpus()
    files = short if call == "short" else long_
    for fmt in (nat.FMT_S16, nat.FMT_F32):
        want = [_decode_expect(oracle, data, fmt) for data in files]
        stats = {}
        got = decode.decode_mp3_files(engine, files, fmt, stats=stats)
        assert (stats["status"] == nat.MP3_JOB_DECODED).all()
        for k, ((g, rate), (w, wr, _, _)) in enumerate(zip(got, want)):
            assert rate == wr and g.tobytes() == w.tobytes(), ("decode_mp3_files", fmt, k)
        offs = np.concatenate([[0], np.cumsum([len(f) for f in files])[:-1]])
        data_t = torch.from_numpy(np.frombuffer(b"".join(files), dtype=np.uint8).copy()).cuda()
        stats = {}
        got = decode.decode_mpeg_files_dev(engine, data_t, list(zip(offs.tolist(), [len(f) for f in files])), fmt, stats=stats)
        assert (stats["status"] == nat.MP3_JOB_DECODED).all()
        for k, ((g, rate), (w, wr, _, _)) in enumerate(zip(got, want)):
            assert rate == wr and g.cpu().numpy().tobytes() == w.tobytes(), ("decode_mpeg_files_dev", fmt, k)
        stats = {}
        got = decode.decode_any_files(engine, files, fmt, device=True, stats=stats)
        assert stats["calls"] == ["mpa"] and (stats["mpa"]["status"] == nat.MP3_JOB_DECODED).all()
        for k, ((g, rate), (w, wr, _, _)) in enumerate(zip(got, want)):
            assert rate == wr and g.cpu().numpy().tobytes() == w.tobytes(), ("decode_any_files", fmt, k)
