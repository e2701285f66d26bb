"""Layer I / II synthesis against the oracle on runs longer than the grid, where the tiles of a CTA hand their history along a
chain.

mpa12_synth_kernel starts a tile's 15 rows of polyphase history in one of three ways: from the stream state (a run's first tile),
from the raw sub-band samples of the 15 slots before the tile (the halo of a share that starts inside a run), or from the previous
tile of the same chain, whose rows are already DCT'd and sit in shared memory (kTileCarryIn).  The planner (symgpu.cpp
build_plan_for, whole frames as units) gives a share more than one tile only once a call holds more tiles than the grid has CTAs:
beyond 132 x 8 Layer II or 132 x 24 Layer I frames on an H100 SXM, 27.6 s of audio at 44.1 kHz.  Every file longer than that goes
through the carried path; shorter calls never do.  Bar: every PCM word bit-identical to the oracle (uint32 view, sign of zero
included).

CPU part: through symgpu_debug_mpa12_plan at the H100 grid, every case has the plan shape its name claims, and the first carried
tile appears one frame past 132 tiles.  GPU part (`gpu` marker): before it compares anything, every test asserts through the same
hook, at the grid of the device it runs on, that its plan holds carried tiles; then synthetic runs through both synthesis entry
points, state across calls, and long files through every Layer I / II file decoder against the file-level oracle chain.
"""
import ctypes

import numpy as np
import pytest

from symphonia_b200 import _native as nat
from symphonia_b200 import workloads
from tests import _mpa12_bitstream as b12
from tests import _oracle

# The launch plans depend on the grid.  The cases below are sized for an H100 SXM: 132 SMs, one 16-warp CTA of the first
# generation per SM (the Layer I / II kernel is launched on the same grid).
H100_SMS, V1_CTAS_PER_SM = 132, 1
GRID = H100_SMS * V1_CTAS_PER_SM
LOAD, STORE, CARRY_IN, CARRY_OUT = 1, 2, 4, 8
TILE_DTYPE = np.dtype([("first_frame", "<u4"), ("stream", "<u4"), ("first_gr", "<u2"), ("n_granules", "<u2"),
                       ("gpf", "u1"), ("n_ch", "u1"), ("flags", "u1"), ("pad", "u1")])
SLOTS = {1: 12, 2: 36}
TILE_FRAMES = {1: 24, 2: 8}   # kMpa12Slots (mp3_kernel.cu): 288 time slots per tile
LONG = [(2, 2400), (2, 11000), (1, 7000)]   # (layer, frames): shares of 3 tiles, of 10+ tiles (a 4.8 minute file), of 3 tiles


# ================================================================================================ plans

def _hook():
    fn = nat.lib().symgpu_debug_mpa12_plan
    fn.restype = ctypes.c_size_t
    fn.argtypes = [ctypes.c_int, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32,
                   ctypes.c_void_p, ctypes.c_size_t] + [ctypes.POINTER(ctypes.c_int)] * 3
    return fn


def _plan(runs, n_frames, layer, grid=GRID):
    """(chain offsets [n_ctas + 1], tiles) of the plan symgpu_mpa12_synth_dev builds; grid <= 0: this device's grid."""
    fn = _hook()
    runs = np.ascontiguousarray(runs, dtype=nat.MPA12_RUN_DTYPE)
    n_streams = int(runs["stream"].max()) + 1
    n_ctas, n_tiles, hdr = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    args = (grid, n_streams, runs.ctypes.data, len(runs), n_frames, SLOTS[layer])
    n = fn(*args, None, 0, n_ctas, n_tiles, hdr)
    assert n > 0
    buf = np.zeros(n, dtype=TILE_DTYPE)
    fn(*args, buf.ctypes.data, n, n_ctas, n_tiles, hdr)
    first = buf[:hdr.value].view(np.uint32)[:n_ctas.value + 1]
    return first, buf[hdr.value:hdr.value + n_tiles.value]


def _chains(tiles):
    """Lengths of the chains: a tile without kTileCarryIn starts one, each kTileCarryIn tile extends it."""
    lengths = []
    for f in tiles["flags"]:
        if f & CARRY_IN:
            lengths[-1] += 1
        else:
            lengths.append(1)
    return np.array(lengths)


def _carried(tiles):
    return int(((tiles["flags"] & CARRY_IN) != 0).sum())


def _runs(lengths, channels=2):
    """One run (and stream) per length, back to back."""
    r = np.zeros(len(lengths), dtype=nat.MPA12_RUN_DTYPE)
    r["stream"] = np.arange(len(lengths))
    r["first_frame"] = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.uint32)
    r["n_frames"] = lengths
    r["channels"] = channels
    return r


def _check_cover(first, tiles, runs, layer):
    """Every frame of every run is in exactly one tile, in run order; a tile holds at most T frames; a chain stays in one run and
    one share; a halo tile (neither loaded nor carried) has two earlier frames of its run in the batch."""
    T = TILE_FRAMES[layer]
    share = np.searchsorted(first, np.arange(len(tiles)), side="right") - 1
    at = 0
    for r in runs:
        f0, n = int(r["first_frame"]), int(r["n_frames"])
        pos = f0
        while pos < f0 + n:
            t = tiles[at]
            assert int(t["first_frame"]) == pos and int(t["stream"]) == int(r["stream"]) and 1 <= int(t["n_granules"]) <= T
            fl = int(t["flags"])
            assert bool(fl & LOAD) == (pos == f0)
            if fl & CARRY_IN:
                assert tiles[at - 1]["flags"] & CARRY_OUT and share[at - 1] == share[at]
            elif not fl & LOAD:
                assert pos - f0 >= 2
            pos += int(t["n_granules"])
            assert bool(fl & STORE) == (pos == f0 + n and not fl & CARRY_OUT)
            at += 1
    assert at == len(tiles)


def _share_end(total, c, n_ctas=GRID):
    return total * (c + 1) // n_ctas


def _short_around_long(layer, seed=4100):
    """Many one- and two-frame runs, one long run, many more short runs; 188 runs before the long one put the long run's first
    chain in a share with one-frame tiles, on both layers."""
    rng = np.random.default_rng(seed + layer)
    long_ = {1: 4000, 2: 1500}[layer]
    return [int(x) for x in rng.integers(1, 3, 188)] + [long_] + [int(x) for x in rng.integers(1, 3, 200)]


def _unequal(layer):
    """Four long runs of unequal length whose starts put a share cut one frame into a run (the keep-two-frames rule moves it to
    the second frame), exactly at a run start, and 37 frames before a cut inside a run.  Returns (lengths, (moved, at_start))."""
    total = {1: 14000, 2: 9000}[layer]
    moved = _share_end(total, 19) - 1
    at_start = _share_end(total, 57)
    inside = _share_end(total, 98) + 37
    bounds = [0, moved, at_start, inside, total]
    return [b - a for a, b in zip(bounds[:-1], bounds[1:])], (moved, at_start)


MIXED = {"short_around_long": lambda layer: (_short_around_long(layer), None), "unequal_long_runs": _unequal}


@pytest.mark.parametrize("layer,frames", LONG)
def test_one_long_run_is_chains_of_carried_tiles(layer, frames):
    runs = _runs([frames])
    first, tiles = _plan(runs, frames, layer)
    _check_cover(first, tiles, runs, layer)
    fl = tiles["flags"]
    assert len(first) == GRID + 1 and _chains(tiles).min() >= 3
    if frames > 10000:
        assert _chains(tiles).min() >= 10
    assert _carried(tiles) >= len(tiles) // 2
    # the run's last chain stores the state from a carried tile; every other chain starts with a halo
    assert (((fl & CARRY_IN) != 0) & ((fl & STORE) != 0)).sum() == 1
    halo = (fl & (LOAD | CARRY_IN)) == 0
    assert halo.sum() == GRID - 1 and ((fl[halo] & CARRY_OUT) != 0).all()
    if layer == 2 and frames == 2400:
        assert len(tiles) == 396 and _carried(tiles) == 264


@pytest.mark.parametrize("layer", [1, 2])
def test_short_runs_around_a_long_run_share_the_plan_with_chains(layer):
    lengths = _short_around_long(layer)
    runs = _runs(lengths)
    first, tiles = _plan(runs, sum(lengths), layer)
    _check_cover(first, tiles, runs, layer)
    fl = tiles["flags"]
    single = ((fl & (LOAD | STORE)) == (LOAD | STORE)) & (tiles["n_granules"] == 1)
    assert single.sum() >= 100, "one-frame tiles that load and store the state (a Layer I one stores older history rows too)"
    assert _carried(tiles) >= 50 and _chains(tiles).max() >= 2
    halo = (fl & (LOAD | CARRY_IN)) == 0
    assert (halo & ((fl & CARRY_OUT) != 0)).sum() >= 20, "halo tiles that start a chain"
    # a share holds one-frame tiles and a chain side by side
    share = np.searchsorted(first, np.arange(len(tiles)), side="right") - 1
    both = {int(s) for s in share[single]} & {int(s) for s in share[(fl & CARRY_IN) != 0]}
    assert both


@pytest.mark.parametrize("layer", [1, 2])
def test_unequal_long_runs_cut_in_every_way(layer):
    lengths, (moved, at_start) = _unequal(layer)
    assert len(set(lengths)) == len(lengths)
    runs = _runs(lengths)
    first, tiles = _plan(runs, sum(lengths), layer)
    _check_cover(first, tiles, runs, layer)
    assert len(first) == GRID + 1 and _carried(tiles) > 0 and _chains(tiles).max() >= 3
    fl, ff = tiles["flags"], tiles["first_frame"].astype(np.int64)
    halo = (fl & (LOAD | CARRY_IN)) == 0
    starts = set(int(x) for x in first[:-1])
    # the cut one frame into the run at `moved` moves to its second frame: a two-frame tile, then a halo at moved + 2
    k = int(np.nonzero(ff == moved)[0][0])
    assert fl[k] == LOAD and tiles["n_granules"][k] == 2 and k + 1 in starts
    assert halo[k + 1] and ff[k + 1] == moved + 2 and not (halo & (ff == moved + 1)).any()
    # the cut at `at_start` starts a share with the run's loaded first tile
    k = int(np.nonzero(ff == at_start)[0][0])
    assert fl[k] & LOAD and k in starts
    # shares that start inside runs
    assert halo.sum() >= GRID // 2 and ((fl[halo] & CARRY_OUT) != 0).any()


@pytest.mark.parametrize("layer", [1, 2])
def test_the_first_carried_tile_comes_one_frame_past_the_grid(layer):
    T = TILE_FRAMES[layer]
    for frames, carried in ((GRID * T, 0), (GRID * T + 1, 1)):
        runs = _runs([frames])
        first, tiles = _plan(runs, frames, layer)
        _check_cover(first, tiles, runs, layer)
        assert (_carried(tiles) > 0) == bool(carried), (layer, frames, _carried(tiles))
    # and a call of many files, each below the threshold, forms chains inside its files once the call is above it
    runs = _runs([40] * 40)
    first, tiles = _plan(runs, 1600, 2)
    _check_cover(first, tiles, runs, 2)
    assert _carried(tiles) > 0


@pytest.mark.parametrize("layer", [1, 2])
def test_shared_launches_of_submitted_frames_never_form_chains(layer):
    """symgpu_mpa12_submit / _wait merge what many threads submit into one launch, but a stream has at most one frame in it
    (symgpu_async.cpp): every slot is a one-frame run.  A chain only forms inside a run longer than a tile, so a shared launch
    never reaches the carried path, however many frames it holds (here 2048, the most a batch takes)."""
    runs = _runs([1] * 2048)
    first, tiles = _plan(runs, 2048, layer)
    _check_cover(first, tiles, runs, layer)
    assert _carried(tiles) == 0 and (tiles["flags"] == (LOAD | STORE)).all()


def test_the_hook_refuses_what_the_launch_refuses():
    fn = _hook()
    runs = _runs([10])
    bad = runs.copy()
    bad["reserved"][0, 1] = 1
    assert fn(GRID, 1, runs.ctypes.data, 1, 10, 36, None, 0, None, None, None) > 0
    assert fn(GRID, 1, runs.ctypes.data, 1, 10, 18, None, 0, None, None, None) == 0   # neither Layer I nor Layer II
    assert fn(GRID, 1, bad.ctypes.data, 1, 10, 36, None, 0, None, None, None) == 0    # reserved bytes set
    assert fn(GRID, 1, runs.ctypes.data, 1, 9, 36, None, 0, None, None, None) == 0    # the run ends beyond the batch


# ================================================================================================ GPU part

@pytest.fixture(scope="module")
def engine():
    import symphonia_b200 as sb
    eng = sb.Engine(0)
    yield eng
    eng.close()


def _device_grid():
    """The grid of a launch on this device: the number of chains of a plan with more tiles than any grid."""
    first, _ = _plan(_runs([1 << 17]), 1 << 17, 2, grid=0)
    return len(first) - 1


def _assert_carried_on_device(runs, n_frames, layer, what):
    first, tiles = _plan(runs, n_frames, layer, grid=0)
    assert _carried(tiles) > 0, f"{what}: the plan on this device ({len(first) - 1} CTAs) has no carried tile"


def _batch(layer, lengths, channels, seed):
    """Sub-band samples of workloads.mpa12_batch for runs of the given lengths; a mono batch has noise in channel 1, which
    the synthesis must not read."""
    total = int(sum(lengths))
    x, _ = workloads.mpa12_batch(1, total, layer=layer, seed=seed)
    if channels == 1:
        x[:, 1] = np.random.default_rng(seed).standard_normal(x[:, 1].shape).astype(np.float32)
    return x, _runs(lengths, channels)


def _want(oracle, x, runs, states=None):
    rc, want, states = _oracle.mpa12_batch(oracle, x, runs, int(runs["stream"].max()) + 1, states)
    assert rc == 0 and np.abs(want).max() > 1e-3
    return want, states


def _same(got, want, layer, channels, what):
    """Bit equality on the frame's samples of every channel the runs hold; channel 1 of a mono run and every plane's tail
    beyond 32 x n_slots samples stay +0.0."""
    n = 32 * SLOTS[layer]
    g, w = got[:, :channels, :n].view(np.uint32), want[:, :channels, :n].view(np.uint32)
    bad = np.nonzero(g != w)
    if len(bad[0]):
        f, c, i = bad[0][0], bad[1][0], bad[2][0]
        raise AssertionError(f"{what}: {len(bad[0])} of {g.size} PCM words differ; first at frame {f} ch {c} sample {i}: "
                             f"gpu {got[f, c, i]!r} oracle {want[f, c, i]!r}")
    assert not got[:, :, n:].view(np.uint32).any(), f"{what}: samples written beyond the frame"
    if channels == 1:
        assert not got[:, 1].view(np.uint32).any(), f"{what}: channel 1 of a mono run is not zero"


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [2, 1])
@pytest.mark.parametrize("layer,frames", LONG)
def test_one_long_run_matches_the_oracle(engine, oracle, layer, frames, channels):
    x, runs = _batch(layer, [frames], channels, 4200 + frames + channels)
    _assert_carried_on_device(runs, frames, layer, f"layer {layer}, {frames} frames")
    want, _ = _want(oracle, x, runs)
    engine.mp3_streams_alloc(1)
    _same(engine.mpa12_synth_host(x, runs), want, layer, channels, f"layer {layer}, one run of {frames} frames, {channels} ch")


@pytest.mark.gpu
@pytest.mark.parametrize("layer", [1, 2])
def test_the_threshold_on_this_device(engine, oracle, layer):
    grid = _device_grid()
    for extra in (0, 1):
        frames = grid * TILE_FRAMES[layer] + extra
        x, runs = _batch(layer, [frames], 2, 4300 + layer + extra)
        _, tiles = _plan(runs, frames, layer, grid=0)
        assert (_carried(tiles) > 0) == bool(extra), (grid, frames, _carried(tiles))
        want, _ = _want(oracle, x, runs)
        engine.mp3_streams_alloc(1)
        _same(engine.mpa12_synth_host(x, runs), want, layer, 2, f"layer {layer}, {frames} frames on a grid of {grid}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(MIXED))
@pytest.mark.parametrize("layer", [1, 2])
def test_mixed_runs_in_one_call(engine, oracle, layer, case):
    lengths, _ = MIXED[case](layer)
    x, runs = _batch(layer, lengths, 2, 4400 + layer)
    runs["channels"][1::3] = 1   # some mono streams among them: their channel 1 input holds samples the kernel must skip
    _assert_carried_on_device(runs, len(x), layer, case)
    want, _ = _want(oracle, x, runs)
    engine.mp3_streams_alloc(len(runs))
    got = engine.mpa12_synth_host(x, runs)
    for ch in (1, 2):
        rows = np.concatenate([np.arange(int(r["first_frame"]), int(r["first_frame"] + r["n_frames"])) for r in runs
                               if int(r["channels"]) == ch])
        _same(got[rows], want[rows], layer, ch, f"layer {layer}, {case}, {ch}-channel runs")


@pytest.mark.gpu
@pytest.mark.parametrize("layer", [1, 2])
def test_state_across_calls_and_reset(engine, oracle, layer):
    """A long run split into two calls, each above the threshold, equals one call; after mp3_stream_reset a third call starts
    from silence."""
    T = TILE_FRAMES[layer]
    n1, n2 = GRID * T + 150, GRID * T + 290
    x, runs = _batch(layer, [n1 + n2], 2, 4500 + layer)
    want, _ = _want(oracle, x, runs)
    engine.mp3_streams_alloc(1)
    got = []
    for lo, hi in ((0, n1), (n1, n1 + n2)):
        r = _runs([hi - lo])
        _assert_carried_on_device(r, hi - lo, layer, f"call of frames {lo}..{hi}")
        got.append(engine.mpa12_synth_host(x[lo:hi], r))
    _same(np.concatenate(got), want, layer, 2, f"layer {layer}, one run in calls of {n1} + {n2} frames")
    engine.mp3_stream_reset(0)
    fresh, _ = _want(oracle, x[n1:], _runs([n2]))
    _same(engine.mpa12_synth_host(x[n1:], _runs([n2])), fresh, layer, 2, f"layer {layer}, after a reset")


@pytest.mark.gpu
@pytest.mark.parametrize("layer,frames", [LONG[0], LONG[2]])
def test_device_entry_point_on_torch_tensors(engine, oracle, layer, frames):
    import torch
    x, runs = _batch(layer, [frames], 2, 4600 + layer)
    _assert_carried_on_device(runs, frames, layer, f"layer {layer}, {frames} frames")
    want, _ = _want(oracle, x, runs)
    sub_t = torch.from_numpy(x).cuda()
    pcm_t = torch.zeros((frames, 2, 1152), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()   # the tensors are torch's, written on its stream
    engine.mp3_streams_alloc(1)
    engine.mpa12_synth_dev(sub_t, runs, SLOTS[layer], pcm_t)
    engine.sync()
    _same(pcm_t.cpu().numpy(), want, layer, 2, f"mpa12_synth_dev, layer {layer}, {frames} frames")


# ------------------------------------------------------------------------------------------------ files

# name: (layer, version, bitrate_idx, rate_idx, mode, protected, frames).  Layer I / II frames are self-contained, so a long
# file repeats a pool of distinct frames (the writer is slow); the synthesis state still differs at every repeat.
FILES = {
    "l2_stereo": (2, "1", 8, 0, 0, False, 1250),
    "l2_joint_crc": (2, "1", 12, 1, 1, True, 1230),   # mode_ext changes from frame to frame
    "l2_mono_crc": (2, "1", 4, 0, 3, True, 1210),
    "l1_stereo": (1, "1", 9, 0, 0, False, 3320),
    "l2_mpeg2": (2, "2", 8, 1, 0, False, 1220),
}
POOL = 150


def _pool(kind, seed):
    layer, version, bitrate_idx, rate_idx, mode, protected, _ = FILES[kind]
    rng = np.random.default_rng(seed)
    gen = b12.gen_layer1_frame if layer == 1 else b12.gen_layer2_frame
    return [gen(rng, version, bitrate_idx, rate_idx, mode, mode_ext=k % 4, protected=protected)[0] for k in range(POOL)]


def _cyclic(pool, n, start=0):
    return b"".join(pool[(start + k) % len(pool)] for k in range(n))


@pytest.fixture(scope="module")
def pools():
    return {kind: _pool(kind, 4700 + k) for k, kind in enumerate(FILES)}


@pytest.fixture(scope="module")
def long_files(pools):
    return {kind: _cyclic(pools[kind], FILES[kind][-1]) for kind in FILES}


def _file_runs(files):
    """Per layer, the runs the many-file decoders synthesise: one run of the file's frames per file (mpa12_decode_kernel.cu)."""
    from symphonia_b200 import decode
    out = {}
    for data in files:
        layer, payload, *_ = decode.mpeg_audio_plan(data)
        out.setdefault(layer, []).append(len(payload))
    return out


def _compare_files(got, want, what):
    for k, ((g, rate), (w, wr, _, _)) in enumerate(zip(got, want)):
        g = g.cpu().numpy() if hasattr(g, "cpu") else g
        assert rate == wr and g.shape == w.shape and g.dtype == w.dtype, (what, k, rate, wr, g.shape, w.shape)
        assert g.tobytes() == w.tobytes(), (what, k)


def _file_decoders(engine, files, fmt, want, with_one_file_decoder=True):
    import torch
    from symphonia_b200 import decode
    for layer, lengths in _file_runs(files).items():
        _assert_carried_on_device(_runs(lengths), sum(lengths), layer, f"the layer {layer} files of the call")
    if with_one_file_decoder:
        engine.mp3_streams_alloc(1)
        _compare_files([decode.decode_mpeg_audio(engine, data, fmt, stream=0) for data in files], want, "decode_mpeg_audio")
    for device in (False, True):
        _compare_files(decode.decode_mpa12_files(engine, files, fmt, device=device), want, f"decode_mpa12_files device={device}")
    offs = np.concatenate([[0], np.cumsum([len(f) for f in files])[:-1]])
    data_t = torch.from_numpy(np.frombuffer(b"".join(files), dtype=np.uint8).copy()).cuda()
    _compare_files(decode.decode_mpeg_files_dev(engine, data_t, list(zip(offs.tolist(), [len(f) for f in files])), fmt), want,
                   "decode_mpeg_files_dev")
    _compare_files(decode.decode_any_files(engine, files, fmt, device=True), want, "decode_any_files")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [nat.FMT_S16, nat.FMT_F32])
def test_long_files_decode_like_the_oracle(engine, oracle, long_files, fmt):
    """Each file alone is above the threshold of its layer, and so is each layer of the many-file calls."""
    from tests.test_zz_file_to_pcm import _decode_expect
    files = list(long_files.values())
    for kind, data in long_files.items():
        layer = FILES[kind][0]
        n = _file_runs([data])[layer][0]
        assert n == FILES[kind][-1]
        _assert_carried_on_device(_runs([n], 1 if FILES[kind][4] == 3 else 2), n, layer, kind)
    want = [_decode_expect(oracle, data, fmt) for data in files]
    _file_decoders(engine, files, fmt, want)


@pytest.mark.gpu
def test_many_short_files_form_chains_inside_files(engine, oracle, pools):
    """40 Layer II files of 40 frames: each file is short, the call is above the threshold, so chains form inside files."""
    from tests.test_zz_file_to_pcm import _decode_expect
    kinds = ["l2_stereo", "l2_joint_crc", "l2_mono_crc"]
    files = [_cyclic(pools[kinds[i % 3]], 40, 11 * i) for i in range(40)]
    for fmt in (nat.FMT_S16, nat.FMT_F32):
        want = [_decode_expect(oracle, data, fmt) for data in files]
        _file_decoders(engine, files, fmt, want, with_one_file_decoder=False)
