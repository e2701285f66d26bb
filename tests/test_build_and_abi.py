"""CPU tier: the C-ABI library loads, exports every symbol include/symgpu.h declares, contains no
fused multiply-add in its SASS (parity depends on it), fails loudly without a GPU, and its host-built
tables equal the oracle's independently written tables bit for bit."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "symgpu.h")).read()
    return sorted(set(re.findall(r"\b(symgpu_[a-z0-9_]+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol():
    import symphonia_b200 as sb
    lib = sb.lib()
    names = _declared_symbols()
    assert len(names) >= 12
    for name in names:
        assert hasattr(lib, name), f"{name} declared in include/symgpu.h but not exported"
    assert lib.symgpu_abi_version() == 1


def _sass_by_function(lib_path):
    sass = subprocess.run(["cuobjdump", "-sass", lib_path], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(ln)
    return sass, {k: "\n".join(v) for k, v in funcs.items()}


def test_no_fused_multiply_add_in_sass():
    """Bit-exact parity needs every product and every sum rounded on its own: -fmad=false, and the channel-pair
    arithmetic of the MP3 kernels is written as separate __fmul_rn / __fadd_rn / __fsub_rn per channel.  Held here:
    the library is sm_90a code only, with no FFMA / DFMA (scalar or packed) in any kernel, and the MP3 kernels keep
    their products and sums as FMUL / FADD."""
    import symphonia_b200 as sb
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    sass, funcs = _sass_by_function(sb.lib_path())
    archs = set(re.findall(r"arch = (sm_\w+)", sass))
    assert archs == {"sm_90a"}, f"kernels built for {sorted(archs)}, not sm_90a only"
    hits = re.findall(r"\b(FFMA|DFMA|FFMA2)\b", sass)
    assert not hits, f"{len(hits)} fused multiply-adds in the kernels: bit-exact parity would break"
    assert re.search(r"\bFMUL\b", sass) and re.search(r"\bFADD\b", sass)
    mp3 = {k: v for k, v in funcs.items() if "mp3v2" in k or "hybrid_mixed" in k or "mp3_synth_kernel" in k}
    assert mp3, "the MP3 synthesis kernels are missing from the library"
    for k, v in mp3.items():
        assert re.search(r"\bFMUL\b", v) and re.search(r"\bFADD\b", v), k


def test_tables_match_oracle(oracle):
    import symphonia_b200 as sb
    lib = sb.lib()
    n = lib.symgpu_tables_host_blob(None, 0)
    blob = np.zeros(n, dtype=np.uint8)
    assert lib.symgpu_tables_host_blob(blob.ctypes.data_as(ctypes.c_void_p), n) == n
    no = oracle.oracle_mp3_tables(None, 0)
    want = np.zeros(no, dtype=np.float32)
    oracle.oracle_mp3_tables(want.ctypes.data_as(ctypes.c_void_p), no)
    got = blob[: 4 * no].view(np.float32)
    assert no == 915
    assert (got.view(np.uint32) == want.view(np.uint32)).all()
    # requantisation scale table: (float)pow(2, 0.25*k), k = -521..46  (requantize.rs:280, :343)
    pow2q = blob[4 * no: 4 * (no + 568)].view(np.float32)
    k = np.arange(-521, 47, dtype=np.float64)
    assert (pow2q == np.exp2(0.25 * k).astype(np.float32)).all()
    pow43 = sb._native.mp3_pow43()
    assert all(pow43[i] == np.float32(oracle.oracle_mp3_pow43(i)) for i in (0, 1, 2, 8, 27, 100, 8206))


def test_engine_fails_loudly_without_gpu():
    import torch
    import symphonia_b200 as sb
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(sb.SymgpuError):
        sb.Engine(0)


def test_workload_generator_is_deterministic_and_well_formed():
    from symphonia_b200 import workloads
    u1, s1, r1 = workloads.mp3_batch(3, 4, seed=5)
    u2, s2, r2 = workloads.mp3_batch(3, 4, seed=5)
    assert (u1.view(np.uint8) == u2.view(np.uint8)).all() and (s1 == s2).all() and (r1 == r2).all()
    assert s1.shape == (12, 2, 2, 576) and u1.shape == (12, 2, 2)
    rz = u1["rzero"]
    line = np.arange(576)
    assert (s1[line[None, None, None, :] >= rz[..., None]] == 0).all()
    assert not np.signbit(s1[s1 == 0]).any()   # zeros are +0.0, as the reference writes them
    # joint stereo requires equal block types in both channels (stereo.rs:503-505)
    assert (u1["block_type"][:, :, 0] == u1["block_type"][:, :, 1]).all()


def test_codec_tables_match_oracle(oracle):
    """FFT / IMDCT twiddles, AAC windows, Vorbis windows and the inverse-dB table built by the product
    (tables.cpp) equal the oracle's independently written ones bit for bit."""
    import symphonia_b200 as sb
    lib = sb.lib()
    n = lib.symgpu_codec_tables_host_blob(None, 0)
    blob = np.zeros(n, dtype=np.uint8)
    lib.symgpu_codec_tables_host_blob(blob.ctypes.data_as(ctypes.c_void_p), n)
    f = blob.view(np.float32)
    pos = 0

    def take(count):
        nonlocal pos
        out = f[pos:pos + count]
        pos += count
        return out

    lit16, lit32, merge = take(16).reshape(8, 2), take(32).reshape(16, 2), take(2 * 2016).reshape(2016, 2)
    tw_long, tw_short, vtw = take(1024).reshape(512, 2), take(128).reshape(64, 2), take(2 * 4080).reshape(4080, 2)
    sine_long, sine_short, kbd_long, kbd_short = take(1024), take(128), take(1024), take(128)
    vwin, inv_db = take(8160), take(256)
    out = (ctypes.c_float * 2)()

    def tw(size, k):
        oracle.oracle_fft_twiddle(size, k, out)
        return np.float32(out[0]), np.float32(out[1])

    for k in range(8):
        assert tuple(lit16[k]) == tw(16, k)
    for k in range(16):
        assert tuple(lit32[k]) == tw(32, k)
    for size in (64, 128, 512, 2048):
        for k in (0, 1, size // 8, size // 4, size // 2 - 1):
            assert tuple(merge[size // 2 - 32 + k]) == tw(size, k), (size, k)
    oracle.oracle_imdct_twiddle.argtypes = [ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_void_p]

    def itw(nn, scale, k):
        oracle.oracle_imdct_twiddle(nn, scale, k, out)
        return np.float32(out[0]), np.float32(out[1])

    for k in (0, 1, 255, 511):
        assert tuple(tw_long[k]) == itw(1024, 1.0 / 2048.0, k)
    for k in (0, 31, 63):
        assert tuple(tw_short[k]) == itw(128, 1.0 / 256.0, k)
    for n2 in (16, 64, 512, 2048):
        for k in (0, n2 // 2, n2 - 1):
            assert tuple(vtw[n2 - 16 + k]) == itw(2 * n2, 1.0, k), (n2, k)
    get = oracle.oracle_aac_window
    for arr, (kbd, short, ln) in ((sine_long, (0, 0, 1024)), (sine_short, (0, 1, 128)), (kbd_long, (1, 0, 1024)),
                                  (kbd_short, (1, 1, 128))):
        want = np.ctypeslib.as_array(get(kbd, short), shape=(ln,))
        assert (arr.view(np.uint32) == want.view(np.uint32)).all()
    for bs in (64, 256, 2048, 8192):
        want = np.ctypeslib.as_array(oracle.oracle_vorbis_window(bs), shape=(bs // 2,))
        got = vwin[bs // 2 - 32: bs // 2 - 32 + bs // 2]
        assert (got.view(np.uint32) == want.view(np.uint32)).all()
    assert all(np.float32(oracle.oracle_vorbis_inverse_db(i)) == inv_db[i] for i in range(256))
    assert pos * 4 == n
