"""The FLAC output stage's sample conversions on the CPU: the oracle's restatement of the reference's FromSample<i32>
(oracle/oracle_conv_i32.cpp; symphonia-core/src/audio/conv.rs:516-531) pinned to the reference's own assertions, and
decode.flac_convert -- the numpy statement of the same table, which the device path is tested against -- equal to the oracle
value for value.

Reference vectors: conv.rs:709-711 (u8), :924-926 (i16), :967-969 (i24), :1096-1098 (f32): from_sample(i32::MAX) == MAX,
(0) == MID, (i32::MIN) == MIN."""
import ctypes
import os
import re

import numpy as np
import pytest

import symphonia_b200 as sb
from symphonia_b200 import _native as nat
from symphonia_b200 import decode

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FORMATS = (nat.FMT_F32, nat.FMT_S16, nat.FMT_S24, nat.FMT_S32, nat.FMT_U8)
I32_MAX, I32_MIN = 2 ** 31 - 1, -2 ** 31


@pytest.fixture(scope="module")
def conv(oracle):
    for name, res in (("u8", ctypes.c_uint8), ("s16", ctypes.c_int16), ("s24", ctypes.c_int32), ("f32", ctypes.c_float)):
        fn = getattr(oracle, "oracle_conv_i32_" + name)
        fn.restype, fn.argtypes = res, [ctypes.c_int32]
    oracle.oracle_conv_i32_pack.restype = ctypes.c_int
    oracle.oracle_conv_i32_pack.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]
    return oracle


def _oracle_pack(conv, s, fmt):
    s = np.ascontiguousarray(s, dtype=np.int32)
    out = np.zeros(s.shape, dtype=nat.FMT_NUMPY[fmt])
    assert conv.oracle_conv_i32_pack(s.ctypes.data_as(ctypes.c_void_p), s.size, fmt, out.ctypes.data_as(ctypes.c_void_p)) == 0
    return out


def test_reference_min_mid_max_vectors(conv):
    assert [conv.oracle_conv_i32_u8(v) for v in (I32_MAX, 0, I32_MIN)] == [255, 128, 0]
    assert [conv.oracle_conv_i32_s16(v) for v in (I32_MAX, 0, I32_MIN)] == [32767, 0, -32768]
    assert [conv.oracle_conv_i32_s24(v) for v in (I32_MAX, 0, I32_MIN)] == [8388607, 0, -8388608]
    assert [conv.oracle_conv_i32_f32(v) for v in (I32_MAX, 0, I32_MIN)] == [float(np.float32(2147483647.0 / 2147483648.0)), 0.0, -1.0]
    # the array form is the scalars in a loop, and refuses a format it does not know
    edge = np.array([I32_MAX, 0, I32_MIN], dtype=np.int32)
    assert _oracle_pack(conv, edge, nat.FMT_U8).tolist() == [255, 128, 0] and _oracle_pack(conv, edge, nat.FMT_S32).tolist() == edge.tolist()
    assert conv.oracle_conv_i32_pack(edge.ctypes.data_as(ctypes.c_void_p), 3, 99, edge.ctypes.data_as(ctypes.c_void_p)) == 1


def test_shifts_are_arithmetic_and_f32_rounds_once(conv):
    assert conv.oracle_conv_i32_s16(-1) == -1 and conv.oracle_conv_i32_s24(-1) == -1 and conv.oracle_conv_i32_u8(-1) == 127
    assert conv.oracle_conv_i32_s16(-65537) == -2 and conv.oracle_conv_i32_s24(-257) == -2 and conv.oracle_conv_i32_s24(255) == 0
    # 2^24 + 1 is not a float: the quotient is rounded to nearest even, once
    assert conv.oracle_conv_i32_f32(2 ** 24 + 1) == 2.0 ** -7 and conv.oracle_conv_i32_f32(2 ** 24 + 3) == float(np.float32(2 ** 24 + 4)) / 2.0 ** 31
    assert conv.oracle_conv_i32_f32(-(2 ** 24) - 1) == -(2.0 ** -7)


def test_flac_convert_equals_the_oracle(conv):
    edge = [I32_MIN, I32_MAX, 0, -1, 1, 255, -255, 256, -256]
    edge += [sign * (2 ** 24 + d) for sign in (1, -1) for d in (-1, 1)]
    rng = np.random.default_rng(20)
    s = np.concatenate([np.array(edge, dtype=np.int32), rng.integers(I32_MIN, I32_MAX, 1_000_000, dtype=np.int64, endpoint=True).astype(np.int32)])
    for fmt in FORMATS:
        got, want = decode.flac_convert(s, fmt), _oracle_pack(conv, s, fmt)
        assert got.dtype == want.dtype == np.dtype(nat.FMT_NUMPY[fmt]) and got.shape == s.shape
        assert (got.view(np.uint8) == want.view(np.uint8)).all(), fmt
    assert decode.flac_convert(s, nat.FMT_S24).dtype == np.int32 and np.abs(decode.flac_convert(s, nat.FMT_S24).astype(np.int64)).max() <= 2 ** 23
    two_d = decode.flac_convert(s[:12].reshape(4, 3), nat.FMT_S16)                 # [frames, channels] in, the same shape out
    assert two_d.shape == (4, 3) and (two_d == decode.flac_convert(s[:12], nat.FMT_S16).reshape(4, 3)).all()
    with pytest.raises(ValueError):
        decode.flac_convert(s[:4], 99)


def test_format_calls_are_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "symgpu.h")).read()
    lib = sb.lib()
    for name in ("symgpu_flac_decode_fmt_host", "symgpu_flac_decode_fmt_dev", "symgpu_flac_decode_host", "symgpu_flac_decode_dev"):
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert hasattr(lib, name), name
    # the format comes before a void* output in the new pair; the old pair keeps its int32_t* output
    assert re.search(r"symgpu_flac_decode_fmt_host\([^;]*int format, void\* out, size_t out_cap", hdr)
    assert re.search(r"symgpu_flac_decode_host\([^;]*int32_t\* out, size_t out_cap", hdr)
