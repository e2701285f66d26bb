"""The thread-safe submission ABI without a device: every new entry point refuses a missing context or buffer with
SYMGPU_ERR_ARG (no C++ exception, no crash), and the per-codec statistics refuse an unknown codec."""
import ctypes

from symphonia_b200 import _native as nat

ERR_ARG = 6


def test_new_entry_points_refuse_missing_arguments():
    L = nat.lib()
    t = nat.Ticket()
    tp = ctypes.byref(t)
    base = ctypes.c_uint32(0)
    assert L.symgpu_aac_submit(None, 0, None, None, 0, None, 2, tp) == ERR_ARG
    assert L.symgpu_mpa12_submit(None, 0, None, 36, 2, tp) == ERR_ARG
    assert L.symgpu_vorbis_submit(None, 0, None, None, None, 1024, tp) == ERR_ARG
    for name in ("symgpu_mp3_wait", "symgpu_aac_wait", "symgpu_mpa12_wait", "symgpu_vorbis_wait"):
        assert getattr(L, name)(None, t, None) == ERR_ARG, name
    assert L.symgpu_vorbis_streams_alloc(None, 4) == ERR_ARG
    assert L.symgpu_vorbis_stream_configure(None, 0, None, None, 0, ctypes.byref(base)) == ERR_ARG
    b, f = ctypes.c_uint64(7), ctypes.c_uint64(7)
    assert L.symgpu_async_stats(None, nat.CODEC_AAC, ctypes.byref(b), ctypes.byref(f)) == ERR_ARG
    L.symgpu_mp3_async_stats.restype = None
    L.symgpu_mp3_async_stats.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    L.symgpu_mp3_async_stats(None, ctypes.byref(b), ctypes.byref(f))
    assert (b.value, f.value) == (0, 0)


def test_ticket_layout_matches_the_header():
    assert ctypes.sizeof(nat.Ticket) == 16
    assert [nat.CODEC_MP3, nat.CODEC_MP1, nat.CODEC_MP2, nat.CODEC_AAC, nat.CODEC_VORBIS] == [0, 1, 2, 3, 4]
