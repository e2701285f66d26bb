"""Seeded ALAC packets from tests/_alac_bitstream.py and the oracle that decodes them (oracle/oracle_alac.cpp), shared by the ALAC
tests."""
import ctypes

import numpy as np

from tests import _alac_bitstream as ab
from tests import _oracle


def oracle_lib():
    lib = _oracle.load()
    lib.oracle_alac_packet.restype = ctypes.c_int
    lib.oracle_alac_packet.argtypes = [ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_uint32] * 6 + [ctypes.c_void_p, ctypes.c_void_p]
    return lib


def oracle_packet(lib, packet, cookie):
    """(refused, samples [frames, channels] int32 scaled to 32 bits) of one packet, as the oracle decodes it."""
    ch, fl = cookie["channels"], cookie["frame_length"]
    planes = np.zeros((ch, max(fl, 1)), dtype=np.int32)
    frames = ctypes.c_uint32(0)
    buf = np.frombuffer(packet, dtype=np.uint8) if len(packet) else np.zeros(1, dtype=np.uint8)
    rc = lib.oracle_alac_packet(buf.ctypes.data_as(ctypes.c_void_p), len(packet), fl, cookie["bit_depth"], cookie["pb"], cookie["mb"],
                                cookie["kb"], ch, planes.ctypes.data_as(ctypes.c_void_p), ctypes.byref(frames))
    return rc != 0, planes[:, :frames.value].T.copy()


def cookie(channels=2, bit_depth=16, frame_length=256, pb=40, mb=10, kb=14):
    return dict(frame_length=frame_length, bit_depth=bit_depth, pb=pb, mb=mb, kb=kb, channels=channels)


def cases(seed=7):
    """[(name, cookie, pcm [frames, channels], packet)] covering the writer's features."""
    rng = np.random.default_rng(seed)
    out = []

    def add(name, ck, pcm, elements=None):
        out.append((name, ck, pcm, ab.encode_packet(pcm, ck, elements)))
    for ch in range(1, 9):
        ck = cookie(channels=ch, frame_length=96)
        add(f"layout{ch}", ck, ab.signal(rng, 96, ch, 16))
    for bd in (16, 20, 24, 32):  # a 32-bit CPE needs tail bits: its coded samples carry one bit more than the depth
        ck = cookie(bit_depth=bd, frame_length=128)
        add(f"bits{bd}", ck, ab.signal(rng, 128, 2, bd), [dict(kind="cpe", shift=8 if bd == 32 else 0, order=4, coeffs=[500, -300, 100, 20], lpc_shift=9)])
        add(f"bits{bd}_mono", cookie(channels=1, bit_depth=bd, frame_length=128), ab.signal(rng, 128, 1, bd))
    for order in list(range(0, 32, 3)) + [31]:
        ck = cookie(channels=1, frame_length=160)
        coeffs = [int(v) for v in rng.integers(-400, 400, size=32)]
        add(f"order{order}", ck, ab.signal(rng, 160, 1, 16), [dict(kind="sce", order=order, coeffs=coeffs, lpc_shift=9)])
    ck = cookie(channels=1, frame_length=160)
    add("mode15", ck, ab.signal(rng, 160, 1, 16), [dict(kind="sce", order=8, mode=15, coeffs=[300, -200, 100, 50, 0, 0, 10, 5], lpc_shift=9)])
    for shift in (8, 16):
        ck = cookie(bit_depth=24, frame_length=128)
        add(f"tail{shift}", ck, ab.signal(rng, 128, 2, 24), [dict(kind="cpe", shift=shift, order=4, coeffs=[500, -300, 100, 20], lpc_shift=9)])
        add(f"tail{shift}_mono", cookie(channels=1, bit_depth=24), ab.signal(rng, 256, 1, 24), [dict(kind="sce", shift=shift, order=2, coeffs=[1000, -500], lpc_shift=10)])
    for w_, s_ in ((1, 1), (2, 3), (-3, 2), (5, 31)):
        ck = cookie(frame_length=128)
        add(f"midside{w_}_{s_}", ck, ab.signal(rng, 128, 2, 16), [dict(kind="cpe", ms_weight=w_, ms_shift=s_, order=4, coeffs=[200, -100, 50, 10], lpc_shift=8)])
    ck = cookie(frame_length=256)
    add("partial", ck, ab.signal(rng, 77, 2, 16), [dict(kind="cpe", partial=True, order=2, coeffs=[700, -300], lpc_shift=9)])
    sil = np.zeros((256, 1), dtype=np.int64)
    sil[5, 0], sil[200, 0] = 3, -2
    add("zero_runs", cookie(channels=1), sil, [dict(kind="sce")])
    add("zero_run_ffff", cookie(channels=1, frame_length=65536), np.zeros((65536, 1), dtype=np.int64), [dict(kind="sce")])
    loud = rng.integers(-30000, 30000, size=(64, 2))
    add("escapes", cookie(frame_length=64, mb=255, kb=4), loud, [dict(kind="cpe")])
    add("uncompressed", cookie(frame_length=64), ab.signal(rng, 64, 2, 16), [dict(kind="cpe", uncompressed=True)])
    add("uncompressed_mono24", cookie(channels=1, bit_depth=24, frame_length=64), ab.signal(rng, 64, 1, 24), [dict(kind="sce", uncompressed=True)])
    add("dse_fil_end", cookie(frame_length=64), ab.signal(rng, 64, 2, 16),
        [dict(kind="dse", count=3, align=True), dict(kind="fil", count=20), dict(kind="dse", count=300), dict(kind="fil", count=4),
         dict(kind="cpe", order=2, coeffs=[300, -100], lpc_shift=8), dict(kind="end")])
    return out
