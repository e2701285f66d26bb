"""A sanitized fuzz pass over the ALAC front-end: random bytes, bit-flipped and spliced writer packets, under random magic
cookies, through tests/cpp/alac_entropy_driver.cpp built with AddressSanitizer + UndefinedBehaviorSanitizer.  No report may
appear, and the front-end, the kernels' call sequence and the oracle must agree on every packet."""
import numpy as np

from tests import _alac_cases as cases
from tests import _alac_driver as drv


def _cookie(rng):
    return dict(frame_length=int(rng.choice([1, 16, 64, 300, 4096])), bit_depth=int(rng.choice([0, 1, 8, 16, 20, 24, 31, 32, 33, 40])),
                pb=int(rng.integers(0, 256)), mb=int(rng.integers(0, 256)), kb=int(rng.integers(0, 256)), channels=int(rng.integers(1, 9)))


def test_fuzz_frontend_sanitized(tmp_path):
    rng = np.random.default_rng(1234)
    seeds = [p for _, _, _, p in cases.cases() if len(p) < 20000]
    items = []
    for k in range(3000):
        ck = _cookie(rng)
        ck["bit_depth"] = min(ck["bit_depth"], 32)
        if k % 3 == 0:
            p = rng.integers(0, 256, size=int(rng.integers(0, 300)), dtype=np.uint8).tobytes()
        else:
            b = bytearray(seeds[int(rng.integers(len(seeds)))])
            for _ in range(int(rng.integers(1, 6))):
                if b:
                    i = int(rng.integers(len(b)))
                    b[i] ^= 1 << int(rng.integers(8))
            if k % 3 == 2:
                b = b[:int(rng.integers(0, len(b) + 1))]
            p = bytes(b)
        items.append((ck, p))
    driver = drv.build(tmp_path, "sanitized")
    n, decoded, refused, bad, text = drv.run(driver, tmp_path, items)
    assert n == len(items) and bad == 0, text[-2000:]
    assert "runtime error" not in text and "AddressSanitizer" not in text
    assert decoded > 0 and refused > 0
