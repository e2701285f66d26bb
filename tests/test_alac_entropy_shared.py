"""The ALAC packet decoder shared by the CPU front-end and the device kernels (symphonia_b200/csrc/alac_entropy.h), on the CPU.

tests/cpp/alac_entropy_driver.cpp decodes every packet through symgpu_alac_fe_decode_packets, through the shared functions called
as the kernels call them (buffers exactly a job's size) and through the oracle, and counts the packets where any two differ.  It
is built plainly, with the device's byte-wise bit window (SYMGPU_MP3E_DEVICE_WINDOW) and with AddressSanitizer +
UndefinedBehaviorSanitizer."""
import numpy as np
import pytest

from tests import _alac_cases as cases
from tests import _alac_driver as drv
from tests.test_alac_frontend import _damaged, _forced


def _corpus():
    rng = np.random.default_rng(17)
    items = []
    for name, ck, pcm, packet in cases.cases():
        if ck["frame_length"] > 4096:
            continue
        items.append((ck, packet))
        for _ in range(10):
            items.append((ck, _damaged(rng, packet)))
        for tag in (2, 5):
            items.append((ck, _forced(packet, 0, 3, tag)))
        items.append((ck, _forced(packet, 7, 12, 1)))
        items.append((ck, _forced(packet, 20, 2, 3)))
        for mode in (1, 14):
            items.append((ck, _forced(packet, 3 + 4 + 12 + 4 + (32 if len(pcm) != ck["frame_length"] else 0) + 16, 4, mode)))
    return items


@pytest.mark.parametrize("kind", list(drv.BUILDS))
def test_shared_decoder_equals_the_oracle(tmp_path, kind):
    driver = drv.build(tmp_path, kind)
    n, decoded, refused, bad, text = drv.run(driver, tmp_path, _corpus())
    assert bad == 0, text[-2000:]
    assert "runtime error" not in text and "AddressSanitizer" not in text
    assert decoded > n // 4 and refused > n // 4
