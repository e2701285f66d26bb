"""The AAC-LC packet rules shared by the CPU front-end and the device kernels (symphonia_b200/csrc/aac_entropy.h), on the CPU.

tests/cpp/aac_entropy_driver.cpp runs the device's schedule -- every packet decoded from a fresh state in a shuffled order, the
per-file walk over the records, the packets that drew noise decoded again from their real generator states, the pulse step with
the scale factors the walk names -- and compares every packet with symgpu_aac_fe_decode called packet by packet in order: status,
units, the TNS records each unit names and the coefficient bits.  The driver is built with -ffp-contract=off and the device's bit
window, and once more with AddressSanitizer + UndefinedBehaviorSanitizer.  The corpus (tests/_aac_corpus.py) has writer streams
at eight rate classes, mono and stereo, with noise, pulses and TNS; truncated and bit-flipped packets between noise packets; a
stereo file whose lone first single-channel element fixes a layout that refuses the pairs behind it; a layout that changes
mid-file; and pulses in bands no section coded, after a decoded packet, after a refused one and with no packet before."""
import os
import struct
import subprocess

import pytest

from tests import _aac_corpus as corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "symphonia_b200", "csrc")


@pytest.fixture(scope="module")
def drivers(tmp_path_factory):
    d = tmp_path_factory.mktemp("aac_entropy")
    src = [os.path.join(ROOT, "tests", "cpp", "aac_entropy_driver.cpp"), os.path.join(CSRC, "aac_frontend.cpp")]
    common = ["g++", "-std=c++17", "-ffp-contract=off", "-DSYMGPU_MP3E_DEVICE_WINDOW", "-I/usr/local/cuda/include", "-pthread"]
    plain, sanitized = str(d / "driver_devwin"), str(d / "driver_sanitized")
    subprocess.check_call(common + ["-O2", "-o", plain] + src)
    subprocess.check_call(common + ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-o", sanitized] + src)
    return d, {"device window": plain, "sanitized": sanitized}


def _run(driver, tmp, files, seed):
    blob = struct.pack("<I", len(files))
    for _, packets, rate, channels in files:
        blob += struct.pack("<3I", rate, channels, len(packets)) + b"".join(struct.pack("<I", len(p)) + p for p in packets)
    src = str(tmp / "in.bin")
    with open(src, "wb") as f:
        f.write(blob)
    res = subprocess.run([driver, src, str(seed)], capture_output=True, text=True, timeout=900,
                         env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=1"))
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    return [int(v) for v in res.stdout.split()]


@pytest.mark.parametrize("build", ["device window", "sanitized"])
def test_device_schedule_equals_the_front_end(drivers, build):
    tmp, exes = drivers
    files = corpus.corpus()
    for seed in (1, 2):
        decoded, refused, unsupported, redecoded, pulses, stale = _run(exes[build], tmp, files, seed)
        assert decoded + refused + unsupported == sum(len(f[1]) for f in files)
        # every kind of packet the corpus is there for was met
        assert decoded > 100 and refused >= 10 and unsupported >= 1
        assert redecoded > 50 and pulses > 10 and stale >= 6


def test_one_file_at_a_time_equals_all_files_at_once(drivers):
    """The schedule across files is independent: each file alone gives the same counts as its share of the whole corpus."""
    tmp, exes = drivers
    files = corpus.corpus()
    whole = _run(exes["device window"], tmp, files, 3)
    parts = [_run(exes["device window"], tmp, [f], 3) for f in files]
    assert [sum(p[i] for p in parts) for i in range(6)] == whole
