"""Builds and runs tests/cpp/alac_entropy_driver.cpp (the shared ALAC packet decoder against the oracle, on the CPU)."""
import os
import struct
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCES = [os.path.join(ROOT, "tests", "cpp", "alac_entropy_driver.cpp"), os.path.join(ROOT, "symphonia_b200", "csrc", "alac_frontend.cpp"),
           os.path.join(ROOT, "oracle", "oracle_alac.cpp")]
BUILDS = {"plain": ["-O2"], "device window": ["-O2", "-DSYMGPU_MP3E_DEVICE_WINDOW"],
          "sanitized": ["-O1", "-g", "-DSYMGPU_MP3E_DEVICE_WINDOW", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"]}


def build(tmp, kind):
    out = str(tmp / ("alac_driver_" + kind.replace(" ", "_")))
    subprocess.check_call(["g++", "-std=c++17", "-ffp-contract=off", "-I/usr/local/cuda/include"] + BUILDS[kind] + ["-o", out] + SOURCES)
    return out


def run(driver, tmp, items):
    """items: [(cookie dict, packet bytes)].  Returns (n, decoded, refused, mismatches, output text)."""
    blob = b"".join(struct.pack("<7I", ck["frame_length"], ck["bit_depth"], ck["pb"], ck["mb"], ck["kb"], ck["channels"], len(p)) + p
                    for ck, p in items)
    src = str(tmp / "alac_in.bin")
    with open(src, "wb") as f:
        f.write(blob)
    res = subprocess.run([driver, src], capture_output=True, text=True, timeout=900,
                         env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=1", UBSAN_OPTIONS="print_stacktrace=1"))
    text = res.stdout + res.stderr
    assert res.returncode in (0, 1), text[-3000:]
    n, dec, ref, bad = (int(v) for v in res.stdout.split()[:4])
    return n, dec, ref, bad, text
