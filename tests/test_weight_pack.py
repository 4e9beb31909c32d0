"""CPU: the 12-bit packed weight format (moe-infinity_b200/csrc/weight_pack.cuh, shared with the GEMM kernels) round-trips.

tests/host/weight_pack_check.cpp encodes and decodes tiles on the host and demands every bf16 bit back: N(0, sigma) tiles at
several sigma, signed zeros and subnormals, 16 patches (coded) and 17 (raw), Inf/NaN (raw), windows across the whole
exponent range, random bit patterns."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_encode_decode_is_bit_exact(tmp_path):
    exe = tmp_path / "weight_pack_check"
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-I", os.path.join(ROOT, "moe-infinity_b200", "csrc"),
                    os.path.join(ROOT, "tests", "host", "weight_pack_check.cpp"), "-o", str(exe)], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.startswith("OK"), r.stdout + r.stderr
