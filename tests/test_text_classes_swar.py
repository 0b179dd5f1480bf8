"""The parse kernels' two-byte clean test (dev_common.cuh utf8_unclean2) flags exactly what utf8_unclean4 flags for
every pair of words it is used on: tests/text_classes_check.cu runs both on the host, exhaustively over an alphabet of
the bytes the rule turns on and over 10^8 random pairs.  No GPU needed; nvcc compiles the check."""
import os
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def test_two_byte_clean_test_matches_the_general_one():
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "text_classes_check")
        subprocess.check_call([NVCC, "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                               os.path.join(HERE, "text_classes_check.cu")])
        r = subprocess.run([exe, "100000000"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("ok:"), r.stdout
