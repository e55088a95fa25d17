"""The row shuttle's content light level on an H100: tests/native/shuttle_light_level_test.cpp against libavifgpu.so, so
every 32-bit PQ save goes through avifgpu_encode_rows_async_light_level, and the `clli` it attaches must equal MaxCLL /
MaxFALL of the CPU oracle's reference-layout codes (checked inside the C++ program)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(tmp_path):
    exe = tmp_path / "shuttle_light_level_test"
    pkg = os.path.join(ROOT, "avif-format_b200")
    cmd = ["g++", "-std=c++17", "-O2", "-mfma", "-ffp-contract=off", "-I", os.path.join(pkg, "host"), "-I", os.path.join(pkg, "csrc"),
           "-I", os.path.join(ROOT, "oracle", "shim"),
           os.path.join(ROOT, "tests", "native", "shuttle_light_level_test.cpp"), os.path.join(pkg, "host", "GpuRowShuttle.cpp"),
           os.path.join(ROOT, "oracle", "shim", "mock_heif.cpp"), os.path.join(ROOT, "tests", "native", "mock_heif_content_light_level.cpp"),
           os.path.join(pkg, "lib", "libavifgpu.so"), os.path.join(ROOT, "oracle", "liboracle.so"),
           "-Wl,-rpath," + os.path.join(pkg, "lib"), "-Wl,-rpath," + os.path.join(ROOT, "oracle"), "-lpthread", "-o", str(exe)]
    subprocess.run(cmd, check=True)
    return str(exe)


@pytest.mark.gpu
def test_shuttle_light_level_matches_oracle(tmp_path):
    out = subprocess.run([build(tmp_path)], capture_output=True, text=True, timeout=600)
    print(out.stdout, out.stderr)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "ALL PASSED" in out.stdout and "FAIL" not in out.stdout
