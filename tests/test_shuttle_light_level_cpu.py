"""The row shuttle's content light level (avifgpu_host::SetContentLightLevelEnabled) on a machine WITHOUT a GPU: the native
program tests/native/shuttle_light_level_test.cpp -- mock Photoshop host, mock libheif, 32-bit PQ saves with the switch on
and off -- linked against tests/native/fake_avifgpu_on_oracle.cpp and tests/native/fake_light_level_on_oracle.cpp, whose
light-level host calls measure the oracle's own reference-layout codes.  What this pins is the shuttle's logic: which
saves measure, one accumulator across every block, the row transform applied first, the values attached with
heif_image_set_content_light_level and reported, nothing after a cancelled save.  The library's own measurement is the GPU tests' business."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(tmp_path):
    exe = tmp_path / "shuttle_light_level_test_cpu"
    pkg = os.path.join(ROOT, "avif-format_b200")
    native = os.path.join(ROOT, "tests", "native")
    cmd = ["g++", "-std=c++17", "-O2", "-mfma", "-ffp-contract=off", "-I", os.path.join(pkg, "host"),
           "-I", os.path.join(pkg, "csrc"), "-I", os.path.join(ROOT, "oracle", "shim"),
           os.path.join(native, "shuttle_light_level_test.cpp"), os.path.join(native, "fake_avifgpu_on_oracle.cpp"),
           os.path.join(native, "fake_light_level_on_oracle.cpp"), os.path.join(native, "mock_heif_content_light_level.cpp"),
           os.path.join(pkg, "host", "GpuRowShuttle.cpp"), os.path.join(ROOT, "oracle", "shim", "mock_heif.cpp"),
           os.path.join(pkg, "lib", "libavifgpu.so"), os.path.join(ROOT, "oracle", "liboracle.so"),
           "-Wl,-rpath," + os.path.join(pkg, "lib"), "-Wl,-rpath," + os.path.join(ROOT, "oracle"), "-lpthread", "-o", str(exe)]
    subprocess.run(cmd, check=True)
    return str(exe)


def test_shuttle_light_level_logic_on_the_cpu(tmp_path):
    out = subprocess.run([build(tmp_path)], capture_output=True, text=True, timeout=600)
    print(out.stdout, out.stderr)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "ALL PASSED" in out.stdout and "FAIL" not in out.stdout
