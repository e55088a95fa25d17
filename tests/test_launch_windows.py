"""The edge-strip windows of the tuned launchers (EncodeWindow / DecodeWindow in csrc/kernel_params.h) against the host
plane geometry (csrc/host_params.cpp), on the CPU.

Every tuned kernel converts an aligned interior of its block and hands the right strip and the odd last 4:2:0 row to the
generic kernel as windows of the block.  tests/native/launch_window_check.cpp takes every valid encode and decode
description, fills it with FillEncodeParams / FillDecodeParams on fake padded planes, and checks windows over a grid of
row blocks (odd decode block starts and odd window starts included): every rows and plane pointer must land where
Encode/DecodePlaneGeometry and Encode/DecodeHostColBytes put that pixel of the image, absent planes stay null, width,
row count and 4:2:0 phase follow, and a window of a window equals the composed window."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "avif-format_b200", "csrc")


def test_windows_match_the_plane_geometry(tmp_path):
    exe = tmp_path / "launch_window_check"
    subprocess.run(["g++", "-std=c++17", "-ffp-contract=off", "-I", "/usr/local/cuda/include", "-I", CSRC,
                    os.path.join(ROOT, "tests", "native", "launch_window_check.cpp"), os.path.join(CSRC, "host_params.cpp"),
                    "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    # every valid description of each direction, each checked at every window of the grid
    assert out.stdout.split("\n")[:2] == ["encode descriptions=120 windows=198720", "decode descriptions=105 windows=196560"], out.stdout
