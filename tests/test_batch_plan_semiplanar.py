"""Semi-planar and MSB-aligned decode sources (avifgpu_decode_desc.source_layout) on the CPU: validation, the API-9-sized
description, plane geometry, and the planning of both batch APIs for them.

tests/native/semiplanar_plan_check.cpp checks the validation of every layout bit set x colour space x bit depth, that an
API-9-sized description is accepted as planar, the interleaved plane's geometry, and, for every YCbCr description into 8-,
16- and 32-bit hosts in each layout, seeded random batches -- odd widths, one-row images, misaligned rows, Y planes and
interleaved chroma planes -- for exact pixel coverage, routing against the block halves (DecodeBlockInterior of
DecodeBatchFamilyOf) and a restatement of the interleaved plane's alignment, plane placement against DecodeWindow, unit
counts, launches per chunk and FindRecord."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "avif-format_b200", "csrc")


def test_semiplanar_sources_validate_route_and_plan(tmp_path):
    exe = tmp_path / "semiplanar_plan_check"
    subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-I", "/usr/local/cuda/include", "-I", CSRC,
                    os.path.join(ROOT, "tests", "native", "semiplanar_plan_check.cpp"), os.path.join(CSRC, "host_params.cpp"),
                    "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    counts = {k: int(v) for k, v in re.findall(r"(\w+)=(\d+)", out.stdout)}
    # 8 layout values x 3 colour spaces x 4 depths, plus 4 geometries
    assert counts["validations"] == 8 * 3 * 4 + 4, out.stdout
    # 8-bit hosts: 8-bit planes, 2 layouts; 16-bit hosts: 10/12-bit planes, 4 layouts; 32-bit hosts: 10/12-bit planes,
    # 4 layouts, 3 curves -- each x 3 alpha states x 3 chroma modes
    assert counts["descriptions"] == 9 * (2 + 2 * 4 + 2 * 4 * 3), out.stdout
    assert counts["images"] > 10000 and counts["units"] > 10000, out.stdout
