"""The planning of batched planar-RGB decodes, on the CPU: PlanDecodeBatch (the host-described batch) and the per-image step
PlanBatchDecodeImage (the device-described batch's plan kernel) for 8-, 16- and 32-bit hosts.

tests/native/rgb_batch_plan_check.cpp plans seeded random batches of 1 to 300 images -- widths 1 to 7, 8, 9, 255 to 257
and random ones, one-row images, misaligned rows and planes -- for every valid planar-RGB description, and checks exact
pixel coverage, routing against the route (DecodeBatchFamilyOf + DecodeBlockInterior) and against a restatement of the
kernels' alignment rules, image order, the launches per chunk, plane placement against DecodeWindow, unit counts with the
256-pixel unit and FindRecord over them.  It also checks that YCbCr and monochrome descriptions route as before."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "avif-format_b200", "csrc")


def test_planar_rgb_decode_plans_cover_route_and_count_every_image(tmp_path):
    exe = tmp_path / "rgb_batch_plan_check"
    subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-I", "/usr/local/cuda/include", "-I", CSRC,
                    os.path.join(ROOT, "tests", "native", "rgb_batch_plan_check.cpp"), os.path.join(CSRC, "host_params.cpp"),
                    "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    counts = {k: int(v) for k, v in re.findall(r"(\w+)=(\d+)", out.stdout)}
    # x 3 alpha states x 2 ranges: 8-bit hosts 8-bit planes; 16-bit hosts 10 / 12 / 16-bit planes; 32-bit hosts 10 / 12 /
    # 16-bit planes x 4 curves
    assert counts["descriptions"] == 3 * 2 * (1 + 3 + 3 * 4), out.stdout
    assert counts["images"] > 10000 and counts["units"] > 10000 and counts["ycbcr"] > 100, out.stdout
