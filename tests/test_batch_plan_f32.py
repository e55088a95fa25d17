"""The planning of batched float-host YCbCr decodes, on the CPU: PlanDecodeBatch (the host-described batch) and the
per-image step PlanBatchDecodeImage (the device-described batch's plan kernel) for 32-bit hosts.

tests/native/f32_batch_plan_check.cpp plans seeded random batches of 1 to 300 images -- widths below 4, one-row images,
misaligned rows and Y planes, unequal Cb / Cr strides -- for every valid YCbCr float-host description, the verified
divisions off and on, and checks exact pixel coverage, routing against DecodeBlockInterior of DecodeBatchFamilyOf, image order, the launches
per chunk, plane placement against DecodeWindow, unit counts with the 128-pixel unit and FindRecord over them."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "avif-format_b200", "csrc")


def test_float_decode_plans_cover_route_and_count_every_image(tmp_path):
    exe = tmp_path / "f32_batch_plan_check"
    subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-I", "/usr/local/cuda/include", "-I", CSRC,
                    os.path.join(ROOT, "tests", "native", "f32_batch_plan_check.cpp"), os.path.join(CSRC, "host_params.cpp"),
                    "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    counts = {k: int(v) for k, v in re.findall(r"(\w+)=(\d+)", out.stdout)}
    # 10 / 12 / 16-bit planes (8-bit ones are refused for float hosts) x 3 alpha states x 3 chroma modes x 4 curves x 2
    assert counts["descriptions"] == 3 * 3 * 3 * 4 * 2, out.stdout
    assert counts["images"] > 10000 and counts["units"] > 10000, out.stdout
