"""The per-image planning step both batch APIs share (PlanBatchEncodeImage / PlanBatchDecodeImage, csrc/batch_plan.h),
and the workspace of the device-described batch, on the CPU.

tests/native/indirect_plan_check.cpp compiles the per-image step -- the same __host__ __device__ functions the plan kernel
runs -- with the host compiler.  Over seeded random image sets (sizes 0 to 600, negative sizes, NULL rows and planes,
misaligned pointers and strides) for every supported encode and decode description it checks that rejected images get
BAD_PARAM and no record; that an accepted image's records cover every pixel exactly once, judged from their rows
pointers, with their planes at their first pixel and chroma site; that an image has an interior exactly when the
single-image predicate of its own block (EncodeBlockInterior / DecodeBlockInterior of the batched family) takes it, with the strips around
it as windows, and is otherwise one whole-image window; and that FindRecord finds the owner of every unit of the
prefix-summed layout."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "avif-format_b200", "csrc")


def test_batch_image_plan_covers_and_routes_every_image(tmp_path):
    exe = tmp_path / "indirect_plan_check"
    subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-I", "/usr/local/cuda/include", "-I", CSRC,
                    os.path.join(ROOT, "tests", "native", "indirect_plan_check.cpp"), os.path.join(CSRC, "host_params.cpp"),
                    "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    encode, decode = [dict(re.findall(r"(\w+)=(\d+)", line)) for line in out.stdout.splitlines()[:2]]
    assert int(encode["descriptions"]) >= 100 and int(encode["images"]) > 5000, out.stdout
    assert int(decode["descriptions"]) >= 20 and int(decode["images"]) > 2000, out.stdout


def test_workspace_bytes_is_host_arithmetic():
    import avifgpu
    sizes = [avifgpu.batch_workspace_bytes(n) for n in (1, 2, 64, 256, 4096)]
    assert sizes == sorted(sizes) and sizes[0] > 0
    assert sizes[-1] < 2 << 20  # about 312 bytes per image
    lib = avifgpu.library()
    out = C.c_size_t()
    for bad in (0, -1, 4097):
        with pytest.raises(avifgpu.AvifGpuError):
            avifgpu.batch_workspace_bytes(bad)
    assert lib.avifgpu_batch_workspace_bytes(1, None) != 0
    assert lib.avifgpu_batch_workspace_bytes(1, C.byref(out)) == 0 and out.value == sizes[0]
