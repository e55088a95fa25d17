"""The batch planners behind avifgpu_encode_batch_device / avifgpu_decode_batch_device (PlanEncodeBatch,
PlanDecodeBatch in csrc/host_params.cpp: chunks packed from the per-image step of csrc/batch_plan.h), on the CPU.

tests/native/batch_plan_check.cpp plans seeded random batches of 1 to 300 images of mixed sizes (1 x 1, widths below 8,
odd widths and heights, misaligned rows) for every valid encode description, on fake padded planes, and checks that
every pixel of every image is covered exactly once by an interior, an edge window or a direct call; that an image is
batched exactly when the single-image launcher's predicate (EncodeBlockInterior of EncodeBatchFamilyOf) takes it; that chunks keep image
order, hold at most 64 images and fit the kernel parameter limit; and that a chunk costs 1 launch, 2 when one of its images has an edge strip; decode batches
get the coverage, routing and launch checks too."""
import ctypes as C
import os
import re
import subprocess

from avifgpu import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "avif-format_b200", "csrc")


def test_chunked_plan_covers_every_pixel_once(tmp_path):
    exe = tmp_path / "batch_plan_check"
    subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-I", "/usr/local/cuda/include", "-I", CSRC,
                    os.path.join(ROOT, "tests", "native", "batch_plan_check.cpp"), os.path.join(CSRC, "host_params.cpp"),
                    "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    encode, decode = [dict(re.findall(r"(\w+)=(\d+)", line)) for line in out.stdout.splitlines()[:2]]
    assert int(encode["descriptions"]) > 100 and int(encode["images"]) > 10000, out.stdout
    assert int(decode["descriptions"]) >= 20 and int(decode["images"]) > 1000, out.stdout


def test_batch_image_struct_matches_the_c_compiler(tmp_path):
    src = tmp_path / "sizes.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "avifgpu.h"\nint main(void){printf("%zu %zu %zu\\n",'
                   'sizeof(avifgpu_batch_image),offsetof(avifgpu_batch_image,row_stride_bytes),offsetof(avifgpu_batch_image,planes));return 0;}\n')
    exe = tmp_path / "sizes"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    sizes = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert sizes == [C.sizeof(abi.BatchImage), abi.BatchImage.row_stride_bytes.offset, abi.BatchImage.planes.offset]
