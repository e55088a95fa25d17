"""The planning of both batch APIs on the CPU: the per-image step PlanBatchEncodeImage / PlanBatchDecodeImage
(csrc/batch_plan.h) that the plan kernel of the device-described batch runs, and the chunks PlanEncodeBatch /
PlanDecodeBatch (csrc/host_params.cpp) build from it for the host-described batch.

tests/native/batch_plan_check.cpp compiles both with the host compiler and runs every description of each slice over
seeded batches of fake images on fake padded planes (widths 1 to 9, 255 to 257, 512, 513 and random ones up to 600; one-row
images; misaligned rows, planes and strides; unequal Cb / Cr strides; misaligned interleaved chroma; and, for the step,
empty, rejected and NULL images).  Every slice gets the same checks from tests/native/plan_harness.h: each record read
back from its rows pointer and its planes held to EncodeWindow / DecodeWindow, exact coverage of every pixel, the route's
interior and strips, unit counts with the family's unit, image order, chunk sizes and launches, and FindRecord over the
prefix-summed layout.  On top of that each slice checks what only holds for its descriptions:
  encode         every valid encode description; a chunk's parameters fit the kernel parameter limit;
  encode_dest    semi-planar and MSB-aligned destinations: validation, the API-10-sized description against an
                 inaccessible page, plane geometry and EncodeWindow, the block halves against the stores' alignment,
                 routing independent of the layout, the plane mask, the interleaved plane's alignment;
  decode_int     YCbCr into 8/16-bit hosts;
  decode_f32     YCbCr into 32-bit hosts: which descriptions the float family takes;
  decode_rgb     planar RGB: which descriptions its families take, their unit width, every interior against the kernels'
                 alignment; YCbCr and monochrome descriptions route as before;
  decode_source  semi-planar and MSB-aligned sources: validation, the API-9-sized description against an inaccessible
                 page, plane geometry, routing, the plane mask, the interleaved plane's alignment;
  indirect       the device-described batch's workspace layout, planar encodes and YCbCr decodes."""
import ctypes as C
import mmap
import os
import re
import subprocess

import pytest

from avifgpu import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "avif-format_b200", "csrc")
LIBRARY = os.path.join(ROOT, "avif-format_b200", "lib", "libavifgpu.so")


@pytest.fixture(scope="module")
def plan_check(tmp_path_factory):
    """The checker, compiled and run once for every slice."""
    exe = tmp_path_factory.mktemp("plans") / "batch_plan_check"
    subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-I", "/usr/local/cuda/include", "-I", CSRC,
                    os.path.join(ROOT, "tests", "native", "batch_plan_check.cpp"), os.path.join(CSRC, "host_params.cpp"),
                    "-o", str(exe)], check=True)
    return subprocess.run([str(exe)], capture_output=True, text=True)


def counts(out, slice_name):
    """The counters the checker printed for `slice_name`, once it has exited cleanly."""
    assert out.returncode == 0, out.stdout + out.stderr
    line = next(line for line in out.stdout.splitlines() if line.split()[0] == slice_name)
    return {k: int(v) for k, v in re.findall(r"(\w+)=(\d+)", line)}


def test_encode_plans(plan_check):
    n = counts(plan_check, "encode")
    assert n["descriptions"] > 100 and n["images"] > 10000, plan_check.stdout


def test_encode_destination_plans(plan_check):
    n = counts(plan_check, "encode_dest")
    # 8 layout values x 3 host depths x 4 channel counts x 2 layout kinds x 3 image depths, the three size checks, and
    # 3 chroma modes x 4 layouts of geometry
    assert n["validations"] == 8 * 3 * 4 * 2 * 3 + 3 + 3 * 4, plan_check.stdout
    # 8/16-bit hosts x 3 alpha cases x 3 chroma modes: 8-bit images in 2 layouts, 10/12-bit ones in 4
    assert n["descriptions"] == 2 * 3 * 3 * (2 + 2 * 4), plan_check.stdout
    assert n["images"] > 10000 and n["units"] > 10000, plan_check.stdout


def test_integer_decode_plans(plan_check):
    n = counts(plan_check, "decode_int")
    assert n["descriptions"] >= 20 and n["images"] > 1000, plan_check.stdout


def test_float_decode_plans(plan_check):
    n = counts(plan_check, "decode_f32")
    # 10 / 12 / 16-bit planes (8-bit ones are refused for float hosts) x 3 alpha states x 3 chroma modes x 4 curves x 2
    assert n["descriptions"] == 3 * 3 * 3 * 4 * 2, plan_check.stdout
    assert n["images"] > 10000 and n["units"] > 10000, plan_check.stdout


def test_planar_rgb_decode_plans(plan_check):
    n = counts(plan_check, "decode_rgb")
    # x 3 alpha states x 2 ranges: 8-bit hosts 8-bit planes; 16-bit hosts 10 / 12 / 16-bit planes; 32-bit hosts 10 / 12 /
    # 16-bit planes x 4 curves
    assert n["descriptions"] == 3 * 2 * (1 + 3 + 3 * 4), plan_check.stdout
    assert n["images"] > 10000 and n["units"] > 10000 and n["ycbcr"] > 100, plan_check.stdout


def test_decode_source_plans(plan_check):
    n = counts(plan_check, "decode_source")
    # 8 layout values x 3 colour spaces x 4 depths, plus 4 geometries
    assert n["validations"] == 8 * 3 * 4 + 4, plan_check.stdout
    # 8-bit hosts: 8-bit planes, 2 layouts; 16-bit hosts: 10/12-bit planes, 4 layouts; 32-bit hosts: 10/12-bit planes,
    # 4 layouts, 3 curves -- each x 3 alpha states x 3 chroma modes
    assert n["descriptions"] == 9 * (2 + 2 * 4 + 2 * 4 * 3), plan_check.stdout
    assert n["images"] > 10000 and n["units"] > 10000, plan_check.stdout


def test_indirect_plans(plan_check):
    n = counts(plan_check, "indirect")
    assert n["encode_descriptions"] >= 100 and n["encode_images"] > 5000, plan_check.stdout
    assert n["decode_descriptions"] >= 20 and n["decode_images"] > 2000, plan_check.stdout


def test_batch_image_struct_matches_the_c_compiler(tmp_path):
    src = tmp_path / "sizes.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "avifgpu.h"\nint main(void){printf("%zu %zu %zu\\n",'
                   'sizeof(avifgpu_batch_image),offsetof(avifgpu_batch_image,row_stride_bytes),offsetof(avifgpu_batch_image,planes));return 0;}\n')
    exe = tmp_path / "sizes"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    sizes = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert sizes == [C.sizeof(abi.BatchImage), abi.BatchImage.row_stride_bytes.offset, abi.BatchImage.planes.offset]


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


@pytest.mark.skipif(not os.path.exists(LIBRARY), reason="the library is built by __graft_entry__.build()")
def test_api10_sized_description_through_the_library_geometry_calls():
    """The library's description-only calls widen an API-10-sized description (one that ends against an inaccessible
    page) before reading it, and read it as planar."""
    import avifgpu

    lib = avifgpu.library()
    size = C.sizeof(abi.EncodeDesc) - 4  # everything before dest_layout
    assert size == 124
    desc = abi.EncodeDesc(9, 5, 16, 4, abi.ALPHA_STRAIGHT, 12, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420,
                          dest_layout=abi.SOURCE_CHROMA_INTERLEAVED | abi.SOURCE_MSB_ALIGNED)
    page = mmap.PAGESIZE
    region = mmap.mmap(-1, 2 * page, prot=mmap.PROT_READ | mmap.PROT_WRITE)
    base = C.addressof(C.c_char.from_buffer(region))
    libc = C.CDLL(None)
    libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    assert libc.mprotect(C.c_void_p(base + page), page, 0) == 0  # PROT_NONE
    try:
        at = base + page - size
        C.memmove(at, C.byref(desc), size)
        C.c_uint32.from_address(at).value = size
        short = C.cast(C.c_void_p(at), C.POINTER(abi.EncodeDesc))
        assert lib.avifgpu_encode_host_col_bytes(short) == 8
        w, h, b = C.c_int32(), C.c_int32(), C.c_int32()
        assert lib.avifgpu_encode_plane_geometry(short, 1, C.byref(w), C.byref(h), C.byref(b)) == 1
        assert (w.value, h.value, b.value) == (5, 3, 2)  # planar Cb: the short description has no layout
        assert lib.avifgpu_encode_plane_geometry(short, 2, C.byref(w), C.byref(h), C.byref(b)) == 1
        # the full-size description with the same fields: interleaved plane 1, no plane 2
        assert lib.avifgpu_encode_plane_geometry(C.byref(desc), 1, C.byref(w), C.byref(h), C.byref(b)) == 1
        assert (w.value, h.value, b.value) == (10, 3, 2)
        assert lib.avifgpu_encode_plane_geometry(C.byref(desc), 2, C.byref(w), C.byref(h), C.byref(b)) == 0
    finally:
        libc.mprotect(C.c_void_p(base + page), page, mmap.PROT_READ | mmap.PROT_WRITE)
