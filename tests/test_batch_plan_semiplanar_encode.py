"""Semi-planar and MSB-aligned encode destinations (avifgpu_encode_desc.dest_layout) on the CPU: validation, the
API-10-sized description, plane geometry and windows, the block halves, and the planning of both batch APIs for them.

tests/native/semiplanar_encode_plan_check.cpp checks the validation of every layout bit set x host depth x channel count x
layout kind x image depth; that an API-10-sized description, ending against an inaccessible page, is validated, widened
and laid out without a read past its end and means planar; the interleaved plane's geometry and EncodeWindow offsets; the
integer and float block halves against a restatement of the stores' alignment rule; and, for every 8/16-bit RGB(A)
description in each layout, seeded random batches -- odd widths, one-row images, misaligned rows, Y planes and interleaved
chroma planes -- for exact pixel coverage, routing against EncodeBlockInterior of EncodeBatchFamilyOf, plane placement against EncodeWindow, unit
counts, launches per chunk and FindRecord."""
import ctypes as C
import mmap
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "avif-format_b200", "csrc")
LIBRARY = os.path.join(ROOT, "avif-format_b200", "lib", "libavifgpu.so")


def test_semiplanar_destinations_validate_route_and_plan(tmp_path):
    exe = tmp_path / "semiplanar_encode_plan_check"
    subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-I", "/usr/local/cuda/include", "-I", CSRC,
                    os.path.join(ROOT, "tests", "native", "semiplanar_encode_plan_check.cpp"), os.path.join(CSRC, "host_params.cpp"),
                    "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    counts = {k: int(v) for k, v in re.findall(r"(\w+)=(\d+)", out.stdout)}
    # 8 layout values x 3 host depths x 4 channel counts x 2 layout kinds x 3 image depths, the three size checks, and
    # 3 chroma modes x 4 layouts of geometry
    assert counts["validations"] == 8 * 3 * 4 * 2 * 3 + 3 + 3 * 4, out.stdout
    # 8/16-bit hosts x 3 alpha cases x 3 chroma modes: 8-bit images in 2 layouts, 10/12-bit ones in 4
    assert counts["descriptions"] == 2 * 3 * 3 * (2 + 2 * 4), out.stdout
    assert counts["images"] > 10000 and counts["units"] > 10000, out.stdout


@pytest.mark.skipif(not os.path.exists(LIBRARY), reason="the library is built by __graft_entry__.build()")
def test_api10_sized_description_through_the_library_geometry_calls():
    """The library's description-only calls widen an API-10-sized description (one that ends against an inaccessible
    page) before reading it, and read it as planar."""
    import avifgpu
    from avifgpu import abi

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
