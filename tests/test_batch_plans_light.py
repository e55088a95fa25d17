"""The planning of the light-level batches on the CPU, and their C ABI without a GPU.

tests/native/light_batch_plan_check.cpp compiles EncodeLightBatchFamilyOf, the per-image step and PlanEncodeLightBatch with
the host compiler and runs every float-host description (PQ and SMPTE 428; every channel count, alpha state, depth, layout,
chroma mode and destination layout; no table, a table the size of the 12-bit PQ one and one too big; row matrix off and
on) over seeded batches through plan_harness.h's three checks, plus which descriptions the family takes, the unit width,
every interior against the batched kernel's loads and stores, the image a record belongs to, and the chunk parameter
limit."""
import ctypes as C
import os
import re
import subprocess

import pytest

from avifgpu import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "avif-format_b200", "csrc")
LIBRARY = os.path.join(ROOT, "avif-format_b200", "lib", "libavifgpu.so")


def test_light_batch_plans(tmp_path):
    exe = tmp_path / "light_batch_plan_check"
    subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-I", "/usr/local/cuda/include", "-I", CSRC,
                    os.path.join(ROOT, "tests", "native", "light_batch_plan_check.cpp"), os.path.join(CSRC, "host_params.cpp"),
                    "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    n = {k: int(v) for k, v in re.findall(r"(\w+)=(\d+)", out.stdout)}
    assert n["descriptions"] > 500 and n["images"] > 50000 and n["units"] > 20000, out.stdout
    # float RGB and RGBA (straight, premultiplied) into planar YCbCr, PQ, 10/12 bits, 3 chroma modes x 4 layouts, with the
    # fitting table and no row matrix
    assert n["tuned"] == 3 * 2 * 3 * 4, out.stdout


@pytest.mark.skipif(not os.path.exists(LIBRARY), reason="the library is built by __graft_entry__.build()")
def test_api_version_and_symbols():
    import avifgpu
    lib = avifgpu.library()
    assert abi.API_VERSION == 13 and lib.avifgpu_api_version() == 13
    for name in ("avifgpu_encode_batch_device_light_level", "avifgpu_encode_batch_indirect_light_level"):
        assert name in avifgpu.EXPORTED_SYMBOLS and hasattr(lib, name)


@pytest.mark.skipif(not os.path.exists(LIBRARY), reason="the library is built by __graft_entry__.build()")
def test_refusals_need_no_device():
    """A NULL context or description is refused before the library touches a device."""
    import avifgpu
    lib = avifgpu.library()
    desc = abi.EncodeDesc(0, 0, 32, 3, abi.ALPHA_NONE, 12, abi.TRANSFER_PQ, 1000, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420)
    images = (abi.BatchImage * 1)()
    assert lib.avifgpu_encode_batch_device_light_level(None, C.byref(desc), images, 1, None, None) == abi.ERR_BAD_PARAM
    assert lib.avifgpu_encode_batch_indirect_light_level(None, C.byref(desc), None, None, 1, None, 0, None, None, None) == abi.ERR_BAD_PARAM
