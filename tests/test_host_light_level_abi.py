"""The C ABI of the light-level host-pointer encodes (avifgpu_encode_rows_light_level, _async_light_level and
_sharded_light_level) without a GPU: additions within API version 13, exported and bound, and refusing a NULL context,
group or description before the library touches a device."""
import ctypes as C
import os

import pytest

from avifgpu import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBRARY = os.path.join(ROOT, "avif-format_b200", "lib", "libavifgpu.so")
NAMES = ("avifgpu_encode_rows_light_level", "avifgpu_encode_rows_async_light_level", "avifgpu_encode_rows_sharded_light_level")


@pytest.mark.skipif(not os.path.exists(LIBRARY), reason="the library is built by __graft_entry__.build()")
def test_additions_within_api_version_13():
    import avifgpu
    lib = avifgpu.library()
    assert abi.API_VERSION == 13 and lib.avifgpu_api_version() == 13
    for name in NAMES:
        assert name in avifgpu.EXPORTED_SYMBOLS and hasattr(lib, name), name


@pytest.mark.skipif(not os.path.exists(LIBRARY), reason="the library is built by __graft_entry__.build()")
def test_refusals_need_no_device():
    """A NULL context, group or description is refused with AVIFGPU_ERR_BAD_PARAM before the library touches a device."""
    import avifgpu
    lib = avifgpu.library()
    desc = abi.EncodeDesc(8, 2, 32, 3, abi.ALPHA_NONE, 12, abi.TRANSFER_PQ, 1000, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420)
    rows = (C.c_float * 48)()
    planes = abi.Planes()
    acc = abi.LightLevel(max_code=7, reserved=8, level_sum=9, pixels=10)
    ticket = C.c_int64(-1)
    for d in (C.byref(desc), None):
        assert lib.avifgpu_encode_rows_light_level(None, d, rows, 96, 0, 2, C.byref(planes), C.byref(acc)) == abi.ERR_BAD_PARAM
        assert lib.avifgpu_encode_rows_async_light_level(None, d, rows, 96, 0, 2, C.byref(planes), C.byref(acc), C.byref(ticket)) == abi.ERR_BAD_PARAM
        assert lib.avifgpu_encode_rows_sharded_light_level(None, d, rows, 96, 0, 2, C.byref(planes), C.byref(acc)) == abi.ERR_BAD_PARAM
    assert ticket.value == -1
    assert acc.as_dict() == {"max_code": 7, "reserved": 8, "level_sum": 9, "pixels": 10}
