"""The C ABI of the sharded device-pointer light-level encode (avifgpu_encode_rows_sharded_device_light_level) without a
GPU: an addition within API version 13, exported, bound with the argument types the header declares, and refusing a NULL
group before the library touches a device."""
import ctypes as C
import os
import re

import pytest

from avifgpu import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBRARY = os.path.join(ROOT, "avif-format_b200", "lib", "libavifgpu.so")
NAME = "avifgpu_encode_rows_sharded_device_light_level"

# The header's parameter types and the ctypes the binding must use for them (device memory is an untyped address).
CTYPES = {
    "avifgpu_shard_group*": C.c_void_p,
    "const avifgpu_encode_desc*": C.POINTER(abi.EncodeDesc),
    "const void* const*": C.POINTER(C.c_void_p),
    "const int64_t*": C.POINTER(C.c_int64),
    "const avifgpu_planes*": C.POINTER(abi.Planes),
    "int32_t": C.c_int32,
    "avifgpu_light_level*": C.c_void_p,
}


def declared_parameters(name):
    text = open(os.path.join(ROOT, "include", "avifgpu.h")).read()
    match = re.search(r"AVIFGPU_EXPORT\s+int\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
    assert match, name
    params = []
    for param in match.group(1).split(","):
        words = " ".join(param.split())
        params.append(re.sub(r"\s*\*", "*", words.rsplit(" ", 1)[0]))  # drop the parameter's name
    return params


@pytest.mark.skipif(not os.path.exists(LIBRARY), reason="the library is built by __graft_entry__.build()")
def test_exported_and_bound_as_declared():
    import avifgpu
    lib = avifgpu.library()
    assert abi.API_VERSION == 13 and lib.avifgpu_api_version() == 13
    assert NAME in avifgpu.EXPORTED_SYMBOLS and hasattr(lib, NAME)
    params = declared_parameters(NAME)
    assert params == ["avifgpu_shard_group*", "const avifgpu_encode_desc*", "const void* const*", "const int64_t*",
                      "const avifgpu_planes*", "int32_t", "avifgpu_light_level*"]
    function = getattr(lib, NAME)
    assert function.restype is C.c_int
    assert list(function.argtypes) == [CTYPES[p] for p in params]
    # the same arguments as the plain call, then the accumulator
    assert list(lib.avifgpu_encode_rows_sharded_device.argtypes) == list(function.argtypes)[:-1]


@pytest.mark.skipif(not os.path.exists(LIBRARY), reason="the library is built by __graft_entry__.build()")
def test_null_group_is_refused_without_a_device():
    import avifgpu
    lib = avifgpu.library()
    desc = abi.EncodeDesc(8, 2, 32, 3, abi.ALPHA_NONE, 12, abi.TRANSFER_PQ, 1000, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420)
    rows = (C.c_void_p * 1)(None)
    strides = (C.c_int64 * 1)(96)
    planes = abi.Planes()
    acc = abi.LightLevel(max_code=7, reserved=8, level_sum=9, pixels=10)
    for d in (C.byref(desc), None):
        for a in (C.addressof(acc), None):
            assert lib.avifgpu_encode_rows_sharded_device_light_level(None, d, rows, strides, C.byref(planes), 0, a) == abi.ERR_BAD_PARAM
    assert acc.as_dict() == {"max_code": 7, "reserved": 8, "level_sum": 9, "pixels": 10}
