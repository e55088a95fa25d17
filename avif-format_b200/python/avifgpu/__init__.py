"""Python binding (ctypes) of the avifgpu C ABI -- see include/avifgpu.h.

This is a thin convenience layer for tests and bench.py: every pixel goes through the shared library
avif-format_b200/lib/libavifgpu.so (CUDA kernels for sm_90a).  There is no Python or CPU implementation behind
it: if the library has not been built, or there is no CUDA device, the calls raise.
"""
import ctypes as C
import os

import numpy as np

from . import abi
from .abi import *  # noqa: F401,F403  (enums and structs)

_PKG_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
LIBRARY_PATH = os.environ.get("AVIFGPU_LIBRARY") or os.path.join(_PKG_ROOT, "lib", "libavifgpu.so")

_lib = None


class AvifGpuError(RuntimeError):
    def __init__(self, status, message):
        super().__init__(f"avifgpu status {status}: {message}")
        self.status = status
        self.message = message


def library():
    """Loads lib/libavifgpu.so (once).  Raises if it is missing -- there is nothing to fall back to."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIBRARY_PATH):
        raise FileNotFoundError(
            f"{LIBRARY_PATH} is missing: build it with `make -C avif-format_b200` (or __graft_entry__.build()). "
            "The avifgpu path has no CPU fallback.")
    lib = C.CDLL(LIBRARY_PATH)
    ctx_p = C.c_void_p

    def sig(name, restype, argtypes):
        fn = getattr(lib, name)
        fn.restype = restype
        fn.argtypes = argtypes

    sig("avifgpu_api_version", C.c_int, [])
    sig("avifgpu_create", C.c_int, [C.c_int, C.POINTER(ctx_p)])
    sig("avifgpu_destroy", None, [ctx_p])
    sig("avifgpu_last_error", C.c_char_p, [ctx_p])
    sig("avifgpu_status_string", C.c_char_p, [C.c_int])
    sig("avifgpu_launch_count", C.c_int64, [ctx_p])
    sig("avifgpu_synchronize", C.c_int, [ctx_p])
    sig("avifgpu_host_alloc", C.c_int, [ctx_p, C.c_size_t, C.POINTER(C.c_void_p)])
    sig("avifgpu_host_free", C.c_int, [ctx_p, C.c_void_p])
    sig("avifgpu_encode_host_col_bytes", C.c_int, [C.POINTER(abi.EncodeDesc)])
    sig("avifgpu_decode_host_col_bytes", C.c_int, [C.POINTER(abi.DecodeDesc)])
    sig("avifgpu_encode_plane_geometry", C.c_int,
        [C.POINTER(abi.EncodeDesc), C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)])
    sig("avifgpu_decode_plane_geometry", C.c_int,
        [C.POINTER(abi.DecodeDesc), C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)])
    sig("avifgpu_get_yuv_coefficients", C.c_int, [C.POINTER(abi.Nclx), C.c_void_p])
    sig("avifgpu_get_hlg_luma_coefficients", C.c_int, [C.c_int32, C.c_void_p])
    sig("avifgpu_build_yuv_tables", C.c_int, [C.POINTER(abi.Nclx), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p])
    sig("avifgpu_encode_rows", C.c_int,
        [ctx_p, C.POINTER(abi.EncodeDesc), C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.POINTER(abi.Planes)])
    sig("avifgpu_decode_rows", C.c_int,
        [ctx_p, C.POINTER(abi.DecodeDesc), C.POINTER(abi.Planes), C.c_int32, C.c_int32, C.c_void_p, C.c_int64])
    sig("avifgpu_encode_rows_device", C.c_int,
        [ctx_p, C.POINTER(abi.EncodeDesc), C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.POINTER(abi.Planes), C.c_void_p])
    sig("avifgpu_decode_rows_device", C.c_int,
        [ctx_p, C.POINTER(abi.DecodeDesc), C.POINTER(abi.Planes), C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p])
    sig("avifgpu_encode_rows_device_light_level", C.c_int,
        [ctx_p, C.POINTER(abi.EncodeDesc), C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.POINTER(abi.Planes), C.c_void_p, C.c_void_p])
    sig("avifgpu_content_light_level", C.c_int,
        [C.POINTER(abi.LightLevel), C.c_int32, C.POINTER(C.c_uint16), C.POINTER(C.c_uint16)])
    sig("avifgpu_encode_batch_device", C.c_int,
        [ctx_p, C.POINTER(abi.EncodeDesc), C.POINTER(abi.BatchImage), C.c_int32, C.c_void_p])
    sig("avifgpu_decode_batch_device", C.c_int,
        [ctx_p, C.POINTER(abi.DecodeDesc), C.POINTER(abi.BatchImage), C.c_int32, C.c_void_p])
    sig("avifgpu_encode_batch_device_light_level", C.c_int,
        [ctx_p, C.POINTER(abi.EncodeDesc), C.POINTER(abi.BatchImage), C.c_int32, C.c_void_p, C.c_void_p])
    sig("avifgpu_batch_workspace_bytes", C.c_int, [C.c_int32, C.POINTER(C.c_size_t)])
    sig("avifgpu_encode_batch_indirect_light_level", C.c_int,
        [ctx_p, C.POINTER(abi.EncodeDesc), C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p])
    for name, desc_type in (("avifgpu_encode_batch_indirect", abi.EncodeDesc), ("avifgpu_decode_batch_indirect", abi.DecodeDesc)):
        sig(name, C.c_int, [ctx_p, C.POINTER(desc_type), C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p])
    sig("avifgpu_transfer_f32", C.c_int, [ctx_p, C.c_int32, C.c_float, C.c_void_p, C.c_void_p, C.c_size_t])
    sig("avifgpu_prepare_encode", C.c_int, [ctx_p, C.POINTER(abi.EncodeDesc), C.POINTER(abi.CurveStats)])
    sig("avifgpu_prepare_decode", C.c_int, [ctx_p, C.POINTER(abi.DecodeDesc)])
    sig("avifgpu_set_table_autobuild", C.c_int, [ctx_p, C.c_int64])
    sig("avifgpu_hlg_ootf_f32", C.c_int, [ctx_p, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_size_t])
    sig("avifgpu_encode_rows_async", C.c_int,
        [ctx_p, C.POINTER(abi.EncodeDesc), C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.POINTER(abi.Planes), C.POINTER(C.c_int64)])
    sig("avifgpu_decode_rows_async", C.c_int,
        [ctx_p, C.POINTER(abi.DecodeDesc), C.POINTER(abi.Planes), C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)])
    sig("avifgpu_wait", C.c_int, [ctx_p, C.c_int64])
    sig("avifgpu_encode_rows_light_level", C.c_int,
        [ctx_p, C.POINTER(abi.EncodeDesc), C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.POINTER(abi.Planes), C.POINTER(abi.LightLevel)])
    sig("avifgpu_encode_rows_async_light_level", C.c_int,
        [ctx_p, C.POINTER(abi.EncodeDesc), C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.POINTER(abi.Planes), C.POINTER(abi.LightLevel),
         C.POINTER(C.c_int64)])
    group_p = C.c_void_p
    sig("avifgpu_shard_group_create", C.c_int, [C.POINTER(C.c_int32), C.c_int32, C.POINTER(group_p)])
    sig("avifgpu_shard_group_destroy", None, [group_p])
    sig("avifgpu_shard_group_size", C.c_int32, [group_p])
    sig("avifgpu_shard_group_context", ctx_p, [group_p, C.c_int32])
    sig("avifgpu_shard_group_peer_access", C.c_int, [group_p, C.c_int32, C.c_int32])
    sig("avifgpu_shard_group_last_error", C.c_char_p, [group_p])
    sig("avifgpu_shard_group_prepare_encode", C.c_int, [group_p, C.POINTER(abi.EncodeDesc)])
    sig("avifgpu_shard_group_synchronize", C.c_int, [group_p])
    sig("avifgpu_shard_row_blocks", C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)])
    sig("avifgpu_encode_rows_sharded", C.c_int,
        [group_p, C.POINTER(abi.EncodeDesc), C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.POINTER(abi.Planes)])
    sig("avifgpu_decode_rows_sharded", C.c_int,
        [group_p, C.POINTER(abi.DecodeDesc), C.POINTER(abi.Planes), C.c_int32, C.c_int32, C.c_void_p, C.c_int64])
    sig("avifgpu_encode_rows_sharded_light_level", C.c_int,
        [group_p, C.POINTER(abi.EncodeDesc), C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.POINTER(abi.Planes), C.POINTER(abi.LightLevel)])
    sig("avifgpu_encode_rows_sharded_device", C.c_int,
        [group_p, C.POINTER(abi.EncodeDesc), C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.POINTER(abi.Planes), C.c_int32])
    sig("avifgpu_icc_to_rec2020_linear_matrix", C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int32)])
    _lib = lib
    return lib


def icc_to_rec2020_linear_matrix(profile_bytes):
    """(3x3 float32 matrix, is_rec2020) for a matrix / TRC RGB profile with linear tone curves; raises for anything else."""
    out = np.zeros(9, np.float32)
    same = C.c_int32(0)
    buf = (C.c_uint8 * len(profile_bytes)).from_buffer_copy(profile_bytes)
    status = library().avifgpu_icc_to_rec2020_linear_matrix(buf, len(profile_bytes), out.ctypes.data, C.byref(same))
    if status != 0:
        raise AvifGpuError(status, "avifgpu_icc_to_rec2020_linear_matrix")
    return out.reshape(3, 3), bool(same.value)


def shard_row_blocks(y0, nrows, parts):
    """[(y0, rows)] * parts as avifgpu_shard_row_blocks cuts rows [y0, y0 + nrows) (pure host arithmetic)."""
    starts = (C.c_int32 * parts)()
    counts = (C.c_int32 * parts)()
    status = library().avifgpu_shard_row_blocks(y0, nrows, parts, starts, counts)
    if status != 0:
        raise AvifGpuError(status, "avifgpu_shard_row_blocks")
    return [(int(starts[i]), int(counts[i])) for i in range(parts)]


EXPORTED_SYMBOLS = [
    "avifgpu_api_version", "avifgpu_create", "avifgpu_destroy", "avifgpu_last_error", "avifgpu_status_string",
    "avifgpu_launch_count", "avifgpu_synchronize", "avifgpu_host_alloc", "avifgpu_host_free",
    "avifgpu_encode_host_col_bytes", "avifgpu_decode_host_col_bytes", "avifgpu_encode_plane_geometry",
    "avifgpu_decode_plane_geometry", "avifgpu_get_yuv_coefficients", "avifgpu_get_hlg_luma_coefficients",
    "avifgpu_build_yuv_tables", "avifgpu_encode_rows", "avifgpu_decode_rows", "avifgpu_encode_rows_device",
    "avifgpu_decode_rows_device", "avifgpu_encode_batch_device", "avifgpu_decode_batch_device",
    "avifgpu_batch_workspace_bytes", "avifgpu_encode_batch_indirect", "avifgpu_decode_batch_indirect", "avifgpu_transfer_f32", "avifgpu_prepare_encode", "avifgpu_set_table_autobuild",
    "avifgpu_hlg_ootf_f32", "avifgpu_prepare_decode",
    "avifgpu_encode_rows_async", "avifgpu_decode_rows_async", "avifgpu_wait",
    "avifgpu_shard_group_create", "avifgpu_shard_group_destroy", "avifgpu_shard_group_size", "avifgpu_shard_group_context",
    "avifgpu_shard_group_peer_access", "avifgpu_shard_group_last_error", "avifgpu_shard_group_prepare_encode",
    "avifgpu_shard_group_synchronize", "avifgpu_shard_row_blocks", "avifgpu_encode_rows_sharded", "avifgpu_decode_rows_sharded",
    "avifgpu_encode_rows_sharded_device", "avifgpu_icc_to_rec2020_linear_matrix",
    "avifgpu_encode_rows_device_light_level", "avifgpu_content_light_level",
    "avifgpu_encode_batch_device_light_level", "avifgpu_encode_batch_indirect_light_level",
    "avifgpu_encode_rows_light_level", "avifgpu_encode_rows_async_light_level", "avifgpu_encode_rows_sharded_light_level",
]


def content_light_level(acc, image_bit_depth):
    """(MaxCLL, MaxFALL) in cd/m2 of an accumulator (abi.LightLevel, a dict with its fields, or the 24 bytes of the device
    accumulator as any buffer) -- avifgpu_content_light_level, pure host arithmetic."""
    if isinstance(acc, dict):
        acc = abi.LightLevel(max_code=acc["max_code"], reserved=acc.get("reserved", 0), level_sum=acc["level_sum"], pixels=acc["pixels"])
    elif not isinstance(acc, abi.LightLevel):
        acc = abi.LightLevel.from_buffer_copy(bytes(memoryview(acc).cast("B")))
    max_cll, max_fall = C.c_uint16(0), C.c_uint16(0)
    status = library().avifgpu_content_light_level(C.byref(acc), image_bit_depth, C.byref(max_cll), C.byref(max_fall))
    if status != 0:
        raise AvifGpuError(status, "avifgpu_content_light_level")
    return int(max_cll.value), int(max_fall.value)


# ---- host-arithmetic helpers (usable without a device) -------------------------------------------------------

def yuv_coefficients(nclx):
    out = np.zeros(3, np.float32)
    status = library().avifgpu_get_yuv_coefficients(C.byref(nclx) if nclx is not None else None, out.ctypes.data)
    if status != 0:
        raise AvifGpuError(status, "avifgpu_get_yuv_coefficients")
    return out


def hlg_luma_coefficients(primaries):
    out = np.zeros(3, np.float32)
    status = library().avifgpu_get_hlg_luma_coefficients(primaries, out.ctypes.data)
    if status != 0:
        raise AvifGpuError(status, "Unsupported color primaries for the HLG Luma Coefficients ")
    return out


def yuv_tables(nclx, bit_depth, monochrome, has_alpha=True):
    n = 1 << bit_depth
    y = np.zeros(n, np.float32)
    uv = None if monochrome else np.zeros(n, np.float32)
    a = np.zeros(n, np.float32) if has_alpha else None
    status = library().avifgpu_build_yuv_tables(
        C.byref(nclx) if nclx is not None else None, bit_depth, int(monochrome), y.ctypes.data,
        uv.ctypes.data if uv is not None else None, a.ctypes.data if a is not None else None)
    if status != 0:
        raise AvifGpuError(status, "avifgpu_build_yuv_tables")
    return y, uv, a


class Context:
    """One avifgpu_context bound to a CUDA device."""

    def __init__(self, device=0):
        self.lib = library()
        handle = C.c_void_p()
        status = self.lib.avifgpu_create(device, C.byref(handle))
        if status != 0:
            raise AvifGpuError(status, self.lib.avifgpu_last_error(None).decode("utf-8", "replace"))
        self.handle = handle
        self.device = device

    def close(self):
        if getattr(self, "handle", None):
            self.lib.avifgpu_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _check(self, status):
        if status != 0:
            raise AvifGpuError(status, self.lib.avifgpu_last_error(self.handle).decode("utf-8", "replace"))

    def launch_count(self):
        return int(self.lib.avifgpu_launch_count(self.handle))

    def synchronize(self):
        self._check(self.lib.avifgpu_synchronize(self.handle))

    # ---- pinned host memory ------------------------------------------------------------------------------------
    def pinned_array(self, shape, dtype):
        """numpy array backed by cudaHostAlloc memory (freed with the returned array's base object)."""
        dtype = np.dtype(dtype)
        count = int(np.prod(shape))
        nbytes = max(count * dtype.itemsize, 1)
        ptr = C.c_void_p()
        self._check(self.lib.avifgpu_host_alloc(self.handle, nbytes, C.byref(ptr)))
        owner = _PinnedOwner(self, ptr.value, nbytes)
        buf = (C.c_uint8 * nbytes).from_address(ptr.value)
        arr = np.frombuffer(buf, dtype=dtype, count=count).reshape(shape)
        owner.buffer = buf
        _pinned_owners[id(buf)] = owner
        return arr

    # ---- host-pointer entry points (numpy) -----------------------------------------------------------------------
    def encode(self, desc, rows, y0=0, nrows=None, planes=None, pad=0):
        """rows: 2-D host array holding rows [y0, y0+nrows).  Returns the 4 whole-image planes (None where absent)."""
        nrows = desc.height - y0 if nrows is None else nrows
        assert rows.dtype == abi.host_dtype(desc.host_depth) and rows.ndim == 2
        assert rows.size == 0 or rows.strides[1] == rows.itemsize
        if planes is None:
            planes = alloc_planes(abi.encode_plane_shapes(desc), abi.code_dtype(desc.image_bit_depth), pad)
        p = abi.planes_from_arrays(planes)
        self._check(self.lib.avifgpu_encode_rows(self.handle, C.byref(desc), rows.ctypes.data, rows.strides[0],
                                                 y0, nrows, C.byref(p)))
        return planes

    def encode_light_level(self, desc, rows, acc, y0=0, nrows=None, planes=None, pad=0):
        """avifgpu_encode_rows_light_level: encode, plus the content light level of the rows added into `acc` (an
        abi.LightLevel in host memory, zeroed by the caller).  Returns the planes."""
        nrows = desc.height - y0 if nrows is None else nrows
        assert rows.dtype == abi.host_dtype(desc.host_depth) and rows.ndim == 2
        assert rows.size == 0 or rows.strides[1] == rows.itemsize
        if planes is None:
            planes = alloc_planes(abi.encode_plane_shapes(desc), abi.code_dtype(desc.image_bit_depth), pad)
        p = abi.planes_from_arrays(planes)
        self._check(self.lib.avifgpu_encode_rows_light_level(self.handle, C.byref(desc), rows.ctypes.data, rows.strides[0],
                                                             y0, nrows, C.byref(p), C.byref(acc)))
        return planes

    def decode(self, desc, planes, y0=0, nrows=None, out=None):
        nrows = desc.height - y0 if nrows is None else nrows
        channels = abi.decode_host_channels(desc)
        if out is None:
            out = np.zeros((nrows, desc.width * channels), abi.host_dtype(desc.host_depth))
        p = abi.planes_from_arrays(planes)
        self._check(self.lib.avifgpu_decode_rows(self.handle, C.byref(desc), C.byref(p), y0, nrows, out.ctypes.data,
                                                 out.strides[0]))
        return out

    def encode_async(self, desc, rows, planes, y0=0, nrows=None):
        """avifgpu_encode_rows_async into caller-provided planes; returns the ticket."""
        nrows = desc.height - y0 if nrows is None else nrows
        p = abi.planes_from_arrays(planes)
        ticket = C.c_int64()
        self._check(self.lib.avifgpu_encode_rows_async(self.handle, C.byref(desc), rows.ctypes.data, rows.strides[0], y0, nrows, C.byref(p),
                                                       C.byref(ticket)))
        return ticket.value

    def encode_async_light_level(self, desc, rows, planes, acc, y0=0, nrows=None):
        """avifgpu_encode_rows_async_light_level: encode_async, plus the content light level of the rows added into `acc`
        (an abi.LightLevel, zeroed by the caller), which is complete -- like the planes -- once wait() with the returned
        ticket has returned; it must stay alive until then."""
        nrows = desc.height - y0 if nrows is None else nrows
        p = abi.planes_from_arrays(planes)
        ticket = C.c_int64()
        self._check(self.lib.avifgpu_encode_rows_async_light_level(self.handle, C.byref(desc), rows.ctypes.data, rows.strides[0], y0, nrows,
                                                                   C.byref(p), C.byref(acc), C.byref(ticket)))
        return ticket.value

    def decode_async(self, desc, planes, out, y0=0, nrows=None):
        nrows = desc.height - y0 if nrows is None else nrows
        p = abi.planes_from_arrays(planes)
        ticket = C.c_int64()
        self._check(self.lib.avifgpu_decode_rows_async(self.handle, C.byref(desc), C.byref(p), y0, nrows, out.ctypes.data, out.strides[0],
                                                       C.byref(ticket)))
        return ticket.value

    def wait(self, ticket=0):
        self._check(self.lib.avifgpu_wait(self.handle, ticket))

    def set_table_autobuild(self, pixels):
        """After how many pixels of one configuration the step tables are built automatically (0 = at first use,
        negative = never); see avifgpu_set_table_autobuild."""
        self._check(self.lib.avifgpu_set_table_autobuild(self.handle, int(pixels)))

    def prepare_encode(self, desc):
        """Builds the device tables `desc` needs and returns their statistics (abi.CurveStats)."""
        stats = abi.CurveStats()
        self._check(self.lib.avifgpu_prepare_encode(self.handle, C.byref(desc), C.byref(stats)))
        return stats

    def prepare_decode(self, desc):
        """Does the first-use work a decode of `desc` would do (the verified divisions); see avifgpu_prepare_decode."""
        self._check(self.lib.avifgpu_prepare_decode(self.handle, C.byref(desc)))

    def transfer(self, function, values, param=0.0):
        values = np.ascontiguousarray(values, dtype=np.float32)
        out = np.empty_like(values)
        self._check(self.lib.avifgpu_transfer_f32(self.handle, function, param, values.ctypes.data, out.ctypes.data,
                                                  values.size))
        return out

    # ---- device-pointer entry points (raw pointers; torch tensors via .data_ptr()) -------------------------------
    def hlg_ootf(self, rgb, primaries, gamma, peak, inverse=False):
        """ApplyHLGOOTF / ApplyInverseHLGOOTF over an array of RGB float triples."""
        rgb = np.ascontiguousarray(rgb, dtype=np.float32)
        out = np.empty_like(rgb)
        self._check(self.lib.avifgpu_hlg_ootf_f32(self.handle, int(inverse), primaries, gamma, peak, rgb.ctypes.data, out.ctypes.data, rgb.size // 3))
        return out

    def encode_device(self, desc, rows_ptr, row_stride, planes_struct, y0=0, nrows=None, stream=0):
        nrows = desc.height - y0 if nrows is None else nrows
        self._check(self.lib.avifgpu_encode_rows_device(self.handle, C.byref(desc), rows_ptr, row_stride, y0, nrows,
                                                        C.byref(planes_struct), stream))

    def encode_device_light_level(self, desc, rows_ptr, row_stride, planes_struct, acc_ptr, y0=0, nrows=None, stream=0):
        """avifgpu_encode_rows_device_light_level: encode_device, plus the content light level of the rows added into the
        device accumulator at `acc_ptr` (24 bytes, zeroed by the caller; see abi.LightLevel)."""
        nrows = desc.height - y0 if nrows is None else nrows
        self._check(self.lib.avifgpu_encode_rows_device_light_level(self.handle, C.byref(desc), rows_ptr, row_stride, y0, nrows,
                                                                    C.byref(planes_struct), acc_ptr, stream))

    def encode_batch_device(self, desc, images, stream=0):
        """avifgpu_encode_batch_device: `images` is a ctypes array of abi.BatchImage (see batch_images_from_tensors)."""
        self._check(self.lib.avifgpu_encode_batch_device(self.handle, C.byref(desc), images, len(images), stream))

    def encode_batch_device_light_level(self, desc, images, acc_ptr, stream=0):
        """avifgpu_encode_batch_device_light_level: encode_batch_device, plus image i's content light level added into the
        device accumulator acc_ptr[i] (len(images) abi.LightLevel entries, zeroed by the caller)."""
        self._check(self.lib.avifgpu_encode_batch_device_light_level(self.handle, C.byref(desc), images, len(images), acc_ptr, stream))

    def decode_batch_device(self, desc, images, stream=0):
        """avifgpu_decode_batch_device: `images` is a ctypes array of abi.BatchImage (planes = source, rows = destination)."""
        self._check(self.lib.avifgpu_decode_batch_device(self.handle, C.byref(desc), images, len(images), stream))

    def encode_batch_indirect(self, desc, images, count, max_count, workspace, status=None, stream=0):
        """avifgpu_encode_batch_indirect: `images` (records, see pack_batch_images), `count` (one int32), `workspace` and
        `status` (max_count int32, or None) are CUDA tensors, read when the work runs on `stream`."""
        self._check(self.lib.avifgpu_encode_batch_indirect(self.handle, C.byref(desc), *_indirect_args(images, count, max_count, workspace, status),
                                                           stream))

    def encode_batch_indirect_light_level(self, desc, images, count, max_count, workspace, acc_ptr, status=None, stream=0):
        """avifgpu_encode_batch_indirect_light_level: encode_batch_indirect, plus image i's content light level added into
        the device accumulator acc_ptr[i] (max_count abi.LightLevel entries, zeroed by the caller)."""
        self._check(self.lib.avifgpu_encode_batch_indirect_light_level(self.handle, C.byref(desc),
                                                                       *_indirect_args(images, count, max_count, workspace, status), acc_ptr,
                                                                       stream))

    def decode_batch_indirect(self, desc, images, count, max_count, workspace, status=None, stream=0):
        """avifgpu_decode_batch_indirect: as encode_batch_indirect (planes = source, rows = destination)."""
        self._check(self.lib.avifgpu_decode_batch_indirect(self.handle, C.byref(desc), *_indirect_args(images, count, max_count, workspace, status),
                                                           stream))

    def decode_device(self, desc, planes_struct, rows_ptr, row_stride, y0=0, nrows=None, stream=0):
        nrows = desc.height - y0 if nrows is None else nrows
        self._check(self.lib.avifgpu_decode_rows_device(self.handle, C.byref(desc), C.byref(planes_struct), y0, nrows,
                                                        rows_ptr, row_stride, stream))


class ShardGroup:
    """avifgpu_shard_group: one context per device of this process, row blocks split between them."""

    def __init__(self, devices):
        self.lib = library()
        devices = list(devices)
        ordinals = (C.c_int32 * len(devices))(*devices)
        handle = C.c_void_p()
        status = self.lib.avifgpu_shard_group_create(ordinals, len(devices), C.byref(handle))
        if status != 0:
            raise AvifGpuError(status, self.lib.avifgpu_shard_group_last_error(None).decode("utf-8", "replace"))
        self.handle = handle
        self.devices = devices

    def close(self):
        if getattr(self, "handle", None):
            self.lib.avifgpu_shard_group_destroy(self.handle)
            self.handle = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, status):
        if status != 0:
            raise AvifGpuError(status, self.lib.avifgpu_shard_group_last_error(self.handle).decode("utf-8", "replace"))

    def size(self):
        return int(self.lib.avifgpu_shard_group_size(self.handle))

    def peer_access(self, source, target):
        return bool(self.lib.avifgpu_shard_group_peer_access(self.handle, source, target))

    def launch_count(self):
        return sum(int(self.lib.avifgpu_launch_count(self.lib.avifgpu_shard_group_context(self.handle, i))) for i in range(self.size()))

    def prepare_encode(self, desc):
        self._check(self.lib.avifgpu_shard_group_prepare_encode(self.handle, C.byref(desc)))

    def synchronize(self):
        self._check(self.lib.avifgpu_shard_group_synchronize(self.handle))

    def encode(self, desc, rows, y0=0, nrows=None, planes=None):
        nrows = desc.height - y0 if nrows is None else nrows
        assert rows.dtype == abi.host_dtype(desc.host_depth) and rows.ndim == 2
        if planes is None:
            planes = alloc_planes(abi.encode_plane_shapes(desc), abi.code_dtype(desc.image_bit_depth))
        p = abi.planes_from_arrays(planes)
        self._check(self.lib.avifgpu_encode_rows_sharded(self.handle, C.byref(desc), rows.ctypes.data, rows.strides[0], y0, nrows, C.byref(p)))
        return planes

    def encode_light_level(self, desc, rows, acc, y0=0, nrows=None, planes=None):
        """avifgpu_encode_rows_sharded_light_level: encode, plus the content light level of the rows added into `acc`
        (an abi.LightLevel, zeroed by the caller) once every member has succeeded.  Returns the planes."""
        nrows = desc.height - y0 if nrows is None else nrows
        assert rows.dtype == abi.host_dtype(desc.host_depth) and rows.ndim == 2
        if planes is None:
            planes = alloc_planes(abi.encode_plane_shapes(desc), abi.code_dtype(desc.image_bit_depth))
        p = abi.planes_from_arrays(planes)
        self._check(self.lib.avifgpu_encode_rows_sharded_light_level(self.handle, C.byref(desc), rows.ctypes.data, rows.strides[0], y0, nrows,
                                                                     C.byref(p), C.byref(acc)))
        return planes

    def decode(self, desc, planes, y0=0, nrows=None, out=None):
        nrows = desc.height - y0 if nrows is None else nrows
        if out is None:
            out = np.zeros((nrows, desc.width * abi.decode_host_channels(desc)), abi.host_dtype(desc.host_depth))
        p = abi.planes_from_arrays(planes)
        self._check(self.lib.avifgpu_decode_rows_sharded(self.handle, C.byref(desc), C.byref(p), y0, nrows, out.ctypes.data, out.strides[0]))
        return out

    def encode_device(self, desc, row_pointers, row_strides, owner_planes, owner=0):
        n = self.size()
        pointers = (C.c_void_p * n)(*[int(v) if v else None for v in row_pointers])
        strides = (C.c_int64 * n)(*[int(v) for v in row_strides])
        self._check(self.lib.avifgpu_encode_rows_sharded_device(self.handle, C.byref(desc), pointers, strides, C.byref(owner_planes), owner))


_pinned_owners = {}


class _PinnedOwner:
    def __init__(self, ctx, ptr, nbytes):
        self.ctx, self.ptr, self.nbytes = ctx, ptr, nbytes
        self.buffer = None

    def free(self):
        if self.ptr and self.ctx.handle:
            self.ctx.lib.avifgpu_host_free(self.ctx.handle, self.ptr)
        self.ptr = None


def alloc_planes(shapes, dtype, pad=0, fill=0xCD):
    out = []
    for shape in shapes:
        if shape is None:
            out.append(None)
            continue
        rows, cols = shape
        backing = np.full((max(rows, 0), cols + pad), fill, dtype=dtype)
        out.append(backing[:, :cols])
    return out


def planes_from_tensors(tensors):
    """abi.Planes pointing at 2-D torch CUDA tensors (None entries stay NULL)."""
    planes = abi.Planes()
    for i, t in enumerate(tensors):
        if t is None:
            planes.data[i] = None
            planes.stride[i] = 0
        else:
            assert t.dim() == 2 and t.stride(1) == 1
            planes.data[i] = t.data_ptr()
            planes.stride[i] = t.stride(0) * t.element_size()
    return planes


def batch_images_from_tensors(images):
    """A ctypes array of abi.BatchImage for [(width, height, rows, planes)]: `rows` a 2-D torch CUDA tensor of host-layout
    rows (or None), `planes` a list of 2-D torch CUDA tensors or None, as for planes_from_tensors.  Encode reads the rows
    and writes the planes, decode the other way round."""
    out = (abi.BatchImage * len(images))()
    for i, (width, height, rows, planes) in enumerate(images):
        out[i].width = width
        out[i].height = height
        if rows is not None:
            assert rows.dim() == 2 and rows.stride(1) == 1
            out[i].rows = rows.data_ptr()
            out[i].row_stride_bytes = rows.stride(0) * rows.element_size()
        out[i].planes = planes_from_tensors(planes)
    return out


def batch_workspace_bytes(max_count):
    """avifgpu_batch_workspace_bytes: the device workspace a device-described batch of up to max_count images needs."""
    out = C.c_size_t()
    status = library().avifgpu_batch_workspace_bytes(max_count, C.byref(out))
    if status != 0:
        raise AvifGpuError(status, f"avifgpu_batch_workspace_bytes({max_count})")
    return out.value


def pack_batch_images(images, capacity=None, out=None):
    """The records of batch_images_from_tensors(images) -- or `images` itself when it already is a ctypes array of
    abi.BatchImage -- as a CUDA uint8 tensor of capacity x sizeof(BatchImage) bytes (records past len(images) zeroed), for
    the device-described batch calls.  With `out` (such a tensor) the records are written into it instead, in stream
    order on the current stream."""
    import torch
    capacity = len(images) if capacity is None else capacity
    assert len(images) <= capacity
    records = images if isinstance(images, C.Array) else batch_images_from_tensors(images)
    host = (abi.BatchImage * capacity)()
    C.memmove(host, records, len(images) * C.sizeof(abi.BatchImage))
    data = torch.frombuffer(bytearray(bytes(host)), dtype=torch.uint8).reshape(capacity, C.sizeof(abi.BatchImage))
    if out is None:
        return data.cuda()
    assert out.dtype == torch.uint8 and out.is_cuda and out.shape == data.shape
    out.copy_(data)
    return out


def _indirect_args(images, count, max_count, workspace, status):
    import torch
    assert images.is_cuda and count.is_cuda and count.dtype == torch.int32 and workspace.is_cuda
    assert images.numel() >= max_count * C.sizeof(abi.BatchImage)
    if status is not None:
        assert status.is_cuda and status.dtype == torch.int32 and status.numel() >= max_count
    return (images.data_ptr(), count.data_ptr(), max_count, workspace.data_ptr(), workspace.numel() * workspace.element_size(),
            None if status is None else status.data_ptr())
