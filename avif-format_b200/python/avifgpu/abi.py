"""ctypes mirror of include/avifgpu.h (structs, enums, plane geometry).

Pure declarations -- importing this module loads no native code.  The oracle loaders under oracle/ reuse these
structures so the same description object can be handed to the GPU library, the C restatement and the compiled
reference.
"""
import ctypes as C

import numpy as np

API_VERSION = 12

# avifgpu_status
OK = 0
ERR_BAD_PARAM = -1
ERR_UNSUPPORTED = -2
ERR_NO_DEVICE = -3
ERR_CUDA = -4
ERR_OOM = -5
ERR_CANCELED = -6

# avifgpu_alpha_state (AlphaState.h:24-29)
ALPHA_NONE, ALPHA_STRAIGHT, ALPHA_PREMULTIPLIED = 0, 1, 2
HLG_REJECT, HLG_OETF, HLG_INVERSE_OOTF_THEN_OETF = 0, 1, 2
# avifgpu_transfer (ColorTransfer.h:28-34)
TRANSFER_PQ, TRANSFER_HLG, TRANSFER_SMPTE428, TRANSFER_CLIP = 0, 1, 2, 3
# avifgpu_chroma (= heif_chroma)
CHROMA_MONOCHROME, CHROMA_420, CHROMA_422, CHROMA_444 = 0, 1, 2, 3
# avifgpu_colorspace (= heif_colorspace)
COLORSPACE_YCBCR, COLORSPACE_RGB, COLORSPACE_MONOCHROME = 0, 1, 2
# avifgpu_layout
LAYOUT_REFERENCE, LAYOUT_PLANAR_YCBCR = 0, 1
# avifgpu_source_layout (bits of DecodeDesc.source_layout and EncodeDesc.dest_layout)
SOURCE_PLANAR, SOURCE_CHROMA_INTERLEAVED, SOURCE_MSB_ALIGNED = 0, 1, 2
# avifgpu_down_filter
DOWN_FILTER_BOX, DOWN_FILTER_TOP_LEFT = 0, 1
# avifgpu_gray16_curve
GRAY16_LUT, GRAY16_SMPTE428 = 0, 1
# avifgpu_function
(FN_LINEAR_TO_PQ, FN_PQ_TO_LINEAR, FN_LINEAR_TO_SMPTE428, FN_SMPTE428_TO_LINEAR, FN_HLG_TO_LINEAR,
 FN_LINEAR_TO_HLG, FN_POWF, FN_EXPF, FN_LOGF) = range(9)

# H.273 code points used by the path
PRIMARIES_BT709, PRIMARIES_BT601, PRIMARIES_BT2020 = 1, 6, 9
TRANSFER_CHAR_SRGB, TRANSFER_CHAR_PQ, TRANSFER_CHAR_SMPTE428, TRANSFER_CHAR_HLG = 13, 16, 17, 18
MATRIX_GBR, MATRIX_BT709, MATRIX_BT601, MATRIX_BT2020_NCL, MATRIX_CHROMA_DERIVED_NCL = 0, 1, 6, 9, 12

MAX_PLANES = 4


class Nclx(C.Structure):
    _fields_ = [
        ("present", C.c_int32),
        ("color_primaries", C.c_int32),
        ("transfer_characteristics", C.c_int32),
        ("matrix_coefficients", C.c_int32),
        ("full_range_flag", C.c_int32),
    ]

    def __init__(self, present=0, color_primaries=2, transfer_characteristics=2, matrix_coefficients=2,
                 full_range_flag=1):
        super().__init__(present, color_primaries, transfer_characteristics, matrix_coefficients, full_range_flag)


class Planes(C.Structure):
    _fields_ = [
        ("data", C.c_void_p * MAX_PLANES),
        ("stride", C.c_int64 * MAX_PLANES),
    ]


class BatchImage(C.Structure):
    """avifgpu_batch_image: one whole image of a batch call (device pointers)."""
    _fields_ = [
        ("width", C.c_int32),
        ("height", C.c_int32),
        ("rows", C.c_void_p),
        ("row_stride_bytes", C.c_int64),
        ("planes", Planes),
    ]


class EncodeDesc(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("width", C.c_int32),
        ("height", C.c_int32),
        ("host_depth", C.c_int32),
        ("host_channels", C.c_int32),
        ("alpha_state", C.c_int32),
        ("image_bit_depth", C.c_int32),
        ("transfer", C.c_int32),
        ("pq_peak_nits", C.c_int32),
        ("layout", C.c_int32),
        ("chroma", C.c_int32),
        ("down_filter", C.c_int32),
        ("gray16_curve", C.c_int32),
        ("nclx", Nclx),
        ("hlg_extension", C.c_int32),
        ("hlg_display_gamma", C.c_float),
        ("hlg_peak_nits", C.c_int32),
        ("row_matrix_enabled", C.c_int32),
        ("row_matrix", C.c_float * 9),
        ("dest_layout", C.c_int32),
    ]

    def __init__(self, width, height, host_depth, host_channels, alpha_state=ALPHA_NONE, image_bit_depth=8,
                 transfer=TRANSFER_CLIP, pq_peak_nits=80, layout=LAYOUT_REFERENCE, chroma=CHROMA_444,
                 down_filter=DOWN_FILTER_BOX, gray16_curve=GRAY16_LUT, nclx=None, hlg_extension=0, hlg_display_gamma=1.2,
                 hlg_peak_nits=1000, *, dest_layout=SOURCE_PLANAR):
        super().__init__()
        self.struct_size = C.sizeof(EncodeDesc)
        self.width, self.height = width, height
        self.host_depth, self.host_channels = host_depth, host_channels
        self.alpha_state = alpha_state
        self.image_bit_depth = image_bit_depth
        self.transfer = transfer
        self.pq_peak_nits = pq_peak_nits
        self.layout = layout
        self.chroma = chroma
        self.down_filter = down_filter
        self.gray16_curve = gray16_curve
        self.nclx = nclx if nclx is not None else Nclx()
        self.hlg_extension = hlg_extension
        self.hlg_display_gamma = hlg_display_gamma
        self.hlg_peak_nits = hlg_peak_nits
        self.dest_layout = dest_layout

    def copy(self, **changes):
        out = EncodeDesc(self.width, self.height, self.host_depth, self.host_channels)
        C.memmove(C.byref(out), C.byref(self), C.sizeof(EncodeDesc))
        for key, value in changes.items():
            setattr(out, key, value)
        return out


class DecodeDesc(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("width", C.c_int32),
        ("height", C.c_int32),
        ("colorspace", C.c_int32),
        ("chroma", C.c_int32),
        ("bit_depth", C.c_int32),
        ("alpha_state", C.c_int32),
        ("host_depth", C.c_int32),
        ("nclx", Nclx),
        ("hlg_apply_ootf", C.c_int32),
        ("hlg_display_gamma", C.c_float),
        ("hlg_peak_nits", C.c_int32),
        ("pq_peak_nits", C.c_int32),
        ("source_layout", C.c_int32),
    ]

    def __init__(self, width, height, colorspace=COLORSPACE_YCBCR, chroma=CHROMA_444, bit_depth=8,
                 alpha_state=ALPHA_NONE, host_depth=8, nclx=None, hlg_apply_ootf=1, hlg_display_gamma=1.2,
                 hlg_peak_nits=1000, pq_peak_nits=80, source_layout=SOURCE_PLANAR):
        super().__init__()
        self.struct_size = C.sizeof(DecodeDesc)
        self.width, self.height = width, height
        self.colorspace, self.chroma = colorspace, chroma
        self.bit_depth = bit_depth
        self.alpha_state = alpha_state
        self.host_depth = host_depth
        self.nclx = nclx if nclx is not None else Nclx()
        self.hlg_apply_ootf = hlg_apply_ootf
        self.hlg_display_gamma = hlg_display_gamma
        self.hlg_peak_nits = hlg_peak_nits
        self.pq_peak_nits = pq_peak_nits
        self.source_layout = source_layout

    def copy(self, **changes):
        out = DecodeDesc(self.width, self.height)
        C.memmove(C.byref(out), C.byref(self), C.sizeof(DecodeDesc))
        for key, value in changes.items():
            setattr(out, key, value)
        return out


class CurveStats(C.Structure):
    _fields_ = [
        ("applicable", C.c_int32),
        ("valid", C.c_int32),
        ("steps", C.c_int32),
        ("bands", C.c_int32),
        ("widest_band_ulps", C.c_uint32),
        ("bucket_count", C.c_int32),
        ("swept_inputs", C.c_uint64),
        ("in_band_inputs", C.c_uint64),
        ("verify_mismatches", C.c_uint64),
        ("build_ms", C.c_double),
    ]

    def as_dict(self):
        return {name: getattr(self, name) for name, _ in self._fields_}


class LightLevel(C.Structure):
    """avifgpu_light_level: the device accumulator of avifgpu_encode_rows_device_light_level (24 bytes)."""
    _fields_ = [
        ("max_code", C.c_uint32),
        ("reserved", C.c_uint32),
        ("level_sum", C.c_uint64),
        ("pixels", C.c_uint64),
    ]

    def as_dict(self):
        return {name: int(getattr(self, name)) for name, _ in self._fields_}


# ---- geometry (mirrors avifgpu_*_plane_geometry / *_host_col_bytes) ---------------------------------------

def host_dtype(host_depth):
    return {8: np.uint8, 16: np.uint16, 32: np.float32}[host_depth]


def code_dtype(bit_depth):
    return np.uint8 if bit_depth <= 8 else np.uint16


def chroma_shifts(chroma):
    return (1 if chroma in (CHROMA_420, CHROMA_422) else 0, 1 if chroma == CHROMA_420 else 0)


def encode_plane_shapes(desc):
    """[(rows, samples_per_row) or None] * 4 for the encode destination of `desc`."""
    w, h = desc.width, desc.height
    has_alpha = desc.alpha_state != ALPHA_NONE
    shapes = [None] * MAX_PLANES
    if desc.layout == LAYOUT_REFERENCE:
        if desc.host_channels <= 2:
            shapes[0] = (h, w)
            if has_alpha:
                shapes[3] = (h, w)
        else:
            shapes[0] = (h, w * desc.host_channels)
    else:
        xs, ys = chroma_shifts(desc.chroma)
        cw, ch = (w + xs) >> xs, (h + ys) >> ys
        shapes[0] = (h, w)
        if desc.dest_layout & SOURCE_CHROMA_INTERLEAVED:
            shapes[1] = (ch, 2 * cw)  # Cb, Cr pairs; no plane 2
        else:
            shapes[1] = (ch, cw)
            shapes[2] = (ch, cw)
        if has_alpha:
            shapes[3] = (h, w)
    return shapes


def decode_plane_shapes(desc):
    w, h = desc.width, desc.height
    has_alpha = desc.alpha_state != ALPHA_NONE
    shapes = [None] * MAX_PLANES
    shapes[0] = (h, w)
    if desc.colorspace == COLORSPACE_YCBCR:
        xs, ys = chroma_shifts(desc.chroma)
        cw, ch = (w + xs) >> xs, (h + ys) >> ys
        if desc.source_layout & SOURCE_CHROMA_INTERLEAVED:
            shapes[1] = (ch, 2 * cw)  # Cb, Cr pairs; no plane 2
        else:
            shapes[1] = (ch, cw)
            shapes[2] = (ch, cw)
    elif desc.colorspace == COLORSPACE_RGB:
        shapes[1] = (h, w)
        shapes[2] = (h, w)
    if has_alpha:
        shapes[3] = (h, w)
    return shapes


def decode_host_channels(desc):
    has_alpha = desc.alpha_state != ALPHA_NONE
    if desc.colorspace == COLORSPACE_MONOCHROME:
        return 2 if has_alpha else 1
    return 4 if has_alpha else 3


def planes_from_arrays(arrays):
    """Planes struct pointing at 2-D numpy arrays (None entries stay NULL).  Keep `arrays` alive."""
    planes = Planes()
    for i, a in enumerate(arrays):
        if a is None:
            planes.data[i] = None
            planes.stride[i] = 0
        else:
            assert a.ndim == 2 and (a.size == 0 or a.strides[1] == a.itemsize)
            planes.data[i] = a.ctypes.data
            planes.stride[i] = a.strides[0]
    return planes
