#!/usr/bin/env python3
"""Device-resident throughput of configurations outside BASELINE.json's bench lines (they run wherever the dispatcher
sends them).  Every launch converts a stack of 8K frames tall enough that its input + output exceed the 50 MB L2
several times over (7680 x 17280 for the 8-bit paths, 7680 x 8640 otherwise), and three such sets rotate, so the GB/s
figures are HBM figures.  Each case is CUDA-event time over at least `--seconds` of back-to-back calls, its window sized
from a 20-call probe, median of `--rounds` windows.  Prints one JSON line per case.

    python profiles/measure_generic_paths.py [--seconds 1.0] [--rounds 3] [--out generic_paths.json]
"""
import collections
import itertools
import os
import statistics

import harness
import torch

import avifgpu
from avifgpu import abi

W, H = 7680, 4320 * 2
H8 = 4320 * 4  # 8-bit paths move 1.5 - 8 bytes per pixel: four frames per launch
ONLY = os.environ.get("AVIFGPU_MEASURE_ONLY")  # run only the cases whose name contains this text
N601 = harness.N601

# `sets` buffer sets rotate; `tables` is None for a case on the shared context, else the case gets its own context with
# automatic table builds off and its tables prepared if True
Case = collections.namedtuple("Case", "name desc bytes_per_px sets tables", defaults=(3, None))


def ycc_decode(bit_depth, host_depth, chroma, nclx, alpha=False):
    return abi.DecodeDesc(W, H8 if bit_depth == 8 else H, abi.COLORSPACE_YCBCR, chroma, bit_depth, abi.ALPHA_STRAIGHT if alpha else abi.ALPHA_NONE,
                          host_depth, nclx)


def ycc_encode(host_depth, channels, image_depth, chroma, nclx, alpha=abi.ALPHA_NONE):
    return abi.EncodeDesc(W, H8 if host_depth == 8 else H, host_depth, channels, alpha, image_depth, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR,
                          chroma, abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, nclx)


def mono_rgb_decode(colorspace, bit_depth, host_depth):
    return abi.DecodeDesc(W, H8 if bit_depth == 8 else H, colorspace, abi.CHROMA_444, bit_depth, abi.ALPHA_NONE, host_depth,
                          abi.Nclx(1, 1, 13, 0 if colorspace == abi.COLORSPACE_RGB else 6, 1))


def float_table_decode(colorspace, transfer, ootf):
    rgb = colorspace == abi.COLORSPACE_RGB
    return abi.DecodeDesc(W, H, colorspace, abi.CHROMA_444 if rgb else abi.CHROMA_MONOCHROME, 10 if rgb else 12, abi.ALPHA_NONE, 32,
                          abi.Nclx(1, abi.PRIMARIES_BT2020, transfer, 0, 1), hlg_apply_ootf=ootf)


def float_encode(channels, layout, depth=12, peak=80, transfer=abi.TRANSFER_PQ):
    alpha = abi.ALPHA_STRAIGHT if channels in (2, 4) else abi.ALPHA_NONE
    return abi.EncodeDesc(W, H, 32, channels, alpha, depth, transfer, peak, layout, abi.CHROMA_420 if layout == abi.LAYOUT_PLANAR_YCBCR else abi.CHROMA_444,
                          abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, abi.Nclx(1, abi.PRIMARIES_BT2020, abi.TRANSFER_CHAR_PQ, abi.MATRIX_BT2020_NCL, 1))


RGB, MONO, PLANAR, REFERENCE = abi.COLORSPACE_RGB, abi.COLORSPACE_MONOCHROME, abi.LAYOUT_PLANAR_YCBCR, abi.LAYOUT_REFERENCE
CASES = [
    Case("decode 8-bit 4:2:0 -> RGB8 (a15)", ycc_decode(8, 8, abi.CHROMA_420, N601), 1.5 + 3),
    Case("decode 8-bit 4:4:4 + alpha -> RGBA8 (a15)", ycc_decode(8, 8, abi.CHROMA_444, N601, alpha=True), 4 + 4),
    Case("decode 10-bit 4:2:0 -> RGB16 (a14)", ycc_decode(10, 16, abi.CHROMA_420, N601), 3 + 6),
    Case("decode 12-bit 4:4:4 -> RGB16 (a14)", ycc_decode(12, 16, abi.CHROMA_444, N601), 6 + 6),
    Case("encode RGB8 -> 8-bit 4:2:0 (a3)", ycc_encode(8, 3, 8, abi.CHROMA_420, N601), 3 + 1.5),
    Case("encode RGBA8 -> 8-bit 4:4:4 + A (config 1 at 8K) (a3)", ycc_encode(8, 4, 8, abi.CHROMA_444, N601, alpha=abi.ALPHA_STRAIGHT), 4 + 4),
    Case("encode RGB8 -> 10-bit 4:2:0 (a3)", ycc_encode(8, 3, 10, abi.CHROMA_420, N601), 3 + 3),
    # monochrome and planar-RGB images (rows a4 / a16 / a18 / a19): still the generic kernels; four sets rotate so that
    # nothing survives in the 50 MB L2
    Case("decode mono 8-bit -> Gray8 (a16)", mono_rgb_decode(MONO, 8, 8), 2, sets=4),
    Case("decode mono 10-bit -> Gray16 (a16)", mono_rgb_decode(MONO, 10, 16), 4, sets=4),
    Case("decode planar RGB 8-bit -> RGB8 (a18)", mono_rgb_decode(RGB, 8, 8), 6, sets=4),
    Case("decode planar RGB 10-bit -> RGB16 (a18)", mono_rgb_decode(RGB, 10, 16), 12, sets=4),
    Case("encode Gray8 -> 8-bit Y (a4)", abi.EncodeDesc(W, H8, 8, 1, abi.ALPHA_NONE, 8), 2, sets=4),
    Case("encode Gray8 -> 10-bit Y (a4)", abi.EncodeDesc(W, H8, 8, 1, abi.ALPHA_NONE, 10), 3, sets=4),
    # float hosts reading planar RGB / monochrome images: kernels_fast_decode_table.cu (per-code EOTF table in shared memory)
    Case("decode planar RGB 10-bit PQ -> RGB32f (a18)", float_table_decode(RGB, abi.TRANSFER_CHAR_PQ, 0), 6 + 12),
    Case("decode planar RGB 10-bit HLG + OOTF -> RGB32f (a18)", float_table_decode(RGB, abi.TRANSFER_CHAR_HLG, 1), 6 + 12),
    Case("decode mono 12-bit PQ -> Gray32f (a16)", float_table_decode(MONO, abi.TRANSFER_CHAR_PQ, 0), 2 + 4),
    # premultiplied alpha on the integer hosts (BASELINE config 4's second variant, SURVEY.md 8(d)): tuned kernel with the verified premultiply
    Case("encode RGBA16 premultiplied -> 10-bit 4:2:2 + A (config 4, premultiplied alpha) (a2, a5)",
         ycc_encode(16, 4, 10, abi.CHROMA_422, None, alpha=abi.ALPHA_PREMULTIPLIED), 8 + 6),
    Case("encode RGBA16 straight -> 10-bit 4:2:2 + A (config 4's own variant, same frame) (a2)",
         ycc_encode(16, 4, 10, abi.CHROMA_422, None, alpha=abi.ALPHA_STRAIGHT), 8 + 6),
    Case("encode RGBA8 premultiplied -> 8-bit 4:2:0 + A (a3, a5)", ycc_encode(8, 4, 8, abi.CHROMA_420, None, alpha=abi.ALPHA_PREMULTIPLIED), 4 + 2.5),
    Case("encode RGBA32f -> 12-bit PQ 4:2:0 + A, exact powf (a1)", float_encode(4, PLANAR), 16 + 5, tables=False),
    Case("encode RGB32f -> interleaved RGB 12-bit PQ (the reference's own layout), exact powf (a1)", float_encode(3, REFERENCE), 12 + 6, tables=False),
    Case("encode RGBA32f -> 12-bit PQ 4:2:0 + A, step tables (a1)", float_encode(4, PLANAR), 16 + 5, tables=True),
    Case("encode RGB32f -> interleaved RGB 12-bit PQ (the reference's own layout), step tables (a1)", float_encode(3, REFERENCE), 12 + 6, tables=True),
    # RGBA in the reference's layout has no tuned kernel: the generic kernel reads the compact step table from global memory
    Case("encode RGBA32f -> interleaved RGBA 12-bit PQ (the reference's own layout), step tables, generic kernel (a1)", float_encode(4, REFERENCE), 16 + 8,
         tables=True),
    Case("encode RGB32f -> 10-bit PQ 4:2:0, tuned kernel (config 2 at 10 bits)", float_encode(3, PLANAR, depth=10), 15, tables=True),
    Case("encode RGB32f -> 12-bit PQ @ 1000 nit 4:2:0, tuned kernel (config 2 at another peak)", float_encode(3, PLANAR, peak=1000), 15, tables=True),
    Case("encode RGB32f -> 12-bit SMPTE 428 4:2:0 (two-level table in the copy-engine kernel)", float_encode(3, PLANAR, transfer=abi.TRANSFER_SMPTE428), 15,
         tables=True),
    Case("encode RGB32f -> 12-bit clip 4:2:0 (no curve)", float_encode(3, PLANAR, transfer=abi.TRANSFER_CLIP), 15, tables=True),
    # Gray(+A) float hosts (row a4 at 32 bits): kernels_fast_gray32.cu, PQ through the compact step table / clip
    Case("encode Gray32f -> 12-bit PQ Y (a4)", float_encode(1, REFERENCE), 4 + 2, tables=True),
    Case("encode GrayA32f -> 12-bit PQ Y + A (a4)", float_encode(2, REFERENCE), 8 + 4, tables=True),
    Case("encode Gray32f -> 12-bit clip Y (a4)", float_encode(1, REFERENCE, transfer=abi.TRANSFER_CLIP), 4 + 2, tables=True),
    Case("encode Gray32f -> 12-bit PQ Y, exact powf (a4)", float_encode(1, REFERENCE), 4 + 2, tables=False),
]


def code_dtype(depth):
    return torch.uint8 if depth == 8 else torch.int16


def buffer_set(desc, generator):
    """(call arguments, tensors) of one buffer set: random host rows or codes, and an empty destination."""
    h, w = desc.height, desc.width
    if isinstance(desc, abi.EncodeDesc):
        shape = (h, w * desc.host_channels)
        if desc.host_depth == 32:
            rows = torch.rand(shape, generator=generator, device="cuda")
        else:
            top = 256 if desc.host_depth == 8 else 32769
            rows = torch.randint(0, top, shape, generator=generator, device="cuda", dtype=torch.int32).to(code_dtype(desc.host_depth))
        planes = [None if s is None else torch.empty(s, dtype=code_dtype(desc.image_bit_depth), device="cuda") for s in abi.encode_plane_shapes(desc)]
        return (desc, rows.data_ptr(), rows.stride(0) * rows.element_size(), avifgpu.planes_from_tensors(planes)), (rows, planes)
    planes = [None if s is None else torch.randint(0, 1 << desc.bit_depth, s, generator=generator, device="cuda", dtype=torch.int32)
              .to(code_dtype(desc.bit_depth)) for s in abi.decode_plane_shapes(desc)]
    out = torch.empty((h, w * abi.decode_host_channels(desc)), dtype={8: torch.uint8, 16: torch.int16, 32: torch.float32}[desc.host_depth], device="cuda")
    return (desc, avifgpu.planes_from_tensors(planes), out.data_ptr(), out.stride(0) * out.element_size()), (planes, out)


def measure(case, ctx, generator, args):
    if case.tables is not None:
        ctx = avifgpu.Context(0)
        ctx.set_table_autobuild(-1)
        if case.tables:
            ctx.prepare_encode(case.desc)
    sets = [buffer_set(case.desc, generator) for _ in range(case.sets)]
    call = ctx.encode_device if isinstance(case.desc, abi.EncodeDesc) else ctx.decode_device
    rotation = itertools.cycle([call_args for call_args, _ in sets])

    def run():
        call(*next(rotation))

    ms = statistics.median(harness.timed({"run": run}, args.seconds, args.rounds)["run"])
    pixels = case.desc.width * case.desc.height
    if case.tables is not None:
        ctx.close()
    return {"case": case.name, "ms": ms, "gpx_s": pixels / ms / 1e6, "gb_s": pixels * case.bytes_per_px / ms / 1e6}


def main():
    args = harness.arguments(rounds=3).parse_args()
    harness.require_gpu()
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    with avifgpu.Context(0) as ctx:
        harness.emit([measure(case, ctx, g, args) for case in CASES if ONLY is None or ONLY in case.name], args.out)


if __name__ == "__main__":
    main()
