#!/usr/bin/env python3
"""Device-resident throughput of configurations outside BASELINE.json's bench lines (they run wherever the dispatcher
sends them).  Every launch converts a stack of 8K frames tall enough that its input + output exceed the 50 MB L2
several times over (7680 x 17280 for the 8-bit paths, 7680 x 8640 otherwise), and three such sets rotate, so the GB/s
figures are HBM figures.  Prints one JSON line per case.

    python profiles/measure_generic_paths.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "avif-format_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import avifgpu  # noqa: E402
from avifgpu import abi  # noqa: E402

W, H = 7680, 4320 * 2
H8 = 4320 * 4  # 8-bit paths move 1.5 - 8 bytes per pixel: four frames per launch
dev = torch.device("cuda", 0)
gpu = avifgpu.Context(0)
g = torch.Generator(device=dev)
g.manual_seed(1)


ONE_LAUNCH = os.environ.get("AVIFGPU_MEASURE_ONE_LAUNCH") == "1"  # under ncu: one warm launch, one measured launch per case
ONLY = os.environ.get("AVIFGPU_MEASURE_ONLY")  # run only the cases whose name contains this text


def wanted(name):
    return ONLY is None or ONLY in name


def timed(fn, steps=30):
    if ONE_LAUNCH:
        steps = 1
    for _ in range(1 if ONE_LAUNCH else 3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def decode_case(name, bit_depth, host_depth, chroma, nclx, bytes_per_px, alpha=False):
    if not wanted(name):
        return
    H = H8 if bit_depth == 8 else globals()["H"]
    desc = abi.DecodeDesc(W, H, abi.COLORSPACE_YCBCR, chroma, bit_depth, abi.ALPHA_STRAIGHT if alpha else abi.ALPHA_NONE, host_depth, nclx)
    shapes = abi.decode_plane_shapes(desc)
    dt = torch.uint8 if bit_depth == 8 else torch.int16
    sets = []
    for _ in range(3):
        planes = [None if s is None else torch.randint(0, 1 << bit_depth, s, generator=g, device=dev, dtype=torch.int32).to(dt) for s in shapes]
        ch = abi.decode_host_channels(desc)
        out = torch.empty((H, W * ch), dtype={8: torch.uint8, 16: torch.int16, 32: torch.float32}[host_depth], device=dev)
        sets.append((avifgpu.planes_from_tensors(planes), planes, out))
    i = [0]

    def run():
        s = sets[i[0] % 3]
        i[0] += 1
        gpu.decode_device(desc, s[0], s[2].data_ptr(), s[2].stride(0) * s[2].element_size())
    ms = timed(run)
    print(json.dumps({"case": name, "ms": ms, "gpx_s": W * H / ms / 1e6, "gb_s": W * H * bytes_per_px / ms / 1e6}))


def encode_case(name, host_depth, channels, image_depth, chroma, nclx, bytes_per_px, alpha=abi.ALPHA_NONE):
    if not wanted(name):
        return
    H = H8 if host_depth == 8 else globals()["H"]
    desc = abi.EncodeDesc(W, H, host_depth, channels, alpha, image_depth, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, chroma,
                          abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, nclx)
    shapes = abi.encode_plane_shapes(desc)
    sets = []
    for _ in range(3):
        if host_depth == 8:
            rows = torch.randint(0, 256, (H, W * channels), generator=g, device=dev, dtype=torch.int32).to(torch.uint8)
        else:
            rows = torch.randint(0, 32769, (H, W * channels), generator=g, device=dev, dtype=torch.int32).to(torch.int16)
        dt = torch.uint8 if image_depth == 8 else torch.int16
        planes = [None if s is None else torch.empty(s, dtype=dt, device=dev) for s in shapes]
        sets.append((rows, avifgpu.planes_from_tensors(planes), planes))
    i = [0]

    def run():
        s = sets[i[0] % 3]
        i[0] += 1
        gpu.encode_device(desc, s[0].data_ptr(), s[0].stride(0) * s[0].element_size(), s[1])
    ms = timed(run)
    print(json.dumps({"case": name, "ms": ms, "gpx_s": W * H / ms / 1e6, "gb_s": W * H * bytes_per_px / ms / 1e6}))


def float_encode_case(name, channels, layout, bytes_per_px, tables, depth=12, peak=80, transfer=abi.TRANSFER_PQ):
    if not wanted(name):
        return
    alpha = abi.ALPHA_STRAIGHT if channels in (2, 4) else abi.ALPHA_NONE
    nclx = abi.Nclx(1, abi.PRIMARIES_BT2020, abi.TRANSFER_CHAR_PQ, abi.MATRIX_BT2020_NCL, 1)
    desc = abi.EncodeDesc(W, H, 32, channels, alpha, depth, transfer, peak, layout, abi.CHROMA_420 if layout == abi.LAYOUT_PLANAR_YCBCR else abi.CHROMA_444,
                          abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, nclx)
    ctx = avifgpu.Context(0)
    ctx.set_table_autobuild(-1)
    if tables:
        ctx.prepare_encode(desc)
    shapes = abi.encode_plane_shapes(desc)
    sets = []
    for _ in range(3):
        rows = torch.rand((H, W * channels), generator=g, device=dev)
        planes = [None if s is None else torch.empty(s, dtype=torch.int16, device=dev) for s in shapes]
        sets.append((rows, avifgpu.planes_from_tensors(planes), planes))
    i = [0]

    def run():
        s = sets[i[0] % 3]
        i[0] += 1
        ctx.encode_device(desc, s[0].data_ptr(), s[0].stride(0) * 4, s[1])
    ms = timed(run, steps=10)
    print(json.dumps({"case": name, "ms": ms, "gpx_s": W * H / ms / 1e6, "gb_s": W * H * bytes_per_px / ms / 1e6}))
    ctx.close()


n601 = abi.Nclx(1, 1, 13, abi.MATRIX_BT601, 1)
decode_case("decode 8-bit 4:2:0 -> RGB8 (a15)", 8, 8, abi.CHROMA_420, n601, 1.5 + 3)
decode_case("decode 8-bit 4:4:4 + alpha -> RGBA8 (a15)", 8, 8, abi.CHROMA_444, n601, 4 + 4, alpha=True)
decode_case("decode 10-bit 4:2:0 -> RGB16 (a14)", 10, 16, abi.CHROMA_420, n601, 3 + 6)
decode_case("decode 12-bit 4:4:4 -> RGB16 (a14)", 12, 16, abi.CHROMA_444, n601, 6 + 6)
encode_case("encode RGB8 -> 8-bit 4:2:0 (a3)", 8, 3, 8, abi.CHROMA_420, n601, 3 + 1.5)
encode_case("encode RGBA8 -> 8-bit 4:4:4 + A (config 1 at 8K) (a3)", 8, 4, 8, abi.CHROMA_444, n601, 4 + 4, alpha=abi.ALPHA_STRAIGHT)
encode_case("encode RGB8 -> 10-bit 4:2:0 (a3)", 8, 3, 10, abi.CHROMA_420, n601, 3 + 3)
def mono_rgb_cases():
    # monochrome and planar-RGB images (rows a4 / a16 / a18 / a19): still the generic kernels
    for name, colorspace, bit_depth, host_depth, bpp in (("decode mono 8-bit -> Gray8 (a16)", abi.COLORSPACE_MONOCHROME, 8, 8, 2),
                                                         ("decode mono 10-bit -> Gray16 (a16)", abi.COLORSPACE_MONOCHROME, 10, 16, 4),
                                                         ("decode planar RGB 8-bit -> RGB8 (a18)", abi.COLORSPACE_RGB, 8, 8, 6),
                                                         ("decode planar RGB 10-bit -> RGB16 (a18)", abi.COLORSPACE_RGB, 10, 16, 12)):
        if not wanted(name):
            continue
        H = H8 if bit_depth == 8 else globals()["H"]
        desc = abi.DecodeDesc(W, H, colorspace, abi.CHROMA_444, bit_depth, abi.ALPHA_NONE, host_depth, abi.Nclx(1, 1, 13, 0 if colorspace == abi.COLORSPACE_RGB else 6, 1))
        shapes = abi.decode_plane_shapes(desc)
        dt = torch.uint8 if bit_depth == 8 else torch.int16
        ch = abi.decode_host_channels(desc)
        sets = []
        for _ in range(4):  # rotate frames so that nothing survives in the 50 MB L2
            planes = [None if s is None else torch.randint(0, 1 << bit_depth, s, generator=g, device=dev, dtype=torch.int32).to(dt) for s in shapes]
            out = torch.empty((H, W * ch), dtype={8: torch.uint8, 16: torch.int16}[host_depth], device=dev)
            sets.append((avifgpu.planes_from_tensors(planes), planes, out))
        i = [0]

        def run():
            s_ = sets[i[0] % 4]
            i[0] += 1
            gpu.decode_device(desc, s_[0], s_[2].data_ptr(), s_[2].stride(0) * s_[2].element_size())
        ms = timed(run)
        print(json.dumps({"case": name, "ms": ms, "gpx_s": W * H / ms / 1e6, "gb_s": W * H * bpp / ms / 1e6}))
    for name, host_depth, depth, bpp in (("encode Gray8 -> 8-bit Y (a4)", 8, 8, 2), ("encode Gray8 -> 10-bit Y (a4)", 8, 10, 3)):
        if not wanted(name):
            continue
        H = H8
        desc = abi.EncodeDesc(W, H, host_depth, 1, abi.ALPHA_NONE, depth)
        shapes = abi.encode_plane_shapes(desc)
        sets = []
        for _ in range(4):
            rows = torch.randint(0, 256, (H, W), generator=g, device=dev, dtype=torch.int32).to(torch.uint8)
            planes = [None if s is None else torch.empty(s, dtype=torch.uint8 if depth == 8 else torch.int16, device=dev) for s in shapes]
            sets.append((rows, avifgpu.planes_from_tensors(planes), planes))
        i = [0]

        def run():
            s_ = sets[i[0] % 4]
            i[0] += 1
            gpu.encode_device(desc, s_[0].data_ptr(), s_[0].stride(0), s_[1])
        ms = timed(run)
        print(json.dumps({"case": name, "ms": ms, "gpx_s": W * H / ms / 1e6, "gb_s": W * H * bpp / ms / 1e6}))


def float_decode_table_cases():
    # float hosts reading planar RGB / monochrome images: kernels_fast_decode_table.cu (per-code EOTF table in shared memory)
    pq = abi.Nclx(1, abi.PRIMARIES_BT2020, abi.TRANSFER_CHAR_PQ, 0, 1)
    hlg = abi.Nclx(1, abi.PRIMARIES_BT2020, abi.TRANSFER_CHAR_HLG, 0, 1)
    for name, colorspace, nclx, ootf, bpp in (("decode planar RGB 10-bit PQ -> RGB32f (a18)", abi.COLORSPACE_RGB, pq, 0, 6 + 12),
                                              ("decode planar RGB 10-bit HLG + OOTF -> RGB32f (a18)", abi.COLORSPACE_RGB, hlg, 1, 6 + 12),
                                              ("decode mono 12-bit PQ -> Gray32f (a16)", abi.COLORSPACE_MONOCHROME, pq, 0, 2 + 4)):
        if not wanted(name):
            continue
        depth = 12 if colorspace == abi.COLORSPACE_MONOCHROME else 10
        desc = abi.DecodeDesc(W, H, colorspace, abi.CHROMA_444 if colorspace == abi.COLORSPACE_RGB else abi.CHROMA_MONOCHROME, depth, abi.ALPHA_NONE, 32, nclx,
                              hlg_apply_ootf=ootf)
        shapes = abi.decode_plane_shapes(desc)
        ch = abi.decode_host_channels(desc)
        sets = []
        for _ in range(3):
            planes = [None if s is None else torch.randint(0, 1 << depth, s, generator=g, device=dev, dtype=torch.int32).to(torch.int16) for s in shapes]
            out = torch.empty((H, W * ch), dtype=torch.float32, device=dev)
            sets.append((avifgpu.planes_from_tensors(planes), planes, out))
        i = [0]

        def run():
            s_ = sets[i[0] % 3]
            i[0] += 1
            gpu.decode_device(desc, s_[0], s_[2].data_ptr(), s_[2].stride(0) * 4)
        ms = timed(run, steps=12)
        print(json.dumps({"case": name, "ms": ms, "gpx_s": W * H / ms / 1e6, "gb_s": W * H * bpp / ms / 1e6}))


mono_rgb_cases()
float_decode_table_cases()
# premultiplied alpha on the integer hosts (BASELINE config 4's second variant, SURVEY.md 8(d)): tuned kernel with the verified premultiply
encode_case("encode RGBA16 premultiplied -> 10-bit 4:2:2 + A (config 4, premultiplied alpha) (a2, a5)", 16, 4, 10, abi.CHROMA_422, None, 8 + 6,
            alpha=abi.ALPHA_PREMULTIPLIED)
encode_case("encode RGBA16 straight -> 10-bit 4:2:2 + A (config 4's own variant, same frame) (a2)", 16, 4, 10, abi.CHROMA_422, None, 8 + 6,
            alpha=abi.ALPHA_STRAIGHT)
encode_case("encode RGBA8 premultiplied -> 8-bit 4:2:0 + A (a3, a5)", 8, 4, 8, abi.CHROMA_420, None, 4 + 2.5, alpha=abi.ALPHA_PREMULTIPLIED)
for tables in (False, True):
    tag = "step tables" if tables else "exact powf"
    float_encode_case(f"encode RGBA32f -> 12-bit PQ 4:2:0 + A, {tag} (a1)", 4, abi.LAYOUT_PLANAR_YCBCR, 16 + 5, tables)
    float_encode_case(f"encode RGB32f -> interleaved RGB 12-bit PQ (the reference's own layout), {tag} (a1)", 3, abi.LAYOUT_REFERENCE, 12 + 6, tables)
# RGBA in the reference's layout has no tuned kernel: the generic kernel reads the compact step table from global memory
float_encode_case("encode RGBA32f -> interleaved RGBA 12-bit PQ (the reference's own layout), step tables, generic kernel (a1)", 4, abi.LAYOUT_REFERENCE, 16 + 8, True)
float_encode_case("encode RGB32f -> 10-bit PQ 4:2:0, tuned kernel (config 2 at 10 bits)", 3, abi.LAYOUT_PLANAR_YCBCR, 15, True, depth=10)
float_encode_case("encode RGB32f -> 12-bit PQ @ 1000 nit 4:2:0, tuned kernel (config 2 at another peak)", 3, abi.LAYOUT_PLANAR_YCBCR, 15, True, peak=1000)
float_encode_case("encode RGB32f -> 12-bit SMPTE 428 4:2:0 (two-level table in the copy-engine kernel)", 3, abi.LAYOUT_PLANAR_YCBCR, 15, True, transfer=abi.TRANSFER_SMPTE428)
float_encode_case("encode RGB32f -> 12-bit clip 4:2:0 (no curve)", 3, abi.LAYOUT_PLANAR_YCBCR, 15, True, transfer=abi.TRANSFER_CLIP)
# Gray(+A) float hosts (row a4 at 32 bits): kernels_fast_gray32.cu, PQ through the compact step table / clip
float_encode_case("encode Gray32f -> 12-bit PQ Y (a4)", 1, abi.LAYOUT_REFERENCE, 4 + 2, True)
float_encode_case("encode GrayA32f -> 12-bit PQ Y + A (a4)", 2, abi.LAYOUT_REFERENCE, 8 + 4, True)
float_encode_case("encode Gray32f -> 12-bit clip Y (a4)", 1, abi.LAYOUT_REFERENCE, 4 + 2, True, transfer=abi.TRANSFER_CLIP)
float_encode_case("encode Gray32f -> 12-bit PQ Y, exact powf (a4)", 1, abi.LAYOUT_REFERENCE, 4 + 2, False)
