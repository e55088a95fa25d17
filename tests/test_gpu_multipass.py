"""The tuned kernels at shapes where their grid-stride loops run more than once, bit for bit against the CPU checker.

Every tuned launcher caps its grid (one persistent CTA per SM, or a few), so a thread or a warp walks the image in
passes.  test_gpu_parity.py runs at most 130 x 5 pixels -- one pass of every loop -- so the walk itself (GroupWalk's
column carry and its degenerate steps, the groups a thread keeps in flight past the end of the image, the flat kernel's
runs of tiles, mbarrier parity and second items) is only exercised here.  Each case:

  * goes through the device entry points on buffers whose row strides are rounded up to 256 bytes (as the host path
    stages them), with a sentinel in the padding that must survive;
  * proves it reached the tuned kernel: its width leaves a right strip (and 4:2:0 an odd last row), so the tuned
    launcher makes 1 + strips launches where the generic kernel alone makes 1;
  * asserts, from the device's SM count and the launcher's grid cap (GRID_CAPS), that the loop runs at least twice;
  * compares with the compiled reference where the reference has the path (the restatement otherwise), with the same
    rule as test_gpu_parity.py."""
import os

import numpy as np
import pytest

import cases
from avifgpu import abi
from gpu_harness import Padded, pick, planes_struct, rgb32_nclx, run_counted, sm_count, strips

pytestmark = pytest.mark.gpu

# How many workers (threads, or warps for the tile kernels) each tuned launcher starts per CTA, and how many CTAs per SM
# at most: (per_cta, ctas_per_sm, in_flight, source of the cap).  in_flight = units a worker loads before it converts
# the first (one outer iteration covers in_flight passes of the grid).
GRID_CAPS = {
    "flat": (28, 1, 1, "kernels_fast_flat.cu:373-377 (warps; kFlatWarps = 28, one CTA per SM)"),
    "rgba": (16, 1, 1, "kernels_fast_rgba.cu:238-242 (warps; kRgbaWarps = 16, one CTA per SM)"),
    "clip": (8, 3, 1, "kernels_fast.cu:116-121 (warps; 8 per CTA, kClipBlocksPerSm = 3)"),
    "gray32_pq": (1024, 1, 2, "kernels_fast_gray32.cu:237-239 (threads; kGroupsInFlight = 2)"),
    "gray32_clip": (256, 8, 2, "kernels_fast_gray32.cu:237-239 (threads; kGroupsInFlight = 2)"),
    "gray16_lut": (1024, 1, 4, "kernels_fast_int.cu:739, 96 (threads; kUnroll = 4)"),
    "gray_int8": (256, 16, 4, "kernels_fast_int.cu:651-653, 607 (threads; kInFlight = 4 for 8-bit hosts)"),
    "gray_int16": (256, 16, 1, "kernels_fast_int.cu:651-653, 607"),
    "rgb_int": (256, 16, 1, "kernels_fast_int.cu:665-667"),
    "stream8": (256, 16, 4, "kernels_fast_decode_int.cu:580-582, 452 (threads; kInFlight = 4 for 8-bit hosts)"),
    "stream16": (256, 16, 1, "kernels_fast_decode_int.cu:580-582, 452"),
    # the occupancy API picks the CTAs per SM (4 at 52 registers, 8 at 32): 8 is the upper bound, so the pass counts
    # asserted with it are lower bounds
    "table": (256, 8, 1, "kernels_fast_decode_table.cu:146-156 (threads; cudaOccupancyMaxActiveBlocksPerMultiprocessor)"),
    "ycc_int": (8, 3, 1, "kernels_fast_decode_int.cu:377-383 (warps; kWarps = 8, kBlocksPerSm = 3)"),
}


def workers(kernel, units, sms):
    """Threads (or warps) in the grid the launcher starts for `units` work units."""
    per_cta, ctas_per_sm, _, _ = GRID_CAPS[kernel]
    ctas = max(1, min(-(-units // per_cta), sms * ctas_per_sm))
    return ctas * per_cta


def passes(kernel, units, sms):
    """Outer iterations of the busiest worker: grid strides, divided by the units it keeps in flight."""
    in_flight = GRID_CAPS[kernel][2]
    return -(-units // (workers(kernel, units, sms) * in_flight))


def assert_passes(kernel, units, sms, at_least=2):
    n = passes(kernel, units, sms)
    assert n >= at_least, f"{kernel}: {units} units make {n} pass(es) at {sms} SMs ({GRID_CAPS[kernel][3]})"


def assert_walk(kernel, groups_per_row, rows, sms, step_rows=None, step_columns=None):
    """GroupWalk's per-thread steps: stride // groupsPerRow rows and stride % groupsPerRow groups."""
    stride = workers(kernel, groups_per_row * rows, sms)
    if step_rows is not None:
        assert stride // groups_per_row == step_rows, (kernel, stride, groups_per_row)
    if step_columns is not None:
        assert stride % groups_per_row == step_columns, (kernel, stride, groups_per_row)
    assert -(-groups_per_row * rows // stride) >= 2, (kernel, stride, groups_per_row, rows)


def flat_schedule(width, rows, sms):
    """FlatSchedule as LaunchFlatKernel builds it (kernels_fast_flat.cu:368-389) for the tuned part (width & ~3)."""
    width4 = width & ~3
    tiles_x = -(-width4 // 128)
    tile_rows = (rows + 1) // 2
    warp_count = workers("flat", tiles_x * tile_rows, sms)
    segments = min(max(warp_count // tiles_x, 1), tile_rows)
    return dict(warp_count=warp_count, tiles_x=tiles_x, items=tiles_x * segments, segment_rows=tile_rows // segments,
                long_segments=tile_rows % segments, unpaired=bool(rows & 1))


def rows_for(kernel, units_per_row_unit, sms, rows_per_unit=1, factor=1.5, odd=False):
    """A height whose units fill `factor` outer iterations of `kernel`'s grid (so the last one is partly past the end)."""
    per_cta, ctas_per_sm, in_flight, _ = GRID_CAPS[kernel]
    capacity = sms * ctas_per_sm * per_cta * in_flight
    h = -(-int(capacity * factor) // units_per_row_unit) * rows_per_unit
    return h | 1 if odd else h


# ---- device calls on buffers with 256-byte row strides and a sentinel in the padding (gpu_harness.Padded) -------------------

def encode_and_compare(gpu, reference, desc, rows, launches, beyond=None):
    """rows: host array; `launches` = what the tuned launcher makes (1 + strips).  beyond: for Gray16 hosts in the
    reference layout, the checker of samples above 32768 -- the reference reads past its 32769-entry tables there, the
    clamp is this project's definition (the restatement's); every other code is the reference's."""
    import torch
    dev = torch.device("cuda", gpu.device)
    src = Padded(dev, rows.shape[0], rows.shape[1], rows.dtype, rows)
    shapes = abi.encode_plane_shapes(desc)
    dtype = abi.code_dtype(desc.image_bit_depth)
    out = [None if s is None else Padded(dev, s[0], s[1], dtype) for s in shapes]
    planes = planes_struct(out)
    delta = run_counted(gpu, lambda: gpu.encode_device(desc, src.ptr(), src.stride, planes))
    assert delta != 1, "the generic kernel served the call: this case tests no tuned kernel"
    assert delta == launches, f"{delta} launches, the tuned launcher makes {launches}"
    expected = reference.encode(desc, rows, threads=os.cpu_count())
    if beyond is not None:
        assert desc.layout == abi.LAYOUT_REFERENCE and desc.host_channels <= 2 and desc.host_depth == 16
        defined = beyond.encode(desc, rows, threads=os.cpu_count())
        for k, channel in ((0, 0), (3, desc.host_channels - 1)):
            if expected[k] is not None:
                outside = rows[:, channel::desc.host_channels] > 32768
                assert np.array_equal(expected[k][~outside], defined[k][~outside]), "the restatement disagrees with the reference"
                expected[k][outside] = defined[k][outside]
    for k, (e, g) in enumerate(zip(expected, out)):
        assert (e is None) == (g is None)
        if e is None:
            continue
        got = g.host()
        assert np.array_equal(e, got), f"plane {k}: {int((e != got).sum())} of {e.size} codes differ; first at {np.argwhere(e != got)[0]}"
        assert g.padding_intact(), f"plane {k}: wrote into the row padding"


def decode_and_compare(gpu, reference, desc, planes, launches, nan_payloads_free=False):
    import torch
    dev = torch.device("cuda", gpu.device)
    src = [None if p is None else Padded(dev, p.shape[0], p.shape[1], p.dtype, p) for p in planes]
    channels = abi.decode_host_channels(desc)
    out = Padded(dev, desc.height, desc.width * channels, abi.host_dtype(desc.host_depth))
    struct = planes_struct(src)
    delta = run_counted(gpu, lambda: gpu.decode_device(desc, struct, out.ptr(), out.stride))
    assert delta != 1, "the generic kernel served the call: this case tests no tuned kernel"
    assert delta == launches, f"{delta} launches, the tuned launcher makes {launches}"
    expected = reference.decode(desc, planes, threads=os.cpu_count())
    got = out.host()
    if expected.dtype == np.float32:
        e, g = expected.view(np.uint32), got.view(np.uint32)
        differ = e != g
        if nan_payloads_free:  # 0 * inf in the OOTF: a NaN on both sides, its payload is the FPU's
            differ &= ~(np.isnan(expected) & np.isnan(got))
            assert np.array_equal(np.isnan(expected), np.isnan(got))
    else:
        differ = expected != got
    assert not differ.any(), f"{int(differ.sum())} of {expected.size} samples differ; first at {np.argwhere(differ)[0]}"
    assert out.padding_intact(), "wrote into the row padding"


_inputs = {}


def cached(key, make):
    """One input per shape, shared by the configurations that read it (the big ones cost a second to draw)."""
    if key not in _inputs:
        _inputs.clear()
        _inputs[key] = make()
    return _inputs[key]


# ---- the flat encode kernel (kernels_fast_flat.cu) ---------------------------------------------------------------------------

INTERLEAVED_CONFIGS = [(depth, transfer, peak) for depth in (10, 12)
                       for transfer, peak in ((abi.TRANSFER_PQ, 80), (abi.TRANSFER_PQ, 1000), (abi.TRANSFER_PQ, 10000), (abi.TRANSFER_SMPTE428, 80))]


@pytest.mark.parametrize("depth,transfer,peak", INTERLEAVED_CONFIGS)
def test_flat_multipass_interleaved(gpu, checker, port, depth, transfer, peak):
    """The reference's interleaved RGB32f -> RGB codes layout through the flat kernel: every warp walks a run of 4-5 tiles
    down one column (runs of unequal length, the mbarrier parity flipping per tile), the last tile row has no second row,
    the last tile column is partial and two columns go to the generic strip."""
    w, h = 4102, 1001
    s = flat_schedule(w, h, sm_count(gpu))
    assert s["segment_rows"] >= 2 and s["long_segments"] > 0 and s["unpaired"], s
    rows = cached(("rgb32", w, h), lambda: cases.float_host_rows(cases.rng_for(f"multipass_rgb32_{w}x{h}"), h, w, 3, specials=True))
    desc = abi.EncodeDesc(w, h, 32, 3, abi.ALPHA_NONE, depth, transfer, peak)
    encode_and_compare(gpu, pick(checker, port, True), desc, rows, strips(w, 4))


def test_flat_multipass_interleaved_several_items(gpu, checker, port):
    """More tile columns than warps in the grid: some warps take a second item (another column) and fetch its first tile
    themselves."""
    sms = sm_count(gpu)
    w = (-(-GRID_CAPS["flat"][0] * sms * 128 * 21 // 20) // 4) * 4 + 2  # ~5 % more tile columns than warps
    h = 3
    s = flat_schedule(w, h, sms)
    assert s["items"] > s["warp_count"], s
    rows = cases.float_host_rows(cases.rng_for(f"multipass_items_{w}"), h, w, 3, specials=True)
    desc = abi.EncodeDesc(w, h, 32, 3, abi.ALPHA_NONE, 12, abi.TRANSFER_PQ, 80)
    encode_and_compare(gpu, pick(checker, port, True), desc, rows, strips(w, 4))


@pytest.mark.parametrize("shape", ["runs", "items"])
@pytest.mark.parametrize("transfer", [abi.TRANSFER_PQ, abi.TRANSFER_SMPTE428])
@pytest.mark.parametrize("chroma", [abi.CHROMA_444, abi.CHROMA_422])
def test_flat_multipass_planar(gpu, port, chroma, transfer, shape):
    """Planar YCbCr through the flat kernel outside config 2's 4:2:0 / 12-bit / PQ 80: 10-bit tables, the matrix and the
    4:2:2 down-filter on every tile of a run, or on a warp's second item.  The reference has no planar YCbCr encoder:
    the restatement is the checker."""
    sms = sm_count(gpu)
    if shape == "runs":
        w, h = 2054, 1203
        s = flat_schedule(w, h, sms)
        assert s["segment_rows"] >= 2 and s["long_segments"] > 0 and s["unpaired"], s
    else:
        w, h = (-(-GRID_CAPS["flat"][0] * sms * 128 * 21 // 20) // 4) * 4 + 2, 3
        s = flat_schedule(w, h, sms)
        assert s["items"] > s["warp_count"], s
    rows = cached(("rgb32", w, h), lambda: cases.float_host_rows(cases.rng_for(f"multipass_rgb32_{w}x{h}"), h, w, 3, specials=True))
    desc = abi.EncodeDesc(w, h, 32, 3, abi.ALPHA_NONE, 10, transfer, 1000, abi.LAYOUT_PLANAR_YCBCR, chroma, abi.DOWN_FILTER_BOX,
                          abi.GRAY16_LUT, cases.NCLX_2020_PQ())
    encode_and_compare(gpu, port, desc, rows, strips(w, 4))


# ---- the RGBA and clip tile kernels (kernels_fast_rgba.cu, kernels_fast.cu) ------------------------------------------------

@pytest.mark.parametrize("chroma", [abi.CHROMA_420, abi.CHROMA_444])
@pytest.mark.parametrize("variant", ["rgba_straight", "rgba_premultiplied", "clip"])
def test_tile_kernels_multipass(gpu, port, variant, chroma):
    """Every warp of EncodeRgbaF32FlatKernel / EncodeRgbF32ClipKernel converts at least two tiles (2 rows x 128 px),
    stepping its tile coordinates with a carry across the row of tiles."""
    sms = sm_count(gpu)
    kernel = "clip" if variant == "clip" else "rgba"
    w = 2053
    tiles_x = -(-(w & ~3) // 128)
    h = rows_for(kernel, tiles_x, sms, rows_per_unit=2, odd=True)
    ys = chroma == abi.CHROMA_420
    assert_passes(kernel, tiles_x * (((h & ~1 if ys else h) + 1) // 2), sms)
    channels = 3 if variant == "clip" else 4
    alpha = {"rgba_straight": abi.ALPHA_STRAIGHT, "rgba_premultiplied": abi.ALPHA_PREMULTIPLIED, "clip": abi.ALPHA_NONE}[variant]
    transfer, depth = (abi.TRANSFER_CLIP, 10) if variant == "clip" else (abi.TRANSFER_PQ, 12)
    rows = cases.float_host_rows(cases.rng_for(f"multipass_{variant}_{chroma}"), h, w, channels, specials=True)
    desc = abi.EncodeDesc(w, h, 32, channels, alpha, depth, transfer, 80, abi.LAYOUT_PLANAR_YCBCR, chroma, abi.DOWN_FILTER_BOX,
                          abi.GRAY16_LUT, cases.NCLX_2020_PQ())
    encode_and_compare(gpu, port, desc, rows, strips(w, 4, odd_rows=ys))


# ---- Gray / GrayA float hosts (kernels_fast_gray32.cu) -------------------------------------------------------------------------

@pytest.mark.parametrize("transfer", [abi.TRANSFER_PQ, abi.TRANSFER_CLIP])
@pytest.mark.parametrize("channels,alpha", [(1, abi.ALPHA_NONE), (2, abi.ALPHA_STRAIGHT), (2, abi.ALPHA_PREMULTIPLIED)])
def test_gray_float_multipass(gpu, checker, port, channels, alpha, transfer):
    """EncodeGrayF32Kernel: two outer iterations of two groups in flight per thread, the second partly past the end."""
    sms = sm_count(gpu)
    kernel = "gray32_pq" if transfer == abi.TRANSFER_PQ else "gray32_clip"
    w = 4099
    h = rows_for(kernel, w // 4, sms)
    assert_passes(kernel, (w // 4) * h, sms)
    rows = cases.float_host_rows(cases.rng_for(f"multipass_gray32_{channels}_{alpha}_{transfer}"), h, w, channels, specials=True)
    desc = abi.EncodeDesc(w, h, 32, channels, alpha, 12, transfer, 80)
    encode_and_compare(gpu, pick(checker, port, True), desc, rows, strips(w, 4))


# ---- integer hosts, encode (kernels_fast_int.cu) -------------------------------------------------------------------------------

@pytest.mark.parametrize("depth", [8, 10, 12])
@pytest.mark.parametrize("channels", [1, 2])
@pytest.mark.parametrize("host_depth", [8, 16])
def test_gray_int_multipass(gpu, checker, port, host_depth, channels, depth):
    """Gray / GrayA integer hosts in the reference layout: EncodeGrayIntKernel (8-bit hosts: four groups in flight, two
    outer iterations), or for Gray16 into 10 / 12 bits the 65536-entry table kernel (four chunks in flight)."""
    sms = sm_count(gpu)
    lut = host_depth == 16 and channels == 1 and depth > 8
    kernel = "gray16_lut" if lut else f"gray_int{host_depth}"
    w = 5003
    h = rows_for(kernel, w // 8, sms)
    assert_passes(kernel, (w // 8) * h, sms)
    rows = cached(("gray", host_depth, channels, w, h),
                  lambda: cases.int_host_rows(cases.rng_for(f"multipass_grayint_{host_depth}_{channels}"), h, w, channels, host_depth, beyond=True))
    alpha = abi.ALPHA_NONE if channels == 1 else abi.ALPHA_STRAIGHT
    desc = abi.EncodeDesc(w, h, host_depth, channels, alpha, depth)
    encode_and_compare(gpu, pick(checker, port, True), desc, rows, strips(w, 8), beyond=port if host_depth == 16 else None)


@pytest.mark.parametrize("host_depth,channels,alpha,depth,chroma", [(16, 4, abi.ALPHA_PREMULTIPLIED, 10, abi.CHROMA_420),
                                                                    (8, 3, abi.ALPHA_NONE, 12, abi.CHROMA_422)])
def test_rgb_int_planar_multipass(gpu, port, host_depth, channels, alpha, depth, chroma):
    """EncodeRgbIntPlanarKernel over two passes of its grid (4:2:0: one group is 8 px x 2 rows)."""
    sms = sm_count(gpu)
    ys = chroma == abi.CHROMA_420
    w = 2053
    h = rows_for("rgb_int", w // 8, sms, rows_per_unit=2 if ys else 1, odd=True)
    assert_passes("rgb_int", (w // 8) * ((h & ~1) >> 1 if ys else h), sms)
    rows = cases.int_host_rows(cases.rng_for(f"multipass_rgbint_{host_depth}_{channels}"), h, w, channels, host_depth, beyond=True)
    desc = abi.EncodeDesc(w, h, host_depth, channels, alpha, depth, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, chroma,
                          abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, cases.NCLX_709())
    encode_and_compare(gpu, port, desc, rows, strips(w, 8, odd_rows=ys))


# ---- integer hosts, decode (kernels_fast_decode_int.cu) ------------------------------------------------------------------------

def nclx_for(colorspace, full_range=1):
    return cases.NCLX_2020_PQ(full_range) if colorspace == abi.COLORSPACE_MONOCHROME else cases.NCLX_GBR()


@pytest.mark.parametrize("alpha", [abi.ALPHA_NONE, abi.ALPHA_STRAIGHT])
@pytest.mark.parametrize("bit_depth,host_depth", [(8, 8), (10, 16), (12, 16)])
@pytest.mark.parametrize("colorspace", [abi.COLORSPACE_MONOCHROME, abi.COLORSPACE_RGB])
def test_stream_decode_multipass(gpu, checker, port, colorspace, bit_depth, host_depth, alpha):
    """StreamDecodeKernel, monochrome and planar RGB: 8-bit images keep four groups in flight over two outer iterations
    (monochrome 8-bit full range is the identity copy, limited range the table); 10 / 12-bit codes into 16-bit hosts
    with out-of-range codes in the containers."""
    sms = sm_count(gpu)
    kernel = f"stream{host_depth}"
    w = 5003
    h = rows_for(kernel, w // 8, sms)
    assert_passes(kernel, (w // 8) * h, sms)
    mono = colorspace == abi.COLORSPACE_MONOCHROME
    desc = abi.DecodeDesc(w, h, colorspace, abi.CHROMA_MONOCHROME if mono else abi.CHROMA_444, bit_depth, alpha, host_depth,
                          nclx_for(colorspace, 1 if alpha == abi.ALPHA_NONE else 0))
    planes = cases.code_planes(cases.rng_for(f"multipass_stream_{colorspace}_{bit_depth}_{alpha}"), desc, overshoot=True)
    decode_and_compare(gpu, pick(checker, port, True), desc, planes, strips(w, 8))


@pytest.mark.parametrize("bit_depth,host_depth", [(8, 8), (10, 16)])
@pytest.mark.parametrize("chroma", [abi.CHROMA_420, abi.CHROMA_422])
def test_ycc_int_decode_multipass(gpu, checker, port, chroma, bit_depth, host_depth):
    """DecodeYccToRgbIntKernel with sub-sampled chroma and straight alpha, two units (256 px x 1-2 rows) per warp."""
    sms = sm_count(gpu)
    ys = chroma == abi.CHROMA_420
    w = 2053
    units_x = -(-(w & ~7) // 256)
    h = rows_for("ycc_int", units_x, sms, rows_per_unit=2 if ys else 1, odd=True)
    assert_passes("ycc_int", units_x * ((h & ~1) >> 1 if ys else h), sms)
    desc = abi.DecodeDesc(w, h, abi.COLORSPACE_YCBCR, chroma, bit_depth, abi.ALPHA_STRAIGHT, host_depth, cases.NCLX_709(0))
    planes = cases.code_planes(cases.rng_for(f"multipass_yccint_{chroma}_{bit_depth}"), desc, overshoot=True)
    decode_and_compare(gpu, pick(checker, port, True), desc, planes, strips(w, 8, odd_rows=ys))


# ---- float hosts, monochrome and planar-RGB decode (kernels_fast_decode_table.cu) ----------------------------------------------

TABLE_CONFIGS = [("rgb", "pq", dict(pq_peak_nits=80)), ("rgb", "pq", dict(pq_peak_nits=1000)), ("rgb", "pq", dict(pq_peak_nits=10000)),
                 ("rgb", "hlg", dict(hlg_apply_ootf=1)), ("rgb", "hlg", dict(hlg_apply_ootf=0)), ("rgb", "428", dict()),
                 ("mono", "full", dict(pq_peak_nits=80)), ("mono", "limited", dict(pq_peak_nits=1000))]


def table_desc(w, h, kind, name, alpha, kwargs):
    if kind == "mono":
        return abi.DecodeDesc(w, h, abi.COLORSPACE_MONOCHROME, abi.CHROMA_MONOCHROME, 12, alpha, 32, cases.NCLX_2020_PQ(int(name == "full")), **kwargs)
    return abi.DecodeDesc(w, h, abi.COLORSPACE_RGB, abi.CHROMA_444, 12 if name == "pq" else 10, alpha, 32, rgb32_nclx(name), **kwargs)


def table_planes(desc, seed):
    # planar RGB float: the reference indexes its 2^depth table with the raw code, so codes above the maximum are out of its
    # contract (test_gpu_parity.py draws them the same way); monochrome clamps them (YuvDecode.cpp) and gets them
    return cases.code_planes(cases.rng_for(seed), desc, overshoot=desc.colorspace == abi.COLORSPACE_MONOCHROME)


@pytest.mark.parametrize("alpha", [abi.ALPHA_NONE, abi.ALPHA_STRAIGHT, abi.ALPHA_PREMULTIPLIED])
@pytest.mark.parametrize("kind,name,kwargs", TABLE_CONFIGS, ids=[f"{k}-{n}-{'-'.join(f'{a}{b}' for a, b in kw.items())}" for k, n, kw in TABLE_CONFIGS])
def test_table_decode_multipass(gpu, checker, port, kind, name, kwargs, alpha):
    """TableDecodeF32Kernel: a table per CTA, then at least two grid strides of 8-pixel groups per thread (asserted with the
    occupancy API's upper bound of 8 CTAs per SM)."""
    sms = sm_count(gpu)
    w, h = 2053, 3001
    assert_passes("table", (w // 8) * h, sms)
    desc = table_desc(w, h, kind, name, alpha, kwargs)
    planes = table_planes(desc, f"multipass_table_{kind}_{name}_{alpha}")
    decode_and_compare(gpu, pick(checker, port, True), desc, planes, strips(w, 8))


@pytest.mark.parametrize("gamma,peak", [(1.2, 1000), (0.85, 100), (1.0, 334), (1.8, 27000), (2.5, 100000)])
@pytest.mark.parametrize("alpha", [abi.ALPHA_NONE, abi.ALPHA_STRAIGHT])
def test_planar_rgb_float_decode_ootf_grid(gpu, checker, port, alpha, gamma, peak):
    """Planar-RGB HLG decode through TableDecodeF32Kernel over the OOTF's gamma / peak grid, black pixels included
    (luma 0: powf(0, gamma - 1), +inf for gamma < 1, then 0 * inf)."""
    w, h = 260, 9
    desc = abi.DecodeDesc(w, h, abi.COLORSPACE_RGB, abi.CHROMA_444, 10, alpha, 32, rgb32_nclx("hlg"), hlg_apply_ootf=1,
                          hlg_display_gamma=gamma, hlg_peak_nits=peak)
    planes = table_planes(desc, f"multipass_ootf_{gamma}_{alpha}")
    for k in range(3):
        planes[k][0, :8] = 0
    decode_and_compare(gpu, pick(checker, port, True), desc, planes, strips(w, 8), nan_payloads_free=True)


# ---- GroupWalk's degenerate steps ---------------------------------------------------------------------------------------------

WALK_KERNELS = ["gray32_pq", "gray_int8", "rgb_int", "stream8", "stream16", "table"]


def walk_case(kernel, w, h, seed):
    """(description, inputs, reference_ok, launches) of one GroupWalk kernel at w x h."""
    if kernel == "gray32_pq":
        desc = abi.EncodeDesc(w, h, 32, 1, abi.ALPHA_NONE, 12, abi.TRANSFER_PQ, 80)
        return desc, cases.float_host_rows(cases.rng_for(seed), h, w, 1, specials=True), True, strips(w, 4)
    if kernel == "gray_int8":
        desc = abi.EncodeDesc(w, h, 8, 2, abi.ALPHA_STRAIGHT, 10)
        return desc, cases.int_host_rows(cases.rng_for(seed), h, w, 2, 8), True, strips(w, 8)
    if kernel == "rgb_int":
        desc = abi.EncodeDesc(w, h, 16, 3, abi.ALPHA_NONE, 10, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_444,
                              abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, cases.NCLX_709())
        return desc, cases.int_host_rows(cases.rng_for(seed), h, w, 3, 16, beyond=True), False, strips(w, 8)
    if kernel == "stream8":
        desc = abi.DecodeDesc(w, h, abi.COLORSPACE_RGB, abi.CHROMA_444, 8, abi.ALPHA_STRAIGHT, 8, cases.NCLX_GBR())
        return desc, cases.code_planes(cases.rng_for(seed), desc), True, strips(w, 8)
    if kernel == "stream16":
        desc = abi.DecodeDesc(w, h, abi.COLORSPACE_MONOCHROME, abi.CHROMA_MONOCHROME, 12, abi.ALPHA_NONE, 16, cases.NCLX_2020_PQ(0))
        return desc, cases.code_planes(cases.rng_for(seed), desc, overshoot=True), True, strips(w, 8)
    desc = abi.DecodeDesc(w, h, abi.COLORSPACE_MONOCHROME, abi.CHROMA_MONOCHROME, 12, abi.ALPHA_STRAIGHT, 32, cases.NCLX_2020_PQ(1))
    return desc, cases.code_planes(cases.rng_for(seed), desc, overshoot=True), True, strips(w, 8)


def group_pixels(kernel):
    return 4 if kernel.startswith("gray32") else 8


def run_walk_case(gpu, checker, port, kernel, w, h, seed):
    desc, inputs, reference_ok, launches = walk_case(kernel, w, h, seed)
    reference = pick(checker, port, reference_ok)
    if isinstance(desc, abi.EncodeDesc):
        encode_and_compare(gpu, reference, desc, inputs, launches)
    else:
        decode_and_compare(gpu, reference, desc, inputs, launches)


@pytest.mark.parametrize("kernel", WALK_KERNELS)
def test_walk_row_longer_than_a_pass(gpu, checker, port, kernel):
    """stepRows = 0: one row holds more groups than the grid has threads, so every step is a column step, and the carry
    takes a thread into the next row."""
    sms = sm_count(gpu)
    per_cta, ctas_per_sm, _, _ = GRID_CAPS[kernel]
    g = group_pixels(kernel)
    groups_per_row = sms * ctas_per_sm * per_cta * 11 // 10
    w, h = groups_per_row * g + 3, 2
    assert_walk(kernel, groups_per_row, h, sms, step_rows=0)
    run_walk_case(gpu, checker, port, kernel, w, h, f"multipass_long_row_{kernel}")


@pytest.mark.parametrize("kernel", WALK_KERNELS)
def test_walk_one_column_of_groups(gpu, checker, port, kernel):
    """stepColumns = 0: a 9 px wide image (one 8-px group, or two 4-px groups, per row) tall enough for two passes."""
    sms = sm_count(gpu)
    g = group_pixels(kernel)
    w = 9
    groups_per_row = w // g
    h = rows_for(kernel, groups_per_row, sms, factor=1.3 / GRID_CAPS[kernel][2])
    assert_walk(kernel, groups_per_row, h, sms, step_columns=0)
    run_walk_case(gpu, checker, port, kernel, w, h, f"multipass_narrow_{kernel}")
