"""The batched kernels (kernels_batch.cu) under their chunk record source held to the CPU checker: every instantiation,
and every grid-stride loop over several passes (test_gpu_batch_indirect.py does the same under the workspace source).

A chunk of avifgpu_{encode,decode}_batch_device launches the instantiation its description selects (host depth, plane
depth, channels / premultiply, chroma) and walks the chunk's concatenated units with a capped, persistent grid, finding
each unit's image as it goes.  test_gpu_batch.py checks the entry points' contract on a few configurations; here:

  * ENCODE_KERNELS and DECODE_KERNELS hold one case per instantiation of EncodeRgbIntBatchKernel (36) and
    DecodeYccToRgbIntBatchKernel (12); test_instantiation_tables_are_complete checks their keys without a GPU.  Each
    case's launch count proves that its eligible images reached the batched kernels;
  * the multi-pass cases make the loops of all four batched kernels run at least twice (asserted from the SM count and
    the launchers' grid caps, BATCH_CAPS), and the edge kernels walk bottom strips of several units per row;
  * a batch led by an empty image, on a fresh context, still does its first-use checks.

Every image is compared bit for bit with the CPU checker -- the restatement for encode (the reference has no planar
YCbCr encoder), the compiled reference for decode -- and with a direct *_rows_device call, and the sentinel in the row
padding must survive.  16-bit hosts carry samples above 32768, 10 / 12-bit planes codes above the maximum."""
import collections
import itertools
import os

import pytest

import cases
from avifgpu import abi
from test_gpu_batch import (CHUNK, DecImage, Image, assert_decode_same_as_direct, assert_same_as_direct, ctx, planar,  # noqa: F401
                            run_batch, run_decode_batch, ycc)
from test_gpu_multipass import pick, run_counted

N601, N709, N2020, GBR = cases.NCLX_601(), cases.NCLX_709(), cases.NCLX_2020_PQ(), cases.NCLX_GBR()
BOX, TOP_LEFT = abi.DOWN_FILTER_BOX, abi.DOWN_FILTER_TOP_LEFT
C444, C422, C420 = abi.CHROMA_444, abi.CHROMA_422, abi.CHROMA_420
NONE, STRAIGHT, PREMUL = abi.ALPHA_NONE, abi.ALPHA_STRAIGHT, abi.ALPHA_PREMULTIPLIED

# ---- the instantiation tables ------------------------------------------------------------------------------------------

# EncodeRgbIntBatchKernel<HostT, PlaneT, CHANNELS, XS, YS, PREMULTIPLY>: one case per (host depth, plane depth,
# channels / alpha, chroma); matrices, down-filters and 10 / 12-bit planes spread over them
ENCODE_KERNELS = [
    ("h8_d8_c3_444_601", planar(8, 3, NONE, 8, C444, N601)),
    ("h8_d8_c3_422_709_box", planar(8, 3, NONE, 8, C422, N709, BOX)),
    ("h8_d8_c3_420_2020_topleft", planar(8, 3, NONE, 8, C420, N2020, TOP_LEFT)),
    ("h8_d8_c4s_444_gbr", planar(8, 4, STRAIGHT, 8, C444, GBR)),
    ("h8_d8_c4s_422_none_topleft", planar(8, 4, STRAIGHT, 8, C422, None, TOP_LEFT)),
    ("h8_d8_c4s_420_601_box", planar(8, 4, STRAIGHT, 8, C420, N601, BOX)),
    ("h8_d8_c4p_444_709", planar(8, 4, PREMUL, 8, C444, N709)),
    ("h8_d8_c4p_422_2020_box", planar(8, 4, PREMUL, 8, C422, N2020, BOX)),
    ("h8_d8_c4p_420_none_topleft", planar(8, 4, PREMUL, 8, C420, None, TOP_LEFT)),
    ("h8_d10_c3_444_2020", planar(8, 3, NONE, 10, C444, N2020)),
    ("h8_d12_c3_422_601_topleft", planar(8, 3, NONE, 12, C422, N601, TOP_LEFT)),
    ("h8_d10_c3_420_709_box", planar(8, 3, NONE, 10, C420, N709, BOX)),
    ("h8_d12_c4s_444_none", planar(8, 4, STRAIGHT, 12, C444, None)),
    ("h8_d10_c4s_422_2020_box", planar(8, 4, STRAIGHT, 10, C422, N2020, BOX)),
    ("h8_d12_c4s_420_601_topleft", planar(8, 4, STRAIGHT, 12, C420, N601, TOP_LEFT)),
    ("h8_d10_c4p_444_gbr", planar(8, 4, PREMUL, 10, C444, GBR)),
    ("h8_d12_c4p_422_709_topleft", planar(8, 4, PREMUL, 12, C422, N709, TOP_LEFT)),
    ("h8_d10_c4p_420_none_box", planar(8, 4, PREMUL, 10, C420, None, BOX)),
    ("h16_d8_c3_444_none", planar(16, 3, NONE, 8, C444, None)),
    ("h16_d8_c3_422_601_box", planar(16, 3, NONE, 8, C422, N601, BOX)),
    ("h16_d8_c3_420_2020_topleft", planar(16, 3, NONE, 8, C420, N2020, TOP_LEFT)),
    ("h16_d8_c4s_444_709", planar(16, 4, STRAIGHT, 8, C444, N709)),
    ("h16_d8_c4s_422_none_topleft", planar(16, 4, STRAIGHT, 8, C422, None, TOP_LEFT)),
    ("h16_d8_c4s_420_709_box", planar(16, 4, STRAIGHT, 8, C420, N709, BOX)),
    ("h16_d8_c4p_444_gbr", planar(16, 4, PREMUL, 8, C444, GBR)),
    ("h16_d8_c4p_422_2020_box", planar(16, 4, PREMUL, 8, C422, N2020, BOX)),
    ("h16_d8_c4p_420_601_topleft", planar(16, 4, PREMUL, 8, C420, N601, TOP_LEFT)),
    ("h16_d12_c3_444_gbr", planar(16, 3, NONE, 12, C444, GBR)),
    ("h16_d10_c3_422_709_topleft", planar(16, 3, NONE, 10, C422, N709, TOP_LEFT)),
    ("h16_d12_c3_420_none_box", planar(16, 3, NONE, 12, C420, None, BOX)),
    ("h16_d10_c4s_444_601", planar(16, 4, STRAIGHT, 10, C444, N601)),
    ("h16_d12_c4s_422_601_box", planar(16, 4, STRAIGHT, 12, C422, N601, BOX)),
    ("h16_d10_c4s_420_2020_topleft", planar(16, 4, STRAIGHT, 10, C420, N2020, TOP_LEFT)),
    ("h16_d12_c4p_444_2020", planar(16, 4, PREMUL, 12, C444, N2020)),
    ("h16_d10_c4p_422_none_box", planar(16, 4, PREMUL, 10, C422, None, BOX)),
    ("h16_d12_c4p_420_709_topleft", planar(16, 4, PREMUL, 12, C420, N709, TOP_LEFT)),
]

# DecodeYccToRgbIntBatchKernel<SampleT, XS, YS, ALPHA>: one case per (8-bit -> 8-bit or 10 / 12-bit -> 16-bit, alpha,
# chroma); full and limited range at both host depths, a 12-bit case with alpha per chroma mode
DECODE_KERNELS = [
    ("h8_d8_a0_444_601lim", ycc(8, 8, C444, NONE, cases.NCLX_601(0))),
    ("h8_d8_a0_422_709", ycc(8, 8, C422, NONE, N709)),
    ("h8_d8_a0_420_none", ycc(8, 8, C420, NONE, None)),
    ("h8_d8_a1_444_gbr", ycc(8, 8, C444, STRAIGHT, GBR)),
    ("h8_d8_a1_422_2020lim", ycc(8, 8, C422, STRAIGHT, cases.NCLX_2020_PQ(0))),
    ("h8_d8_a1_420_601", ycc(8, 8, C420, STRAIGHT, N601)),
    ("h16_d10_a0_444_gbr", ycc(16, 10, C444, NONE, GBR)),
    ("h16_d12_a0_422_none", ycc(16, 12, C422, NONE, None)),
    ("h16_d10_a0_420_709lim", ycc(16, 10, C420, NONE, cases.NCLX_709(0))),
    ("h16_d12_a1_444_601lim", ycc(16, 12, C444, STRAIGHT, cases.NCLX_601(0))),
    ("h16_d12_a1_422_709", ycc(16, 12, C422, STRAIGHT, N709)),
    ("h16_d12_a1_420_2020lim", ycc(16, 12, C420, STRAIGHT, cases.NCLX_2020_PQ(0))),
]

CHANNELS = {(3, NONE): "c3", (4, STRAIGHT): "c4s", (4, PREMUL): "c4p"}


def encode_key(desc):
    """The template arguments WithRgbIntKey (launch_keys.h) picks for `desc`: host depth, plane bytes, channels /
    premultiply, chroma."""
    return desc.host_depth, 2 if desc.image_bit_depth > 8 else 1, CHANNELS[(desc.host_channels, desc.alpha_state)], desc.chroma


def decode_key(desc):
    """The template arguments WithYccIntKey (launch_keys.h) picks for `desc`: sample type, alpha, chroma."""
    assert desc.alpha_state != PREMUL and (desc.host_depth == 8) == (desc.bit_depth == 8)
    return desc.host_depth, desc.alpha_state == STRAIGHT, desc.chroma


def matrix_name(nclx):
    return "none" if not nclx.present else {abi.MATRIX_BT601: "601", abi.MATRIX_BT709: "709", abi.MATRIX_BT2020_NCL: "2020",
                                             abi.MATRIX_GBR: "gbr"}[nclx.matrix_coefficients]


def test_instantiation_tables_are_complete():
    """Each table has exactly one case per instantiation, and spreads every runtime parameter over at least two cases."""
    encode = [encode_key(d) for _, d in ENCODE_KERNELS]
    assert sorted(encode) == sorted(itertools.product((8, 16), (1, 2), ("c3", "c4s", "c4p"), (C444, C422, C420)))
    decode = [decode_key(d) for _, d in DECODE_KERNELS]
    assert sorted(decode) == sorted(itertools.product((8, 16), (False, True), (C444, C422, C420)))
    assert len({name for name, _ in ENCODE_KERNELS + DECODE_KERNELS}) == len(ENCODE_KERNELS) + len(DECODE_KERNELS)

    def at_least_twice(values, expected):
        counts = collections.Counter(values)
        assert set(counts) == set(expected) and min(counts.values()) >= 2, counts

    at_least_twice([matrix_name(d.nclx) for _, d in ENCODE_KERNELS], ("none", "601", "709", "2020", "gbr"))
    at_least_twice([matrix_name(d.nclx) for _, d in DECODE_KERNELS], ("none", "601", "709", "2020", "gbr"))
    assert all(d.chroma == C444 for _, d in ENCODE_KERNELS + DECODE_KERNELS if matrix_name(d.nclx) == "gbr")
    at_least_twice([d.down_filter for _, d in ENCODE_KERNELS if d.chroma != C444], (BOX, TOP_LEFT))
    at_least_twice([d.image_bit_depth for _, d in ENCODE_KERNELS if d.image_bit_depth > 8], (10, 12))
    at_least_twice([d.bit_depth for _, d in DECODE_KERNELS if d.bit_depth > 8], (10, 12))
    at_least_twice([(d.host_depth, bool(d.nclx.full_range_flag) or not d.nclx.present) for _, d in DECODE_KERNELS],
                   ((8, True), (8, False), (16, True), (16, False)))
    assert {d.chroma for _, d in DECODE_KERNELS if d.bit_depth == 12 and d.alpha_state == STRAIGHT} == {C444, C422, C420}


# ---- launches: proof that the eligible images reached the batched kernels ------------------------------------------------

# widths 8 (one group), 264 and 520 (the last 256-px unit has one active lane), right strips (37, 95, 130), odd heights
# (a bottom strip in 4:2:0), and images the batch hands to direct calls: narrower than 8, or 1 row in 4:2:0
MIXED = [(264, 3), (8, 2), (37, 9), (7, 5), (130, 1), (520, 4), (95, 6), (1, 1), (64, 7)]


def ys_of(desc):
    return 1 if desc.chroma == C420 else 0


def eligible(im, ys):
    """EncodeBlockInterior / DecodeBlockInterior of the batched family on these aligned buffers: an 8-px group and a (4:2:0) row pair."""
    return im.w >= 8 and im.h >= 1 + ys


def has_edge(im, ys):
    return im.w % 8 != 0 or (ys and im.h % 2 != 0)


def fresh_output(im):
    return im.fresh_planes() if isinstance(im, Image) else im.alloc()


def expected_launches(ctx, images, ys):
    """Per chunk of eligible images one launch, one more when any of them has an edge strip; plus the direct calls of
    the others, counted by making them."""
    chosen = [im for im in images if eligible(im, ys)]
    total = sum(1 + any(has_edge(im, ys) for im in chosen[i:i + CHUNK]) for i in range(0, len(chosen), CHUNK))
    for im in images:
        if im.w and im.h and not eligible(im, ys):
            before = ctx.launch_count()
            im.direct(ctx, fresh_output(im))
            total += ctx.launch_count() - before
    return total


def assert_batched(ctx, run, images, ys):
    """The second of two runs (first-use checks happen in the first) makes exactly the launches of the chunk rule: an
    eligible image that fell back would add its own direct launches instead."""
    launches = run_counted(ctx, run)
    assert any(eligible(im, ys) for im in images)
    assert launches == expected_launches(ctx, images, ys), f"{launches} launches"


@pytest.mark.gpu
@pytest.mark.parametrize("name,desc", ENCODE_KERNELS, ids=[c[0] for c in ENCODE_KERNELS])
def test_encode_instantiation(ctx, port, name, desc):
    images = [Image(desc, w, h, f"kernels_{name}_{i}", beyond=True) for i, (w, h) in enumerate(MIXED)]
    assert_batched(ctx, lambda: run_batch(ctx, desc, images), images, ys_of(desc))
    assert_same_as_direct(ctx, images, port)


@pytest.mark.gpu
@pytest.mark.parametrize("name,desc", DECODE_KERNELS, ids=[c[0] for c in DECODE_KERNELS])
def test_decode_instantiation(ctx, checker, port, name, desc):
    images = [DecImage(desc, w, h, f"kernels_{name}_{i}", overshoot=True) for i, (w, h) in enumerate(MIXED)]
    assert_batched(ctx, lambda: run_decode_batch(ctx, desc, images), images, ys_of(desc))
    assert_decode_same_as_direct(ctx, images, pick(checker, port, True))


# ---- several passes of every loop -----------------------------------------------------------------------------------------

# Workers per CTA and CTAs per SM at most, for each batched launch: (per_cta, ctas_per_sm, source of the cap).  An
# interior worker is a warp taking one 256-px unit at a time, an edge worker a CTA taking one run of 256 sites or pixels.
BATCH_CAPS = {
    "encode_interior": (8, 16, "LaunchEncodeBatchChunk (warps; 8 per CTA, kStreamBlocksPerSm = 16)"),
    "encode_edge": (1, 16, "LaunchEncodeBatchChunk (CTAs; kStreamBlocksPerSm = 16)"),
    "decode_interior": (8, 3, "LaunchDecodeBatchChunk (warps; 8 per CTA, kYccBlocksPerSm = 3)"),
    "decode_edge": (1, 16, "LaunchDecodeBatchChunk (CTAs; kStreamBlocksPerSm = 16)"),
}


def assert_passes(kernel, units, sms):
    """The grid the launcher starts for `units` units has at most half as many workers (GridFor's cap)."""
    per_cta, ctas_per_sm, source = BATCH_CAPS[kernel]
    workers = max(1, min(-(-units // per_cta), sms * ctas_per_sm)) * per_cta
    assert units >= 2 * workers, f"{kernel}: {units} units, {workers} workers at {sms} SMs ({source})"


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def interior_units(w, h, ys):
    """BatchInteriorUnits of an image's aligned interior."""
    return -(-(w & ~7) // 256) * ((h >> 1) if ys else h)


def edge_units(w, h, chroma, decode):
    """BatchEdgeUnits of the right strip (w % 8 columns, every row) and, for 4:2:0 with an odd height, of the last row:
    runs of 256 chroma sites of a row (pair) on encode, of 256 pixels of a row on decode."""
    xs, ys = abi.chroma_shifts(chroma)
    odd_row = ys and h % 2
    if decode:
        xs = ys = 0
    units = -(-(((w % 8) + xs) >> xs) // 256) * ((h + ys) >> ys) if w % 8 else 0
    return units + (bottom_units(w, chroma, decode) if odd_row else 0)


def bottom_units(w, chroma, decode):
    """Units of the odd last 4:2:0 row: the interior's width in runs of 256 sites (encode) or pixels (decode)."""
    xs = 0 if decode else abi.chroma_shifts(chroma)[0]
    return -(-(((w & ~7) + xs) >> xs) // 256)


def run_multipass_encode(ctx, port, desc, n, w, h, seed):
    sms = sm_count()
    ys = ys_of(desc)
    assert_passes("encode_interior", n * interior_units(w, h, ys), sms)
    assert_passes("encode_edge", n * edge_units(w, h, desc.chroma, False), sms)
    images = [Image(desc, w, h, f"{seed}_{i}", beyond=True) for i in range(n)]
    assert_batched(ctx, lambda: run_batch(ctx, desc, images), images, ys)
    assert_same_as_direct(ctx, images, port, threads=os.cpu_count())


def run_multipass_decode(ctx, checker, desc, n, w, h, seed):
    sms = sm_count()
    ys = ys_of(desc)
    assert_passes("decode_interior", n * interior_units(w, h, ys), sms)
    assert_passes("decode_edge", n * edge_units(w, h, desc.chroma, True), sms)
    images = [DecImage(desc, w, h, f"{seed}_{i}", overshoot=True) for i in range(n)]
    assert_batched(ctx, lambda: run_decode_batch(ctx, desc, images), images, ys)
    assert_decode_same_as_direct(ctx, images, checker, threads=os.cpu_count())


@pytest.mark.gpu
@pytest.mark.parametrize("chroma,h", [(C444, 264), (C420, 527)], ids=["444", "420"])
def test_encode_batch_multipass(ctx, port, chroma, h):
    """64 images of 527 px: three 256-px units per interior row (the last with one active lane) and a 7-px right strip.
    The interior walk takes about 3 passes of its grid, the edge walk about 8; in 4:2:0 the odd last rows' bottom strips
    join the edge walk."""
    desc = planar(16, 4, STRAIGHT, 10, chroma, N709 if chroma == C444 else N2020)
    run_multipass_encode(ctx, port, desc, CHUNK, 527, h, f"kernels_multipass_{chroma}")


@pytest.mark.gpu
@pytest.mark.parametrize("bit_depth,host_depth,nclx", [(8, 8, N601), (10, 16, cases.NCLX_2020_PQ(0))], ids=["8to8", "10to16"])
def test_decode_batch_multipass(ctx, checker, port, bit_depth, host_depth, nclx):
    """64 images of 527 x 263, 4:2:0 with alpha: 393 interior units (row pairs) and 266 edge units (263 right-strip rows,
    3 units of the last row) per image -- about 8 passes of both grids."""
    desc = ycc(host_depth, bit_depth, C420, STRAIGHT, nclx)
    run_multipass_decode(ctx, pick(checker, port, True), desc, CHUNK, 527, 263, f"kernels_multipass_{bit_depth}")


@pytest.mark.gpu
def test_encode_bottom_strip_of_several_units(ctx, port):
    """Odd 4:2:0 heights 1289 px wide: each bottom strip is 644 chroma sites, three edge units, the last one partial."""
    w = 1289
    desc = planar(8, 4, STRAIGHT, 8, C420, N601)
    assert bottom_units(w, C420, False) == 3
    images = [Image(desc, w, h, f"kernels_bottom_{i}") for i, h in enumerate((5, 3, 9, 2))]
    assert_batched(ctx, lambda: run_batch(ctx, desc, images), images, 1)
    assert_same_as_direct(ctx, images, port, threads=os.cpu_count())


@pytest.mark.gpu
def test_decode_bottom_strip_of_several_units(ctx, checker, port):
    """Odd 4:2:0 heights 1289 px wide: each bottom strip is 1288 pixels, six edge units, the last one partial."""
    w = 1289
    desc = ycc(16, 12, C420, STRAIGHT, N709)
    assert bottom_units(w, C420, True) == 6
    images = [DecImage(desc, w, h, f"kernels_bottom_{i}", overshoot=True) for i, h in enumerate((5, 3, 9, 2))]
    assert_batched(ctx, lambda: run_decode_batch(ctx, desc, images), images, 1)
    assert_decode_same_as_direct(ctx, images, pick(checker, port, True), threads=os.cpu_count())


# ---- the first image is empty ---------------------------------------------------------------------------------------------

class Empty:
    """A 0 x 5 image: valid, converts nothing."""
    w, h = 0, 5

    def record(self):
        return (0, 5, None, [None] * abi.MAX_PLANES)


def first_call_launches(ctx, run):
    import torch
    before = ctx.launch_count()
    run()
    torch.cuda.synchronize()
    return ctx.launch_count() - before


@pytest.mark.gpu
def test_encode_batch_led_by_an_empty_image_on_a_fresh_context(port):
    """The first call of a premultiplied configuration verifies the fast premultiply (one launch) before it plans the
    batch; the first image converting nothing must not change that."""
    import avifgpu
    desc = planar(8, 4, PREMUL, 10, C422, N709, BOX)
    with avifgpu.Context(0) as fresh:
        images = [Image(desc, w, h, f"kernels_empty_first_{i}") for i, (w, h) in enumerate(MIXED)]
        launches = first_call_launches(fresh, lambda: run_batch(fresh, desc, [Empty()] + images))
        assert launches == 1 + expected_launches(fresh, images, 0)
        assert_same_as_direct(fresh, images, port)


@pytest.mark.gpu
def test_decode_batch_led_by_an_empty_image_on_a_fresh_context(checker, port):
    """The first decode call of a YCbCr configuration verifies the fast green-channel division (one launch) with the
    first image's parameters; a first image that converts nothing must still carry the description's matrix and range."""
    import avifgpu
    desc = ycc(16, 12, C420, STRAIGHT, cases.NCLX_2020_PQ(0))
    with avifgpu.Context(0) as fresh:
        images = [DecImage(desc, w, h, f"kernels_empty_first_{i}", overshoot=True) for i, (w, h) in enumerate(MIXED)]
        launches = first_call_launches(fresh, lambda: run_decode_batch(fresh, desc, [Empty()] + images))
        assert launches == 1 + expected_launches(fresh, images, 1)
        assert_decode_same_as_direct(fresh, images, pick(checker, port, True))
