"""The planar and project-defined encodes on an H100, held to the independent model of encode_spec.py rather than to the
C restatement: the tuned encode kernels (flat, RGBA, clip, integer planar, Gray16 table), both batch APIs, the generic
kernel on the HLG save path, the row matrix and unaligned buffers, and the two full-size configurations.

Every case runs on random rows and on extreme_rows(), whose saturated chroma sites reach the tuned kernels' one packed
min on chroma and the luma path that has no upper clamp.  Shapes are 259 x 37: a right strip for every tuned kernel
(groups of 4 or 8 pixels) and an odd last row, so the launch count of a second call proves the route -- the tuned
launcher makes 1 + strips launches, the generic kernel 1.  Float hosts run on `gpu` (step tables: the tuned kernels)
and on `gpu_exact` (no tables: the generic kernel, except for the clip kernel, which needs none)."""
import numpy as np
import pytest

import cases
import encode_spec
from avifgpu import abi
from gpu_harness import ctx  # noqa: F401
from gpu_harness import (ENCODE_KERNELS, MIXED, SENTINEL, EncodeImage, Indirect, Padded, assert_batched, launches_of, planes_struct, run_batch,
                         run_counted, strips, whole, ys_of)

pytestmark = pytest.mark.gpu

W, H = 259, 37
BOX, TOP_LEFT = abi.DOWN_FILTER_BOX, abi.DOWN_FILTER_TOP_LEFT
C444, C422, C420 = abi.CHROMA_444, abi.CHROMA_422, abi.CHROMA_420
NONE, STRAIGHT, PREMUL = abi.ALPHA_NONE, abi.ALPHA_STRAIGHT, abi.ALPHA_PREMULTIPLIED
PQ, SMPTE428, CLIP, HLG = abi.TRANSFER_PQ, abi.TRANSFER_SMPTE428, abi.TRANSFER_CLIP, abi.TRANSFER_HLG
MATRICES = {"none": lambda: None, "709": cases.NCLX_709, "2020": cases.NCLX_2020_PQ, "derived": cases.NCLX_DERIVED}


@pytest.fixture(scope="module")
def ref():
    checker = encode_spec.load()
    if checker is None:
        pytest.fail("oracle/_ref/libavifref.so is not loaded: the encode model is built on the compiled reference -- build it "
                    "where the reference tree is mounted (make -C oracle); it ships with the tree")
    return checker


def inputs(desc, seed):
    """The seeded random rows of cases.py and extreme_rows(), both W x H."""
    rng = cases.rng_for(seed)
    if desc.host_depth == 32:
        rows = cases.float_host_rows(rng, desc.height, desc.width, desc.host_channels)
    else:
        rows = cases.int_host_rows(rng, desc.height, desc.width, desc.host_channels, desc.host_depth, beyond=True)
    return [("random", rows), ("extreme", encode_spec.extreme_rows(desc, desc.width, desc.height, seed))]


def encode_counted(ctx, desc, rows, launches, misalign=0):
    """Converts host `rows` through avifgpu_encode_rows_device on 256-byte-strided buffers (the source `misalign` bytes
    off), asserts the second call's launch count and that the row padding kept its sentinel; returns the planes."""
    import torch
    dev = torch.device("cuda", ctx.device)
    src = Padded(dev, rows.shape[0], rows.shape[1] + (misalign and 16 // rows.itemsize), rows.dtype)
    src.bytes[:, misalign:misalign + rows.shape[1] * rows.itemsize] = torch.from_numpy(
        np.ascontiguousarray(rows).view(np.uint8).reshape(rows.shape[0], -1)).to(dev)
    out = [None if s is None else Padded(dev, s[0], s[1], abi.code_dtype(desc.image_bit_depth)) for s in abi.encode_plane_shapes(desc)]
    planes = planes_struct(out)
    delta = run_counted(ctx, lambda: ctx.encode_device(desc, src.ptr() + misalign, src.stride, planes))
    assert delta == launches, f"{delta} launches, expected {launches}"
    for k, p in enumerate(out):
        assert p is None or p.padding_intact(), f"plane {k}: wrote into the row padding"
    return [None if p is None else p.host() for p in out]


def check_all_inputs(ref, contexts, desc, seed, group=None):
    """Every (context, input) pair against the model; `contexts` maps a context to whether the tuned launcher (with
    pixel groups of `group`) serves it there."""
    ys = desc.layout == abi.LAYOUT_PLANAR_YCBCR and desc.chroma == C420
    for ctx, tuned in contexts:
        launches = strips(desc.width, group, odd_rows=ys) if tuned else 1
        for label, rows in inputs(desc, seed):
            got = encode_counted(ctx, desc, rows, launches)
            encode_spec.assert_matches(ref, desc, rows, got, f"{label} rows, {'tuned' if tuned else 'generic'} route")


def planar_float(channels, alpha, depth, transfer, chroma, down, nclx, peak=None):
    return abi.EncodeDesc(W, H, 32, channels, alpha, depth, transfer, peak or (80 if depth == 12 else 1000), abi.LAYOUT_PLANAR_YCBCR,
                          chroma, down, abi.GRAY16_LUT, nclx)


# ---- EncodeRgbF32FlatKernel: planar RGB32f with a curve -----------------------------------------------------------------------

FLAT = [(transfer, depth, chroma, down, m) for transfer in (PQ, SMPTE428) for depth in (10, 12) for chroma in (C444, C422, C420)
        for down in ((BOX,) if chroma == C444 else (BOX, TOP_LEFT)) for m in MATRICES]


@pytest.mark.parametrize("transfer,depth,chroma,down,matrix", FLAT, ids=[f"t{t}_d{d}_ch{c}_f{f}_{m}" for t, d, c, f, m in FLAT])
def test_flat_kernel(gpu, gpu_exact, ref, transfer, depth, chroma, down, matrix):
    desc = planar_float(3, NONE, depth, transfer, chroma, down, MATRICES[matrix]())
    check_all_inputs(ref, ((gpu, True), (gpu_exact, False)), desc, f"spec_flat_{transfer}_{depth}_{chroma}_{down}_{matrix}", 4)


# ---- EncodeRgbaF32FlatKernel: straight and premultiplied alpha --------------------------------------------------------------------

RGBA = [(alpha, chroma, transfer, depth, m) for alpha in (STRAIGHT, PREMUL) for chroma, m in ((C444, "709"), (C422, "2020"), (C420, "derived"))
        for transfer, depth in ((PQ, 12), (SMPTE428, 10))]


@pytest.mark.parametrize("alpha,chroma,transfer,depth,matrix", RGBA, ids=[f"a{a}_ch{c}_t{t}_d{d}_{m}" for a, c, t, d, m in RGBA])
def test_rgba_kernel(gpu, gpu_exact, ref, alpha, chroma, transfer, depth, matrix):
    desc = planar_float(4, alpha, depth, transfer, chroma, BOX, MATRICES[matrix]())
    check_all_inputs(ref, ((gpu, True), (gpu_exact, False)), desc, f"spec_rgba_{alpha}_{chroma}_{transfer}_{depth}", 4)


# ---- EncodeRgbF32ClipKernel: no curve (needs no table, so the exact context takes it too) ------------------------------------------

CLIP_CASES = [(depth, chroma, down, m) for (depth, chroma, down), m in zip(
    ((10, C444, BOX), (12, C444, BOX), (10, C422, TOP_LEFT), (12, C422, BOX), (10, C420, BOX), (12, C420, TOP_LEFT)),
    ("2020", "none", "709", "derived", "2020", "709"))]


@pytest.mark.parametrize("depth,chroma,down,matrix", CLIP_CASES, ids=[f"d{d}_ch{c}_f{f}_{m}" for d, c, f, m in CLIP_CASES])
def test_clip_kernel(gpu, gpu_exact, ref, depth, chroma, down, matrix):
    desc = planar_float(3, NONE, depth, CLIP, chroma, down, MATRICES[matrix]())
    check_all_inputs(ref, ((gpu, True), (gpu_exact, True)), desc, f"spec_clip_{depth}_{chroma}_{down}_{matrix}", 4)


# ---- EncodeRgbIntPlanarKernel: one case per instantiation key -------------------------------------------------------------------

@pytest.mark.parametrize("name,desc", ENCODE_KERNELS, ids=[c[0] for c in ENCODE_KERNELS])
def test_int_planar_kernel(gpu, ref, name, desc):
    """Host depth, plane bytes, channels / premultiply and chroma as gpu_harness.ENCODE_KERNELS spreads them,
    with its matrices, down-filters and 10 / 12-bit planes; 16-bit random rows carry samples above 32768, extreme rows
    65535."""
    check_all_inputs(ref, ((gpu, True),), desc.copy(width=W, height=H), f"spec_int_{name}", 8)


# ---- the batched integer kernels, both APIs -------------------------------------------------------------------------------------

BATCH_SIZES = MIXED + [(W, H), (520, 9), (16, 2)]


def assert_images_match(ref, images):
    for im in images:
        if im.w and im.h:
            got = [None if p is None else p.cpu().numpy().view(abi.code_dtype(im.desc.image_bit_depth)) for p in im.planes]
            encode_spec.assert_matches(ref, im.desc, im.host, got, f"{im.w} x {im.h} image")
            for p in im.planes:
                if p is not None:
                    assert (whole(p)[:, p.shape[1]:] == SENTINEL).all()


@pytest.mark.parametrize("api", ["device", "indirect"])
@pytest.mark.parametrize("name,desc", ENCODE_KERNELS, ids=[c[0] for c in ENCODE_KERNELS])
def test_batch_kernels(ctx, ref, name, desc, api):
    """Batches of extreme images of several sizes: aligned interiors, right strips, odd 4:2:0 heights, and images too
    small for the interior kernel."""
    # host rows: extreme_rows() of f"spec_batch_{name}_{i}_{w}x{h}"
    images = [EncodeImage(desc, w, h, f"{name}_{i}_{w}x{h}", prefix="spec_batch_", extreme=True) for i, (w, h) in enumerate(BATCH_SIZES)]
    if api == "device":
        assert_batched(ctx, lambda: run_batch(ctx, desc, images), images, ys_of(desc))
    else:
        batch = Indirect(len(images))
        batch.load(images)
        batch.encode(ctx, desc)  # the first call of a premultiplied description also makes the premultiply check
        assert launches_of(ctx, lambda: batch.encode(ctx, desc)) == 3
        assert (batch.statuses() == 0).all()
    assert_images_match(ref, images)


# ---- EncodeGray16LutKernel: Gray16 -> SMPTE 428 ------------------------------------------------------------------------------------

@pytest.mark.parametrize("depth", [10, 12])
def test_gray16_smpte428_every_input(gpu, ref, depth):
    """All 65536 samples, 259 wide: the table kernel takes 256 columns, the generic kernel the 3-column right strip."""
    h = -(-65536 // W)
    rows = (np.arange(W * h) % 65536).astype(np.uint16).reshape(h, W)
    rows[:, -3:] = rows[::-1, :3]  # the right strip sees the whole range too
    desc = abi.EncodeDesc(W, h, 16, 1, NONE, depth, gray16_curve=abi.GRAY16_SMPTE428)
    got = encode_counted(gpu, desc, rows, strips(W, 8))
    encode_spec.assert_matches(ref, desc, rows, got)


# ---- the generic kernel: HLG save path, row matrix, unaligned buffers --------------------------------------------------------------

HLG_CASES = [(channels, alpha, extension, layout) for channels, alpha in ((3, NONE), (4, STRAIGHT), (4, PREMUL))
             for extension in (abi.HLG_OETF, abi.HLG_INVERSE_OOTF_THEN_OETF) for layout in (abi.LAYOUT_REFERENCE, abi.LAYOUT_PLANAR_YCBCR)]


@pytest.mark.parametrize("channels,alpha,extension,layout", HLG_CASES, ids=[f"c{c}_a{a}_x{x}_l{l}" for c, a, x, l in HLG_CASES])
def test_hlg_save(gpu, gpu_exact, ref, channels, alpha, extension, layout):
    depth = 10 if extension == abi.HLG_OETF else 12
    desc = abi.EncodeDesc(W, H, 32, channels, alpha, depth, HLG, 80, layout, C420, BOX, abi.GRAY16_LUT, cases.NCLX_2020_HLG(),
                          hlg_extension=extension, hlg_display_gamma=1.2, hlg_peak_nits=1000)
    check_all_inputs(ref, ((gpu, False), (gpu_exact, False)), desc, f"spec_hlg_{channels}_{alpha}_{extension}_{layout}")


ROW_MATRIX = [(3, NONE, abi.LAYOUT_PLANAR_YCBCR, PQ), (4, PREMUL, abi.LAYOUT_PLANAR_YCBCR, PQ), (4, STRAIGHT, abi.LAYOUT_REFERENCE, SMPTE428),
              (3, NONE, abi.LAYOUT_REFERENCE, CLIP)]


@pytest.mark.parametrize("channels,alpha,layout,transfer", ROW_MATRIX, ids=[f"c{c}_a{a}_l{l}_t{t}" for c, a, l, t in ROW_MATRIX])
def test_row_matrix(gpu, gpu_exact, ref, channels, alpha, layout, transfer):
    desc = abi.EncodeDesc(W, H, 32, channels, alpha, 12, transfer, 1000, layout, C420, BOX, abi.GRAY16_LUT, cases.NCLX_2020_PQ())
    desc.row_matrix_enabled = 1
    desc.row_matrix = type(desc.row_matrix)(*cases.ROW_MATRIX_709_TO_2020)
    check_all_inputs(ref, ((gpu, False), (gpu_exact, False)), desc, f"spec_rowmatrix_{channels}_{alpha}_{layout}_{transfer}")


@pytest.mark.parametrize("kind", ["float", "int"])
def test_planar_on_unaligned_rows(gpu, ref, kind):
    """A source 4 bytes off its alignment: no tuned kernel may read it, the generic kernel converts the whole image."""
    if kind == "float":
        desc = planar_float(4, PREMUL, 12, PQ, C420, BOX, cases.NCLX_2020_PQ())
    else:
        desc = abi.EncodeDesc(W, H, 16, 3, NONE, 10, CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, C422, BOX, abi.GRAY16_LUT, cases.NCLX_709())
    for label, rows in inputs(desc, f"spec_unaligned_{kind}"):
        got = encode_counted(gpu, desc, rows, 1, misalign=4)
        encode_spec.assert_matches(ref, desc, rows, got, label)


# ---- full size: BASELINE configs 2 and 4, extreme bands at the top, middle and bottom --------------------------------------------

BAND = 64


def banded_frame(desc, block, seed):
    """The frame tiled from `block` (random rows), with 32 extreme rows at the top, from the middle and at the very
    bottom; returns it and the three 64-row bands the test compares."""
    h = desc.height
    rows = np.tile(block, (-(-h // block.shape[0]), 1))[:h]
    middle = (h // 2) & ~1
    for y0 in (0, middle, h - 32):
        rows[y0:y0 + 32] = encode_spec.extreme_rows(desc.copy(height=32), desc.width, 32, f"{seed}_{y0}")
    return rows, (0, middle - 32, h - BAND)


def check_bands(ref, desc, rows, got, bands):
    _, ys = abi.chroma_shifts(desc.chroma)
    for y0 in bands:
        band = desc.copy(height=BAND)
        planes = [None if p is None else p[(y0 >> ys if k in (1, 2) else y0):][:(BAND >> ys if k in (1, 2) else BAND)]
                  for k, p in enumerate(got)]
        encode_spec.assert_matches(ref, band, rows[y0:y0 + BAND], planes, f"rows {y0}..{y0 + BAND}")


def test_config2_8k_rgb32f_12bit_pq_420(gpu, ref):
    desc = abi.EncodeDesc(7680, 4320, 32, 3, NONE, 12, PQ, 80, abi.LAYOUT_PLANAR_YCBCR, C420, BOX, abi.GRAY16_LUT, cases.NCLX_2020_PQ())
    block = cases.float_host_rows(cases.rng_for("spec_config2"), 128, desc.width, 3)
    rows, bands = banded_frame(desc, block, "spec_config2")
    check_bands(ref, desc, rows, gpu.encode(desc, rows), bands)


def test_config4_16k_rgba16_10bit_422_alpha(gpu, ref):
    desc = abi.EncodeDesc(16384, 16384, 16, 4, STRAIGHT, 10, CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, C422, BOX, abi.GRAY16_LUT, None)
    block = cases.int_host_rows(cases.rng_for("spec_config4"), 64, desc.width, 4, 16, beyond=True)
    rows, bands = banded_frame(desc, block, "spec_config4")
    check_bands(ref, desc, rows, gpu.encode(desc, rows), bands)
