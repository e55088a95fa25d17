"""Batched HDR decodes: 10 / 12-bit YCbCr into 32-bit float hosts (PQ, HLG with and without the OOTF, SMPTE 428) through
both batch APIs, run by DecodeYccToRgbF32BatchKernel (kernels_batch.cu) and, for the windows, by DecodeBatchKernel's
float-host instantiation.

  * KERNELS holds one case per instantiation of the batched kernel: 3 chroma modes x (PQ with the verified division, PQ
    with the IEEE division, HLG, SMPTE 428) x alpha = 24.  test_kernel_table_is_complete checks it without a GPU, and that
    matrices, bit depths, full / limited range and OOTF on / off each appear in at least two cases;
  * every case runs a mix of sizes (widths 4, 127, 128, 129, 260, right strips, odd 4:2:0 heights) and of images the
    tuned kernel does not take (width 3, one 4:2:0 row, misaligned rows or planes, unequal Cb / Cr strides) under the
    host-described call, whose launch count proves the batched route, and under the device-described one;
  * the IEEE-division PQ kernel is what a call captured before the PQ division is verified runs, so those cases capture
    the call on a fresh context and replay it;
  * multi-pass batches make both grids walk at least twice, rejected images keep their outputs, one captured call is
    replayed on 1, 64 and 256 images at new addresses, and an HLG capture made before the divisions are verified sends
    every image to the edge kernel with the same bits.

Every image equals a direct avifgpu_decode_rows_device call bit for bit and the compiled reference in float bits, codes
above the maximum included; the sentinel in the row padding must survive."""
import collections
import itertools
import os

import pytest

from avifgpu import abi
from gpu_harness import ctx  # noqa: F401
from gpu_harness import (DECODE_FAULTS, DecodeImage, Empty, Indirect, assert_decode_same_as_direct, assert_passes, captured, capture_and_replay,
                         chunk_launches, direct_launches, host_or_device, launches_of, padded, pick, rejected_records, replay_sets,
                         run_decode_batch, sm_count)

C444, C422, C420 = abi.CHROMA_444, abi.CHROMA_422, abi.CHROMA_420
NONE, STRAIGHT = abi.ALPHA_NONE, abi.ALPHA_STRAIGHT
TRANSFERS = {"pq": abi.TRANSFER_CHAR_PQ, "pq_ieee": abi.TRANSFER_CHAR_PQ, "hlg": abi.TRANSFER_CHAR_HLG, "428": abi.TRANSFER_CHAR_SMPTE428}
CHROMA_NAMES = {C444: "444", C422: "422", C420: "420"}
MATRICES = {"601": abi.MATRIX_BT601, "709": abi.MATRIX_BT709, "2020": abi.MATRIX_BT2020_NCL}


def hdr(variant, chroma, alpha, depth, matrix, full, ootf=1):
    nclx = abi.Nclx(1, abi.PRIMARIES_BT2020, TRANSFERS[variant], MATRICES[matrix], full)
    return abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, chroma, depth, alpha, 32, nclx, hlg_apply_ootf=ootf, pq_peak_nits=1000)


def kernel_cases():
    """(name, variant, desc): the runtime parameters rotate over the 24 instantiations."""
    out = []
    for i, (chroma, variant, alpha) in enumerate(itertools.product((C444, C422, C420), ("pq", "pq_ieee", "hlg", "428"), (NONE, STRAIGHT))):
        depth, matrix, full, ootf = (10, 12)[i % 2], ("601", "709", "2020")[i % 3], (i // 2) % 2, (i // 3) % 2
        name = f"{CHROMA_NAMES[chroma]}_{variant}_a{int(alpha == STRAIGHT)}_d{depth}_{matrix}{'full' if full else 'lim'}"
        if variant == "hlg":
            name += "_ootf" if ootf else "_noootf"
        out.append((name, variant, hdr(variant, chroma, alpha, depth, matrix, full, ootf)))
    return out


KERNELS = kernel_cases()


def test_kernel_table_is_complete():
    keys = [(d.chroma, v, d.alpha_state) for _, v, d in KERNELS]
    assert sorted(keys) == sorted(itertools.product((C444, C422, C420), TRANSFERS, (NONE, STRAIGHT)))
    assert len({name for name, _, _ in KERNELS}) == 24

    def at_least_twice(values, expected):
        counts = collections.Counter(values)
        assert set(counts) == set(expected) and min(counts.values()) >= 2, counts

    at_least_twice([d.nclx.matrix_coefficients for _, _, d in KERNELS], MATRICES.values())
    at_least_twice([d.bit_depth for _, _, d in KERNELS], (10, 12))
    at_least_twice([d.nclx.full_range_flag for _, _, d in KERNELS], (0, 1))
    at_least_twice([d.hlg_apply_ootf for _, v, d in KERNELS if v == "hlg"], (0, 1))


# ---- images -------------------------------------------------------------------------------------------------------------

# widths 4 (one lane), 127 / 129 / 130 (right strips), 128 (one tile), 260 (a tile with one active lane); odd heights (a
# bottom strip in 4:2:0); width 3, 1 x 1 and a 4:2:0 image one row high are not the tuned kernel's
MIXED = [(4, 3), (127, 5), (128, 2), (129, 7), (260, 4), (130, 1), (3, 6), (1, 1), (64, 9)]


def unequal_chroma_strides(im):
    """Gives the Cr plane 64 more bytes of row stride than Cb."""
    import torch
    cr = im.planes[2]
    backing = torch.zeros((max(cr.shape[0], 1), padded(cr.shape[1]) + 64), dtype=torch.uint8, device="cuda")
    im.planes[2] = backing[:cr.shape[0], :cr.shape[1]]
    im.planes[2].copy_(cr)
    im.unequal = True
    return im


def mix(desc, seed):
    images = [DecodeImage(desc, w, h, f"{seed}_{i}", overshoot=True) for i, (w, h) in enumerate(MIXED)]
    images.append(DecodeImage(desc, 64, 7, f"{seed}_rows", overshoot=True, rows_offset=4))
    images.append(DecodeImage(desc, 68, 6, f"{seed}_planes", overshoot=True, planes_misalign=2))
    images.append(unequal_chroma_strides(DecodeImage(desc, 72, 8, f"{seed}_strides", overshoot=True)))
    return images


def ys_of(desc):
    return 1 if desc.chroma == C420 else 0


def eligible(im):
    """DecodeYccF32BlockInterior on these buffers: 4-pixel groups, a (4:2:0) row pair, aligned, equal Cb / Cr strides."""
    aligned = im.rows.data_ptr() % 16 == 0 and all(p is None or p.data_ptr() % 8 == 0 for p in im.planes)
    return im.w >= 4 and im.h >= 1 + ys_of(im.desc) and aligned and not getattr(im, "unequal", False)


def has_edge(im):
    return im.w % 4 != 0 or (ys_of(im.desc) and im.h % 2 != 0)


# ---- 1. every instantiation, host-described and device-described ------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name,variant,desc", KERNELS, ids=[c[0] for c in KERNELS])
def test_host_described_instantiation(checker, port, name, variant, desc):
    import avifgpu
    images = mix(desc, f"f32_host_{name}")
    fallbacks = [im for im in images if im.w and im.h and not eligible(im)]
    assert len(fallbacks) >= 5 and any(has_edge(im) for im in images if eligible(im))
    with avifgpu.Context(0) as fresh:
        if variant == "pq_ieee":
            # before the PQ division is verified: the IEEE-division kernel; every fallback is one generic launch
            launches = captured(fresh, lambda stream: run_decode_batch(fresh, desc, images, stream))
            assert launches == chunk_launches(images, eligible, has_edge) + len(fallbacks)
        else:
            fresh.prepare_decode(desc)
            # into the image's own rows: their alignment is part of its route
            direct = direct_launches(fresh, fallbacks, into=lambda im: im.rows)
            assert launches_of(fresh, lambda: run_decode_batch(fresh, desc, images)) == chunk_launches(images, eligible, has_edge) + direct
        assert_decode_same_as_direct(fresh, images, pick(checker, port, True))


@pytest.mark.gpu
@pytest.mark.parametrize("name,variant,desc", KERNELS, ids=[c[0] for c in KERNELS])
def test_device_described_instantiation(checker, port, name, variant, desc):
    import avifgpu
    images = mix(desc, f"f32_indirect_{name}")
    batch = Indirect(16)
    batch.load(images[:5] + [Empty()] + images[5:])
    with avifgpu.Context(0) as fresh:
        if variant == "pq_ieee":
            assert captured(fresh, lambda stream: batch.decode(fresh, desc, stream)) == 3
        else:
            fresh.prepare_decode(desc)
            assert launches_of(fresh, lambda: batch.decode(fresh, desc)) == 3
        assert (batch.statuses()[:len(images) + 1] == 0).all()
        assert_decode_same_as_direct(fresh, images, pick(checker, port, True))


# ---- 2. several passes of both grids -------------------------------------------------------------------------------------------

def interior_units(w, h, ys):
    """BatchInteriorUnits of an image's aligned interior with the 128-pixel unit."""
    return -(-(w & ~3) // 128) * ((h >> 1) if ys else h)


def edge_units(w, h, ys):
    """Runs of 256 pixels of one row: the right strip's rows, and the odd last 4:2:0 row's interior width."""
    right = h if w % 4 else 0
    return right + (-(-(w & ~3) // 256) if ys and h % 2 else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("api", ["host", "device"])
def test_multipass(ctx, checker, port, api):
    """64 images of 515 x 263, 4:2:0 with alpha, PQ: 524 interior units (4 tiles x 131 row pairs) and 265 edge units per
    image.  The interior grid has kDecodeBlocksPerSm = 2 CTAs of 8 warps per SM, the edge grid 16 one-CTA workers per SM
    (kernels_batch.cu): both walk their units at least twice."""
    desc = hdr("pq", C420, STRAIGHT, 12, "2020", 0)
    n, w, h = 64, 515, 263
    sms = sm_count(ctx)
    assert_passes("ycc_f32_interior", n * interior_units(w, h, 1), sms)
    assert_passes("decode_edge", n * edge_units(w, h, 1), sms)
    images = [DecodeImage(desc, w, h, f"f32_multipass_{api}_{i}", overshoot=True) for i in range(n)]
    ctx.prepare_decode(desc)
    host_or_device(ctx, desc, "decode", api, images,
                   lambda done: assert_decode_same_as_direct(ctx, done, pick(checker, port, True), threads=os.cpu_count()))


# ---- 3. device-described specifics ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_rejected_images_keep_their_outputs(ctx, checker, port):
    desc = hdr("hlg", C422, STRAIGHT, 10, "709", 1)
    images = [DecodeImage(desc, w, h, f"f32_bad_{i}") for i, (w, h) in enumerate([(64, 16), (37, 9), (64, 4), (8, 2), (130, 5), (7, 5)])]
    ctx.prepare_decode(desc)
    rejected_records(ctx, desc, "decode", images, DECODE_FAULTS, lambda good: assert_decode_same_as_direct(ctx, good, pick(checker, port, True)))


def replay(ctx, desc, tag, reference, prepare):
    """One capture of a device-described call, replayed on 1, 64 and 256 images at new addresses."""
    sets = replay_sets(lambda w, h, seed: DecodeImage(desc, w, h, seed, overshoot=True), tag, (136, 34), MIXED)
    capture_and_replay(ctx, desc, "decode", DecodeImage(desc, 64, 16, f"{tag}_capture"), sets,
                       lambda images: assert_decode_same_as_direct(ctx, images, reference, threads=os.cpu_count()),
                       (lambda: ctx.prepare_decode(desc)) if prepare else None)


@pytest.mark.gpu
def test_captured_call_replays_new_image_sets(checker, port):
    import avifgpu
    desc = hdr("hlg", C420, NONE, 10, "2020", 1)
    with avifgpu.Context(0) as fresh:
        replay(fresh, desc, "f32_replay", pick(checker, port, True), prepare=True)


@pytest.mark.gpu
def test_unprepared_hlg_capture_runs_the_edge_kernel(checker, port):
    """Captured before the HLG divisions are verified, the description has no tuned interior: every image is one whole-image
    window of the edge kernel (the generic kernel's code, what a direct call of it would run then) -- the same bits."""
    import avifgpu
    desc = hdr("hlg", C422, STRAIGHT, 12, "709", 0)
    with avifgpu.Context(0) as fresh:
        replay(fresh, desc, "f32_unprepared", pick(checker, port, True), prepare=False)


@pytest.mark.gpu
def test_premultiplied_float_decode_stays_unsupported(ctx):
    import avifgpu
    desc = hdr("pq", C420, abi.ALPHA_PREMULTIPLIED, 10, "2020", 1)
    batch = Indirect(4)
    before = ctx.launch_count()
    with pytest.raises(avifgpu.AvifGpuError) as info:
        batch.decode(ctx, desc)
    assert info.value.status == abi.ERR_UNSUPPORTED and ctx.launch_count() == before
