"""Batched planar-RGB (lossless) decodes through both batch APIs: 8-bit planes into 8-bit hosts and 10 / 12-bit planes into
16-bit hosts, run by DecodePlanarRgbIntBatchKernel, and 10 / 12-bit planes with PQ, HLG (with and without the OOTF) or
SMPTE 428 into 32-bit hosts, run by TableDecodeF32BatchKernel (kernels_batch.cu); right strips and images the tuned
kernels do not take run DecodeBatchKernel.

  * KERNELS holds one case per instantiation of the two batched kernels (host depth x alpha, and for 32-bit hosts alpha,
    with the curves as runtime values spread over the cases); each runs under the host-described call, whose launch count
    proves the batched route (1 + (edges ? 1 : 0) per chunk, plus the direct calls of the other images), and under the
    device-described one (always 3 launches);
  * the images mix widths 8, 9, 255, 256, 257, 7 and 1 x 1, one-row images, rows misaligned by 4 or 8 bytes (RGB8 stores
    8-byte words, so 8 keeps it tuned), misaligned planes and codes above the maximum;
  * multi-pass batches make the interior and edge grids walk at least twice, rejected images keep their outputs, one
    captured call is replayed on 1, 64 and 256 images at new addresses, premultiplied alpha keeps its direct calls, and the
    device-described call still refuses monochrome and premultiplied planar RGB without a launch.

Every image equals a direct avifgpu_decode_rows_device call bit for bit (the row padding's sentinel included) and the
compiled reference.  For 32-bit hosts the reference indexes its 2^depth table with the raw code, so codes above the
maximum are out of its contract: those images are held to the direct call only (test_gpu_multipass.table_planes)."""
import os

import pytest

import cases
from avifgpu import abi
from gpu_harness import ctx  # noqa: F401
from gpu_harness import (DECODE_FAULTS, DecodeImage, Empty, Indirect, assert_decode_same_as_direct, assert_passes, capture_and_replay, captured,
                         chunk_launches, direct_launches, host_or_device, launches_of, pick, rejected_records, replay_sets, rgb32_nclx,
                         run_decode_batch, sm_count)

NONE, STRAIGHT, PREMUL = abi.ALPHA_NONE, abi.ALPHA_STRAIGHT, abi.ALPHA_PREMULTIPLIED


def rgb(host_depth, depth, alpha, curve=None, **kwargs):
    nclx = cases.NCLX_GBR() if host_depth != 32 else rgb32_nclx(curve)
    return abi.DecodeDesc(0, 0, abi.COLORSPACE_RGB, abi.CHROMA_444, depth, alpha, host_depth, nclx, **kwargs)


# (name, desc): DecodePlanarRgbIntBatchKernel<uint8_t / uint16_t, 3 / 4>, TableDecodeF32BatchKernel<0 / 1> twice each
KERNELS = [
    ("h8_rgb", rgb(8, 8, NONE)),
    ("h8_rgba", rgb(8, 8, STRAIGHT)),
    ("h16_rgb_d10", rgb(16, 10, NONE)),
    ("h16_rgba_d12", rgb(16, 12, STRAIGHT)),
    ("f32_rgb_pq_d12", rgb(32, 12, NONE, "pq", pq_peak_nits=1000)),
    ("f32_rgb_428_d10", rgb(32, 10, NONE, "428")),
    ("f32_rgba_hlg_ootf_d10", rgb(32, 10, STRAIGHT, "hlg", hlg_apply_ootf=1)),
    ("f32_rgba_hlg_d12", rgb(32, 12, STRAIGHT, "hlg", hlg_apply_ootf=0)),
]


def test_kernel_table_is_complete():
    keys = {(d.host_depth, d.alpha_state) for _, d in KERNELS}
    assert keys == {(h, a) for h in (8, 16, 32) for a in (NONE, STRAIGHT)}
    curves = {d.nclx.transfer_characteristics for _, d in KERNELS if d.host_depth == 32}
    assert curves == {abi.TRANSFER_CHAR_PQ, abi.TRANSFER_CHAR_HLG, abi.TRANSFER_CHAR_SMPTE428}


# ---- images -------------------------------------------------------------------------------------------------------------

# widths 8 (one lane), 9 / 255 / 257 (right strips), 256 (one unit), 264 (a unit with one active lane), 520; width 7 and 1 x 1
# are not the tuned kernels'
MIXED = [(8, 3), (9, 5), (255, 2), (256, 4), (257, 3), (264, 1), (520, 2), (7, 6), (1, 1)]


def overshoot_ok(desc):
    return desc.host_depth != 32


def mix(desc, seed):
    over = overshoot_ok(desc)
    images = [DecodeImage(desc, w, h, f"{seed}_{i}", overshoot=over) for i, (w, h) in enumerate(MIXED)]
    images.append(DecodeImage(desc, 64, 7, f"{seed}_rows4", overshoot=over, rows_offset=4))
    images.append(DecodeImage(desc, 72, 5, f"{seed}_rows8", overshoot=over, rows_offset=8))
    images.append(DecodeImage(desc, 68, 6, f"{seed}_planes", overshoot=over, planes_misalign=2))
    if not over:
        over_image = DecodeImage(desc, 136, 3, f"{seed}_over", overshoot=True)
        over_image.direct_only = True
        images.append(over_image)
    return images


def eligible(im):
    """DecodePlanarRgbBlockInterior on these buffers: 8-pixel groups, planes on 8 samples, rows on the kernel's stores."""
    d = im.desc
    plane_align = 16 if d.bit_depth > 8 else 8
    row_align = 8 if d.host_depth == 8 and d.alpha_state == NONE else 16
    aligned = im.rows.data_ptr() % row_align == 0 and all(p is None or p.data_ptr() % plane_align == 0 for p in im.planes)
    return im.w >= 8 and im.h >= 1 and aligned and d.alpha_state != PREMUL


def has_edge(im):
    return im.w % 8 != 0


# ---- 1. every instantiation, host-described and device-described ------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name,desc", KERNELS, ids=[c[0] for c in KERNELS])
def test_host_described_instantiation(ctx, checker, port, name, desc):
    images = mix(desc, f"rgb_host_{name}")
    fallbacks = [im for im in images if im.w and im.h and not eligible(im)]
    assert len(fallbacks) >= 4 and any(has_edge(im) for im in images if eligible(im))
    if desc.host_depth == 8 and desc.alpha_state == NONE:
        assert eligible(images[len(MIXED) + 1])  # RGB8 rows 8 bytes off 16 stay tuned
    ctx.prepare_decode(desc)
    # into the image's own rows: their alignment is part of its route
    direct = direct_launches(ctx, fallbacks, into=lambda im: im.rows)
    assert launches_of(ctx, lambda: run_decode_batch(ctx, desc, images)) == chunk_launches(images, eligible, has_edge) + direct
    assert_decode_same_as_direct(ctx, images, pick(checker, port, True))


@pytest.mark.gpu
@pytest.mark.parametrize("name,desc", KERNELS, ids=[c[0] for c in KERNELS])
def test_device_described_instantiation(ctx, checker, port, name, desc):
    images = mix(desc, f"rgb_indirect_{name}")
    batch = Indirect(16)
    batch.load(images[:5] + [Empty()] + images[5:])
    ctx.prepare_decode(desc)
    assert launches_of(ctx, lambda: batch.decode(ctx, desc)) == 3
    assert (batch.statuses()[:len(images) + 1] == 0).all()
    assert_decode_same_as_direct(ctx, images, pick(checker, port, True))


@pytest.mark.gpu
def test_chunks_of_many_images(ctx, checker, port):
    """130 images: three chunks, the last two with right strips, in one host-described call."""
    desc = KERNELS[3][1]
    images = [DecodeImage(desc, 64 if i < 64 else 67, 3, f"rgb_chunks_{i}", overshoot=True) for i in range(130)]
    assert launches_of(ctx, lambda: run_decode_batch(ctx, desc, images)) == 1 + 2 + 2
    assert_decode_same_as_direct(ctx, images, pick(checker, port, True))


# ---- 2. several passes of both grids -------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("api", ["host", "device"])
@pytest.mark.parametrize("name", ["h16_rgba_d12", "f32_rgb_pq_d12"])
def test_multipass(ctx, checker, port, api, name):
    """64 images of 525 x 300: 3 units of 256 pixels per row, 900 interior units and 300 one-row edge units per image.  The
    integer interior grid is capped at 16 CTAs of 8 warps per SM, the table one at its residency (at most 8 CTAs per SM at
    these registers), the edge grid at 16 one-CTA workers per SM: all walk their units at least twice."""
    desc = dict(KERNELS)[name]
    n, w, h = 64, 525, 300
    assert -(-(w & ~7) // 256) == 3 and w % 8
    sms = sm_count(ctx)
    assert_passes("rgb_f32_interior" if desc.host_depth == 32 else "rgb_int_interior", n * 3 * h, sms)
    assert_passes("decode_edge", n * h, sms)
    images = [DecodeImage(desc, w, h, f"rgb_multipass_{api}_{name}_{i}", overshoot=overshoot_ok(desc)) for i in range(n)]
    ctx.prepare_decode(desc)
    host_or_device(ctx, desc, "decode", api, images,
                   lambda done: assert_decode_same_as_direct(ctx, done, pick(checker, port, True), threads=os.cpu_count()))


# ---- 3. device-described specifics ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["h8_rgba", "f32_rgba_hlg_ootf_d10"])
def test_rejected_images_keep_their_outputs(ctx, checker, port, name):
    desc = dict(KERNELS)[name]
    images = [DecodeImage(desc, w, h, f"rgb_bad_{name}_{i}") for i, (w, h) in enumerate([(64, 16), (37, 9), (64, 4), (8, 2), (130, 5), (7, 5)])]
    ctx.prepare_decode(desc)
    rejected_records(ctx, desc, "decode", images, DECODE_FAULTS, lambda good: assert_decode_same_as_direct(ctx, good, pick(checker, port, True)))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["h16_rgb_d10", "f32_rgba_hlg_d12"])
def test_captured_call_replays_new_image_sets(checker, port, name):
    """One capture of a device-described call, replayed on 1, 64 and 256 images at new addresses."""
    import avifgpu
    desc = dict(KERNELS)[name]
    over = overshoot_ok(desc)
    reference = pick(checker, port, True)
    tag = f"rgb_replay_{name}"
    sets = replay_sets(lambda w, h, seed: DecodeImage(desc, w, h, seed, overshoot=over), tag, (136, 34), MIXED)
    with avifgpu.Context(0) as fresh:
        capture_and_replay(fresh, desc, "decode", DecodeImage(desc, 64, 16, f"{tag}_capture"), sets,
                           lambda images: assert_decode_same_as_direct(fresh, images, reference, threads=os.cpu_count()),
                           lambda: fresh.prepare_decode(desc))


@pytest.mark.gpu
def test_captured_host_described_call_replays_like_direct_calls(checker, port):
    """A host-described planar-RGB batch captured into a graph: the same launches as the call itself, the same bits."""
    import avifgpu
    desc = dict(KERNELS)["f32_rgb_428_d10"]
    images = mix(desc, "rgb_captured_host")
    with avifgpu.Context(0) as fresh:
        fresh.prepare_decode(desc)
        before = fresh.launch_count()
        run_decode_batch(fresh, desc, images)
        calls = fresh.launch_count() - before
        assert captured(fresh, lambda stream: run_decode_batch(fresh, desc, images, stream)) == calls
        assert_decode_same_as_direct(fresh, images, pick(checker, port, True))


# ---- 4. what stays as it was -----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("host_depth", [16, 32])
def test_premultiplied_planar_rgb_keeps_its_direct_calls(ctx, checker, port, host_depth):
    desc = rgb(16, 10, PREMUL) if host_depth == 16 else rgb(32, 12, PREMUL, "pq")
    images = [DecodeImage(desc, w, h, f"rgb_premul_{host_depth}_{i}") for i, (w, h) in enumerate(MIXED)]
    ctx.prepare_decode(desc)
    direct = direct_launches(ctx, images, into=lambda im: im.rows)
    assert launches_of(ctx, lambda: run_decode_batch(ctx, desc, images)) == direct
    assert_decode_same_as_direct(ctx, images, pick(checker, port, True))


@pytest.mark.gpu
@pytest.mark.parametrize("name,desc", [
    ("premultiplied_rgb8", rgb(8, 8, PREMUL)),
    ("premultiplied_rgb32", rgb(32, 10, PREMUL, "hlg")),
    ("monochrome16", abi.DecodeDesc(0, 0, abi.COLORSPACE_MONOCHROME, abi.CHROMA_MONOCHROME, 12, NONE, 16, cases.NCLX_2020_PQ())),
    ("monochrome32", abi.DecodeDesc(0, 0, abi.COLORSPACE_MONOCHROME, abi.CHROMA_MONOCHROME, 10, STRAIGHT, 32, cases.NCLX_2020_PQ())),
], ids=["premultiplied_rgb8", "premultiplied_rgb32", "monochrome16", "monochrome32"])
def test_indirect_refuses_monochrome_and_premultiplied(ctx, name, desc):
    import avifgpu
    batch = Indirect(4)
    before = ctx.launch_count()
    with pytest.raises(avifgpu.AvifGpuError) as info:
        batch.decode(ctx, desc)
    assert info.value.status == abi.ERR_UNSUPPORTED and ctx.launch_count() == before
