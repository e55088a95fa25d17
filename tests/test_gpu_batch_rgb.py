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

import numpy as np
import pytest

import cases
from avifgpu import abi
from test_gpu_batch import CHUNK, SENTINEL, DecImage, ctx, padded, run_decode_batch, whole  # noqa: F401
from test_gpu_batch_f32 import captured
from test_gpu_batch_indirect import Empty, Indirect, launches_of
from test_gpu_multipass import pick, rgb32_nclx

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


def offset_rows(im, offset):
    """Moves a decode image's destination rows `offset` bytes off their alignment, keeping the row stride."""
    import torch
    stride = padded(im.row_bytes)
    backing = torch.full(((im.h + 1) * stride,), SENTINEL, dtype=torch.uint8, device="cuda")
    im.rows = backing[offset:offset + im.h * stride].view(im.h, stride)[:, :im.row_bytes]
    return im


def mix(desc, seed):
    over = overshoot_ok(desc)
    images = [DecImage(desc, w, h, f"{seed}_{i}", overshoot=over) for i, (w, h) in enumerate(MIXED)]
    images.append(offset_rows(DecImage(desc, 64, 7, f"{seed}_rows4", overshoot=over), 4))
    images.append(offset_rows(DecImage(desc, 72, 5, f"{seed}_rows8", overshoot=over), 8))
    images.append(DecImage(desc, 68, 6, f"{seed}_planes", misalign=2, overshoot=over))
    if not over:
        over_image = DecImage(desc, 136, 3, f"{seed}_over", overshoot=True)
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


def chunk_launches(images):
    chosen = [im for im in images if eligible(im)]
    return sum(1 + any(has_edge(im) for im in chosen[i:i + CHUNK]) for i in range(0, len(chosen), CHUNK))


def bits(a):
    return a.view(np.uint32) if a.dtype == np.float32 else a


def assert_same_as_direct_and_reference(ctx, images, reference, threads=1):
    """Each image: its rows (padding included) equal a direct call's, and the reference's output bit for bit."""
    import torch
    for im in images:
        direct = im.alloc()
        im.direct(ctx, direct)
        torch.cuda.synchronize()
        got = whole(im.rows)
        assert np.array_equal(got, whole(direct)), (im.w, im.h)
        assert (got[:, im.row_bytes:] == SENTINEL).all(), ("padding overwritten", im.w, im.h)
        if im.w and im.h and not getattr(im, "direct_only", False):
            expected = bits(reference.decode(im.desc, im.codes, threads=threads))
            values = bits(im.rows.cpu().numpy().view(abi.host_dtype(im.desc.host_depth)))
            differ = values != expected
            assert not differ.any(), ("reference", im.w, im.h, int(differ.sum()), np.argwhere(differ)[0])


def direct_launches(ctx, images):
    """The launches of one direct call of each image, made into the image's own rows (their alignment is part of its
    route); the batch overwrites them with the same bits."""
    total = 0
    for im in images:
        before = ctx.launch_count()
        im.direct(ctx, im.rows)
        total += ctx.launch_count() - before
    return total


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
    direct = direct_launches(ctx, fallbacks)
    assert launches_of(ctx, lambda: run_decode_batch(ctx, desc, images)) == chunk_launches(images) + direct
    assert_same_as_direct_and_reference(ctx, images, pick(checker, port, True))


@pytest.mark.gpu
@pytest.mark.parametrize("name,desc", KERNELS, ids=[c[0] for c in KERNELS])
def test_device_described_instantiation(ctx, checker, port, name, desc):
    images = mix(desc, f"rgb_indirect_{name}")
    batch = Indirect(16)
    batch.load(images[:5] + [Empty()] + images[5:])
    ctx.prepare_decode(desc)
    assert launches_of(ctx, lambda: batch.decode(ctx, desc)) == 3
    assert (batch.statuses()[:len(images) + 1] == 0).all()
    assert_same_as_direct_and_reference(ctx, images, pick(checker, port, True))


@pytest.mark.gpu
def test_chunks_of_many_images(ctx, checker, port):
    """130 images: three chunks, the last two with right strips, in one host-described call."""
    desc = KERNELS[3][1]
    images = [DecImage(desc, 64 if i < 64 else 67, 3, f"rgb_chunks_{i}", overshoot=True) for i in range(130)]
    assert launches_of(ctx, lambda: run_decode_batch(ctx, desc, images)) == 1 + 2 + 2
    assert_same_as_direct_and_reference(ctx, images, pick(checker, port, True))


# ---- 2. several passes of both grids -------------------------------------------------------------------------------------------

def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


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
    sms = sm_count()
    assert n * 3 * h >= 2 * sms * 16 * 8
    assert n * h >= 2 * sms * 16
    images = [DecImage(desc, w, h, f"rgb_multipass_{api}_{name}_{i}", overshoot=overshoot_ok(desc)) for i in range(n)]
    ctx.prepare_decode(desc)
    if api == "host":
        assert launches_of(ctx, lambda: run_decode_batch(ctx, desc, images)) == 2
    else:
        batch = Indirect(n)
        batch.load(images)
        assert launches_of(ctx, lambda: batch.decode(ctx, desc)) == 3
        assert (batch.statuses() == 0).all()
    assert_same_as_direct_and_reference(ctx, images, pick(checker, port, True), threads=os.cpu_count())


# ---- 3. device-described specifics ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["h8_rgba", "f32_rgba_hlg_ootf_d10"])
def test_rejected_images_keep_their_outputs(ctx, checker, port, name):
    import avifgpu
    import torch
    desc = dict(KERNELS)[name]
    images = [DecImage(desc, w, h, f"rgb_bad_{name}_{i}") for i, (w, h) in enumerate([(64, 16), (37, 9), (64, 4), (8, 2), (130, 5), (7, 5)])]
    records = avifgpu.batch_images_from_tensors([im.record() for im in images])
    records[1].rows = None
    records[3].planes.data[3] = None
    records[5].width = -1
    batch = Indirect(6)
    batch.load(records)
    ctx.prepare_decode(desc)
    assert launches_of(ctx, lambda: batch.decode(ctx, desc)) == 3
    bad = abi.ERR_BAD_PARAM
    assert list(batch.statuses()) == [0, bad, 0, bad, 0, bad]
    torch.cuda.synchronize()
    assert all((whole(images[i].rows) == SENTINEL).all() for i in (1, 3, 5))
    assert_same_as_direct_and_reference(ctx, [images[i] for i in (0, 2, 4)], pick(checker, port, True))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["h16_rgb_d10", "f32_rgba_hlg_d12"])
def test_captured_call_replays_new_image_sets(checker, port, name):
    """One capture of a device-described call, replayed on 1, 64 and 256 images at new addresses."""
    import avifgpu
    import torch
    desc = dict(KERNELS)[name]
    over = overshoot_ok(desc)
    reference = pick(checker, port, True)
    with avifgpu.Context(0) as fresh:
        batch = Indirect(256)
        stream = torch.cuda.Stream()
        with torch.cuda.stream(stream):
            batch.load([DecImage(desc, 64, 16, f"rgb_replay_{name}_capture")])
        fresh.prepare_decode(desc)
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        before = fresh.launch_count()
        with torch.cuda.graph(graph, stream=stream):
            batch.decode(fresh, desc, stream.cuda_stream)
        assert fresh.launch_count() - before == 3
        sets = [[DecImage(desc, 96, 10, f"rgb_replay_{name}_one", overshoot=over)],
                [DecImage(desc, 136, 34, f"rgb_replay_{name}_64_{i}", overshoot=over) for i in range(64)],
                [DecImage(desc, *MIXED[i % len(MIXED)], f"rgb_replay_{name}_256_{i}", overshoot=over) for i in range(256)]]
        for images in sets:
            with torch.cuda.stream(stream):
                batch.load(images)
                before = fresh.launch_count()
                graph.replay()
            torch.cuda.synchronize()
            assert fresh.launch_count() == before
            assert (batch.statuses()[:len(images)] == 0).all()
            assert_same_as_direct_and_reference(fresh, images, reference, threads=os.cpu_count())
        del graph


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
        assert_same_as_direct_and_reference(fresh, images, pick(checker, port, True))


# ---- 4. what stays as it was -----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("host_depth", [16, 32])
def test_premultiplied_planar_rgb_keeps_its_direct_calls(ctx, checker, port, host_depth):
    desc = rgb(16, 10, PREMUL) if host_depth == 16 else rgb(32, 12, PREMUL, "pq")
    images = [DecImage(desc, w, h, f"rgb_premul_{host_depth}_{i}") for i, (w, h) in enumerate(MIXED)]
    ctx.prepare_decode(desc)
    direct = direct_launches(ctx, images)
    assert launches_of(ctx, lambda: run_decode_batch(ctx, desc, images)) == direct
    assert_same_as_direct_and_reference(ctx, images, pick(checker, port, True))


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
