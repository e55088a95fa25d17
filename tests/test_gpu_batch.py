"""avifgpu_encode_batch_device: many whole images per launch (include/avifgpu.h, "batches of small device-resident
images").

Every batched image must equal, bit for bit, a direct avifgpu_encode_rows_device call of the same image -- and the CPU
checker.  Plane rows are padded with a sentinel that must survive.  Launch counts follow the chunk rule: one launch for
a chunk's interiors, one more when any of its images has an edge strip, one direct call per image the tuned integer
kernel does not take."""
import pytest

import cases
from avifgpu import abi
from gpu_harness import ctx  # noqa: F401
from gpu_harness import (CHUNK, SIZES, DecodeImage, EncodeImage, assert_decode_same_as_direct, assert_passes, assert_same_as_direct, capture,
                         direct_launches, pick, planar, run_batch, run_decode_batch, sm_count, ycc)

pytestmark = pytest.mark.gpu

N601 = abi.Nclx(1, 1, 13, abi.MATRIX_BT601, 1)
PARITY = [
    ("h8c4_straight_d8_444_601", planar(8, 4, abi.ALPHA_STRAIGHT, 8, abi.CHROMA_444, N601)),
    ("h8c3_d8_420_709", planar(8, 3, abi.ALPHA_NONE, 8, abi.CHROMA_420, cases.NCLX_709())),
    ("h8c4_premul_d10_422_2020", planar(8, 4, abi.ALPHA_PREMULTIPLIED, 10, abi.CHROMA_422, cases.NCLX_2020_PQ())),
    ("h8c3_d12_444_gbr", planar(8, 3, abi.ALPHA_NONE, 12, abi.CHROMA_444, cases.NCLX_GBR())),
    ("h16c4_straight_d10_422_2020", planar(16, 4, abi.ALPHA_STRAIGHT, 10, abi.CHROMA_422, cases.NCLX_2020_PQ())),
    ("h16c3_d12_420_709", planar(16, 3, abi.ALPHA_NONE, 12, abi.CHROMA_420, cases.NCLX_709())),
    ("h16c4_premul_d8_420_601_topleft", planar(16, 4, abi.ALPHA_PREMULTIPLIED, 8, abi.CHROMA_420, N601, abi.DOWN_FILTER_TOP_LEFT)),
    ("h16c4_premul_d12_444_none", planar(16, 4, abi.ALPHA_PREMULTIPLIED, 12, abi.CHROMA_444, None)),
    ("h8c4_straight_d10_444_gbr", planar(8, 4, abi.ALPHA_STRAIGHT, 10, abi.CHROMA_444, cases.NCLX_GBR())),
    ("h16c3_d8_422_601", planar(16, 3, abi.ALPHA_NONE, 8, abi.CHROMA_422, N601)),
]


@pytest.mark.parametrize("name,desc", PARITY, ids=[p[0] for p in PARITY])
def test_batch_equals_direct_calls_and_checker(ctx, port, name, desc):
    images = [EncodeImage(desc, w, h, f"{name}_{i}") for i, (w, h) in enumerate(SIZES)]
    run_batch(ctx, desc, images)
    assert_same_as_direct(ctx, images, port)


def eligible_images(desc, n, w=64, h=16, seed="count"):
    return [EncodeImage(desc, w, h, f"{seed}_{i}") for i in range(n)]


@pytest.mark.parametrize("n", [1, 8, 64])
@pytest.mark.parametrize("edges", [False, True])
def test_one_chunk_costs_one_or_two_launches(ctx, n, edges):
    desc = PARITY[0][1]
    images = eligible_images(desc, n, 69 if edges else 64, 16, f"count_{n}_{edges}")
    before = ctx.launch_count()
    run_batch(ctx, desc, images)
    assert ctx.launch_count() - before == (2 if edges else 1)
    assert_same_as_direct(ctx, images)


@pytest.mark.parametrize("kind", ["float_pq", "gray16", "reference_layout"])
def test_fallback_only_batch_costs_the_direct_calls(ctx, kind):
    desc = {"float_pq": planar(32, 3, abi.ALPHA_NONE, 12, abi.CHROMA_420, cases.NCLX_2020_PQ()),
            "gray16": abi.EncodeDesc(0, 0, 16, 1, abi.ALPHA_NONE, 10),
            "reference_layout": abi.EncodeDesc(0, 0, 8, 4, abi.ALPHA_STRAIGHT, 8)}[kind]
    if kind == "float_pq":
        desc.transfer = abi.TRANSFER_PQ
    images = [EncodeImage(desc, w, h, f"fallback_{kind}_{i}") for i, (w, h) in enumerate(SIZES)]
    ctx.prepare_encode(desc)
    expected = direct_launches(ctx, images)
    before = ctx.launch_count()
    run_batch(ctx, desc, images)
    assert ctx.launch_count() - before == expected
    assert_same_as_direct(ctx, images)


def test_mixed_batch_with_an_unaligned_image(ctx):
    desc = PARITY[0][1]
    images = eligible_images(desc, 5, 64, 16, "mixed")
    odd = EncodeImage(desc, 64, 16, "mixed_odd", rows_misalign=4)
    images.insert(2, odd)
    expected_direct = direct_launches(ctx, [odd])
    before = ctx.launch_count()
    run_batch(ctx, desc, images)
    assert ctx.launch_count() - before == 1 + expected_direct
    assert_same_as_direct(ctx, images)


def test_batch_over_two_chunks(ctx):
    desc = PARITY[4][1]
    # a fallback image (width < 8) inside the run, and the chunk boundary inside the eligible images
    images = eligible_images(desc, CHUNK + 6, 44, 6, "chunks")
    images.insert(30, EncodeImage(desc, 5, 3, "chunks_narrow"))
    expected_direct = direct_launches(ctx, [images[30]])
    before = ctx.launch_count()
    run_batch(ctx, desc, images)
    assert ctx.launch_count() - before == 2 + 2 + expected_direct
    assert_same_as_direct(ctx, images)


def test_persistent_walk_runs_several_passes(ctx):
    desc = PARITY[0][1]
    images = eligible_images(desc, 64, 512, 512, "passes")
    assert_passes("encode_interior", len(images) * 2 * 512, sm_count(ctx))  # two 256-pixel units per row
    run_batch(ctx, desc, images)
    assert_same_as_direct(ctx, images[:: 7])


@pytest.mark.parametrize("fault", ["null_plane", "negative_size", "null_rows"])
def test_one_bad_image_fails_the_call_before_any_launch(ctx, fault):
    import avifgpu
    desc = PARITY[0][1]
    images = eligible_images(desc, 6, 64, 16, f"bad_{fault}")
    records = avifgpu.batch_images_from_tensors([im.record() for im in images])
    if fault == "null_plane":
        records[4].planes.data[1] = None
    elif fault == "negative_size":
        records[4].height = -2
    else:
        records[4].rows = None
    before = ctx.launch_count()
    with pytest.raises(avifgpu.AvifGpuError) as info:
        ctx.encode_batch_device(desc, records)
    assert info.value.status == abi.ERR_BAD_PARAM
    assert ctx.launch_count() == before
    assert all(im.untouched() for im in images)


def test_empty_batch_is_ok_without_a_launch(ctx):
    import avifgpu
    desc = PARITY[0][1]
    before = ctx.launch_count()
    ctx.encode_batch_device(desc, avifgpu.batch_images_from_tensors([]))
    ctx.encode_batch_device(desc, avifgpu.batch_images_from_tensors([(0, 5, None, [None] * 4), (7, 0, None, [None] * 4)]))
    assert ctx.launch_count() == before


def test_captured_batch_replays_like_direct_calls(ctx):
    import torch
    desc = PARITY[2][1]  # premultiplied: the check is prepared by one batch call outside the capture
    images = [EncodeImage(desc, w, h, f"capture_{i}") for i, (w, h) in enumerate(SIZES)]
    stream = torch.cuda.Stream()
    before = ctx.launch_count()
    run_batch(ctx, desc, images, stream.cuda_stream)
    torch.cuda.synchronize()
    direct = ctx.launch_count() - before - 1  # the first call also ran the premultiply check
    graph, launches = capture(ctx, lambda s: run_batch(ctx, desc, images, s), stream)
    assert launches == direct
    for seed in (1, 2):
        for i, im in enumerate(images):
            if im.w and im.h:
                fresh = EncodeImage(desc, im.w, im.h, f"capture_{i}_replay{seed}")
                im.rows.copy_(fresh.rows)
                im.host = fresh.host
        before = ctx.launch_count()
        graph.replay()
        torch.cuda.synchronize()
        assert ctx.launch_count() == before
        assert_same_as_direct(ctx, images)


# ---- decode ---------------------------------------------------------------------------------------------------------

DECODE = [
    ("h8_d8_420_a1_601", ycc(8, 8, abi.CHROMA_420, abi.ALPHA_STRAIGHT, N601)),
    ("h8_d8_444_a0_709", ycc(8, 8, abi.CHROMA_444, abi.ALPHA_NONE, cases.NCLX_709())),
    ("h16_d10_422_a1_2020", ycc(16, 10, abi.CHROMA_422, abi.ALPHA_STRAIGHT, cases.NCLX_2020_PQ())),
    ("h16_d12_420_a0_601", ycc(16, 12, abi.CHROMA_420, abi.ALPHA_NONE, N601)),
    ("h16_d10_444_a0_gbr", ycc(16, 10, abi.CHROMA_444, abi.ALPHA_NONE, cases.NCLX_GBR())),
    ("h8_d8_422_a2_709_premultiplied", ycc(8, 8, abi.CHROMA_422, abi.ALPHA_PREMULTIPLIED, cases.NCLX_709())),
]


@pytest.mark.parametrize("name,desc", DECODE, ids=[p[0] for p in DECODE])
def test_decode_batch_equals_direct_calls_and_checker(ctx, checker, port, name, desc):
    images = [DecodeImage(desc, w, h, f"{name}_{i}") for i, (w, h) in enumerate(SIZES)]
    run_decode_batch(ctx, desc, images)
    assert_decode_same_as_direct(ctx, images, pick(checker, port, True))


@pytest.mark.parametrize("n", [1, 8, 64])
@pytest.mark.parametrize("edges", [False, True])
def test_decode_chunk_costs_one_or_two_launches(ctx, n, edges):
    desc = DECODE[0][1]
    images = [DecodeImage(desc, 69 if edges else 64, 16, f"dcount_{n}_{edges}_{i}") for i in range(n)]
    ctx.prepare_decode(desc)
    before = ctx.launch_count()
    run_decode_batch(ctx, desc, images)
    assert ctx.launch_count() - before == (2 if edges else 1)
    assert_decode_same_as_direct(ctx, images)


def test_decode_fallback_and_mixed_batches(ctx):
    mono = abi.DecodeDesc(0, 0, abi.COLORSPACE_MONOCHROME, abi.CHROMA_MONOCHROME, 10, abi.ALPHA_NONE, 32, cases.NCLX_2020_PQ())
    images = [DecodeImage(mono, w, h, f"dmono_{i}") for i, (w, h) in enumerate(SIZES)]
    ctx.prepare_decode(mono)
    expected = direct_launches(ctx, images)
    before = ctx.launch_count()
    run_decode_batch(ctx, mono, images)
    assert ctx.launch_count() - before == expected
    assert_decode_same_as_direct(ctx, images)
    desc = DECODE[0][1]
    mixed = [DecodeImage(desc, 64, 16, f"dmixed_{i}") for i in range(CHUNK + 3)]
    mixed.insert(10, DecodeImage(desc, 64, 16, "dmixed_odd", planes_misalign=2))
    before = ctx.launch_count()
    run_decode_batch(ctx, desc, mixed)
    odd_launches = ctx.launch_count() - before - 2  # two chunks without edges
    assert odd_launches >= 1
    assert_decode_same_as_direct(ctx, mixed)


def test_decode_bad_image_and_empty_batch(ctx):
    import avifgpu
    desc = DECODE[0][1]
    images = [DecodeImage(desc, 64, 16, f"dbad_{i}") for i in range(4)]
    records = avifgpu.batch_images_from_tensors([im.record() for im in images])
    records[2].planes.data[3] = None
    before = ctx.launch_count()
    with pytest.raises(avifgpu.AvifGpuError) as info:
        ctx.decode_batch_device(desc, records)
    assert info.value.status == abi.ERR_BAD_PARAM and ctx.launch_count() == before
    assert all(im.untouched() for im in images)
    ctx.decode_batch_device(desc, avifgpu.batch_images_from_tensors([]))
    assert ctx.launch_count() == before


def test_captured_decode_batch_replays_like_direct_calls(ctx):
    import torch
    desc = DECODE[2][1]
    images = [DecodeImage(desc, w, h, f"dcapture_{i}") for i, (w, h) in enumerate(SIZES)]
    ctx.prepare_decode(desc)
    stream = torch.cuda.Stream()
    before = ctx.launch_count()
    run_decode_batch(ctx, desc, images, stream.cuda_stream)
    torch.cuda.synchronize()
    direct = ctx.launch_count() - before
    graph, launches = capture(ctx, lambda s: run_decode_batch(ctx, desc, images, s), stream)
    assert launches == direct
    for seed in (1, 2):
        for i, im in enumerate(images):
            fresh = DecodeImage(desc, im.w, im.h, f"dcapture_{i}_replay{seed}")
            for p, q in zip(im.planes, fresh.planes):
                if p is not None:
                    p.copy_(q)
        graph.replay()
        torch.cuda.synchronize()
        assert_decode_same_as_direct(ctx, images)
