"""avifgpu_encode_batch_device: many whole images per launch (include/avifgpu.h, "batches of small device-resident
images").

Every batched image must equal, bit for bit, a direct avifgpu_encode_rows_device call of the same image -- and the CPU
checker.  Plane rows are padded with a sentinel that must survive.  Launch counts follow the chunk rule: one launch for
a chunk's interiors, one more when any of its images has an edge strip, one direct call per image the tuned integer
kernel does not take."""
import numpy as np
import pytest

import cases
from avifgpu import abi
from test_gpu_multipass import pick

pytestmark = pytest.mark.gpu

SENTINEL = 0xCD
CHUNK = 64  # kBatchChunkImages
# mixed sizes: aligned interiors with and without right strips, odd 4:2:0 heights, widths below 8, a 1 x 1 image
SIZES = [(64, 16), (37, 9), (8, 2), (1, 1), (130, 33), (7, 5), (256, 64), (95, 4)]


@pytest.fixture
def ctx():
    import avifgpu
    context = avifgpu.Context(0)
    yield context
    context.close()


def padded(n):
    return (n + 63) // 64 * 64 + 64


class Image:
    """One image's seeded host rows and sentinel-padded planes, as byte tensors on the GPU."""

    def __init__(self, desc, w, h, seed, misalign=0, beyond=False):
        import torch
        self.w, self.h = w, h
        d = self.desc = batch_desc(desc, w, h)
        rng = cases.rng_for(f"batch_{seed}_{w}x{h}")
        if d.host_depth == 32:
            self.host = cases.float_host_rows(rng, h, w, d.host_channels)
        else:
            self.host = cases.int_host_rows(rng, h, w, d.host_channels, d.host_depth, beyond=beyond)
        row_bytes = w * d.host_channels * d.host_depth // 8
        backing = torch.zeros((max(h, 1), padded(row_bytes) + misalign), dtype=torch.uint8, device="cuda")
        self.rows = backing[:, misalign:misalign + row_bytes]
        if h and w:
            self.rows.copy_(torch.from_numpy(np.ascontiguousarray(self.host).view(np.uint8).reshape(h, row_bytes)).cuda())
        self.sample_bytes = 2 if d.image_bit_depth > 8 else 1
        self.planes = [self.alloc(s) for s in abi.encode_plane_shapes(d)]

    def alloc(self, shape):
        import torch
        if shape is None:
            return None
        rows, cols = shape
        backing = torch.full((max(rows, 1), padded(cols * self.sample_bytes)), SENTINEL, dtype=torch.uint8, device="cuda")
        return backing[:rows, :cols * self.sample_bytes]

    def fresh_planes(self):
        return [None if p is None else self.alloc((p.shape[0], p.shape[1] // self.sample_bytes)) for p in self.planes]

    def record(self):
        return (self.w, self.h, self.rows, self.planes)

    def direct(self, ctx, planes):
        import avifgpu
        stride = self.rows.stride(0)
        ctx.encode_device(self.desc, self.rows.data_ptr(), stride, avifgpu.planes_from_tensors(planes))


def batch_desc(desc, w, h):
    d = abi.EncodeDesc.from_buffer_copy(desc)
    d.width, d.height = w, h
    return d


def whole(plane):
    """The plane's bytes with the row padding (the sentinel) included."""
    return plane.as_strided((plane.shape[0], plane.stride(0)), (plane.stride(0), 1)).cpu().numpy()


def run_batch(ctx, desc, images, stream=0):
    import avifgpu
    ctx.encode_batch_device(desc, avifgpu.batch_images_from_tensors([im.record() for im in images]), stream=stream)


def assert_same_as_direct(ctx, images, checker=None, threads=1):
    import torch
    for im in images:
        reference = im.fresh_planes()
        im.direct(ctx, reference)
        torch.cuda.synchronize()
        for k, (got, want) in enumerate(zip(im.planes, reference)):
            if got is None:
                continue
            a, b = whole(got), whole(want)
            assert np.array_equal(a, b), (im.w, im.h, k)
            assert (a[:, got.shape[1]:] == SENTINEL).all(), ("padding overwritten", im.w, im.h, k)
        if checker is not None and im.w and im.h:
            expected = checker.encode(im.desc, im.host, threads=threads)
            for k, got in enumerate(im.planes):
                if got is not None:
                    codes = got.cpu().numpy().view(abi.code_dtype(im.desc.image_bit_depth))
                    assert np.array_equal(codes, expected[k]), ("checker", im.w, im.h, k)


def planar(host_depth, channels, alpha, depth, chroma, nclx, down=abi.DOWN_FILTER_BOX):
    return abi.EncodeDesc(0, 0, host_depth, channels, alpha, depth, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, chroma, down,
                          abi.GRAY16_LUT, nclx)


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
    images = [Image(desc, w, h, f"{name}_{i}") for i, (w, h) in enumerate(SIZES)]
    run_batch(ctx, desc, images)
    assert_same_as_direct(ctx, images, port)


def eligible_images(desc, n, w=64, h=16, seed="count"):
    return [Image(desc, w, h, f"{seed}_{i}") for i in range(n)]


@pytest.mark.parametrize("n", [1, 8, 64])
@pytest.mark.parametrize("edges", [False, True])
def test_one_chunk_costs_one_or_two_launches(ctx, n, edges):
    desc = PARITY[0][1]
    images = eligible_images(desc, n, 69 if edges else 64, 16, f"count_{n}_{edges}")
    before = ctx.launch_count()
    run_batch(ctx, desc, images)
    assert ctx.launch_count() - before == (2 if edges else 1)
    assert_same_as_direct(ctx, images)


def direct_launches(ctx, images):
    total = 0
    for im in images:
        before = ctx.launch_count()
        im.direct(ctx, im.fresh_planes())
        total += ctx.launch_count() - before
    return total


@pytest.mark.parametrize("kind", ["float_pq", "gray16", "reference_layout"])
def test_fallback_only_batch_costs_the_direct_calls(ctx, kind):
    desc = {"float_pq": planar(32, 3, abi.ALPHA_NONE, 12, abi.CHROMA_420, cases.NCLX_2020_PQ()),
            "gray16": abi.EncodeDesc(0, 0, 16, 1, abi.ALPHA_NONE, 10),
            "reference_layout": abi.EncodeDesc(0, 0, 8, 4, abi.ALPHA_STRAIGHT, 8)}[kind]
    if kind == "float_pq":
        desc.transfer = abi.TRANSFER_PQ
    images = [Image(desc, w, h, f"fallback_{kind}_{i}") for i, (w, h) in enumerate(SIZES)]
    ctx.prepare_encode(desc)
    expected = direct_launches(ctx, images)
    before = ctx.launch_count()
    run_batch(ctx, desc, images)
    assert ctx.launch_count() - before == expected
    assert_same_as_direct(ctx, images)


def test_mixed_batch_with_an_unaligned_image(ctx):
    desc = PARITY[0][1]
    images = eligible_images(desc, 5, 64, 16, "mixed")
    odd = Image(desc, 64, 16, "mixed_odd", misalign=4)
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
    images.insert(30, Image(desc, 5, 3, "chunks_narrow"))
    expected_direct = direct_launches(ctx, [images[30]])
    before = ctx.launch_count()
    run_batch(ctx, desc, images)
    assert ctx.launch_count() - before == 2 + 2 + expected_direct
    assert_same_as_direct(ctx, images)


def test_persistent_walk_runs_several_passes(ctx):
    import torch
    desc = PARITY[0][1]
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    # interior grid: at most 16 CTAs of 8 warps per SM (LaunchEncodeBatchChunk, kernels_batch.cu), one 256-pixel unit per warp
    warps = sm * 16 * 8
    images = eligible_images(desc, 64, 512, 512, "passes")
    units = len(images) * 2 * 512
    assert units >= 2 * warps
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
    import torch
    torch.cuda.synchronize()
    for im in images:
        for p in im.planes:
            if p is not None:
                assert (whole(p) == SENTINEL).all()


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
    images = [Image(desc, w, h, f"capture_{i}") for i, (w, h) in enumerate(SIZES)]
    stream = torch.cuda.Stream()
    before = ctx.launch_count()
    run_batch(ctx, desc, images, stream.cuda_stream)
    torch.cuda.synchronize()
    direct = ctx.launch_count() - before - 1  # the first call also ran the premultiply check
    graph = torch.cuda.CUDAGraph()
    before = ctx.launch_count()
    with torch.cuda.graph(graph, stream=stream):
        run_batch(ctx, desc, images, stream.cuda_stream)
    assert ctx.launch_count() - before == direct
    for seed in (1, 2):
        for i, im in enumerate(images):
            if im.w and im.h:
                fresh = Image(desc, im.w, im.h, f"capture_{i}_replay{seed}")
                im.rows.copy_(fresh.rows)
                im.host = fresh.host
        before = ctx.launch_count()
        graph.replay()
        torch.cuda.synchronize()
        assert ctx.launch_count() == before
        assert_same_as_direct(ctx, images)


# ---- decode ---------------------------------------------------------------------------------------------------------

class DecImage:
    """One image's seeded source planes and sentinel-padded destination rows, as byte tensors on the GPU."""

    def __init__(self, desc, w, h, seed, misalign=0, overshoot=False):
        import torch
        self.w, self.h = w, h
        d = self.desc = abi.DecodeDesc.from_buffer_copy(desc)
        d.width, d.height = w, h
        self.codes = cases.code_planes(cases.rng_for(f"dbatch_{seed}_{w}x{h}"), d, overshoot=overshoot)
        self.planes = []
        for c in self.codes:
            if c is None:
                self.planes.append(None)
                continue
            raw = np.ascontiguousarray(c).view(np.uint8)
            backing = torch.zeros((max(raw.shape[0], 1), padded(raw.shape[1]) + misalign), dtype=torch.uint8, device="cuda")
            plane = backing[:raw.shape[0], misalign:misalign + raw.shape[1]]
            plane.copy_(torch.from_numpy(raw).cuda())
            self.planes.append(plane)
        self.row_bytes = w * abi.decode_host_channels(d) * d.host_depth // 8
        self.rows = self.alloc()

    def alloc(self):
        import torch
        return torch.full((max(self.h, 1), padded(self.row_bytes)), SENTINEL, dtype=torch.uint8, device="cuda")[:self.h, :self.row_bytes]

    def record(self):
        return (self.w, self.h, self.rows, self.planes)

    def direct(self, ctx, rows):
        import avifgpu
        ctx.decode_device(self.desc, avifgpu.planes_from_tensors(self.planes), rows.data_ptr(), rows.stride(0))


def run_decode_batch(ctx, desc, images, stream=0):
    import avifgpu
    ctx.decode_batch_device(desc, avifgpu.batch_images_from_tensors([im.record() for im in images]), stream=stream)


def assert_decode_same_as_direct(ctx, images, checker=None, threads=1):
    import torch
    for im in images:
        reference = im.alloc()
        im.direct(ctx, reference)
        torch.cuda.synchronize()
        a, b = whole(im.rows), whole(reference)
        assert np.array_equal(a, b), (im.w, im.h)
        assert (a[:, im.row_bytes:] == SENTINEL).all(), ("padding overwritten", im.w, im.h)
        if checker is not None and im.w and im.h:
            expected = checker.decode(im.desc, im.codes, threads=threads)
            got = im.rows.cpu().numpy().view(abi.host_dtype(im.desc.host_depth))
            assert np.array_equal(got, expected), ("checker", im.w, im.h)


def ycc(host_depth, bit_depth, chroma, alpha, nclx):
    return abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, chroma, bit_depth, alpha, host_depth, nclx)


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
    images = [DecImage(desc, w, h, f"{name}_{i}") for i, (w, h) in enumerate(SIZES)]
    run_decode_batch(ctx, desc, images)
    assert_decode_same_as_direct(ctx, images, pick(checker, port, True))


@pytest.mark.parametrize("n", [1, 8, 64])
@pytest.mark.parametrize("edges", [False, True])
def test_decode_chunk_costs_one_or_two_launches(ctx, n, edges):
    desc = DECODE[0][1]
    images = [DecImage(desc, 69 if edges else 64, 16, f"dcount_{n}_{edges}_{i}") for i in range(n)]
    ctx.prepare_decode(desc)
    before = ctx.launch_count()
    run_decode_batch(ctx, desc, images)
    assert ctx.launch_count() - before == (2 if edges else 1)
    assert_decode_same_as_direct(ctx, images)


def test_decode_fallback_and_mixed_batches(ctx):
    mono = abi.DecodeDesc(0, 0, abi.COLORSPACE_MONOCHROME, abi.CHROMA_MONOCHROME, 10, abi.ALPHA_NONE, 32, cases.NCLX_2020_PQ())
    images = [DecImage(mono, w, h, f"dmono_{i}") for i, (w, h) in enumerate(SIZES)]
    ctx.prepare_decode(mono)
    expected = 0
    for im in images:
        before = ctx.launch_count()
        im.direct(ctx, im.alloc())
        expected += ctx.launch_count() - before
    before = ctx.launch_count()
    run_decode_batch(ctx, mono, images)
    assert ctx.launch_count() - before == expected
    assert_decode_same_as_direct(ctx, images)
    desc = DECODE[0][1]
    mixed = [DecImage(desc, 64, 16, f"dmixed_{i}") for i in range(CHUNK + 3)]
    mixed.insert(10, DecImage(desc, 64, 16, "dmixed_odd", misalign=2))
    before = ctx.launch_count()
    run_decode_batch(ctx, desc, mixed)
    odd_launches = ctx.launch_count() - before - 2  # two chunks without edges
    assert odd_launches >= 1
    assert_decode_same_as_direct(ctx, mixed)


def test_decode_bad_image_and_empty_batch(ctx):
    import avifgpu
    import torch
    desc = DECODE[0][1]
    images = [DecImage(desc, 64, 16, f"dbad_{i}") for i in range(4)]
    records = avifgpu.batch_images_from_tensors([im.record() for im in images])
    records[2].planes.data[3] = None
    before = ctx.launch_count()
    with pytest.raises(avifgpu.AvifGpuError) as info:
        ctx.decode_batch_device(desc, records)
    assert info.value.status == abi.ERR_BAD_PARAM and ctx.launch_count() == before
    torch.cuda.synchronize()
    assert all((whole(im.rows) == SENTINEL).all() for im in images)
    ctx.decode_batch_device(desc, avifgpu.batch_images_from_tensors([]))
    assert ctx.launch_count() == before


def test_captured_decode_batch_replays_like_direct_calls(ctx):
    import torch
    desc = DECODE[2][1]
    images = [DecImage(desc, w, h, f"dcapture_{i}") for i, (w, h) in enumerate(SIZES)]
    ctx.prepare_decode(desc)
    stream = torch.cuda.Stream()
    before = ctx.launch_count()
    run_decode_batch(ctx, desc, images, stream.cuda_stream)
    torch.cuda.synchronize()
    direct = ctx.launch_count() - before
    graph = torch.cuda.CUDAGraph()
    before = ctx.launch_count()
    with torch.cuda.graph(graph, stream=stream):
        run_decode_batch(ctx, desc, images, stream.cuda_stream)
    assert ctx.launch_count() - before == direct
    for seed in (1, 2):
        for i, im in enumerate(images):
            fresh = DecImage(desc, im.w, im.h, f"dcapture_{i}_replay{seed}")
            for p, q in zip(im.planes, fresh.planes):
                if p is not None:
                    p.copy_(q)
        graph.replay()
        torch.cuda.synchronize()
        assert_decode_same_as_direct(ctx, images)
