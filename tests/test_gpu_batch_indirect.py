"""avifgpu_encode_batch_indirect / avifgpu_decode_batch_indirect: batches whose image records and count are read from
device memory when the work runs (include/avifgpu.h, "batches described in device memory"), run by the batched kernels
of kernels_batch.cu under their workspace record source.

Every accepted image is compared bit for bit with a direct *_rows_device call of the same image and with the CPU checker
(the restatement for encode, the compiled reference for decode, by pick()), and the sentinel in the row padding must
survive.  A call is always three launches; a captured call replays whatever the records and count hold at replay.

  * every instantiation of the interior kernels (the tables of test_gpu_batch_kernels.py), on a mix of aligned images,
    right strips, odd 4:2:0 heights, height 1, width < 8, a misaligned rows pointer and a 0 x 5 image;
  * rejected images (NULL rows, NULL plane, negative width) get BAD_PARAM and keep the sentinel;
  * a count of 0, max_count, max_count + 1 and -1;
  * one capture replayed on 1, 64 and 256 images at new addresses -- encode with premultiplied alpha, prepared and
    unprepared, and decode;
  * loops of both kernels over several passes of their grids;
  * host rejections, with no launch."""
import ctypes as C
import os

import pytest

import cases
from avifgpu import abi
from test_gpu_batch import SENTINEL, SIZES, DecImage, Image, assert_decode_same_as_direct, assert_same_as_direct, ctx, padded, planar, whole, ycc  # noqa: F401
from test_gpu_batch_kernels import DECODE_KERNELS, ENCODE_KERNELS, MIXED, assert_passes, edge_units, interior_units, sm_count
from test_gpu_multipass import pick

pytestmark = pytest.mark.gpu

BAD = abi.ERR_BAD_PARAM
UNTOUCHED = 7  # a status value the call never writes


class Empty:
    """A 0 x 5 image: accepted, converts nothing."""
    w, h = 0, 5

    def record(self):
        return (0, 5, None, [None] * abi.MAX_PLANES)


class Indirect:
    """Device-side records, count, workspace and status array for batches of up to `capacity` images."""

    def __init__(self, capacity):
        import avifgpu
        import torch
        self.capacity = capacity
        self.records = torch.zeros((capacity, C.sizeof(abi.BatchImage)), dtype=torch.uint8, device="cuda")
        self.count = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.workspace = torch.empty(avifgpu.batch_workspace_bytes(capacity), dtype=torch.uint8, device="cuda")
        self.status = torch.full((capacity,), UNTOUCHED, dtype=torch.int32, device="cuda")

    def load(self, images, count=None):
        """Writes the records (image objects or a ctypes record array) and the count, on the current stream."""
        import avifgpu
        records = images if isinstance(images, C.Array) else [im.record() for im in images]
        avifgpu.pack_batch_images(records, self.capacity, out=self.records)
        self.count.fill_(len(images) if count is None else count)
        self.status.fill_(UNTOUCHED)

    def encode(self, ctx, desc, stream=0):
        ctx.encode_batch_indirect(desc, self.records, self.count, self.capacity, self.workspace, self.status, stream)

    def decode(self, ctx, desc, stream=0):
        ctx.decode_batch_indirect(desc, self.records, self.count, self.capacity, self.workspace, self.status, stream)

    def statuses(self):
        return self.status.cpu().numpy()


def launches_of(ctx, call):
    import torch
    before = ctx.launch_count()
    call()
    torch.cuda.synchronize()
    return ctx.launch_count() - before


def misaligned_rows(im):
    """Moves a decode image's destination rows 4 bytes off their alignment, keeping the row stride."""
    import torch
    stride = padded(im.row_bytes)
    backing = torch.full(((im.h + 1) * stride,), SENTINEL, dtype=torch.uint8, device="cuda")
    im.rows = backing[4:4 + im.h * stride].view(im.h, stride)[:, :im.row_bytes]
    return im


def encode_mix(desc, seed):
    images = [Image(desc, w, h, f"{seed}_{i}", beyond=True) for i, (w, h) in enumerate(MIXED)]
    images.append(Image(desc, 64, 7, f"{seed}_misaligned", misalign=4))
    return images


def decode_mix(desc, seed):
    images = [DecImage(desc, w, h, f"{seed}_{i}", overshoot=True) for i, (w, h) in enumerate(MIXED)]
    images.append(misaligned_rows(DecImage(desc, 64, 7, f"{seed}_misaligned", overshoot=True)))
    return images


# ---- 1. every instantiation ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name,desc", ENCODE_KERNELS, ids=[c[0] for c in ENCODE_KERNELS])
def test_encode_indirect_instantiation(ctx, port, name, desc):
    images = encode_mix(desc, f"indirect_{name}")
    batch = Indirect(16)
    batch.load(images[:5] + [Empty()] + images[5:])
    batch.encode(ctx, desc)  # the first call of a premultiplied description also makes the premultiply check
    assert launches_of(ctx, lambda: batch.encode(ctx, desc)) == 3
    assert (batch.statuses()[:len(images) + 1] == 0).all()
    assert (batch.statuses()[len(images) + 1:] == UNTOUCHED).all()
    assert_same_as_direct(ctx, images, port)


@pytest.mark.parametrize("name,desc", DECODE_KERNELS, ids=[c[0] for c in DECODE_KERNELS])
def test_decode_indirect_instantiation(ctx, checker, port, name, desc):
    images = decode_mix(desc, f"indirect_{name}")
    batch = Indirect(16)
    batch.load(images[:5] + [Empty()] + images[5:])
    ctx.prepare_decode(desc)
    assert launches_of(ctx, lambda: batch.decode(ctx, desc)) == 3
    assert (batch.statuses()[:len(images) + 1] == 0).all()
    assert_decode_same_as_direct(ctx, images, pick(checker, port, True))


def test_decode_of_16_bit_planes_runs_in_the_edge_kernel(ctx, checker, port):
    """16-bit planes have no tuned integer kernel: every image is one whole-image window."""
    desc = ycc(16, 16, abi.CHROMA_420, abi.ALPHA_STRAIGHT, cases.NCLX_709())
    images = decode_mix(desc, "indirect_d16")
    batch = Indirect(16)
    batch.load(images)
    assert launches_of(ctx, lambda: batch.decode(ctx, desc)) == 3
    assert (batch.statuses()[:len(images)] == 0).all()
    assert_decode_same_as_direct(ctx, images, pick(checker, port, True))


# ---- 2. rejected images -------------------------------------------------------------------------------------------------------

def untouched(im):
    outputs = [p for p in im.planes if p is not None] if isinstance(im, Image) else [im.rows]
    return all((whole(p) == SENTINEL).all() for p in outputs)


def test_encode_rejects_bad_images_and_converts_the_rest(ctx, port):
    import avifgpu
    desc = ENCODE_KERNELS[5][1]
    images = [Image(desc, w, h, f"indirect_bad_{i}") for i, (w, h) in enumerate([(64, 16), (37, 9), (64, 4), (8, 2), (130, 5), (7, 5), (96, 3), (520, 4)])]
    records = avifgpu.batch_images_from_tensors([im.record() for im in images])
    records[2].rows = None
    records[4].planes.data[1] = None
    records[6].width = -3
    batch = Indirect(8)
    batch.load(records)
    assert launches_of(ctx, lambda: batch.encode(ctx, desc)) == 3
    status = batch.statuses()
    assert list(status) == [0, 0, BAD, 0, BAD, 0, BAD, 0]
    assert all(untouched(images[i]) for i in (2, 4, 6))
    assert_same_as_direct(ctx, [images[i] for i in (0, 1, 3, 5, 7)], port)


def test_decode_rejects_bad_images_and_converts_the_rest(ctx, checker, port):
    import avifgpu
    desc = DECODE_KERNELS[5][1]
    images = [DecImage(desc, w, h, f"indirect_dbad_{i}") for i, (w, h) in enumerate([(64, 16), (37, 9), (64, 4), (8, 2), (130, 5), (7, 5), (96, 3)])]
    records = avifgpu.batch_images_from_tensors([im.record() for im in images])
    records[1].rows = None
    records[3].planes.data[3] = None
    records[5].width = -1
    batch = Indirect(7)
    batch.load(records)
    ctx.prepare_decode(desc)
    assert launches_of(ctx, lambda: batch.decode(ctx, desc)) == 3
    assert list(batch.statuses()) == [0, BAD, 0, BAD, 0, BAD, 0]
    assert all(untouched(images[i]) for i in (1, 3, 5))
    assert_decode_same_as_direct(ctx, [images[i] for i in (0, 2, 4, 6)], pick(checker, port, True))


# ---- 3. the count -----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("direction", ["encode", "decode"])
def test_count_zero_full_and_out_of_range(ctx, checker, port, direction):
    encode = direction == "encode"
    desc = ENCODE_KERNELS[3][1] if encode else DECODE_KERNELS[2][1]
    make = Image if encode else DecImage
    images = [make(desc, w, h, f"indirect_count_{direction}_{i}") for i, (w, h) in enumerate(SIZES)]
    batch = Indirect(len(images))
    run = (lambda: batch.encode(ctx, desc)) if encode else (lambda: batch.decode(ctx, desc))
    if not encode:
        ctx.prepare_decode(desc)
    for count in (0, len(images) + 1, -1):
        batch.load(images, count)
        assert launches_of(ctx, run) == 3
        assert all(untouched(im) for im in images if im.w and im.h), count
        expected = UNTOUCHED if count == 0 else BAD
        assert (batch.statuses() == expected).all(), count
    batch.load(images)
    assert launches_of(ctx, run) == 3
    assert (batch.statuses() == 0).all()
    if encode:
        assert_same_as_direct(ctx, images, port)
    else:
        assert_decode_same_as_direct(ctx, images, pick(checker, port, True))


# ---- 4. capture once, replay many -----------------------------------------------------------------------------------------------

def replay_sets(make, desc, tag):
    """1 image; 64 images of 512 x 512; 256 mixed images -- fresh buffers, so new addresses, each time."""
    mixed = [(264, 3), (37, 9), (7, 5), (130, 1), (95, 6), (64, 7), (8, 2), (1, 1)]
    return [
        [make(desc, 96, 10, f"{tag}_one")],
        [make(desc, 512, 512, f"{tag}_big_{i}") for i in range(64)],
        [make(desc, *mixed[i % len(mixed)], f"{tag}_mixed_{i}") for i in range(256)],
    ]


def capture_and_replay(ctx, desc, encode, check, tag, before_capture=None):
    import torch
    make = Image if encode else DecImage
    batch = Indirect(256)
    stream = torch.cuda.Stream()
    run = (lambda: batch.encode(ctx, desc, stream.cuda_stream)) if encode else (lambda: batch.decode(ctx, desc, stream.cuda_stream))
    with torch.cuda.stream(stream):
        batch.load([make(desc, 64, 16, f"{tag}_capture")])
    if before_capture is not None:
        before_capture()
    stream.synchronize()
    graph = torch.cuda.CUDAGraph()
    before = ctx.launch_count()
    with torch.cuda.graph(graph, stream=stream):
        run()
    assert ctx.launch_count() - before == 3
    for images in replay_sets(make, desc, tag):
        with torch.cuda.stream(stream):
            batch.load(images)
            before = ctx.launch_count()
            graph.replay()
        torch.cuda.synchronize()
        assert ctx.launch_count() == before
        assert (batch.statuses()[:len(images)] == 0).all()
        check(images)
    del graph


@pytest.mark.parametrize("prepared", [True, False], ids=["prepared", "unprepared"])
def test_captured_encode_replays_new_image_sets(port, prepared):
    """Premultiplied alpha: prepared by one call outside the capture, the graph holds the interior kernel; captured on a
    fresh context before the premultiply check, every image goes through the edge kernel -- the same bits."""
    import avifgpu
    desc = ENCODE_KERNELS[7][1]
    assert desc.alpha_state == abi.ALPHA_PREMULTIPLIED
    with avifgpu.Context(0) as fresh:
        def prepare():
            warm = Indirect(1)
            warm.load([Image(desc, 64, 16, "indirect_warm")])
            warm.encode(fresh, desc)
        capture_and_replay(fresh, desc, True, lambda images: assert_same_as_direct(fresh, images, port, threads=os.cpu_count()),
                           f"indirect_replay_{prepared}", prepare if prepared else None)


def test_captured_decode_replays_new_image_sets(checker, port):
    import avifgpu
    desc = DECODE_KERNELS[11][1]
    with avifgpu.Context(0) as fresh:
        capture_and_replay(fresh, desc, False,
                           lambda images: assert_decode_same_as_direct(fresh, images, pick(checker, port, True), threads=os.cpu_count()),
                           "indirect_dreplay", lambda: fresh.prepare_decode(desc))


# ---- 5. several passes of every loop ------------------------------------------------------------------------------------------

def test_encode_indirect_multipass(ctx, port):
    desc = planar(16, 4, abi.ALPHA_STRAIGHT, 10, abi.CHROMA_444, cases.NCLX_709())
    n, w, h = 64, 527, 264
    assert_passes("encode_interior", n * interior_units(w, h, 0), sm_count())
    assert_passes("encode_edge", n * edge_units(w, h, desc.chroma, False), sm_count())
    images = [Image(desc, w, h, f"indirect_multipass_{i}", beyond=True) for i in range(n)]
    batch = Indirect(n)
    batch.load(images)
    assert launches_of(ctx, lambda: batch.encode(ctx, desc)) == 3
    assert (batch.statuses() == 0).all()
    assert_same_as_direct(ctx, images, port, threads=os.cpu_count())


def test_decode_indirect_multipass(ctx, checker, port):
    desc = ycc(16, 10, abi.CHROMA_420, abi.ALPHA_STRAIGHT, cases.NCLX_2020_PQ(0))
    n, w, h = 64, 527, 263
    assert_passes("decode_interior", n * interior_units(w, h, 1), sm_count())
    assert_passes("decode_edge", n * edge_units(w, h, desc.chroma, True), sm_count())
    images = [DecImage(desc, w, h, f"indirect_dmultipass_{i}", overshoot=True) for i in range(n)]
    batch = Indirect(n)
    batch.load(images)
    ctx.prepare_decode(desc)
    assert launches_of(ctx, lambda: batch.decode(ctx, desc)) == 3
    assert (batch.statuses() == 0).all()
    assert_decode_same_as_direct(ctx, images, pick(checker, port, True), threads=os.cpu_count())


# ---- 6. host rejections, before any launch --------------------------------------------------------------------------------------

def unsupported_descriptions():
    float_pq = planar(32, 3, abi.ALPHA_NONE, 12, abi.CHROMA_420, cases.NCLX_2020_PQ())
    float_pq.transfer = abi.TRANSFER_PQ
    return [("float_pq", float_pq, True), ("gray16", abi.EncodeDesc(0, 0, 16, 1, abi.ALPHA_NONE, 10), True),
            ("reference_layout", abi.EncodeDesc(0, 0, 8, 4, abi.ALPHA_STRAIGHT, 8), True),
            ("premultiplied_ycbcr_decode", ycc(8, 8, abi.CHROMA_422, abi.ALPHA_PREMULTIPLIED, cases.NCLX_709()), False)]


@pytest.mark.parametrize("name,desc,encode", unsupported_descriptions(), ids=[u[0] for u in unsupported_descriptions()])
def test_unsupported_description_launches_nothing(ctx, name, desc, encode):
    import avifgpu
    batch = Indirect(4)
    call = batch.encode if encode else batch.decode
    before = ctx.launch_count()
    with pytest.raises(avifgpu.AvifGpuError) as info:
        call(ctx, desc)
    assert info.value.status == abi.ERR_UNSUPPORTED and ctx.launch_count() == before


def test_bad_arguments_launch_nothing(ctx):
    import avifgpu
    desc = ENCODE_KERNELS[0][1]
    ddesc = DECODE_KERNELS[0][1]
    batch = Indirect(8)
    lib = ctx.lib
    before = ctx.launch_count()
    for max_count in (0, 4097):
        for call in (ctx.encode_batch_indirect, ctx.decode_batch_indirect):
            d = desc if call == ctx.encode_batch_indirect else ddesc
            with pytest.raises(avifgpu.AvifGpuError) as info:
                call(d, batch.records, batch.count, max_count, batch.workspace, batch.status) if max_count == 0 else \
                    lib_call(lib, ctx, call == ctx.encode_batch_indirect, d, batch, max_count, batch.workspace.numel())
            assert info.value.status == BAD
    small = batch.workspace[:avifgpu.batch_workspace_bytes(8) - 1]
    with pytest.raises(avifgpu.AvifGpuError) as info:
        ctx.encode_batch_indirect(desc, batch.records, batch.count, 8, small, batch.status)
    assert info.value.status == BAD
    with pytest.raises(avifgpu.AvifGpuError) as info:
        ctx.decode_batch_indirect(ddesc, batch.records, batch.count, 8, small, batch.status)
    assert info.value.status == BAD
    pointers = [batch.records.data_ptr(), batch.count.data_ptr(), batch.workspace.data_ptr()]
    for encode in (True, False):
        fn = lib.avifgpu_encode_batch_indirect if encode else lib.avifgpu_decode_batch_indirect
        d = desc if encode else ddesc
        for k in range(3):
            args = list(pointers)
            args[k] = None
            assert fn(ctx.handle, C.byref(d), args[0], args[1], 8, args[2], batch.workspace.numel(), None, 0) == BAD
        assert fn(ctx.handle, None, *pointers[:2], 8, pointers[2], batch.workspace.numel(), None, 0) == BAD
    assert lib.avifgpu_encode_batch_indirect(None, C.byref(desc), *pointers[:2], 8, pointers[2], batch.workspace.numel(), None, 0) == BAD
    assert ctx.launch_count() == before


def lib_call(lib, ctx, encode, desc, batch, max_count, workspace_bytes):
    """A call with a max_count the binding's own capacity asserts would refuse."""
    fn = lib.avifgpu_encode_batch_indirect if encode else lib.avifgpu_decode_batch_indirect
    ctx._check(fn(ctx.handle, C.byref(desc), batch.records.data_ptr(), batch.count.data_ptr(), max_count, batch.workspace.data_ptr(),
                  workspace_bytes, batch.status.data_ptr(), 0))
