"""avifgpu_encode_batch_indirect / avifgpu_decode_batch_indirect: batches whose image records and count are read from
device memory when the work runs (include/avifgpu.h, "batches described in device memory"), run by the batched kernels
of kernels_batch.cu under their workspace record source.

Every accepted image is compared bit for bit with a direct *_rows_device call of the same image and with the CPU checker
(the restatement for encode, the compiled reference for decode, by pick()), and the sentinel in the row padding must
survive.  A call is always three launches; a captured call replays whatever the records and count hold at replay.

  * every instantiation of the interior kernels (gpu_harness.ENCODE_KERNELS / DECODE_KERNELS), on a mix of aligned images,
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
from gpu_harness import ctx  # noqa: F401
from gpu_harness import (BAD, DECODE_FAULTS, DECODE_KERNELS, ENCODE_KERNELS, MIXED, SIZES, UNTOUCHED, DecodeImage, EncodeImage, Empty, Indirect,
                         assert_decode_same_as_direct, assert_passes, assert_same_as_direct, capture_and_replay, edge_units, host_or_device,
                         interior_units, launches_of, pick, planar, rejected_records, replay_sets, sm_count, ycc)

pytestmark = pytest.mark.gpu


def encode_mix(desc, seed):
    images = [EncodeImage(desc, w, h, f"{seed}_{i}", beyond=True) for i, (w, h) in enumerate(MIXED)]
    images.append(EncodeImage(desc, 64, 7, f"{seed}_misaligned", rows_misalign=4))
    return images


def decode_mix(desc, seed):
    images = [DecodeImage(desc, w, h, f"{seed}_{i}", overshoot=True) for i, (w, h) in enumerate(MIXED)]
    images.append(DecodeImage(desc, 64, 7, f"{seed}_misaligned", overshoot=True, rows_offset=4))
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

SIZES_8 = [(64, 16), (37, 9), (64, 4), (8, 2), (130, 5), (7, 5), (96, 3), (520, 4)]


def test_encode_rejects_bad_images_and_converts_the_rest(ctx, port):
    desc = ENCODE_KERNELS[5][1]
    images = [EncodeImage(desc, w, h, f"indirect_bad_{i}") for i, (w, h) in enumerate(SIZES_8)]
    rejected_records(ctx, desc, "encode", images, {2: ("rows", None), 4: ("plane", 1), 6: ("width", -3)},
                     lambda good: assert_same_as_direct(ctx, good, port))


def test_decode_rejects_bad_images_and_converts_the_rest(ctx, checker, port):
    desc = DECODE_KERNELS[5][1]
    images = [DecodeImage(desc, w, h, f"indirect_dbad_{i}") for i, (w, h) in enumerate(SIZES_8[:7])]
    ctx.prepare_decode(desc)
    rejected_records(ctx, desc, "decode", images, DECODE_FAULTS, lambda good: assert_decode_same_as_direct(ctx, good, pick(checker, port, True)))


# ---- 3. the count -----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("direction", ["encode", "decode"])
def test_count_zero_full_and_out_of_range(ctx, checker, port, direction):
    encode = direction == "encode"
    desc = ENCODE_KERNELS[3][1] if encode else DECODE_KERNELS[2][1]
    make = EncodeImage if encode else DecodeImage
    images = [make(desc, w, h, f"indirect_count_{direction}_{i}") for i, (w, h) in enumerate(SIZES)]
    batch = Indirect(len(images))
    run = (lambda: batch.encode(ctx, desc)) if encode else (lambda: batch.decode(ctx, desc))
    if not encode:
        ctx.prepare_decode(desc)
    for count in (0, len(images) + 1, -1):
        batch.load(images, count)
        assert launches_of(ctx, run) == 3
        assert all(im.untouched() for im in images if im.w and im.h), count
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

def replay(ctx, desc, direction, tag, check, prepare=None):
    """One capture replayed on 1 image; 64 images of 512 x 512; 256 mixed images."""
    make = EncodeImage if direction == "encode" else DecodeImage
    mixed = [(264, 3), (37, 9), (7, 5), (130, 1), (95, 6), (64, 7), (8, 2), (1, 1)]
    sets = replay_sets(lambda w, h, seed: make(desc, w, h, seed), tag, (512, 512), mixed, ("one", "big", "mixed"))
    capture_and_replay(ctx, desc, direction, make(desc, 64, 16, f"{tag}_capture"), sets, check, prepare)


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
            warm.load([EncodeImage(desc, 64, 16, "indirect_warm")])
            warm.encode(fresh, desc)
        replay(fresh, desc, "encode", f"indirect_replay_{prepared}", lambda images: assert_same_as_direct(fresh, images, port, threads=os.cpu_count()),
               prepare if prepared else None)


def test_captured_decode_replays_new_image_sets(checker, port):
    import avifgpu
    desc = DECODE_KERNELS[11][1]
    with avifgpu.Context(0) as fresh:
        replay(fresh, desc, "decode", "indirect_dreplay",
               lambda images: assert_decode_same_as_direct(fresh, images, pick(checker, port, True), threads=os.cpu_count()),
               lambda: fresh.prepare_decode(desc))


# ---- 5. several passes of every loop ------------------------------------------------------------------------------------------

def test_encode_indirect_multipass(ctx, port):
    desc = planar(16, 4, abi.ALPHA_STRAIGHT, 10, abi.CHROMA_444, cases.NCLX_709())
    n, w, h = 64, 527, 264
    assert_passes("encode_interior", n * interior_units(w, h, 0), sm_count(ctx))
    assert_passes("encode_edge", n * edge_units(w, h, desc.chroma, False), sm_count(ctx))
    images = [EncodeImage(desc, w, h, f"indirect_multipass_{i}", beyond=True) for i in range(n)]
    host_or_device(ctx, desc, "encode", "device", images, lambda done: assert_same_as_direct(ctx, done, port, threads=os.cpu_count()))


def test_decode_indirect_multipass(ctx, checker, port):
    desc = ycc(16, 10, abi.CHROMA_420, abi.ALPHA_STRAIGHT, cases.NCLX_2020_PQ(0))
    n, w, h = 64, 527, 263
    assert_passes("ycc_int_interior", n * interior_units(w, h, 1), sm_count(ctx))
    assert_passes("decode_edge", n * edge_units(w, h, desc.chroma, True), sm_count(ctx))
    images = [DecodeImage(desc, w, h, f"indirect_dmultipass_{i}", overshoot=True) for i in range(n)]
    ctx.prepare_decode(desc)
    host_or_device(ctx, desc, "decode", "device", images,
                   lambda done: assert_decode_same_as_direct(ctx, done, pick(checker, port, True), threads=os.cpu_count()))


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
