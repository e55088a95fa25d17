"""Semi-planar and MSB-aligned decode sources (avifgpu_decode_desc.source_layout): NV12 / NV16 / P010 / P016-style Cb, Cr
pairs in plane 1 and 16-bit samples with the code in their top bits, read straight from device memory by the direct device
call and both batch APIs.

  * CASES holds one case per new instantiation of the tuned YCbCr decode kernels: integer (8-bit hosts x alpha x chroma,
    interleaved; 16-bit hosts x alpha x chroma x interleaved / MSB-aligned / both) and float (PQ with the verified and the
    IEEE division, HLG, SMPTE 428 x alpha x chroma x the three layouts).  test_case_table_is_complete checks it without a GPU;
  * every case runs a mix of sizes (odd widths, so odd chroma pair counts; odd 4:2:0 heights; right strips) and of images
    the tuned kernels do not take (a misaligned interleaved plane, misaligned rows, a 1 x 1 image) under the direct call,
    whose launch counts prove the tuned and generic routes, and under both batch APIs;
  * every output row, padding sentinel included, equals today's planar decode of the same image with its planes
    de-interleaved and shifted by torch, and the compiled reference on those planes -- codes above the maximum included
    where the layout can hold them (interleaved, low-bit samples);
  * the low bits of MSB-aligned samples are random and a second set of random low bits changes no output bit; direct
    calls in row blocks with odd y0; grids that walk at least twice; one captured device-described call replayed on 1, 64
    and 256 images; the host-pointer, async and sharded calls refuse a non-zero layout with no launch; an API-9-sized
    description still decodes."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest

import cases
from avifgpu import abi
from gpu_harness import ctx  # noqa: F401
from gpu_harness import (SENTINEL, DecodeImage, Indirect, assert_passes, capture_and_replay, captured, chunk_launches, host_or_device, launches_of,
                         pick, replay_sets, run_decode_batch, sm_count, whole)

C444, C422, C420 = abi.CHROMA_444, abi.CHROMA_422, abi.CHROMA_420
NONE, STRAIGHT = abi.ALPHA_NONE, abi.ALPHA_STRAIGHT
NV, MSB, NVMSB = abi.SOURCE_CHROMA_INTERLEAVED, abi.SOURCE_MSB_ALIGNED, abi.SOURCE_CHROMA_INTERLEAVED | abi.SOURCE_MSB_ALIGNED
LAYOUT_NAMES = {NV: "nv", MSB: "msb", NVMSB: "nvmsb"}
CHROMA_NAMES = {C444: "444", C422: "422", C420: "420"}
TRANSFERS = {"pq": abi.TRANSFER_CHAR_PQ, "pq_ieee": abi.TRANSFER_CHAR_PQ, "hlg": abi.TRANSFER_CHAR_HLG, "428": abi.TRANSFER_CHAR_SMPTE428}
MATRICES = (abi.MATRIX_BT601, abi.MATRIX_BT709, abi.MATRIX_BT2020_NCL)


def ycc(host, depth, chroma, alpha, layout, matrix, full, transfer=abi.TRANSFER_CHAR_PQ, ootf=1):
    nclx = abi.Nclx(1, abi.PRIMARIES_BT2020, transfer, matrix, full)
    return abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, chroma, depth, alpha, host, nclx, hlg_apply_ootf=ootf, pq_peak_nits=1000,
                          source_layout=layout)


def case_table():
    """(name, variant, desc): variant is "int" or the float curve; depth, matrix and range rotate over the cases."""
    out = []
    keys = [(8, "int", a, c, NV) for a in (NONE, STRAIGHT) for c in (C444, C422, C420)]
    keys += [(16, "int", a, c, l) for a in (NONE, STRAIGHT) for c in (C444, C422, C420) for l in (NV, MSB, NVMSB)]
    keys += [(32, v, a, c, l) for v in TRANSFERS for a in (NONE, STRAIGHT) for c in (C444, C422, C420) for l in (NV, MSB, NVMSB)]
    for i, (host, variant, alpha, chroma, layout) in enumerate(keys):
        depth = 8 if host == 8 else (10, 12)[i % 2]
        matrix, full, ootf = MATRICES[i % 3], (i // 2) % 2, (i // 3) % 2
        transfer = TRANSFERS.get(variant, abi.TRANSFER_CHAR_PQ)
        name = f"h{host}_{variant}_{CHROMA_NAMES[chroma]}_a{int(alpha == STRAIGHT)}_{LAYOUT_NAMES[layout]}_d{depth}"
        out.append((name, variant, ycc(host, depth, chroma, alpha, layout, matrix, full, transfer, ootf)))
    return out


CASES = case_table()


def test_case_table_is_complete():
    keys = {(d.host_depth, v, d.alpha_state, d.chroma, d.source_layout) for _, v, d in CASES}
    expected = set(itertools.product([8], ["int"], (NONE, STRAIGHT), (C444, C422, C420), [NV]))
    expected |= set(itertools.product([16], ["int"], (NONE, STRAIGHT), (C444, C422, C420), (NV, MSB, NVMSB)))
    expected |= set(itertools.product([32], TRANSFERS, (NONE, STRAIGHT), (C444, C422, C420), (NV, MSB, NVMSB)))
    assert keys == expected and len(CASES) == len(expected) == 6 + 18 + 72
    assert {d.bit_depth for _, _, d in CASES if d.host_depth != 8} == {10, 12}
    assert {d.nclx.matrix_coefficients for _, _, d in CASES} == set(MATRICES)
    assert {d.nclx.full_range_flag for _, _, d in CASES} == {0, 1}


# ---- images -------------------------------------------------------------------------------------------------------------

def image(desc, w, h, seed, **kwargs):
    """A DecodeImage of seed "semi_...": codes above the maximum where the layout holds them (low-bit samples)."""
    return DecodeImage(desc, w, h, seed, prefix="semi_", overshoot=not desc.source_layout & MSB, **kwargs)


def mix(desc, seed):
    # odd widths (odd chroma pair counts), odd 4:2:0 heights, right strips, a 1 x 1 image; one image whose interleaved
    # plane is 2 bytes off the pair loads' alignment, one with misaligned rows
    sizes = [(8, 2), (37, 5), (64, 7), (129, 4), (256, 3), (7, 3), (1, 1), (100, 6)]
    images = [image(desc, w, h, f"{seed}_{i}") for i, (w, h) in enumerate(sizes)]
    images.append(image(desc, 70, 6, f"{seed}_chroma", chroma_misalign=2))
    images.append(image(desc, 64, 5, f"{seed}_rows", rows_offset=4))
    return images


def ys_of(desc):
    return 1 if desc.chroma == C420 else 0


def pair_alignment(desc):
    """DecodeYccIntBlockInterior / DecodeYccF32BlockInterior: the interleaved plane's pair loads."""
    planar = (4 if desc.chroma != C444 else 8) * (1 if desc.host_depth == 8 else 2)
    if desc.host_depth == 32:
        planar = 4 if desc.chroma != C444 else 8
        return 2 * planar
    return min(16, 2 * planar)


def eligible(im):
    d = im.desc
    f32 = d.host_depth == 32
    sample = 1 if d.host_depth == 8 else 2
    row_align = 16 if f32 or d.alpha_state == STRAIGHT else 8 * sample
    luma = 8 if f32 else 8 * sample
    chroma = pair_alignment(d) if d.source_layout & NV else (4 if d.chroma != C444 else 8) * (1 if f32 else sample)
    planes = [p for p in im.planes if p is not None]
    aligned = (im.rows.data_ptr() % row_align == 0 and im.rows.stride(0) % row_align == 0 and planes[0].data_ptr() % luma == 0 and
               im.planes[1].data_ptr() % chroma == 0 and im.planes[1].stride(0) % chroma == 0)
    return im.w >= (4 if f32 else 8) and im.h >= 1 + ys_of(d) and aligned


def has_edge(im):
    step = 4 if im.desc.host_depth == 32 else 8
    return im.w % step != 0 or (ys_of(im.desc) and im.h % 2 != 0)


def direct_launches(im):
    """A direct call: the tuned interior plus its right and bottom strips, or one generic launch."""
    if not eligible(im):
        return 1
    step = 4 if im.desc.host_depth == 32 else 8
    return 1 + (im.w % step != 0) + (ys_of(im.desc) and im.h % 2 != 0)


def assert_planar_and_reference(ctx, images, reference, threads=1):
    """Each image's rows, padding included, equal the planar decode of its torch-made planar planes, and the reference."""
    import avifgpu
    import torch
    torch.cuda.synchronize()
    for im in images:
        expected = im.alloc()
        ctx.decode_device(im.planar_desc, avifgpu.planes_from_tensors(im.torch_planar()), expected.data_ptr(), expected.stride(0), 0, im.h)
        torch.cuda.synchronize()
        got = whole(im.rows)
        assert np.array_equal(got, whole(expected)), ("planar decode", im.w, im.h)
        assert (got[:, im.row_bytes:] == SENTINEL).all(), ("padding overwritten", im.w, im.h)
        if im.w and im.h:
            want = np.ascontiguousarray(reference.decode(im.planar_desc, im.codes, threads=threads)).view(np.uint8).reshape(im.h, -1)
            assert np.array_equal(got[:, :im.row_bytes], want), ("reference", im.w, im.h)


# ---- 1. every new instantiation, under the direct call and both batch APIs ------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name,variant,desc", CASES, ids=[c[0] for c in CASES])
def test_instantiation(checker, port, name, variant, desc):
    import avifgpu
    reference = pick(checker, port, True)
    images = mix(desc, name)
    fallbacks = [im for im in images if not eligible(im)]
    assert len(fallbacks) >= 3 and any(has_edge(im) for im in images if eligible(im))
    with avifgpu.Context(0) as fresh:
        ieee = variant == "pq_ieee"  # the IEEE-division kernel: what a call captured before the PQ division is verified runs
        run = (lambda call: captured(fresh, call)) if ieee else (lambda call: launches_of(fresh, lambda: call(0)))
        if not ieee:
            fresh.prepare_decode(desc)
        # direct calls: a tuned image is its interior and strips, an image the tuned kernel does not take one generic launch
        for im in images:
            launches = run(lambda stream: im.direct(fresh, im.rows, stream=stream))
            assert launches == direct_launches(im), (im.w, im.h, launches)
        assert_planar_and_reference(fresh, images, reference)
        for im in images:
            im.rows.fill_(0)
        # the host-described batch: one chunk of one or two launches, then one direct call per image it does not take
        direct = sum(1 for im in fallbacks if im.w and im.h)
        assert run(lambda stream: run_decode_batch(fresh, desc, images, stream)) == chunk_launches(images, eligible, has_edge) + direct
        assert_planar_and_reference(fresh, images, reference)
        for im in images:
            im.rows.fill_(0)
        # the device-described batch: three launches
        batch = Indirect(16)
        batch.load(images)
        assert run(lambda stream: batch.decode(fresh, desc, stream)) == 3
        assert (batch.statuses()[:len(images)] == 0).all()
        assert_planar_and_reference(fresh, images, reference)


# ---- 2. low bits, row blocks, grids that walk twice, capture and replay ------------------------------------------------------

P010 = ycc(16, 10, C420, STRAIGHT, NVMSB, abi.MATRIX_BT2020_NCL, 0)
P016_F32 = ycc(32, 12, C420, NONE, NVMSB, abi.MATRIX_BT2020_NCL, 0)
NV12 = ycc(8, 8, C420, STRAIGHT, NV, abi.MATRIX_BT709, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("desc", [P010, P016_F32, ycc(16, 12, C444, STRAIGHT, MSB, abi.MATRIX_BT601, 1)], ids=["p010_h16", "p016_h32", "yuv444_16bit"])
def test_low_bits_change_nothing(ctx, desc):
    import torch
    ctx.prepare_decode(desc)
    a = [image(desc, w, h, "lowbits", low_bits_seed=1) for w, h in ((136, 10), (37, 5))]
    b = [image(desc, w, h, "lowbits", low_bits_seed=2) for w, h in ((136, 10), (37, 5))]
    assert not all(torch.equal(x, y) for x, y in zip(a[0].planes, b[0].planes) if x is not None)
    for images in (a, b):
        run_decode_batch(ctx, desc, images)
    for im in a + b:
        direct = im.alloc()
        im.direct(ctx, direct)
        torch.cuda.synchronize()
        assert np.array_equal(whole(direct), whole(im.rows))
    for x, y in zip(a, b):
        assert np.array_equal(whole(x.rows), whole(y.rows))


@pytest.mark.gpu
@pytest.mark.parametrize("desc", [NV12, P010, P016_F32], ids=["nv12", "p010", "p016_f32"])
def test_row_blocks_with_odd_y0(ctx, checker, port, desc):
    ctx.prepare_decode(desc)
    im = image(desc, 203, 21, "blocks")
    for y0, y1 in ((0, 3), (3, 8), (8, 9), (9, 16), (16, 21)):
        im.direct(ctx, im.rows, y0, y1 - y0)
    assert_planar_and_reference(ctx, [im], pick(checker, port, True))


@pytest.mark.gpu
@pytest.mark.parametrize("api", ["host", "device"])
@pytest.mark.parametrize("desc", [NV12, P016_F32], ids=["nv12", "p016_f32"])
def test_multipass(ctx, checker, port, api, desc):
    """64 images of 515 x 263 (4:2:0): 2 (5 for float hosts) interior units x 131 row pairs and 264 edge units per image;
    the interior grids have 3 (integer) or 2 (float) CTAs of 8 warps per SM, the edge grid 16 one-CTA workers per SM."""
    n, w, h = 64, 515, 263
    f32 = desc.host_depth == 32
    interior = -(-(w & ~(3 if f32 else 7)) // (128 if f32 else 256)) * (h // 2)
    assert_passes("ycc_f32_interior" if f32 else "ycc_int_interior", n * interior, sm_count(ctx))
    assert_passes("decode_edge", n * (h + 1), sm_count(ctx))
    images = [image(desc, w, h, f"multipass_{api}_{i}") for i in range(n)]
    ctx.prepare_decode(desc)
    host_or_device(ctx, desc, "decode", api, images, lambda done: assert_planar_and_reference(ctx, done, pick(checker, port, True), threads=os.cpu_count()))


@pytest.mark.gpu
@pytest.mark.parametrize("desc", [NV12, P016_F32], ids=["nv12", "p016_f32"])
def test_captured_call_replays_new_image_sets(checker, port, desc):
    import avifgpu
    reference = pick(checker, port, True)
    sizes = [(8, 2), (37, 5), (129, 4), (7, 3), (100, 6)]
    sets = replay_sets(lambda w, h, seed: image(desc, w, h, seed), "replay", (136, 34), sizes)
    with avifgpu.Context(0) as fresh:
        capture_and_replay(fresh, desc, "decode", image(desc, 64, 16, "replay_capture"), sets,
                           lambda images: assert_planar_and_reference(fresh, images, reference, threads=os.cpu_count()),
                           lambda: fresh.prepare_decode(desc))


# ---- 3. refusals and the API-9-sized description ----------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("call", ["sync", "async", "sharded"])
def test_host_async_and_sharded_calls_refuse_a_layout(ctx, call):
    import avifgpu
    desc = abi.DecodeDesc.from_buffer_copy(P010)
    desc.width, desc.height = 32, 8
    planar = abi.DecodeDesc.from_buffer_copy(desc)
    planar.source_layout = abi.SOURCE_PLANAR
    planes = cases.code_planes(cases.rng_for("refuse"), planar)
    planes = [planes[0], np.repeat(planes[1], 2, axis=1), None, planes[3]]
    out = np.zeros((8, 32 * 4), dtype=np.uint16)
    before = ctx.launch_count()
    with pytest.raises(avifgpu.AvifGpuError) as failure:
        if call == "sync":
            ctx.decode(desc, planes, out=out)
        elif call == "async":
            ctx.decode_async(desc, planes, out)
        else:
            with avifgpu.ShardGroup([0]) as group:
                group.decode(desc, planes, out=out)
    assert failure.value.status == abi.ERR_UNSUPPORTED
    assert ctx.launch_count() == before and not out.any()


@pytest.mark.gpu
def test_api9_sized_description_decodes(ctx, checker, port):
    """A caller built against API version 9 passes the shorter struct; it means the planar layout, whatever follows it."""
    import avifgpu
    import torch
    desc = ycc(16, 10, C420, STRAIGHT, abi.SOURCE_PLANAR, abi.MATRIX_BT709, 1)
    images = [image(desc, 77, 9, "v9")]
    old = abi.DecodeDesc.from_buffer_copy(images[0].desc)
    old.struct_size = C.sizeof(abi.DecodeDesc) - 4
    old.source_layout = NVMSB  # past the end of an API-9 struct: never read
    ctx.decode_device(old, avifgpu.planes_from_tensors(images[0].planes), images[0].rows.data_ptr(), images[0].rows.stride(0), 0, 9)
    torch.cuda.synchronize()
    assert_planar_and_reference(ctx, images, pick(checker, port, True))
    for im in images:
        im.rows.fill_(0)
    run_decode_batch(ctx, old, images)
    assert_planar_and_reference(ctx, images, pick(checker, port, True))
