"""Semi-planar and MSB-aligned encode destinations (avifgpu_encode_desc.dest_layout): NV12 / NV16 / P010 / P016-style Cb, Cr
pairs in plane 1 and 16-bit samples with the code in their top bits, written straight into device memory by the direct
device call and both batch APIs.

  * CASES holds one case per new tuned instantiation: integer planar (8/16-bit hosts x 8-bit planes interleaved, or 10/12-
    bit planes interleaved / MSB-aligned / both x channels and alpha x chroma), flat (PQ on the compact table at 12 and 10
    bits, SMPTE 428 on the compact table at 10 bits and the two-level one at 12 bits), RGBA (PQ, SMPTE 428) and clip, each
    float family x chroma x the three layouts.  test_case_table_is_complete checks it without a GPU;
  * every case runs a mix of sizes (odd widths, so right strips and odd chroma pair counts; odd 4:2:0 heights) and of
    images the tuned kernels do not take (a misaligned interleaved plane, misaligned rows, narrow images) under the direct
    call, whose launch counts prove the tuned and generic routes, and under both batch APIs (float hosts: the host-described
    one runs direct calls, the device-described one refuses them, as for planar planes);
  * planes 0, 1 and 3 of every image, row padding included, equal the planar encode of the same description and rows with
    its planes re-interleaved and shifted by torch; a sentinel-filled plane-2 buffer passed with an interleaved layout
    comes back untouched; one case per family is also held to the independent model (encode_spec.py) on random and
    saturated-site rows;
  * untuned descriptions (HLG save, row matrix) in the generic kernel; row blocks at several even y0; grids that walk at
    least twice; one captured device-described call replayed on 1, 64 and 256 images; every refusal (host-pointer, async,
    both sharded calls, the reference layout, 8-bit MSB-aligned, unknown bits) launches nothing; an API-10-sized
    description encodes planar."""
import ctypes as C
import itertools

import numpy as np
import pytest

import cases
import encode_spec
from avifgpu import abi
from gpu_harness import ctx  # noqa: F401
from gpu_harness import (SENTINEL, EncodeImage, Indirect, assert_passes, capture_and_replay, chunk_launches, host_or_device, launches_of,
                         replay_sets, run_batch, sm_count, whole)

C444, C422, C420 = abi.CHROMA_444, abi.CHROMA_422, abi.CHROMA_420
NONE, STRAIGHT, PREMUL = abi.ALPHA_NONE, abi.ALPHA_STRAIGHT, abi.ALPHA_PREMULTIPLIED
NV, MSB, NVMSB = abi.SOURCE_CHROMA_INTERLEAVED, abi.SOURCE_MSB_ALIGNED, abi.SOURCE_CHROMA_INTERLEAVED | abi.SOURCE_MSB_ALIGNED
LAYOUT_NAMES = {NV: "nv", MSB: "msb", NVMSB: "nvmsb"}
CHROMA_NAMES = {C444: "444", C422: "422", C420: "420"}
ALPHA_NAMES = {(3, NONE): "rgb", (4, STRAIGHT): "rgba", (4, PREMUL): "premul"}
NCLX = (cases.NCLX_709, cases.NCLX_2020_PQ, cases.NCLX_DERIVED)
# float families: (name, transfer, image depth, channels) -- the flat kernel's reachable (curve, table) pairs, RGBA, clip
FLOAT_FAMILIES = [("flat_pq12", abi.TRANSFER_PQ, 12, 3), ("flat_pq10", abi.TRANSFER_PQ, 10, 3), ("flat_428_10", abi.TRANSFER_SMPTE428, 10, 3),
                  ("flat_428_12", abi.TRANSFER_SMPTE428, 12, 3), ("rgba_pq", abi.TRANSFER_PQ, 12, 4), ("rgba_428", abi.TRANSFER_SMPTE428, 10, 4),
                  ("clip", abi.TRANSFER_CLIP, 12, 3)]


def encode_desc(host, channels, alpha, depth, chroma, dest, nclx, transfer=abi.TRANSFER_CLIP, down=abi.DOWN_FILTER_BOX):
    return abi.EncodeDesc(0, 0, host, channels, alpha, depth, transfer, 80, abi.LAYOUT_PLANAR_YCBCR, chroma, down, abi.GRAY16_LUT, nclx,
                          dest_layout=dest)


def case_table():
    """(name, family, desc): family is "int" or a float family; matrix, depth and down filter rotate over the cases."""
    out = []
    keys = [(h, "int", ca, 8, c, NV) for h in (8, 16) for ca in ALPHA_NAMES for c in (C444, C422, C420)]
    keys += [(h, "int", ca, None, c, l) for h in (8, 16) for ca in ALPHA_NAMES for c in (C444, C422, C420) for l in (NV, MSB, NVMSB)]
    keys += [(32, f, None, None, c, l) for f in FLOAT_FAMILIES for c in (C444, C422, C420) for l in (NV, MSB, NVMSB)]
    for i, (host, family, channel_alpha, depth, chroma, layout) in enumerate(keys):
        nclx = NCLX[i % 3]()
        down = abi.DOWN_FILTER_TOP_LEFT if i % 5 == 4 and chroma != C444 else abi.DOWN_FILTER_BOX
        if family == "int":
            channels, alpha = channel_alpha
            depth = depth or (10, 12)[i % 2]
            name = f"h{host}_{ALPHA_NAMES[channel_alpha]}_d{depth}_{CHROMA_NAMES[chroma]}_{LAYOUT_NAMES[layout]}"
            out.append((name, "int", encode_desc(host, channels, alpha, depth, chroma, layout, nclx, down=down)))
        else:
            fname, transfer, depth, channels = family
            alpha = (NONE, STRAIGHT, PREMUL)[i % 3] if channels == 4 else NONE
            if alpha == NONE and channels == 4:
                alpha = STRAIGHT
            name = f"h32_{fname}_{CHROMA_NAMES[chroma]}_{LAYOUT_NAMES[layout]}"
            out.append((name, fname, encode_desc(32, channels, alpha, depth, chroma, layout, cases.NCLX_2020_PQ(), transfer, down)))
    return out


CASES = case_table()


def test_case_table_is_complete():
    ints = {(d.host_depth, d.host_channels, d.alpha_state, d.image_bit_depth > 8, d.chroma, d.dest_layout) for _, f, d in CASES if f == "int"}
    expected = set(itertools.product((8, 16), [(3, NONE), (4, STRAIGHT), (4, PREMUL)], [False], (C444, C422, C420), [NV]))
    expected |= set(itertools.product((8, 16), [(3, NONE), (4, STRAIGHT), (4, PREMUL)], [True], (C444, C422, C420), (NV, MSB, NVMSB)))
    assert ints == {(h, c, a, wide, ch, l) for h, (c, a), wide, ch, l in expected} and len(ints) == 18 + 54
    floats = {(f, d.chroma, d.dest_layout) for _, f, d in CASES if f != "int"}
    assert floats == set(itertools.product([f[0] for f in FLOAT_FAMILIES], (C444, C422, C420), (NV, MSB, NVMSB)))
    assert len(CASES) == 72 + 63 == len({name for name, _, _ in CASES})
    assert {d.image_bit_depth for _, f, d in CASES if f == "int" and d.image_bit_depth > 8} == {10, 12}


# ---- images -------------------------------------------------------------------------------------------------------------

def image(desc, w, h, seed, **kwargs):
    """An EncodeImage of seed "semi_encode_...", 16-bit hosts with samples above 32768."""
    return EncodeImage(desc, w, h, seed, prefix="semi_encode_", beyond=True, **kwargs)


def assert_layout_of_planar(ctx, images):
    """Planes 0, 1 and 3 of every image, padding included, are the planar encode re-laid; plane 2 of an interleaved layout
    is untouched."""
    import torch
    torch.cuda.synchronize()
    for im in images:
        want = im.expected(ctx)
        for k, plane in enumerate(im.planes):
            if plane is None:
                continue
            got = whole(plane)
            if k == 2 and im.desc.dest_layout & NV:
                assert (got == SENTINEL).all(), ("plane 2 written", im.w, im.h)
                continue
            assert np.array_equal(got[:, :plane.shape[1]], want[k]), ("planar encode, re-laid", im.w, im.h, k)
            assert (got[:, plane.shape[1]:] == SENTINEL).all(), ("padding overwritten", im.w, im.h, k)


def reset(images):
    for im in images:
        for p in im.planes:
            if p is not None:
                p.fill_(SENTINEL)


def mix(desc, seed):
    # right strips and odd chroma pair counts, odd 4:2:0 heights, narrow images, a 1 x 1 image; one image whose
    # interleaved plane is 2 bytes off the paired stores' alignment, one with misaligned rows
    sizes = [(8, 2), (37, 5), (64, 7), (129, 4), (256, 3), (7, 3), (1, 1), (100, 6)]
    images = [image(desc, w, h, f"{seed}_{i}") for i, (w, h) in enumerate(sizes)]
    images.append(image(desc, 70, 6, f"{seed}_chroma", chroma_misalign=2))
    images.append(image(desc, 64, 5, f"{seed}_rows", rows_misalign=4))
    return images


def ys_of(desc):
    return 1 if desc.chroma == C420 else 0


def eligible(im):
    """EncodeRgbIntBlockInterior / EncodeRgbF32BlockInterior, restated."""
    d = im.desc
    f32 = d.host_depth == 32
    sample = im.sample_bytes
    sites = 4 if d.chroma != C444 else 8
    if f32:
        row_align, luma, chroma = 16, 8, (2 if d.dest_layout & NV else 1) * (4 if d.chroma != C444 else 8)
    else:
        row_align = 16 if (8 * d.host_channels * d.host_depth // 8) % 16 == 0 else 8
        luma = 8 * sample
        chroma = min(16, 2 * sites * sample) if d.dest_layout & NV else sites * sample
    p = im.planes
    aligned = (im.rows.data_ptr() % row_align == 0 and im.rows.stride(0) % row_align == 0 and p[0].data_ptr() % luma == 0 and
               p[1].data_ptr() % chroma == 0 and p[1].stride(0) % chroma == 0 and
               (p[3] is None or (p[3].data_ptr() % luma == 0 and p[3].stride(0) % luma == 0)))
    return im.w >= (4 if f32 else 8) and im.h >= 1 + ys_of(d) and aligned


def has_edge(im):
    step = 4 if im.desc.host_depth == 32 else 8
    return im.w % step != 0 or (ys_of(im.desc) and im.h % 2 != 0)


def direct_launches(im):
    if not eligible(im):
        return 1
    step = 4 if im.desc.host_depth == 32 else 8
    return 1 + (im.w % step != 0) + (ys_of(im.desc) and im.h % 2 != 0)


@pytest.fixture(scope="module")
def tables():
    """One context for the float cases, so each (curve, depth) builds its step table once."""
    import avifgpu
    context = avifgpu.Context(0)
    yield context
    context.close()


# ---- 1. every new instantiation, under the direct call and both batch APIs ------------------------------------------------

SPEC_CASES = {"h16_premul_d12_420_nvmsb", "h8_rgb_d8_420_nv", "h32_flat_pq12_420_nvmsb", "h32_flat_428_12_422_nv", "h32_rgba_pq_420_nvmsb",
              "h32_clip_444_msb"}


@pytest.mark.gpu
@pytest.mark.parametrize("name,family,desc", CASES, ids=[c[0] for c in CASES])
def test_instantiation(tables, request, name, family, desc):
    import avifgpu
    images = mix(desc, name)
    fallbacks = [im for im in images if not eligible(im)]
    assert len(fallbacks) >= 3 and any(has_edge(im) for im in images if eligible(im))
    if family == "int":
        ctx = avifgpu.Context(0)
        images[0].direct(ctx)  # the first call of a premultiplied description makes the premultiply check
        reset(images[:1])
    else:
        ctx = tables
        stats = ctx.prepare_encode(desc).as_dict() if family != "clip" else None
        assert stats is None or (stats["valid"] == 1 and stats["verify_mismatches"] == 0)
    try:
        # direct calls: a tuned image is its interior and strips, an image the tuned kernel does not take one generic launch
        for im in images:
            assert launches_of(ctx, lambda: im.direct(ctx)) == direct_launches(im), (im.w, im.h)
        assert_layout_of_planar(ctx, images)
        reset(images)
        # the host-described batch: one chunk of one or two launches (integer hosts), one direct call per other image
        direct = sum(direct_launches(im) for im in images if im.w and im.h and (family != "int" or not eligible(im)))
        chunks = chunk_launches(images, eligible, has_edge) if family == "int" else 0
        assert launches_of(ctx, lambda: run_batch(ctx, desc, images)) == chunks + direct
        assert_layout_of_planar(ctx, images)
        reset(images)
        # the device-described batch: three launches for integer hosts; float hosts are refused, as for planar planes
        batch = Indirect(16)
        batch.load(images)
        if family == "int":
            assert launches_of(ctx, lambda: batch.encode(ctx, desc)) == 3
            assert (batch.statuses()[:len(images)] == 0).all()
            assert_layout_of_planar(ctx, images)
        else:
            before = ctx.launch_count()
            with pytest.raises(avifgpu.AvifGpuError) as failure:
                batch.encode(ctx, desc)
            assert failure.value.status == abi.ERR_UNSUPPORTED and ctx.launch_count() == before
        # the independent model, on random and saturated-site rows
        if name in SPEC_CASES:
            ref = request.getfixturevalue("ref")
            for extreme in (False, True):
                im = image(desc, 259, 37, f"{name}_spec", extreme=extreme)
                im.direct(ctx)
                import torch
                torch.cuda.synchronize()
                encode_spec.assert_matches(ref, im.planar_desc, im.host, im.codes_of_output(), f"{name} extreme={extreme}")
    finally:
        if family == "int":
            ctx.close()


# ---- 2. untuned descriptions, row blocks, grids that walk twice, capture and replay -------------------------------------------

P010 = encode_desc(16, 4, STRAIGHT, 10, C420, NVMSB, cases.NCLX_2020_PQ())
NV12 = encode_desc(8, 3, NONE, 8, C420, NV, cases.NCLX_709())
P016_F32 = encode_desc(32, 3, NONE, 12, C420, NVMSB, cases.NCLX_2020_PQ(), abi.TRANSFER_PQ)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hlg", "row_matrix"])
def test_untuned_descriptions_take_the_generic_kernel(tables, kind):
    desc = abi.EncodeDesc.from_buffer_copy(P016_F32)
    if kind == "hlg":
        desc.transfer, desc.hlg_extension = abi.TRANSFER_HLG, 1
    else:
        desc.row_matrix_enabled = 1
        desc.row_matrix[:] = [0.9, 0.05, 0.05, 0.1, 0.8, 0.1, 0.0, 0.1, 0.9]
    tables.prepare_encode(desc)
    images = [image(desc, w, h, f"untuned_{kind}") for w, h in ((136, 10), (37, 5))]
    for im in images:
        assert launches_of(tables, lambda: im.direct(tables)) == 1
    assert_layout_of_planar(tables, images)


@pytest.mark.gpu
@pytest.mark.parametrize("desc", [NV12, P010, P016_F32], ids=["nv12", "p010", "p016_f32"])
def test_row_blocks(tables, desc):
    tables.prepare_encode(desc)
    im = image(desc, 203, 21, "blocks")
    for y0, y1 in ((0, 4), (4, 10), (10, 12), (12, 20), (20, 21)):
        im.direct(tables, y0=y0, nrows=y1 - y0)
    assert_layout_of_planar(tables, [im])


@pytest.mark.gpu
@pytest.mark.parametrize("api", ["host", "device"])
@pytest.mark.parametrize("desc", [NV12, P010], ids=["nv12", "p010"])
def test_multipass(ctx, api, desc):
    """64 images of 1031 x 300 (4:2:0): 4 interior units x 150 row pairs and 150 edge units per image; the interior grid
    has 16 CTAs of 8 warps per SM, the edge grid 16 one-CTA workers per SM -- both walk at least twice."""
    n, w, h = 64, 1031, 300
    assert_passes("encode_interior", n * 4 * (h // 2), sm_count(ctx))
    assert_passes("encode_edge", n * (h // 2), sm_count(ctx))
    images = [image(desc, w, h, f"multipass_{api}_{i}") for i in range(n)]
    images[0].direct(ctx)
    host_or_device(ctx, desc, "encode", api, images, lambda done: assert_layout_of_planar(ctx, done))


@pytest.mark.gpu
@pytest.mark.parametrize("desc", [NV12, P010], ids=["nv12", "p010"])
def test_captured_call_replays_new_image_sets(desc):
    import avifgpu
    sizes = [(8, 2), (37, 5), (129, 4), (7, 3), (100, 6)]
    sets = replay_sets(lambda w, h, seed: image(desc, w, h, seed), "replay", (136, 34), sizes)
    warm = image(desc, 64, 16, "replay_capture")
    with avifgpu.Context(0) as fresh:
        # the premultiply check, outside the capture
        capture_and_replay(fresh, desc, "encode", warm, sets, lambda images: assert_layout_of_planar(fresh, images), lambda: warm.direct(fresh))


# ---- 3. refusals and the API-10-sized description ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("call", ["sync", "async", "sharded", "sharded_device"])
def test_host_async_and_sharded_calls_refuse_a_layout(ctx, call):
    import avifgpu
    desc = abi.EncodeDesc.from_buffer_copy(P010)
    desc.width, desc.height = 32, 8
    rows = cases.int_host_rows(cases.rng_for("refuse"), 8, 32, 4, 16)
    planes = avifgpu.alloc_planes(abi.encode_plane_shapes(desc), np.uint16)
    before = ctx.launch_count()
    with pytest.raises(avifgpu.AvifGpuError) as failure:
        if call == "sync":
            ctx.encode(desc, rows, planes=planes)
        elif call == "async":
            ctx.encode_async(desc, rows, planes)
        else:
            with avifgpu.ShardGroup([0]) as group:
                try:
                    if call == "sharded":
                        group.encode(desc, rows, planes=planes)
                    else:
                        im = image(desc, 32, 8, "refuse_device")
                        group.encode_device(desc, [im.rows.data_ptr()], [im.rows.stride(0)], avifgpu.planes_from_tensors(im.planes))
                finally:
                    assert group.launch_count() == 0
    assert failure.value.status == abi.ERR_UNSUPPORTED
    assert ctx.launch_count() == before and all((p == 0xCD).all() for p in planes if p is not None)


@pytest.mark.gpu
@pytest.mark.parametrize("fault,status", [("reference_layout", abi.ERR_UNSUPPORTED), ("msb_8bit", abi.ERR_BAD_PARAM), ("unknown_bits", abi.ERR_BAD_PARAM)])
def test_device_calls_refuse_bad_layouts(ctx, fault, status):
    import avifgpu
    desc = abi.EncodeDesc.from_buffer_copy(NV12)
    if fault == "reference_layout":
        desc.layout = abi.LAYOUT_REFERENCE
    elif fault == "msb_8bit":
        desc.dest_layout = NVMSB
    else:
        desc.dest_layout = 4
    im = image(NV12, 64, 8, "bad_layout")
    before = ctx.launch_count()
    for call in (lambda: im.direct(ctx, desc=desc), lambda: run_batch(ctx, desc, [im]), lambda: Indirect(4).encode(ctx, desc)):
        with pytest.raises(avifgpu.AvifGpuError) as failure:
            call()
        assert failure.value.status == status
    assert ctx.launch_count() == before
    assert all((whole(p) == SENTINEL).all() for p in im.planes if p is not None)


@pytest.mark.gpu
@pytest.mark.parametrize("desc", [P010, P016_F32], ids=["p010", "p016_f32"])
def test_api10_sized_description_encodes_planar(tables, desc):
    """A caller built against API version 10 passes the shorter struct; it means the planar layout, whatever follows it."""
    tables.prepare_encode(desc)
    planar = abi.EncodeDesc.from_buffer_copy(desc)
    planar.dest_layout = abi.SOURCE_PLANAR
    images = [image(planar, 77, 9, "v10"), image(planar, 136, 10, "v10b")]
    old = abi.EncodeDesc.from_buffer_copy(images[0].desc)
    old.struct_size = C.sizeof(abi.EncodeDesc) - 4
    old.dest_layout = NVMSB  # past the end of an API-10 struct: never read
    images[0].direct(tables, desc=old)
    run_batch(tables, old, images[1:])
    assert_layout_of_planar(tables, images)
