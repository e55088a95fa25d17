"""Batches of HDR images with each image's content light level (avifgpu_encode_batch_device_light_level,
avifgpu_encode_batch_indirect_light_level; DESIGN.md sections 4.4 and 5).

Every case converts one batch of SIZES and MIXED images (padded planes, sentinels) through both calls and holds them to
three things: the planes equal avifgpu_encode_batch_device's of the same images, padding included; each device_acc[i]
equals a zeroed accumulator after one avifgpu_encode_rows_device_light_level call of image i; and that accumulator equals
light_level_spec.accumulate of the checker's own R'G'B' codes.  CASES covers every instantiation of the batched
light-level interior kernel (RGB, RGBA straight, RGBA premultiplied x chroma x destination layout), each under both
record sources (a host chunk and the workspace), and the edge kernel under both.  On top: NaN / +-inf / negatives /
over-peak / saturated inputs and values inside the step table's fuzzy bands, launch counts, grids that walk the units at
least twice, more than 64 images, the device-described call's rejections, a captured graph replayed on a new image set
after an in-graph memset, a capture before avifgpu_prepare_encode, and the refusals, which launch nothing."""
import ctypes as C

import numpy as np
import pytest

import cases
import light_level_spec as spec
from avifgpu import abi
from gpu_harness import BAD, CHUNK, MIXED, SENTINEL, SIZES, UNTOUCHED, EncodeImage, Empty, Indirect, launches_of, sm_count, whole

pytestmark = pytest.mark.gpu

C444, C422, C420 = abi.CHROMA_444, abi.CHROMA_422, abi.CHROMA_420
NONE, STRAIGHT, PREMUL = abi.ALPHA_NONE, abi.ALPHA_STRAIGHT, abi.ALPHA_PREMULTIPLIED
NV, MSB = abi.SOURCE_CHROMA_INTERLEAVED, abi.SOURCE_MSB_ALIGNED
LAYOUTS = {"planar": 0, "nv": NV, "msb": MSB, "nvmsb": NV | MSB}
CHROMAS = {"444": C444, "422": C422, "420": C420}
HOSTS = {"rgb": (3, NONE), "rgba": (4, STRAIGHT), "premul": (4, PREMUL)}
ACC_BYTES = C.sizeof(abi.LightLevel)
# EncodeLightF32BatchKernel's grid (LaunchEncodeLightBatchChunk): one CTA of kLightBatchWarps = 16 warps per SM at most, a
# warp taking one unit at a time
LIGHT_WARPS_PER_CTA, LIGHT_CTAS_PER_SM = 16, 1


def assert_light_interior_passes(units, sms):
    """The interior grid the launcher starts for `units` units has at most half as many warps (GridFor's cap)."""
    warps = max(1, min(-(-units // LIGHT_WARPS_PER_CTA), sms * LIGHT_CTAS_PER_SM)) * LIGHT_WARPS_PER_CTA
    assert units >= 2 * warps, f"{units} units, {warps} warps at {sms} SMs"


def desc_of(channels, alpha, depth, chroma=C420, dest=0, layout=abi.LAYOUT_PLANAR_YCBCR, transfer=abi.TRANSFER_PQ, down=abi.DOWN_FILTER_BOX):
    return abi.EncodeDesc(0, 0, 32, channels, alpha, depth, transfer, 1000, layout, chroma if layout == abi.LAYOUT_PLANAR_YCBCR else C444, down,
                          abi.GRAY16_LUT, cases.NCLX_2020_PQ(), dest_layout=dest)


# (name, desc): every (host, chroma, layout) of EncodeLightF32BatchKernel, the depth alternating between 12 and 10 bits
CASES = []
for i, (hname, (channels, alpha)) in enumerate(HOSTS.items()):
    for j, (cname, chroma) in enumerate(CHROMAS.items()):
        for k, (lname, dest) in enumerate(LAYOUTS.items()):
            depth = 12 if (i + j + k) % 2 == 0 else 10
            down = abi.DOWN_FILTER_TOP_LEFT if lname == "nv" and chroma != C444 else abi.DOWN_FILTER_BOX
            CASES.append((f"{hname}_d{depth}_{cname}_{lname}", desc_of(channels, alpha, depth, chroma, dest, down=down)))


def test_case_table_covers_every_light_instantiation():
    keys = {(d.host_channels, d.alpha_state, d.chroma, d.dest_layout) for _, d in CASES}
    assert keys == {(c, a, ch, l) for c, a in HOSTS.values() for ch in CHROMAS.values() for l in LAYOUTS.values()}
    assert {d.image_bit_depth for _, d in CASES} == {10, 12}
    assert len({n for n, _ in CASES}) == len(CASES)


@pytest.fixture(scope="module")
def gpu():
    import avifgpu
    ctx = avifgpu.Context(0)
    yield ctx
    ctx.close()


def accs(n):
    import torch
    return torch.zeros((max(n, 1), 3), dtype=torch.int64, device="cuda")


def acc_list(tensor, n):
    import torch
    torch.cuda.synchronize()
    raw = tensor.cpu().numpy()
    return [{"max_code": int(raw[i, 0] & 0xFFFFFFFF), "reserved": int(raw[i, 0] >> 32), "level_sum": int(raw[i, 1]), "pixels": int(raw[i, 2])}
            for i in range(n)]


ZERO = {"max_code": 0, "reserved": 0, "level_sum": 0, "pixels": 0}


def band_rows(port, desc, rng, h, w):
    """Samples right at the PQ steps of the image depth: linear values whose code changes there, nudged by a few ulps, so
    that many samples fall inside the step table's fuzzy bands."""
    max_code = (1 << desc.image_bit_depth) - 1
    codes = rng.integers(1, max_code, h * w * desc.host_channels)
    # PQ inverse of (k - 0.5) / max at the description's peak: the decision points of the quantiser
    e = np.clip((codes - 0.5) / max_code, 0, 1).astype(np.float64)
    m1, m2, c1, c2, c3 = 0.1593017578125, 78.84375, 0.8359375, 18.8515625, 18.6875
    p = e ** (1 / m2)
    linear = (np.maximum(p - c1, 0) / (c2 - c3 * p)) ** (1 / m1) * (10000.0 / desc.pq_peak_nits)
    v = linear.astype(np.float32).view(np.int32) + rng.integers(-3, 4, linear.shape).astype(np.int32)
    out = v.view(np.float32).reshape(h, w, desc.host_channels)
    if desc.host_channels == 4:
        out[..., 3] = np.where(rng.random((h, w)) < 0.3, np.float32(0.5), np.float32(1.0))
    return out


def special_rows(rng, h, w, channels):
    pool = np.array([np.nan, -np.nan, np.inf, -np.inf, -1.0, -0.0, 0.0, 1.0, 100.0, 1e30, 7.5, 1e-38, 3.4e38], np.float32)
    v = rng.choice(pool, h * w * channels).astype(np.float32).reshape(h, w, channels)
    saturated = rng.random((h, w)) < 0.2  # pure red / blue at peak: chroma at its clip
    v[saturated, 0] = 100.0
    v[saturated, 1] = 0.0
    if channels == 4:
        v[..., 3] = np.where(rng.random((h, w)) < 0.3, np.float32(0.5), np.float32(1.0))
    return v


def make_images(desc, sizes, tag, port=None, rows_misalign=0):
    """Images of `sizes`: seeded random rows, every third one special values and every third one fuzzy-band values."""
    import torch
    images = []
    for i, (w, h) in enumerate(sizes):
        im = EncodeImage(desc, w, h, f"{tag}_{i}", prefix="lbatch_", rows_misalign=rows_misalign if i % 4 == 3 else 0)
        if w and h and i % 3 != 0:
            rng = cases.rng_for(f"lbatch_{tag}_{i}_values")
            host = special_rows(rng, h, w, desc.host_channels) if i % 3 == 1 else band_rows(port, desc, rng, h, w)
            im.host = np.ascontiguousarray(host.reshape(h, w * desc.host_channels))
            im.rows.copy_(torch.from_numpy(im.host.view(np.uint8).reshape(h, im.row_bytes)).cuda())
        images.append(im)
    return images


def records(images):
    import avifgpu
    return avifgpu.batch_images_from_tensors([im.record() for im in images])


def reference_desc(desc, w, h):
    d = abi.EncodeDesc.from_buffer_copy(desc)
    d.layout, d.dest_layout, d.chroma = abi.LAYOUT_REFERENCE, 0, C444
    d.width, d.height = w, h
    return d


def spec_acc(port, im):
    if im.w == 0 or im.h == 0:
        return ZERO
    codes = port.encode(reference_desc(im.desc, im.w, im.h), im.host, threads=8)[0]
    channels = im.desc.host_channels
    return spec.accumulate(codes, channels if channels >= 3 else 1, spec.levels(port, im.desc.image_bit_depth))


def direct_accs(ctx, images):
    """One zeroed accumulator per image after its own avifgpu_encode_rows_device_light_level call (into scratch planes)."""
    import avifgpu
    acc = accs(len(images))
    for i, im in enumerate(images):
        if im.w and im.h:
            scratch = im.fresh_planes()
            ctx.encode_device_light_level(im.desc, im.rows.data_ptr(), im.rows.stride(0), avifgpu.planes_from_tensors(scratch),
                                          acc.data_ptr() + i * ACC_BYTES)
    return acc_list(acc, len(images))


def plain_planes(ctx, desc, images):
    """avifgpu_encode_batch_device of the same images, into fresh sentinel planes: each plane's whole bytes."""
    import avifgpu
    outs = [im.fresh_planes() for im in images]
    recs = [(im.w, im.h, im.rows, out) for im, out in zip(images, outs)]
    ctx.encode_batch_device(desc, avifgpu.batch_images_from_tensors(recs))
    return [[None if p is None else whole(p) for p in out] for out in outs]


def assert_planes(images, expected, skip=()):
    for i, (im, want) in enumerate(zip(images, expected)):
        for k, (got, w) in enumerate(zip(im.planes, want)):
            if got is None:
                continue
            if i in skip:
                assert (whole(got) == SENTINEL).all(), ("a skipped image was written", i, k)
            else:
                assert np.array_equal(whole(got), w), ("planes differ from avifgpu_encode_batch_device", i, k, im.w, im.h)


def reset(images):
    for im in images:
        for p in im.planes:
            if p is not None:
                p.fill_(SENTINEL)


def host_launches(images):
    """The host-described light-level batch's launches: per chunk of up to 64 tuned images one, one more when one of them
    has a right strip or an odd last 4:2:0 row; one generic launch for every other non-empty image (width < 4, misaligned
    rows, a one-row 4:2:0 image)."""
    ys = 1 if images[0].desc.chroma == C420 else 0
    tuned = [im for im in images if im.w >= 4 and im.h >> ys and im.rows.data_ptr() % 16 == 0]
    direct = sum(1 for im in images if im.w and im.h and im not in tuned)
    edges = [(im.w % 4 != 0) or (ys and im.h % 2 == 1) for im in tuned]
    return sum(1 + any(edges[i:i + CHUNK]) for i in range(0, len(tuned), CHUNK)) + direct


@pytest.mark.parametrize("name, desc", CASES, ids=[c[0] for c in CASES])
def test_both_calls_match_the_direct_calls(gpu, port, name, desc):
    import avifgpu
    d = abi.EncodeDesc.from_buffer_copy(desc)
    gpu.prepare_encode(d)
    images = make_images(d, SIZES + MIXED, name, port, rows_misalign=4)
    expected = plain_planes(gpu, d, images)
    direct = direct_accs(gpu, images)
    for i, im in enumerate(images):
        assert direct[i] == spec_acc(port, im), ("direct call vs the checker's codes", i, im.w, im.h)
        assert direct[i]["pixels"] == im.w * im.h
    listed = images[:3] + [Empty()] + images[3:]  # an empty image leaves its entry alone
    n = len(listed)
    want = direct[:3] + [ZERO] + direct[3:]

    # host-described
    acc = accs(n)
    launches = launches_of(gpu, lambda: gpu.encode_batch_device_light_level(d, records(listed), acc.data_ptr()))
    assert launches == host_launches(images), launches
    assert_planes(images, expected)
    assert acc_list(acc, n) == want

    # device-described
    reset(images)
    batch = Indirect(n)
    batch.load(listed)
    acc = accs(n)
    launches = launches_of(gpu, lambda: gpu.encode_batch_indirect_light_level(d, batch.records, batch.count, n, batch.workspace, acc.data_ptr(),
                                                                              batch.status))
    assert launches == 3
    assert (batch.statuses() == 0).all()
    assert_planes(images, expected)
    assert acc_list(acc, n) == want


@pytest.mark.parametrize("name", ["rgb_d12_420_planar", "premul_d10_444_nv", "rgba_d12_422_msb"])
def test_grids_walk_the_units_twice_and_batches_pass_64(gpu, port, name):
    """A batch whose interior units are at least twice the interior grid's warps (one CTA of 16 warps per SM), with more
    than one chunk, and edges on every image."""
    d = abi.EncodeDesc.from_buffer_copy(next(c for n, c in CASES if n == name))
    gpu.prepare_encode(d)
    sms = sm_count(gpu)
    ys = 1 if d.chroma == C420 else 0
    w = 1024 + 3
    h = 2 * ((2 * 16 * sms) // (70 * (w // 128)) + 2)  # rows per image so that 70 images hold 2 x warps units
    sizes = [(w, h + 1)] * 70
    per_image = (w // 128) * (h >> ys)  # the interior: 1024 x h pixels (h even), units of 128 pixels x (1 << ys) rows
    assert_light_interior_passes(CHUNK * per_image, sms)
    images = make_images(d, sizes, f"walk_{name}", port)
    expected = plain_planes(gpu, d, images)
    direct = direct_accs(gpu, images)
    acc = accs(len(images))
    launches = launches_of(gpu, lambda: gpu.encode_batch_device_light_level(d, records(images), acc.data_ptr()))
    assert launches == 4  # two chunks of interiors and strips
    assert_planes(images, expected)
    assert acc_list(acc, len(images)) == direct
    reset(images)
    batch = Indirect(len(images))
    batch.load(images)
    acc = accs(len(images))
    assert launches_of(gpu, lambda: gpu.encode_batch_indirect_light_level(d, batch.records, batch.count, len(images), batch.workspace,
                                                                          acc.data_ptr(), batch.status)) == 3
    assert_planes(images, expected)
    assert acc_list(acc, len(images)) == direct


def test_device_rejections_leave_their_entries(gpu, port):
    import torch
    d = abi.EncodeDesc.from_buffer_copy(CASES[0][1])
    gpu.prepare_encode(d)
    images = make_images(d, [(64, 8), (37, 9), (130, 6), (8, 2), (95, 4)], "reject", port)
    expected = plain_planes(gpu, d, images)
    direct = direct_accs(gpu, images)
    recs = records(images)
    recs[1].rows = None
    recs[2].planes.data[1] = None
    recs[3].width = -1
    batch = Indirect(len(images))
    batch.load(recs)
    acc = accs(len(images))
    acc.fill_(5)
    gpu.encode_batch_indirect_light_level(d, batch.records, batch.count, len(images), batch.workspace, acc.data_ptr(), batch.status)
    torch.cuda.synchronize()
    assert list(batch.statuses()) == [0, BAD, BAD, BAD, 0]
    got = acc_list(acc, len(images))
    five = {"max_code": 5, "reserved": 0, "level_sum": 5, "pixels": 5}
    for i in (1, 2, 3):
        assert got[i] == five, i
    for i in (0, 4):
        want = direct[i]
        assert got[i] == {"max_code": max(5, want["max_code"]), "reserved": 0, "level_sum": want["level_sum"] + 5, "pixels": want["pixels"] + 5}
    assert_planes(images, expected, skip=(1, 2, 3))
    # a count out of range touches nothing
    reset(images)
    batch.load(images, count=len(images) + 1)
    acc.fill_(0)
    assert launches_of(gpu, lambda: gpu.encode_batch_indirect_light_level(d, batch.records, batch.count, len(images), batch.workspace,
                                                                          acc.data_ptr(), batch.status)) == 3
    assert (batch.statuses() == BAD).all()
    assert acc_list(acc, len(images)) == [ZERO] * len(images)
    assert all(im.untouched() for im in images)


@pytest.mark.parametrize("prepared", [True, False], ids=["tuned", "before_prepare"])
def test_captured_graph_replays_on_a_new_image_set(port, prepared):
    import avifgpu
    import torch
    ctx = avifgpu.Context(0)
    try:
        if not prepared:
            ctx.set_table_autobuild(-1)
        d = desc_of(3, NONE, 12, C420, NV | MSB)
        if prepared:
            ctx.prepare_encode(d)
        cap = 24
        batch = Indirect(cap)
        acc = accs(cap)
        first = make_images(d, SIZES, "capture_a", port)
        batch.load(first)
        stream = torch.cuda.Stream()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        before = ctx.launch_count()
        with torch.cuda.graph(graph, stream=stream):
            acc.zero_()  # an in-graph memset of the accumulators
            ctx.encode_batch_indirect_light_level(d, batch.records, batch.count, cap, batch.workspace, acc.data_ptr(), batch.status,
                                                  torch.cuda.current_stream().cuda_stream)
        assert ctx.launch_count() - before == 3
        for tag, sizes in (("capture_b", MIXED), ("capture_c", SIZES + MIXED)):
            images = make_images(d, sizes, tag, port)
            batch.load(images)
            acc.fill_(12345)
            torch.cuda.synchronize()
            graph.replay()
            torch.cuda.synchronize()
            got = acc_list(acc, len(images))
            for i, im in enumerate(images):
                assert got[i] == spec_acc(port, im), (tag, i)
            assert acc_list(acc, cap)[len(images):] == [ZERO] * (cap - len(images))
            expected = plain_planes(ctx, d, images)
            assert_planes(images, expected)
        del graph
        if not prepared:
            # before prepare every image goes through the edge kernel: host-described, every image is one direct call
            images = make_images(d, [(64, 8), (37, 9)], "capture_host", port)
            acc = accs(2)
            assert launches_of(ctx, lambda: ctx.encode_batch_device_light_level(d, records(images), acc.data_ptr())) == 2
            assert acc_list(acc, 2) == [spec_acc(port, im) for im in images]
    finally:
        ctx.close()


REFUSALS = [("int8", dict(host_depth=8, transfer=abi.TRANSFER_CLIP)), ("int16", dict(host_depth=16, transfer=abi.TRANSFER_CLIP)),
            ("hlg", dict(transfer=abi.TRANSFER_HLG)), ("smpte428", dict(transfer=abi.TRANSFER_SMPTE428)), ("clip", dict(transfer=abi.TRANSFER_CLIP))]


@pytest.mark.parametrize("what, change", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refusals_launch_nothing(gpu, what, change):
    import avifgpu
    d = desc_of(3, NONE, 10)
    for k, v in change.items():
        setattr(d, k, v)
    if what == "hlg":
        d.hlg_extension = abi.HLG_OETF
        d.nclx = cases.NCLX_2020_HLG()
    images = [EncodeImage(d, 64, 4, f"refuse_{what}")]
    batch = Indirect(1)
    batch.load(images)
    acc = accs(1)
    for call in (lambda: gpu.encode_batch_device_light_level(d, records(images), acc.data_ptr()),
                 lambda: gpu.encode_batch_indirect_light_level(d, batch.records, batch.count, 1, batch.workspace, acc.data_ptr(), batch.status)):
        before = gpu.launch_count()
        with pytest.raises(avifgpu.AvifGpuError) as failure:
            call()
        assert failure.value.status == abi.ERR_UNSUPPORTED and gpu.launch_count() == before
    assert acc_list(acc, 1) == [ZERO] and images[0].untouched() and (batch.statuses() == UNTOUCHED).all()


@pytest.mark.parametrize("what", ["reference", "gray"])
def test_device_described_refuses_reference_layout_and_gray(gpu, what):
    import avifgpu
    d = desc_of(3, NONE, 12, layout=abi.LAYOUT_REFERENCE) if what == "reference" else desc_of(1, NONE, 12, layout=abi.LAYOUT_REFERENCE)
    images = [EncodeImage(d, 64, 4, f"refuse_{what}")]
    batch = Indirect(1)
    batch.load(images)
    acc = accs(1)
    before = gpu.launch_count()
    with pytest.raises(avifgpu.AvifGpuError) as failure:
        gpu.encode_batch_indirect_light_level(d, batch.records, batch.count, 1, batch.workspace, acc.data_ptr(), batch.status)
    assert failure.value.status == abi.ERR_UNSUPPORTED and gpu.launch_count() == before
    assert images[0].untouched()


def test_host_described_takes_reference_layout_and_gray_through_direct_calls(gpu, port):
    for d in (desc_of(3, NONE, 12, layout=abi.LAYOUT_REFERENCE), desc_of(2, STRAIGHT, 10, layout=abi.LAYOUT_REFERENCE)):
        gpu.prepare_encode(d)
        images = make_images(d, [(64, 8), (37, 9)], f"ref_{d.host_channels}", port)
        expected = plain_planes(gpu, d, images)
        direct = direct_accs(gpu, images)
        assert direct == [spec_acc(port, im) for im in images]
        acc = accs(2)
        gpu.encode_batch_device_light_level(d, records(images), acc.data_ptr())
        assert_planes(images, expected)
        assert acc_list(acc, 2) == direct


def test_null_accumulator_is_a_bad_parameter(gpu):
    d = desc_of(3, NONE, 12)
    images = [EncodeImage(d, 64, 4, "null_acc")]
    batch = Indirect(1)
    batch.load(images)
    before = gpu.launch_count()
    assert gpu.lib.avifgpu_encode_batch_device_light_level(gpu.handle, C.byref(d), records(images), 1, None, None) == BAD
    assert gpu.lib.avifgpu_encode_batch_indirect_light_level(gpu.handle, C.byref(d), batch.records.data_ptr(), batch.count.data_ptr(), 1,
                                                             batch.workspace.data_ptr(), batch.workspace.numel(), None, None, None) == BAD
    assert gpu.launch_count() == before and images[0].untouched()
