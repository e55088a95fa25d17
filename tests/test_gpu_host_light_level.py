"""The content light level measured by the host-pointer encodes (avifgpu_encode_rows_light_level, _async_light_level and
_sharded_light_level; include/avifgpu.h, DESIGN.md sections 5 and 6), on an H100.

The light-level host calls run the plain host calls' slice loop, with one device accumulator per pipeline slot that each
slice clears, feeds and copies into a pinned mirror; merging a mirror into the caller's host accumulator is a debt of the
slot, paid on retire or before the slot's next slice rewrites the mirror.  Every case checks:
  * the planes, row padding included, are bit-identical to the plain host call's, with equal launch counts;
  * the accumulator equals the one avifgpu_encode_rows_device_light_level adds over the same rows -- and, on small
    shapes, the one computed from the restatement's reference-layout codes (light_level_spec.py);
  * `reserved` is never written.
ROUTES has the routes of the device light-level cases that the host calls take (planar destination only): the flat
kernel at 12 and 10 bits in every chroma mode and the interleaved reference layout, RGBA straight and premultiplied,
Gray and Gray+A, and the generic kernel with no table or with a row matrix.  Then: blocks of at least three slices
with a short last slice (pinned and pageable rows, padded strides), row blocks that add up across sync and async calls,
two images' blocks interleaved on one context with decodes and plain encodes between them (complete after
avifgpu_wait of a ticket, and after avifgpu_synchronize), the refusals, and the shard group."""
import ctypes as C

import numpy as np
import pytest

import cases
import light_level_spec as spec
from avifgpu import abi

pytestmark = pytest.mark.gpu

C444, C422, C420 = abi.CHROMA_444, abi.CHROMA_422, abi.CHROMA_420
NONE, STRAIGHT, PREMUL = abi.ALPHA_NONE, abi.ALPHA_STRAIGHT, abi.ALPHA_PREMULTIPLIED
CHROMAS = {"444": C444, "422": C422, "420": C420}
SLICE_BYTES = 32 << 20  # SliceRows, avifgpu_api.cu: 32 MiB of host rows per slice, at least 2 rows, even
RESERVED = 0x5A5A5A5A  # what every accumulator's `reserved` starts with, and must keep


def slice_rows(nrows, row_bytes):
    return min(max(SLICE_BYTES // row_bytes, 2) & ~1, nrows)


def desc_of(channels, alpha, depth, layout=abi.LAYOUT_PLANAR_YCBCR, chroma=C420, transfer=abi.TRANSFER_PQ, row_matrix=None):
    d = abi.EncodeDesc(0, 0, 32, channels, alpha, depth, transfer, 1000, layout, chroma if layout == abi.LAYOUT_PLANAR_YCBCR else C444,
                       abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, cases.NCLX_2020_PQ())
    if row_matrix is not None:
        d.row_matrix_enabled = 1
        for i, v in enumerate(row_matrix):
            d.row_matrix[i] = v
    return d


# (name, desc, route): "tuned" = a prepared context, "generic" = a context that never builds tables (the generic kernel)
ROUTES = []
for depth in (12, 10):
    for cname, chroma in CHROMAS.items():
        ROUTES.append((f"flat_d{depth}_{cname}", desc_of(3, NONE, depth, chroma=chroma), "tuned"))
    ROUTES.append((f"flat_d{depth}_interleaved", desc_of(3, NONE, depth, layout=abi.LAYOUT_REFERENCE), "tuned"))
for alpha, aname in ((STRAIGHT, "straight"), (PREMUL, "premul")):
    for cname, chroma in CHROMAS.items():
        ROUTES.append((f"rgba_{aname}_{cname}", desc_of(4, alpha, 12, chroma=chroma), "tuned"))
ROUTES += [("gray", desc_of(1, NONE, 12, layout=abi.LAYOUT_REFERENCE), "tuned"),
           ("gray_alpha", desc_of(2, STRAIGHT, 12, layout=abi.LAYOUT_REFERENCE), "tuned"),
           ("gray_alpha_premul", desc_of(2, PREMUL, 10, layout=abi.LAYOUT_REFERENCE), "tuned"),
           ("generic_no_table_planar", desc_of(3, NONE, 12), "generic"),
           ("generic_no_table_rgba", desc_of(4, PREMUL, 10, chroma=C422), "generic"),
           ("generic_no_table_interleaved", desc_of(4, STRAIGHT, 12, layout=abi.LAYOUT_REFERENCE), "generic"),
           ("generic_no_table_gray", desc_of(1, NONE, 10, layout=abi.LAYOUT_REFERENCE), "generic"),
           ("generic_row_matrix", desc_of(3, NONE, 12, row_matrix=[0.6274, 0.3293, 0.0433, 0.0691, 0.9195, 0.0114, 0.0164, 0.0880, 0.8956]), "tuned"),
           ("generic_row_matrix_rgba", desc_of(4, STRAIGHT, 10, chroma=C444, row_matrix=[1.2, -0.1, -0.1, -0.05, 1.1, -0.05, 0.0, -0.2, 1.2]), "tuned")]


def route(name):
    return next(r for r in ROUTES if r[0] == name)


@pytest.fixture(scope="module")
def contexts():
    import avifgpu
    tuned, generic = avifgpu.Context(0), avifgpu.Context(0)
    generic.set_table_autobuild(-1)
    yield {"tuned": tuned, "generic": generic}
    tuned.close()
    generic.close()


def sized(desc, w, h):
    d = abi.EncodeDesc.from_buffer_copy(desc)
    d.width, d.height = w, h
    return d


def new_acc():
    return abi.LightLevel(reserved=RESERVED)


def acc_dict(acc):
    got = acc.as_dict()
    assert got.pop("reserved") == RESERVED, "reserved was written"
    return got


def without_reserved(acc):
    return {k: v for k, v in acc.items() if k != "reserved"}


def host_rows(desc, w, h, seed, specials=False, row_pad=0, ctx=None):
    """Seeded float rows of (h, w * channels), on a stride `row_pad` floats wider than the payload; page-locked when `ctx`
    is given."""
    data = cases.float_host_rows(cases.rng_for(f"host_light_{seed}"), h, w, desc.host_channels, specials=specials).reshape(h, -1)
    shape = (h, data.shape[1] + row_pad)
    backing = ctx.pinned_array(shape, np.float32) if ctx is not None else np.zeros(shape, np.float32)
    backing[:, :data.shape[1]] = data
    return backing[:, :data.shape[1]]


def device_acc(ctx, desc, rows):
    """What avifgpu_encode_rows_device_light_level adds over the same rows (a whole-image call)."""
    import avifgpu
    import torch
    dev = torch.from_numpy(np.ascontiguousarray(rows).view(np.uint8)).cuda()
    planes = [None if s is None else torch.empty((s[0], s[1] * 2), dtype=torch.uint8, device="cuda") for s in abi.encode_plane_shapes(desc)]
    acc = torch.zeros(3, dtype=torch.int64, device="cuda")
    ctx.encode_device_light_level(desc, dev.data_ptr(), dev.stride(0), avifgpu.planes_from_tensors(planes), acc.data_ptr())
    torch.cuda.synchronize()
    raw = acc.cpu().numpy()
    return {"max_code": int(raw.view(np.uint32)[0]), "level_sum": int(raw[1]), "pixels": int(raw[2])}


def spec_acc(port, desc, rows):
    """The accumulator from the restatement's reference-layout codes of the same rows."""
    ref = abi.EncodeDesc.from_buffer_copy(desc)
    ref.layout, ref.dest_layout, ref.chroma = abi.LAYOUT_REFERENCE, 0, C444
    codes = port.encode(ref, np.ascontiguousarray(rows), threads=8)[0]
    return without_reserved(spec.accumulate(codes, desc.host_channels if desc.host_channels >= 3 else 1, spec.levels(port, desc.image_bit_depth)))


def planes_for(desc, pad=0):
    import avifgpu
    return avifgpu.alloc_planes(abi.encode_plane_shapes(desc), abi.code_dtype(desc.image_bit_depth), pad)


def backing(planes):
    return [None if p is None else p.base.copy() for p in planes]


def same_planes(a, b):
    return all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(backing(a), backing(b)))


def launches(ctx, call):
    before = ctx.launch_count()
    result = call()
    return ctx.launch_count() - before, result


def check_against_plain(ctx, desc, rows, pad=0):
    """Plain host call vs light-level host call of the same rows: planes (padding included) and launches; returns the
    light-level call's accumulator."""
    plain_launches, plain = launches(ctx, lambda: ctx.encode(desc, rows, planes=planes_for(desc, pad)))
    acc = new_acc()
    light_launches, light = launches(ctx, lambda: ctx.encode_light_level(desc, rows, acc, planes=planes_for(desc, pad)))
    assert light_launches == plain_launches, (light_launches, plain_launches)
    assert same_planes(light, plain), "planes differ from the plain host call"
    return acc_dict(acc)


@pytest.mark.parametrize("name, desc, kind", ROUTES, ids=[r[0] for r in ROUTES])
def test_route(contexts, port, name, desc, kind):
    ctx = contexts[kind]
    for i, (w, h) in enumerate([(509, 66), (37, 9)]):
        d = sized(desc, w, h)
        if kind == "tuned":
            ctx.prepare_encode(d)
        rows = host_rows(d, w, h, f"{name}_{i}", specials=i == 0)
        got = check_against_plain(ctx, d, rows, pad=5)
        assert got == device_acc(ctx, d, rows), name
        assert got == spec_acc(port, d, rows), name
        assert got["pixels"] == w * h


@pytest.mark.parametrize("memory", ["pinned", "pageable"])
@pytest.mark.parametrize("name", ["flat_d12_420", "rgba_premul_422", "gray_alpha", "generic_no_table_planar"])
def test_frames_over_several_slices(contexts, name, memory):
    _, desc, kind = route(name)
    ctx = contexts[kind]
    w = 4096
    row_bytes = w * desc.host_channels * 4
    step = slice_rows(1 << 20, row_bytes)
    h = (2 * step + step // 3) | 1  # three slices, the last one short, with an odd last row
    d = sized(desc, w, h)
    assert -(-h // slice_rows(h, row_bytes)) >= 3 and h % slice_rows(h, row_bytes) != 0
    if kind == "tuned":
        ctx.prepare_encode(d)
    rows = host_rows(d, w, h, f"slices_{name}", row_pad=7, ctx=ctx if memory == "pinned" else None)
    got = check_against_plain(ctx, d, rows, pad=3)
    assert got == device_acc(ctx, d, rows)


@pytest.mark.parametrize("name", ["flat_d12_420", "rgba_straight_444", "gray", "generic_no_table_rgba"])
def test_row_blocks_add_up(contexts, port, name):
    _, desc, kind = route(name)
    ctx = contexts[kind]
    w, h = 300, 39
    d = sized(desc, w, h)
    if kind == "tuned":
        ctx.prepare_encode(d)
    rows = host_rows(d, w, h, f"blocks_{name}", ctx=ctx)
    whole_planes = ctx.encode(d, rows, planes=planes_for(d, 4))
    acc = new_acc()
    planes = planes_for(d, 4)
    for i, (y0, n) in enumerate([(0, 12), (12, 0), (12, 20), (32, 7)]):  # an empty block, an odd last row
        if i % 2:
            ctx.wait(ctx.encode_async_light_level(d, rows[y0:y0 + n], planes, acc, y0=y0, nrows=n))
        else:
            ctx.encode_light_level(d, rows[y0:y0 + n], acc, y0=y0, nrows=n, planes=planes)
    assert same_planes(planes, whole_planes)
    assert acc_dict(acc) == device_acc(ctx, d, rows) == spec_acc(port, d, rows)


def interleaved_saves(ctx, d, images, block, finish):
    """Two images' row blocks sent in turn through two page-locked row buffers that alternate like the shuttle's, each
    image into its own accumulator, with a pageable decode and a plain asynchronous encode on the same context between
    them.  finish(tickets, accs) completes the accumulators.  Returns the accumulators and planes."""
    w, h = d.width, d.height
    buffers = [ctx.pinned_array((block, w * d.host_channels), np.float32) for _ in range(2)]
    accs = [new_acc(), new_acc()]
    planes = [planes_for(d, 2), planes_for(d, 2)]
    ddesc = abi.DecodeDesc(w, 64, abi.COLORSPACE_YCBCR, C420, 10, abi.ALPHA_NONE, 32, cases.NCLX_2020_HLG())
    codes = cases.code_planes(np.random.default_rng(7), ddesc)
    decoded = np.zeros((64, w * 3), np.float32)
    other = host_rows(d, w, h, "interleaved_other")
    other_planes = planes_for(d)
    tickets = [[], []]
    calls = 0
    for top in range(0, h, block):
        n = min(block, h - top)
        for i, rows in enumerate(images):
            buffer = buffers[calls & 1]
            buffer[:n] = rows[top:top + n]
            tickets[i].append(ctx.encode_async_light_level(d, buffer[:n], planes[i], accs[i], y0=top, nrows=n))
            calls += 1
        ctx.decode_async(ddesc, codes, decoded)
        ctx.encode_async(d, other[top:top + n], other_planes, y0=top, nrows=n)
    finish(tickets, accs)
    ctx.wait()  # the decodes and plain encodes after the last light-level call, before their buffers go
    return accs, planes


@pytest.mark.parametrize("finish", ["wait", "synchronize"])
def test_async_blocks_of_two_images_interleaved(contexts, finish):
    ctx = contexts["tuned"]
    _, desc, _ = route("flat_d12_420")
    w, h, block = 4096, 3101, 1500  # blocks of three slices, the last block short with an odd last row
    d = sized(desc, w, h)
    ctx.prepare_encode(d)
    images = [host_rows(d, w, h, f"interleaved_{i}") for i in range(2)]
    expected = [device_acc(ctx, d, rows) for rows in images]

    def complete(tickets, accs):
        if finish == "synchronize":
            ctx.synchronize()
            return
        for i in range(2):  # image 0's last ticket comes first: waiting for it does not cover image 1's last block
            ctx.wait(tickets[i][-1])
            assert acc_dict(accs[i]) == expected[i], i

    accs, planes = interleaved_saves(ctx, d, images, block, complete)
    for i in range(2):
        assert acc_dict(accs[i]) == expected[i], i
        assert same_planes(planes[i], ctx.encode(d, images[i], planes=planes_for(d, 2))), i


def refusal_cases():
    out = []
    for host_depth in (8, 16):
        d = desc_of(3, NONE, 10, transfer=abi.TRANSFER_CLIP)
        d.host_depth = host_depth
        out.append((f"host{host_depth}", d, abi.ERR_UNSUPPORTED))
    out.append(("smpte428", desc_of(3, NONE, 12, transfer=abi.TRANSFER_SMPTE428), abi.ERR_UNSUPPORTED))
    out.append(("clip", desc_of(3, NONE, 12, transfer=abi.TRANSFER_CLIP), abi.ERR_UNSUPPORTED))
    nv = desc_of(3, NONE, 12)
    nv.dest_layout = abi.SOURCE_CHROMA_INTERLEAVED
    out.append(("dest_layout", nv, abi.ERR_UNSUPPORTED))
    out.append(("null_acc", desc_of(3, NONE, 12), abi.ERR_BAD_PARAM))
    return out


SENTINEL_ACC = dict(max_code=0xA5A5A5A5, reserved=0x5A5A5A5A, level_sum=0x0123456789ABCDEF, pixels=0xFEDCBA9876543210)


@pytest.mark.parametrize("form", ["sync", "async", "sharded"])
@pytest.mark.parametrize("name, desc, status", refusal_cases(), ids=[c[0] for c in refusal_cases()])
def test_refusals(contexts, name, desc, status, form):
    import avifgpu
    w, h = 64, 4
    d = sized(desc, w, h)
    rows = np.zeros((h, w * d.host_channels), abi.host_dtype(d.host_depth))
    planes = planes_for(d)
    before = backing(planes)
    acc = abi.LightLevel(**SENTINEL_ACC)
    ref = None if name == "null_acc" else C.byref(acc)
    p = abi.planes_from_arrays(planes)
    if form == "sharded":
        group = avifgpu.ShardGroup([0])
        try:
            got = group.lib.avifgpu_encode_rows_sharded_light_level(group.handle, C.byref(d), rows.ctypes.data, rows.strides[0], 0, h, C.byref(p), ref)
            assert group.launch_count() == 0
        finally:
            group.close()
    else:
        ctx = contexts["tuned"]
        before_launches, ticket = ctx.launch_count(), C.c_int64(-1)
        if form == "sync":
            got = ctx.lib.avifgpu_encode_rows_light_level(ctx.handle, C.byref(d), rows.ctypes.data, rows.strides[0], 0, h, C.byref(p), ref)
        else:
            got = ctx.lib.avifgpu_encode_rows_async_light_level(ctx.handle, C.byref(d), rows.ctypes.data, rows.strides[0], 0, h, C.byref(p), ref,
                                                                C.byref(ticket))
            assert ticket.value == -1, "a refused call takes no ticket"
        assert ctx.launch_count() == before_launches
    assert got == status, (got, status)
    assert acc.as_dict() == SENTINEL_ACC
    assert all((a is None and b is None) or np.array_equal(a, b) for a, b in zip(backing(planes), before))


def group_devices():
    import torch
    return [[0]] + ([list(range(torch.cuda.device_count()))] if torch.cuda.device_count() > 1 else [])


@pytest.mark.parametrize("devices", ["one", "all"])
def test_sharded(contexts, devices):
    import avifgpu
    sets = group_devices()
    if devices == "all" and len(sets) == 1:
        pytest.skip("one visible GPU")
    _, desc, _ = route("rgba_straight_420")
    w, h = 777, 301
    d = sized(desc, w, h)
    rows = host_rows(d, w, h, "sharded")
    single = new_acc()
    single_planes = contexts["tuned"].encode_light_level(d, rows, single, planes=planes_for(d, 2))
    with avifgpu.ShardGroup(sets[0] if devices == "one" else sets[1]) as group:
        acc = new_acc()
        planes = group.encode_light_level(d, rows, acc, planes=planes_for(d, 2))
        assert acc_dict(acc) == acc_dict(single) == device_acc(contexts["tuned"], d, rows)
        assert same_planes(planes, single_planes)
        refused = sized(desc_of(3, NONE, 12, transfer=abi.TRANSFER_SMPTE428), w, h)
        kept = abi.LightLevel(**SENTINEL_ACC)
        with pytest.raises(avifgpu.AvifGpuError) as failure:
            group.encode_light_level(refused, np.zeros((h, w * 3), np.float32), kept)
        assert failure.value.status == abi.ERR_UNSUPPORTED and kept.as_dict() == SENTINEL_ACC
