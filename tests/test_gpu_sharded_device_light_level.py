"""The content light level measured by the sharded device-pointer encode (avifgpu_encode_rows_sharded_device_light_level;
include/avifgpu.h, DESIGN.md sections 5 and 7), on H100s.

Each member with a non-empty row block measures it into a partial in its own memory and copies the partial into a gather
array in the owner's memory; the owner's stream waits for every member and one single-warp kernel adds the partials into
the caller's accumulator.  Every case runs on a one-member group, and on two-member and all-device groups where the box
has them, and checks:
  * the accumulator equals what one avifgpu_encode_rows_device_light_level call over the whole image adds on one device,
    and (small shapes) what the restatement's reference-layout codes give (light_level_spec.py); `reserved` is never
    written;
  * the planes, row padding included, are bit-identical to the plain sharded device call's;
  * every member launches what the plain call launches there, and the owner one more (the merge).
Both routes: a prepared group (tuned kernels, level tables) and a fresh group that never builds tables (the generic
kernel evaluates the levels).  Then heights with uneven blocks, an odd last 4:2:0 row and empty blocks;
back-to-back calls with no synchronize between them; and the refusals, which launch nothing and leave the accumulator as
it was."""
import ctypes as C

import numpy as np
import pytest

import cases
import light_level_spec as spec
from avifgpu import abi

pytestmark = pytest.mark.gpu

C444, C422, C420 = abi.CHROMA_444, abi.CHROMA_422, abi.CHROMA_420
NONE, STRAIGHT, PREMUL = abi.ALPHA_NONE, abi.ALPHA_STRAIGHT, abi.ALPHA_PREMULTIPLIED
RESERVED = 0x5A5A5A5A  # what every accumulator's `reserved` starts with, and must keep
PAD = 6                # bytes of row padding after every plane row; the calls must leave them alone
FILL = 0xCD


def device_count():
    import torch
    return torch.cuda.device_count()


def groups():
    n = device_count()
    return [[0]] + ([[0, 1]] if n >= 2 else []) + ([list(range(n))] if n > 2 else [])


def desc_of(channels, alpha, depth, chroma=C420, layout=abi.LAYOUT_PLANAR_YCBCR, transfer=abi.TRANSFER_PQ, nclx=None):
    return abi.EncodeDesc(0, 0, 32, channels, alpha, depth, transfer, 1000, layout, chroma if layout == abi.LAYOUT_PLANAR_YCBCR else C444,
                          abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, nclx if nclx is not None else cases.NCLX_2020_PQ())


DESCS = {
    "rgb_d12_420": desc_of(3, NONE, 12, C420),
    "rgba_straight_d10_444": desc_of(4, STRAIGHT, 10, C444),
    "rgba_premul_d12_422": desc_of(4, PREMUL, 12, C422),
    "gray_alpha_reference": desc_of(2, STRAIGHT, 12, layout=abi.LAYOUT_REFERENCE),
}


def sized(desc, w, h):
    d = abi.EncodeDesc.from_buffer_copy(desc)
    d.width, d.height = w, h
    return d


def host_rows(desc, seed, specials=True):
    return cases.float_host_rows(cases.rng_for(f"sharded_device_light_{seed}"), desc.height, desc.width, desc.host_channels, specials=specials)


class Group:
    """A shard group with the frame's row blocks resident on their members; `generic`: members never build tables."""

    def __init__(self, devices, generic=False):
        import avifgpu
        self.group = avifgpu.ShardGroup(devices)
        self.devices = devices
        self.lib = self.group.lib
        if generic:
            for i in range(len(devices)):
                assert self.lib.avifgpu_set_table_autobuild(self.context(i), -1) == 0

    def close(self):
        self.group.close()

    def context(self, i):
        return self.lib.avifgpu_shard_group_context(self.group.handle, i)

    def launches(self):
        return [int(self.lib.avifgpu_launch_count(self.context(i))) for i in range(len(self.devices))]

    def settle(self):
        """torch's uploads and fills done: the library's streams do not wait for torch's."""
        import torch
        for device in self.devices:
            torch.cuda.synchronize(device)

    def upload(self, desc, rows):
        """Member r's row block in member r's memory: (pointers, strides, tensors)."""
        import avifgpu
        import torch
        pointers, strides, keep = [], [], []
        for member, (y0, count) in enumerate(avifgpu.shard_row_blocks(0, desc.height, len(self.devices))):
            t = torch.from_numpy(np.ascontiguousarray(rows[y0:y0 + count])).to(f"cuda:{self.devices[member]}")
            keep.append(t)
            pointers.append(t.data_ptr() if count > 0 else None)
            strides.append(t.stride(0) * 4 if count > 0 else 0)
        return pointers, strides, keep

    def owner_planes(self, desc, owner=0):
        """Whole-image planes in the owner's memory, PAD bytes of FILL after every row: (padded backings, abi.Planes)."""
        import avifgpu
        import torch
        backings, views = [], []
        for shape in abi.encode_plane_shapes(desc):
            if shape is None:
                backings.append(None)
                views.append(None)
                continue
            b = torch.full((shape[0], shape[1] * 2 + PAD), FILL, dtype=torch.uint8, device=f"cuda:{self.devices[owner]}")
            backings.append(b)
            views.append(b[:, :shape[1] * 2])
        return backings, avifgpu.planes_from_tensors(views)

    def new_acc(self, owner=0):
        import torch
        acc = torch.zeros(3, dtype=torch.int64, device=f"cuda:{self.devices[owner]}")
        acc[0] = RESERVED << 32
        return acc

    def plain(self, desc, rows, owner=0):
        """The plain sharded device call: (planes, launches per member)."""
        pointers, strides, _keep = self.upload(desc, rows)
        backings, planes = self.owner_planes(desc, owner)
        before = self.launches()
        self.settle()
        self.group.encode_device(desc, pointers, strides, planes, owner=owner)
        self.group.synchronize()
        return host_planes(backings), [a - b for a, b in zip(self.launches(), before)]

    def light(self, desc, rows, acc, owner=0):
        """The light-level call into `acc`: (planes, launches per member)."""
        pointers, strides, _keep = self.upload(desc, rows)
        backings, planes = self.owner_planes(desc, owner)
        before = self.launches()
        self.settle()
        self.group.encode_device_light_level(desc, pointers, strides, planes, acc.data_ptr(), owner=owner)
        self.group.synchronize()
        return host_planes(backings), [a - b for a, b in zip(self.launches(), before)]


def host_planes(backings):
    return [None if b is None else b.cpu().numpy() for b in backings]


def same_planes(a, b):
    return all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(a, b))


def acc_dict(acc):
    raw = acc.cpu().numpy()
    words = raw.view(np.uint32)
    assert int(words[1]) == RESERVED, "reserved was written"
    return {"max_code": int(words[0]), "level_sum": int(raw[1]), "pixels": int(raw[2])}


def single_device_acc(gpu, desc, rows):
    """What one avifgpu_encode_rows_device_light_level call over the whole image adds on one device."""
    import avifgpu
    import torch
    dev = torch.from_numpy(np.ascontiguousarray(rows)).cuda()
    planes = [None if s is None else torch.empty((s[0], s[1] * 2), dtype=torch.uint8, device="cuda") for s in abi.encode_plane_shapes(desc)]
    acc = torch.zeros(3, dtype=torch.int64, device="cuda")
    acc[0] = RESERVED << 32
    gpu.encode_device_light_level(desc, dev.data_ptr(), dev.stride(0) * 4, avifgpu.planes_from_tensors(planes), acc.data_ptr())
    torch.cuda.synchronize()
    return acc_dict(acc)


def spec_acc(port, desc, rows):
    ref = abi.EncodeDesc.from_buffer_copy(desc)
    ref.layout, ref.dest_layout, ref.chroma = abi.LAYOUT_REFERENCE, 0, C444
    codes = port.encode(ref, np.ascontiguousarray(rows), threads=8)[0]
    got = spec.accumulate(codes, desc.host_channels if desc.host_channels >= 3 else 1, spec.levels(port, desc.image_bit_depth))
    return {k: v for k, v in got.items() if k != "reserved"}


def check_against_plain(g, desc, rows, owner=0):
    """Plain call (once to warm first-use work, once counted) vs the light-level call: planes with padding, launches per
    member; returns the light-level call's accumulator."""
    g.plain(desc, rows, owner)
    plain_planes, plain_launches = g.plain(desc, rows, owner)
    acc = g.new_acc(owner)
    light_planes, light_launches = g.light(desc, rows, acc, owner)
    assert same_planes(light_planes, plain_planes), "planes differ from the plain sharded device call"
    expected = list(plain_launches)
    expected[owner] += 1
    assert light_launches == expected, (light_launches, plain_launches)
    return acc_dict(acc)


@pytest.mark.parametrize("route", ["tuned", "generic"])
@pytest.mark.parametrize("name", list(DESCS))
@pytest.mark.parametrize("devices", groups(), ids=lambda d: f"{len(d)}gpu")
def test_equals_the_single_device_call(gpu, port, devices, name, route):
    d = sized(DESCS[name], 509, 66)
    rows = host_rows(d, name)
    g = Group(devices, generic=route == "generic")
    try:
        if route == "tuned":
            g.group.prepare_encode(d)
        got = check_against_plain(g, d, rows)
    finally:
        g.close()
    assert got == single_device_acc(gpu, d, rows) == spec_acc(port, d, rows), name
    assert got["pixels"] == d.width * d.height


@pytest.mark.parametrize("height", [1, 2, 3, 5, 67, 1031])
@pytest.mark.parametrize("devices", groups(), ids=lambda d: f"{len(d)}gpu")
def test_uneven_and_empty_blocks(gpu, devices, height):
    """Uneven blocks, an odd last 4:2:0 row, and (on a group of two or more) heights that leave members with empty
    blocks; the rows carry NaN, +-inf, negative and above-peak samples."""
    import avifgpu
    d = sized(DESCS["rgb_d12_420"], 300, height)
    rows = host_rows(d, f"height_{height}")
    blocks = avifgpu.shard_row_blocks(0, height, len(devices))
    if len(devices) > 1 and height <= 3:
        assert any(count == 0 for _, count in blocks), blocks
    g = Group(devices)
    try:
        g.group.prepare_encode(d)
        got = check_against_plain(g, d, rows)
    finally:
        g.close()
    assert got == single_device_acc(gpu, d, rows)
    assert got["pixels"] == d.width * height


@pytest.mark.parametrize("devices", groups(), ids=lambda d: f"{len(d)}gpu")
def test_back_to_back_calls_without_a_synchronize(gpu, devices):
    """Calls that follow each other with no synchronize reuse the partials and the owner's gather array: each call's
    copies wait for the previous merge.  Two frames into two accumulators get their own values; one frame twice into one
    accumulator keeps max_code and doubles the sums."""
    d = sized(DESCS["rgb_d12_420"], 3840, 2161)
    frames = [host_rows(d, f"back_to_back_{i}", specials=i == 0) for i in range(2)]
    expected = [single_device_acc(gpu, d, rows) for rows in frames]
    assert expected[0] != expected[1]
    g = Group(devices)
    try:
        g.group.prepare_encode(d)
        uploads = [g.upload(d, rows) for rows in frames]
        backings, planes = g.owner_planes(d)
        accs = [g.new_acc(), g.new_acc()]
        g.settle()
        for i in range(2):
            g.group.encode_device_light_level(d, uploads[i][0], uploads[i][1], planes, accs[i].data_ptr())
        g.group.synchronize()
        assert [acc_dict(a) for a in accs] == expected
        twice = g.new_acc()
        g.settle()
        for _ in range(2):
            g.group.encode_device_light_level(d, uploads[0][0], uploads[0][1], planes, twice.data_ptr())
        # the owner's stream waits for every member before the merge: its context's synchronize completes the call
        assert g.lib.avifgpu_synchronize(g.context(0)) == 0
        assert acc_dict(twice) == {"max_code": expected[0]["max_code"], "level_sum": 2 * expected[0]["level_sum"],
                                   "pixels": 2 * expected[0]["pixels"]}
        single_planes, _ = g.plain(d, frames[0])
        assert same_planes(host_planes(backings), single_planes)
        g.group.synchronize()
    finally:
        g.close()


def refusal_cases():
    out = [("hlg", desc_of(3, NONE, 10, transfer=abi.TRANSFER_HLG, nclx=cases.NCLX_2020_HLG()), abi.ERR_UNSUPPORTED),
           ("smpte428", desc_of(3, NONE, 12, transfer=abi.TRANSFER_SMPTE428), abi.ERR_UNSUPPORTED),
           ("clip", desc_of(3, NONE, 12, transfer=abi.TRANSFER_CLIP), abi.ERR_UNSUPPORTED)]
    for host_depth in (8, 16):
        d = desc_of(3, NONE, 10, transfer=abi.TRANSFER_CLIP)
        d.host_depth = host_depth
        out.append((f"host{host_depth}", d, abi.ERR_UNSUPPORTED))
    nv = desc_of(3, NONE, 12)
    nv.dest_layout = abi.SOURCE_CHROMA_INTERLEAVED
    out.append(("dest_layout", nv, abi.ERR_UNSUPPORTED))
    out.append(("null_acc", desc_of(3, NONE, 12), abi.ERR_BAD_PARAM))
    out.append(("owner_outside", desc_of(3, NONE, 12), abi.ERR_BAD_PARAM))
    return out


SENTINEL = [0x5A5A5A5AA5A5A5A5, 0x0123456789ABCDEF, 0x7EDCBA9876543210]


@pytest.mark.parametrize("name, desc, status", refusal_cases(), ids=[c[0] for c in refusal_cases()])
@pytest.mark.parametrize("devices", groups(), ids=lambda d: f"{len(d)}gpu")
def test_refusals_launch_nothing_and_leave_the_accumulator(devices, name, desc, status):
    import torch
    d = sized(desc, 64, 6)
    rows = np.zeros((d.height, d.width * d.host_channels), abi.host_dtype(d.host_depth))
    g = Group(devices)
    try:
        pointers, strides, _keep = g.upload(d, rows.astype(np.float32))  # refused before the rows are read: any device memory
        backings, planes = g.owner_planes(d)
        acc = torch.tensor(SENTINEL, dtype=torch.int64, device=f"cuda:{devices[0]}")
        before = g.launches()
        g.settle()
        n = len(devices)
        owner = n if name == "owner_outside" else 0
        got = g.lib.avifgpu_encode_rows_sharded_device_light_level(
            g.group.handle, C.byref(d), (C.c_void_p * n)(*pointers), (C.c_int64 * n)(*strides), C.byref(planes), owner,
            None if name == "null_acc" else acc.data_ptr())
        g.group.synchronize()
        assert got == status, (got, status, g.lib.avifgpu_shard_group_last_error(g.group.handle))
        assert g.launches() == before
        assert acc.cpu().tolist() == SENTINEL
        assert all(b is None or np.all(b == FILL) for b in host_planes(backings))
    finally:
        g.close()
