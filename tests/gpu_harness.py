"""What the GPU tests of the device entry points share: sentinel-padded device buffers, seeded batch images, the batch
calls and their launch counts, the batched kernels' grid caps, the scenarios several batched families run, and the
comparators.

A plain module, imported like cases.py.  Importing it touches no GPU: torch is imported inside the functions, so the
table checks of the modules that import it run without one.  pytest rewrites asserts only in test modules, so every
assert here carries its own message."""
import ctypes as C
import os

import numpy as np
import pytest

import cases
import encode_spec
from avifgpu import abi

SENTINEL = 0xCD
CHUNK = 64  # kBatchChunkImages
NV, MSB = abi.SOURCE_CHROMA_INTERLEAVED, abi.SOURCE_MSB_ALIGNED
BAD = abi.ERR_BAD_PARAM
UNTOUCHED = 7  # a status value the device-described calls never write


@pytest.fixture
def ctx():
    import avifgpu
    context = avifgpu.Context(0)
    yield context
    context.close()


def pick(checker, port, reference_ok):
    """test_gpu_parity.pick(): the compiled reference wherever the reference has the path; a missing oracle/_ref is a
    failure unless AVIFGPU_ALLOW_RESTATEMENT=1."""
    if not reference_ok:
        return port
    if checker.kind != "reference":
        if os.environ.get("AVIFGPU_ALLOW_RESTATEMENT") == "1":
            return port
        pytest.fail("oracle/_ref/libavifref.so is not loaded: build it where the reference tree is mounted (make -C oracle) -- "
                    "or set AVIFGPU_ALLOW_RESTATEMENT=1 to compare against the restatement")
    return checker


def sm_count(ctx):
    import torch
    return torch.cuda.get_device_properties(torch.device("cuda", ctx.device)).multi_processor_count


def padded(n):
    """A row stride for `n` bytes: rounded up to 64, plus 64 bytes of sentinel."""
    return (n + 63) // 64 * 64 + 64


def aligned_rows(dev, rows, cols, dtype, fill):
    """A (rows, cols) torch view on `dev` whose rows start 256 bytes apart (what the tuned kernels' vector loads and stores
    need), filled with `fill`."""
    import torch
    per_line = 256 // torch.empty((), dtype=dtype).element_size()
    return torch.full((rows, -(-cols // per_line) * per_line), fill, dtype=dtype, device=dev)[:, :cols]


def whole(plane):
    """The plane's bytes with the row padding (the sentinel) included."""
    return plane.as_strided((plane.shape[0], plane.stride(0)), (plane.stride(0), 1)).cpu().numpy()


def device_bytes(raw, misalign=0):
    """A copy of the 2-D uint8 array `raw` on the GPU, its rows on a padded stride, `misalign` bytes off the alignment."""
    import torch
    backing = torch.zeros((max(raw.shape[0], 1), padded(raw.shape[1]) + misalign), dtype=torch.uint8, device="cuda")
    plane = backing[:raw.shape[0], misalign:misalign + raw.shape[1]]
    plane.copy_(torch.from_numpy(raw).cuda())
    return plane


def launches_of(ctx, call):
    """The launches `call` makes."""
    import torch
    before = ctx.launch_count()
    call()
    torch.cuda.synchronize()
    return ctx.launch_count() - before


def run_counted(ctx, call):
    """Runs `call` twice and returns the launches of the second: table builds and first-use checks happen in the first."""
    import torch
    call()
    torch.cuda.synchronize()
    return launches_of(ctx, call)


def strips(width, group, odd_rows=False):
    """Launches of a tuned launcher: the kernel, a right strip when width % group != 0, an odd last 4:2:0 row."""
    return 1 + (width % group != 0) + bool(odd_rows)


def rgb32_nclx(transfer_name):
    nclx = {"pq": cases.NCLX_2020_PQ, "hlg": cases.NCLX_2020_HLG, "428": cases.NCLX_2020_428}[transfer_name]()
    nclx.matrix_coefficients = abi.MATRIX_GBR
    return nclx


# ---- device buffers with 256-byte row strides and a sentinel in the padding -----------------------------------------------

class Padded:
    """A (rows, cols) array of `dtype` on the device, each row 256-byte aligned, the padding filled with SENTINEL."""

    def __init__(self, dev, rows, cols, dtype, source=None):
        import torch
        self.dtype = np.dtype(dtype)
        self.payload = cols * self.dtype.itemsize
        self.stride = -(-self.payload // 256) * 256
        self.bytes = torch.full((rows, self.stride), SENTINEL, dtype=torch.uint8, device=dev)
        if source is not None:
            assert source.shape == (rows, cols) and source.dtype == self.dtype, "source shape or type"
            self.bytes[:, :self.payload] = torch.from_numpy(np.ascontiguousarray(source).view(np.uint8).reshape(rows, self.payload)).to(dev)
        self.view = self.bytes[:, :self.payload]
        self.shape = (rows, cols)

    def ptr(self):
        return self.bytes.data_ptr()

    def host(self):
        return self.view.contiguous().cpu().numpy().view(self.dtype).reshape(self.shape)

    def padding_intact(self):
        return self.payload == self.stride or bool((self.bytes[:, self.payload:] == SENTINEL).all().item())


def planes_struct(padded):
    planes = abi.Planes()
    for k, p in enumerate(padded):
        planes.data[k] = None if p is None else p.ptr()
        planes.stride[k] = 0 if p is None else p.stride
    return planes


# ---- batch images -------------------------------------------------------------------------------------------------------

class EncodeImage:
    """One image's seeded host rows and sentinel-padded destination planes of `desc`'s layout, as byte tensors on the GPU.
    The rows are drawn from the seed f"{prefix}{seed}_{w}x{h}", or are extreme_rows() of f"{prefix}{seed}".  With
    interleaved chroma, plane 2 is a sentinel-filled buffer of the planar size, passed to every call, that must stay
    untouched."""

    def __init__(self, desc, w, h, seed, prefix="batch_", beyond=False, rows_misalign=0, chroma_misalign=0, extreme=False):
        import torch
        self.w, self.h = w, h
        d = self.desc = abi.EncodeDesc.from_buffer_copy(desc)
        d.width, d.height = w, h
        self.planar_desc = abi.EncodeDesc.from_buffer_copy(d)
        self.planar_desc.dest_layout = abi.SOURCE_PLANAR
        if extreme:
            self.host = encode_spec.extreme_rows(d, w, h, f"{prefix}{seed}")
        elif d.host_depth == 32:
            self.host = cases.float_host_rows(cases.rng_for(f"{prefix}{seed}_{w}x{h}"), h, w, d.host_channels)
        else:
            self.host = cases.int_host_rows(cases.rng_for(f"{prefix}{seed}_{w}x{h}"), h, w, d.host_channels, d.host_depth, beyond=beyond)
        self.row_bytes = w * d.host_channels * d.host_depth // 8
        backing = torch.zeros((max(h, 1), padded(self.row_bytes) + rows_misalign), dtype=torch.uint8, device="cuda")
        self.rows = backing[:h, rows_misalign:rows_misalign + self.row_bytes]
        if w and h:
            self.rows.copy_(torch.from_numpy(np.ascontiguousarray(self.host).view(np.uint8).reshape(h, self.row_bytes)).cuda())
        self.sample_bytes = 2 if d.image_bit_depth > 8 else 1
        self.planes = [self.alloc(s, chroma_misalign if k == 1 else 0) for k, s in enumerate(abi.encode_plane_shapes(d))]
        if d.dest_layout & NV:
            self.planes[2] = self.alloc(abi.encode_plane_shapes(self.planar_desc)[2])

    def alloc(self, shape, misalign=0):
        import torch
        if shape is None:
            return None
        rows, cols = shape
        # one spare row: whole() reads a full stride from the view's first byte, `misalign` bytes past the last row
        backing = torch.full((max(rows, 1) + 1, padded(cols * self.sample_bytes) + misalign), SENTINEL, dtype=torch.uint8, device="cuda")
        return backing[:rows, misalign:misalign + cols * self.sample_bytes]

    def fresh_planes(self):
        return [None if p is None else self.alloc((p.shape[0], p.shape[1] // self.sample_bytes)) for p in self.planes]

    fresh_output = fresh_planes

    def record(self):
        return (self.w, self.h, self.rows, self.planes)

    def direct(self, ctx, planes=None, desc=None, y0=0, nrows=None, stream=0):
        import avifgpu
        ctx.encode_device(desc or self.desc, self.rows.data_ptr() + y0 * self.rows.stride(0), self.rows.stride(0),
                          avifgpu.planes_from_tensors(planes or self.planes), y0, nrows, stream)

    def untouched(self):
        return all((whole(p) == SENTINEL).all() for p in self.planes if p is not None)

    def expected(self, ctx):
        """The planar encode of the same description and rows, then re-interleaved and shifted by torch: per plane of the
        layout, its visible bytes (numpy, uint8)."""
        import torch
        planar = [self.alloc(s) for s in abi.encode_plane_shapes(self.planar_desc)]
        self.direct(ctx, planar, self.planar_desc)
        torch.cuda.synchronize()
        wide = self.sample_bytes == 2
        codes = [None if p is None else p.contiguous().view(torch.int16 if wide else torch.uint8).to(torch.int32) & (0xFFFF if wide else 0xFF)
                 for p in planar]
        if self.desc.dest_layout & MSB:
            shift = 16 - self.desc.image_bit_depth
            codes = [None if c is None else c << shift for c in codes]
        if self.desc.dest_layout & NV:
            codes[1] = torch.stack([codes[1], codes[2]], dim=-1).reshape(codes[1].shape[0], -1)
            codes[2] = None
        dtype = np.uint16 if wide else np.uint8
        return [None if c is None else c.cpu().numpy().astype(dtype).view(np.uint8).reshape(c.shape[0], -1) for c in codes]

    def codes_of_output(self):
        """The output turned back into planar, low-bit codes (numpy), for the independent model."""
        wide = self.sample_bytes == 2
        out = [None if p is None else p.cpu().numpy().view(np.uint16 if wide else np.uint8).astype(np.int64) for p in self.planes]
        if self.desc.dest_layout & NV:
            out[1], out[2] = out[1][:, 0::2], out[1][:, 1::2]
        if self.desc.dest_layout & MSB:
            out = [None if c is None else c >> (16 - self.desc.image_bit_depth) for c in out]
        return out


class DecodeImage:
    """One image's seeded codes (from f"{prefix}{seed}_{w}x{h}"), the source planes of `desc`'s layout made from them
    (random low bits under MSB-aligned codes) as byte tensors on the GPU, and sentinel-padded destination rows.

    planes_misalign moves every source plane, chroma_misalign plane 1 too, rows_offset the destination rows (keeping
    their stride) that many bytes off their alignment.  A direct_only image is held to the direct call, not the
    reference."""

    def __init__(self, desc, w, h, seed, prefix="dbatch_", overshoot=False, planes_misalign=0, chroma_misalign=0, rows_offset=0,
                 low_bits_seed=None):
        import torch
        self.w, self.h = w, h
        d = self.desc = abi.DecodeDesc.from_buffer_copy(desc)
        d.width, d.height = w, h
        self.planar_desc = abi.DecodeDesc.from_buffer_copy(d)
        self.planar_desc.source_layout = abi.SOURCE_PLANAR
        rng = cases.rng_for(f"{prefix}{seed}_{w}x{h}")
        self.codes = cases.code_planes(rng, self.planar_desc, overshoot=overshoot)
        source = list(self.codes)
        if d.source_layout & MSB:
            shift = 16 - d.bit_depth
            noise = np.random.default_rng(low_bits_seed if low_bits_seed is not None else rng.integers(1 << 31))
            source = [None if c is None else ((c.astype(np.uint32) << shift) | noise.integers(0, 1 << shift, c.shape)).astype(np.uint16)
                      for c in source]
        if d.source_layout & NV:
            pairs = np.empty((source[1].shape[0], 2 * source[1].shape[1]), dtype=source[1].dtype)
            pairs[:, 0::2], pairs[:, 1::2] = source[1], source[2]
            source[1], source[2] = pairs, None
        self.planes = [None if s is None else device_bytes(np.ascontiguousarray(s).view(np.uint8), planes_misalign + (chroma_misalign if k == 1 else 0))
                       for k, s in enumerate(source)]
        self.row_bytes = w * abi.decode_host_channels(d) * d.host_depth // 8
        if rows_offset:
            stride = padded(self.row_bytes)
            backing = torch.full(((h + 1) * stride,), SENTINEL, dtype=torch.uint8, device="cuda")
            self.rows = backing[rows_offset:rows_offset + h * stride].view(h, stride)[:, :self.row_bytes]
        else:
            self.rows = self.alloc()
        self.direct_only = False

    def alloc(self):
        import torch
        return torch.full((max(self.h, 1), padded(self.row_bytes)), SENTINEL, dtype=torch.uint8, device="cuda")[:self.h, :self.row_bytes]

    fresh_output = alloc

    def record(self):
        return (self.w, self.h, self.rows, self.planes)

    def direct(self, ctx, rows, y0=0, nrows=None, stream=0):
        import avifgpu
        ctx.decode_device(self.desc, avifgpu.planes_from_tensors(self.planes), rows.data_ptr() + y0 * rows.stride(0), rows.stride(0), y0, nrows,
                          stream)

    def untouched(self):
        return bool((whole(self.rows) == SENTINEL).all())

    def torch_planar(self):
        """The planar, low-bit planes of the same image, made on the GPU by torch: de-interleave, then shift."""
        import torch
        wide = self.desc.bit_depth > 8
        dtype = torch.int16 if wide else torch.uint8
        samples = [None if p is None else p.contiguous().view(dtype) for p in self.planes]
        if self.desc.source_layout & NV:
            samples[1], samples[2] = samples[1][:, 0::2], samples[1][:, 1::2]
        if self.desc.source_layout & MSB:
            shift = 16 - self.desc.bit_depth
            samples = [None if s is None else ((s.to(torch.int32) & 0xFFFF) >> shift).to(torch.int16) for s in samples]
        out = []
        for s in samples:
            if s is None:
                out.append(None)
                continue
            raw = torch.empty(s.shape, dtype=s.dtype, device="cuda").copy_(s).view(torch.uint8)  # dense, whatever s's strides
            backing = torch.zeros((max(raw.shape[0], 1), padded(raw.shape[1])), dtype=torch.uint8, device="cuda")
            backing[:raw.shape[0], :raw.shape[1]].copy_(raw)
            out.append(backing[:raw.shape[0], :raw.shape[1]])
        return out


class Empty:
    """A 0 x 5 image: valid, converts nothing."""
    w, h = 0, 5

    def record(self):
        return (0, 5, None, [None] * abi.MAX_PLANES)


# ---- calls and counts -------------------------------------------------------------------------------------------------------

def run_batch(ctx, desc, images, stream=0):
    import avifgpu
    ctx.encode_batch_device(desc, avifgpu.batch_images_from_tensors([im.record() for im in images]), stream=stream)


def run_decode_batch(ctx, desc, images, stream=0):
    import avifgpu
    ctx.decode_batch_device(desc, avifgpu.batch_images_from_tensors([im.record() for im in images]), stream=stream)


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


def capture(ctx, call, stream=None):
    """Records call(stream handle) into a CUDA graph on `stream` (torch's capture stream when None), in torch's default
    global capture mode; returns the graph and the launches counted while capturing."""
    import torch
    graph = torch.cuda.CUDAGraph()
    before = ctx.launch_count()
    with torch.cuda.graph(graph, stream=stream):
        call(torch.cuda.current_stream().cuda_stream)
    return graph, ctx.launch_count() - before


def captured(ctx, call):
    """Captures `call` on a side stream, replays it once, and returns the launches captured."""
    import torch
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    graph, launches = capture(ctx, call, stream)
    graph.replay()
    torch.cuda.synchronize()
    del graph
    return launches


def chunk_launches(images, eligible, has_edge):
    """The host-described batch's launches for its eligible images: per chunk of them one, one more when any of the
    chunk's images has an edge strip."""
    chosen = [im for im in images if eligible(im)]
    return sum(1 + any(has_edge(im) for im in chosen[i:i + CHUNK]) for i in range(0, len(chosen), CHUNK))


def direct_launches(ctx, images, into=None):
    """The launches of one direct call of each image, counted by making them into `into(image)` -- by default a fresh
    output buffer."""
    total = 0
    for im in images:
        before = ctx.launch_count()
        im.direct(ctx, im.fresh_output() if into is None else into(im))
        total += ctx.launch_count() - before
    return total


# ---- the integer batched kernels' instantiation tables and route (EncodeRgbIntBatchKernel, DecodeYccToRgbIntBatchKernel) ------

def planar(host_depth, channels, alpha, depth, chroma, nclx, down=abi.DOWN_FILTER_BOX):
    return abi.EncodeDesc(0, 0, host_depth, channels, alpha, depth, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, chroma, down,
                          abi.GRAY16_LUT, nclx)


def ycc(host_depth, bit_depth, chroma, alpha, nclx):
    return abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, chroma, bit_depth, alpha, host_depth, nclx)


N601, N709, N2020, GBR = cases.NCLX_601(), cases.NCLX_709(), cases.NCLX_2020_PQ(), cases.NCLX_GBR()
BOX, TOP_LEFT = abi.DOWN_FILTER_BOX, abi.DOWN_FILTER_TOP_LEFT
C444, C422, C420 = abi.CHROMA_444, abi.CHROMA_422, abi.CHROMA_420
NONE, STRAIGHT, PREMUL = abi.ALPHA_NONE, abi.ALPHA_STRAIGHT, abi.ALPHA_PREMULTIPLIED

# EncodeRgbIntBatchKernel<HostT, PlaneT, CHANNELS, XS, YS, PREMULTIPLY>: one case per (host depth, plane depth,
# channels / alpha, chroma); matrices, down-filters and 10 / 12-bit planes spread over them
ENCODE_KERNELS = [
    ("h8_d8_c3_444_601", planar(8, 3, NONE, 8, C444, N601)),
    ("h8_d8_c3_422_709_box", planar(8, 3, NONE, 8, C422, N709, BOX)),
    ("h8_d8_c3_420_2020_topleft", planar(8, 3, NONE, 8, C420, N2020, TOP_LEFT)),
    ("h8_d8_c4s_444_gbr", planar(8, 4, STRAIGHT, 8, C444, GBR)),
    ("h8_d8_c4s_422_none_topleft", planar(8, 4, STRAIGHT, 8, C422, None, TOP_LEFT)),
    ("h8_d8_c4s_420_601_box", planar(8, 4, STRAIGHT, 8, C420, N601, BOX)),
    ("h8_d8_c4p_444_709", planar(8, 4, PREMUL, 8, C444, N709)),
    ("h8_d8_c4p_422_2020_box", planar(8, 4, PREMUL, 8, C422, N2020, BOX)),
    ("h8_d8_c4p_420_none_topleft", planar(8, 4, PREMUL, 8, C420, None, TOP_LEFT)),
    ("h8_d10_c3_444_2020", planar(8, 3, NONE, 10, C444, N2020)),
    ("h8_d12_c3_422_601_topleft", planar(8, 3, NONE, 12, C422, N601, TOP_LEFT)),
    ("h8_d10_c3_420_709_box", planar(8, 3, NONE, 10, C420, N709, BOX)),
    ("h8_d12_c4s_444_none", planar(8, 4, STRAIGHT, 12, C444, None)),
    ("h8_d10_c4s_422_2020_box", planar(8, 4, STRAIGHT, 10, C422, N2020, BOX)),
    ("h8_d12_c4s_420_601_topleft", planar(8, 4, STRAIGHT, 12, C420, N601, TOP_LEFT)),
    ("h8_d10_c4p_444_gbr", planar(8, 4, PREMUL, 10, C444, GBR)),
    ("h8_d12_c4p_422_709_topleft", planar(8, 4, PREMUL, 12, C422, N709, TOP_LEFT)),
    ("h8_d10_c4p_420_none_box", planar(8, 4, PREMUL, 10, C420, None, BOX)),
    ("h16_d8_c3_444_none", planar(16, 3, NONE, 8, C444, None)),
    ("h16_d8_c3_422_601_box", planar(16, 3, NONE, 8, C422, N601, BOX)),
    ("h16_d8_c3_420_2020_topleft", planar(16, 3, NONE, 8, C420, N2020, TOP_LEFT)),
    ("h16_d8_c4s_444_709", planar(16, 4, STRAIGHT, 8, C444, N709)),
    ("h16_d8_c4s_422_none_topleft", planar(16, 4, STRAIGHT, 8, C422, None, TOP_LEFT)),
    ("h16_d8_c4s_420_709_box", planar(16, 4, STRAIGHT, 8, C420, N709, BOX)),
    ("h16_d8_c4p_444_gbr", planar(16, 4, PREMUL, 8, C444, GBR)),
    ("h16_d8_c4p_422_2020_box", planar(16, 4, PREMUL, 8, C422, N2020, BOX)),
    ("h16_d8_c4p_420_601_topleft", planar(16, 4, PREMUL, 8, C420, N601, TOP_LEFT)),
    ("h16_d12_c3_444_gbr", planar(16, 3, NONE, 12, C444, GBR)),
    ("h16_d10_c3_422_709_topleft", planar(16, 3, NONE, 10, C422, N709, TOP_LEFT)),
    ("h16_d12_c3_420_none_box", planar(16, 3, NONE, 12, C420, None, BOX)),
    ("h16_d10_c4s_444_601", planar(16, 4, STRAIGHT, 10, C444, N601)),
    ("h16_d12_c4s_422_601_box", planar(16, 4, STRAIGHT, 12, C422, N601, BOX)),
    ("h16_d10_c4s_420_2020_topleft", planar(16, 4, STRAIGHT, 10, C420, N2020, TOP_LEFT)),
    ("h16_d12_c4p_444_2020", planar(16, 4, PREMUL, 12, C444, N2020)),
    ("h16_d10_c4p_422_none_box", planar(16, 4, PREMUL, 10, C422, None, BOX)),
    ("h16_d12_c4p_420_709_topleft", planar(16, 4, PREMUL, 12, C420, N709, TOP_LEFT)),
]

# DecodeYccToRgbIntBatchKernel<SampleT, XS, YS, ALPHA>: one case per (8-bit -> 8-bit or 10 / 12-bit -> 16-bit, alpha,
# chroma); full and limited range at both host depths, a 12-bit case with alpha per chroma mode
DECODE_KERNELS = [
    ("h8_d8_a0_444_601lim", ycc(8, 8, C444, NONE, cases.NCLX_601(0))),
    ("h8_d8_a0_422_709", ycc(8, 8, C422, NONE, N709)),
    ("h8_d8_a0_420_none", ycc(8, 8, C420, NONE, None)),
    ("h8_d8_a1_444_gbr", ycc(8, 8, C444, STRAIGHT, GBR)),
    ("h8_d8_a1_422_2020lim", ycc(8, 8, C422, STRAIGHT, cases.NCLX_2020_PQ(0))),
    ("h8_d8_a1_420_601", ycc(8, 8, C420, STRAIGHT, N601)),
    ("h16_d10_a0_444_gbr", ycc(16, 10, C444, NONE, GBR)),
    ("h16_d12_a0_422_none", ycc(16, 12, C422, NONE, None)),
    ("h16_d10_a0_420_709lim", ycc(16, 10, C420, NONE, cases.NCLX_709(0))),
    ("h16_d12_a1_444_601lim", ycc(16, 12, C444, STRAIGHT, cases.NCLX_601(0))),
    ("h16_d12_a1_422_709", ycc(16, 12, C422, STRAIGHT, N709)),
    ("h16_d12_a1_420_2020lim", ycc(16, 12, C420, STRAIGHT, cases.NCLX_2020_PQ(0))),
]

# mixed sizes: aligned interiors with and without right strips, odd 4:2:0 heights, widths below 8, a 1 x 1 image
SIZES = [(64, 16), (37, 9), (8, 2), (1, 1), (130, 33), (7, 5), (256, 64), (95, 4)]

# widths 8 (one group), 264 and 520 (the last 256-px unit has one active lane), right strips (37, 95, 130), odd heights
# (a bottom strip in 4:2:0), and images the batch hands to direct calls: narrower than 8, or 1 row in 4:2:0
MIXED = [(264, 3), (8, 2), (37, 9), (7, 5), (130, 1), (520, 4), (95, 6), (1, 1), (64, 7)]


def ys_of(desc):
    return 1 if desc.chroma == C420 else 0


def int_eligible(im, ys):
    """EncodeBlockInterior / DecodeBlockInterior of the integer batched family on aligned buffers: an 8-px group and a
    (4:2:0) row pair."""
    return im.w >= 8 and im.h >= 1 + ys


def int_has_edge(im, ys):
    return im.w % 8 != 0 or (ys and im.h % 2 != 0)


def expected_launches(ctx, images, ys):
    """The integer family's chunk launches, plus the direct calls of the other images, counted by making them."""
    others = [im for im in images if im.w and im.h and not int_eligible(im, ys)]
    return chunk_launches(images, lambda im: int_eligible(im, ys), lambda im: int_has_edge(im, ys)) + direct_launches(ctx, others)


def assert_batched(ctx, run, images, ys):
    """The second of two runs (first-use checks happen in the first) makes exactly the launches of the chunk rule: an
    eligible image that fell back would add its own direct launches instead."""
    launches = run_counted(ctx, run)
    assert any(int_eligible(im, ys) for im in images), "no image is the batched kernels'"
    expected = expected_launches(ctx, images, ys)
    assert launches == expected, f"{launches} launches, the chunk rule makes {expected}"


def interior_units(w, h, ys):
    """BatchInteriorUnits of an image's aligned interior (the integer family's 256-px units)."""
    return -(-(w & ~7) // 256) * ((h >> 1) if ys else h)


def edge_units(w, h, chroma, decode):
    """BatchEdgeUnits of the right strip (w % 8 columns, every row) and, for 4:2:0 with an odd height, of the last row:
    runs of 256 chroma sites of a row (pair) on encode, of 256 pixels of a row on decode."""
    xs, ys = abi.chroma_shifts(chroma)
    odd_row = ys and h % 2
    if decode:
        xs = ys = 0
    units = -(-(((w % 8) + xs) >> xs) // 256) * ((h + ys) >> ys) if w % 8 else 0
    return units + (bottom_units(w, chroma, decode) if odd_row else 0)


def bottom_units(w, chroma, decode):
    """Units of the odd last 4:2:0 row: the interior's width in runs of 256 sites (encode) or pixels (decode)."""
    xs = 0 if decode else abi.chroma_shifts(chroma)[0]
    return -(-(((w & ~7) + xs) >> xs) // 256)


# ---- grid walks -----------------------------------------------------------------------------------------------------------

# Workers per CTA and CTAs per SM at most, for each batched launch of kernels_batch.cu: (per_cta, ctas_per_sm, source of
# the cap).  An interior worker is a warp taking one unit at a time, an edge worker a CTA taking one run of 256 sites or
# pixels.
BATCH_CAPS = {
    "encode_interior": (8, 16, "LaunchEncodeBatchChunk (warps; 8 per CTA, kStreamBlocksPerSm = 16)"),
    "encode_edge": (1, 16, "LaunchEncodeBatchChunk (CTAs; kStreamBlocksPerSm = 16)"),
    "ycc_int_interior": (8, 3, "LaunchDecodeBatchChunk, LaunchYccInt (warps; 8 per CTA, kYccBlocksPerSm = 3)"),
    "ycc_f32_interior": (8, 2, "LaunchDecodeBatchChunk, LaunchYccF32 (warps; 8 per CTA, kDecodeBlocksPerSm = 2)"),
    "rgb_int_interior": (8, 16, "LaunchPlanarRgbInt (warps; 8 per CTA, kStreamBlocksPerSm = 16)"),
    # CodeTableGridCap asks the occupancy API; 8 CTAs of 256 threads fill an SM's 2048 threads, so 8 bounds it from above
    # and the passes asserted with it are lower bounds
    "rgb_f32_interior": (8, 8, "LaunchPlanarRgbF32, CodeTableGridCap (warps; 8 per CTA, at most 8 CTAs per SM)"),
    "decode_edge": (1, 16, "LaunchDecodeBatchChunk, LaunchDecodeEdge (CTAs; kStreamBlocksPerSm = 16)"),
}


def assert_passes(kernel, units, sms):
    """The grid the launcher starts for `units` units has at most half as many workers (GridFor's cap)."""
    per_cta, ctas_per_sm, source = BATCH_CAPS[kernel]
    workers = max(1, min(-(-units // per_cta), sms * ctas_per_sm)) * per_cta
    assert units >= 2 * workers, f"{kernel}: {units} units, {workers} workers at {sms} SMs ({source})"


# ---- scenarios shared by the batched families -----------------------------------------------------------------------------

def batch_call(ctx, desc, direction, images=None, batch=None):
    """A call of `images` through the host-described API, or of the loaded `batch` through the device-described one:
    a function of the stream."""
    encode = direction == "encode"
    if batch is None:
        run = run_batch if encode else run_decode_batch
        return lambda stream=0: run(ctx, desc, images, stream)
    call = batch.encode if encode else batch.decode
    return lambda stream=0: call(ctx, desc, stream)


def host_or_device(ctx, desc, direction, api, images, check):
    """One call of `images`, one chunk with edges: two launches through the host-described API ("host"), or three through
    the device-described one with every status 0; then check(images)."""
    if api == "host":
        launches = launches_of(ctx, batch_call(ctx, desc, direction, images))
        assert launches == 2, f"{launches} launches of a host-described chunk with edges"
    else:
        batch = Indirect(len(images))
        batch.load(images)
        launches = launches_of(ctx, batch_call(ctx, desc, direction, batch=batch))
        assert launches == 3, f"{launches} launches of a device-described call"
        assert (batch.statuses() == 0).all(), f"statuses {batch.statuses()}"
    check(images)


# The rejected records of the decode families: NULL rows, a NULL alpha plane, a negative width.
DECODE_FAULTS = {1: ("rows", None), 3: ("plane", 3), 5: ("width", -1)}


def rejected_records(ctx, desc, direction, images, faults, check):
    """One device-described call of `images` with `faults` ({index: ("rows" | "width", value) or ("plane", k)}) set in
    their records: three launches, BAD_PARAM for each faulted image and 0 for the others, the faulted images' outputs
    keep their sentinel, and check(the others)."""
    import avifgpu
    records = avifgpu.batch_images_from_tensors([im.record() for im in images])
    for i, (field, value) in faults.items():
        if field == "plane":
            records[i].planes.data[value] = None
        else:
            setattr(records[i], field, value)
    batch = Indirect(len(images))
    batch.load(records)
    launches = launches_of(ctx, batch_call(ctx, desc, direction, batch=batch))
    assert launches == 3, f"{launches} launches of a device-described call"
    status = list(batch.statuses())
    assert status == [BAD if i in faults else 0 for i in range(len(images))], f"statuses {status}"
    assert all(images[i].untouched() for i in faults), "a rejected image's output was written"
    check([im for i, im in enumerate(images) if i not in faults])


def replay_sets(make, tag, big, mixed, names=("one", "64", "256")):
    """1 image of 96 x 10; 64 images of `big`; 256 images cycling through `mixed` -- fresh buffers, so new addresses.
    make(w, h, seed) builds one image."""
    return [[make(96, 10, f"{tag}_{names[0]}")],
            [make(*big, f"{tag}_{names[1]}_{i}") for i in range(64)],
            [make(*mixed[i % len(mixed)], f"{tag}_{names[2]}_{i}") for i in range(256)]]


def capture_and_replay(ctx, desc, direction, first, sets, check, prepare=None):
    """Captures one device-described call of the image `first` on a side stream (after prepare(), when given): three
    launches.  Replays it on each image set, loaded into the same records: no launch counted, every status 0, and
    check(images)."""
    import torch
    batch = Indirect(256)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        batch.load([first])
    if prepare is not None:
        prepare()
    stream.synchronize()
    graph, launches = capture(ctx, batch_call(ctx, desc, direction, batch=batch), stream)
    assert launches == 3, f"{launches} launches captured"
    for images in sets:
        with torch.cuda.stream(stream):
            batch.load(images)
            before = ctx.launch_count()
            graph.replay()
        torch.cuda.synchronize()
        assert ctx.launch_count() == before, "a replay must not count launches"
        assert (batch.statuses()[:len(images)] == 0).all(), f"statuses {batch.statuses()[:len(images)]}"
        check(images)
    del graph


# ---- comparators -------------------------------------------------------------------------------------------------------------

def assert_same_as_direct(ctx, images, checker=None, threads=1):
    """Each encode image: its planes, padding included, equal a direct call's, and the checker's codes when given."""
    import torch
    for im in images:
        reference = im.fresh_planes()
        im.direct(ctx, reference)
        torch.cuda.synchronize()
        for k, (got, want) in enumerate(zip(im.planes, reference)):
            if got is None:
                continue
            a, b = whole(got), whole(want)
            assert np.array_equal(a, b), ("direct call", im.w, im.h, k)
            assert (a[:, got.shape[1]:] == SENTINEL).all(), ("padding overwritten", im.w, im.h, k)
        if checker is not None and im.w and im.h:
            expected = checker.encode(im.desc, im.host, threads=threads)
            for k, got in enumerate(im.planes):
                if got is not None:
                    codes = got.cpu().numpy().view(abi.code_dtype(im.desc.image_bit_depth))
                    assert np.array_equal(codes, expected[k]), ("checker", im.w, im.h, k)


def decode_counted(gpu, desc, planes, what):
    """Decodes host `planes` through avifgpu_decode_rows_device from and into 256-byte aligned rows, asserts that the
    tuned launcher served it (its kernel + the generic right strip: 2 launches; the generic kernel alone makes 1) and
    returns the host floats."""
    import torch
    import avifgpu
    dev = torch.device("cuda", gpu.device)
    device_planes = []
    for p in planes:
        device_planes.append(None if p is None else aligned_rows(dev, p.shape[0], p.shape[1], torch.int16, 0))
        if p is not None:
            device_planes[-1].copy_(torch.from_numpy(p.view(np.int16)))
    out = aligned_rows(dev, desc.height, desc.width * abi.decode_host_channels(desc), torch.float32, 0.0)
    gpu.prepare_decode(desc)
    before = gpu.launch_count()
    gpu.decode_device(desc, avifgpu.planes_from_tensors(device_planes), out.data_ptr(), out.stride(0) * 4)
    torch.cuda.synchronize(dev)
    made = gpu.launch_count() - before
    assert made == 2, f"{made} launches: {what} and its right strip make 2, the generic kernel alone 1"
    return out.contiguous().cpu().numpy()


def differing_samples(expected, got):
    """Where two host arrays of decoded samples differ: floats bit for bit with NaN on both sides counting as equal,
    integers as they are."""
    if expected.dtype != np.float32:
        return expected != got
    nan_e, nan_g = np.isnan(expected), np.isnan(got)
    return (nan_e != nan_g) | (~nan_e & (expected.view(np.uint32) != got.view(np.uint32)))


def assert_same_floats(expected, got, planes, what):
    """Bit for bit, NaN on both sides counting as equal; names the first differing pixels by their codes."""
    bad = differing_samples(expected, got)
    if bad.any():
        channels = expected.shape[1] // planes[0].shape[1]
        at = np.argwhere(bad)[:6]
        shown = [f"codes {tuple(int(p[y, x // channels]) for p in planes if p is not None)} channel {x % channels}: "
                 f"{expected[y, x]!r} expected, {got[y, x]!r}" for y, x in at]
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.size} samples differ; " + "; ".join(shown))


def bits(a):
    return a.view(np.uint32) if a.dtype == np.float32 else a


def assert_decode_same_as_direct(ctx, images, reference=None, threads=1):
    """Each decode image: its rows, padding included, equal a direct call's, and unless it is direct_only the reference's
    output bit for bit (float hosts compared as bit patterns)."""
    import torch
    for im in images:
        direct = im.alloc()
        im.direct(ctx, direct)
        torch.cuda.synchronize()
        got = whole(im.rows)
        assert np.array_equal(got, whole(direct)), ("direct call", im.w, im.h)
        assert (got[:, im.row_bytes:] == SENTINEL).all(), ("padding overwritten", im.w, im.h)
        if reference is not None and im.w and im.h and not im.direct_only:
            expected = bits(reference.decode(im.desc, im.codes, threads=threads))
            values = bits(im.rows.cpu().numpy().view(abi.host_dtype(im.desc.host_depth)))
            assert values.shape == expected.shape, ("reference shape", im.w, im.h, values.shape, expected.shape)
            differ = values != expected
            assert not differ.any(), ("reference", im.w, im.h, int(differ.sum()), np.argwhere(differ)[0])
