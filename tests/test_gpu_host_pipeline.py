"""The host-pointer pipeline with encode and decode calls sharing one context (H100).

avifgpu_encode_rows / avifgpu_decode_rows and their _async forms run through pipeline state the context owns and both
directions share (avifgpu_api.cu, "host-pointer entry points"): SLOTS slots, each with a stream, device staging and
grow-only pinned bounce buffers; the copies out of a slot's pinned buffers into pageable caller memory that the slot
owes until it is retired; and the release of the page-locked rows the previous asynchronous encode handed over.  Each
case makes a call meet what an earlier one left behind: which slice lands on which slot, and that the slot still
holds the earlier call's slice, are asserted from the rules below (Pipeline).  Every output is held bit for bit to the
CPU checker (gpu_harness.pick), which a plain call of the whole image on a separate context must match too.  Every test
makes a fresh context, so its slots start at 0."""
import os

import numpy as np
import pytest

import cases
from avifgpu import abi
from gpu_harness import ctx  # noqa: F401
from gpu_harness import BAD, SENTINEL, pick

pytestmark = pytest.mark.gpu
THREADS = os.cpu_count() or 8

# The pipeline's rules.
SLOTS = 3               # kPipelineStreams, avifgpu_api.cu: slice i of a call takes slot (first + i) % SLOTS
SLICE_BYTES = 32 << 20  # SliceRows, avifgpu_api.cu: 32 MiB / row payload rows per slice, at least 2, even


def slice_rows(nrows, row_bytes):
    return min(max(SLICE_BYTES // row_bytes, 2) & ~1, nrows)


class Pipeline:
    """The slots as the rules place a context's calls on them: which call's slice each slot holds, and whether that
    slice owes a copy into pageable caller memory.  A synchronous call retires every slot (RetireThrough of its own
    ticket, the newest)."""

    def __init__(self):
        self.next = 0
        self.held = {}  # slot -> (call, slice index, slice bytes, owes)

    def issue(self, call, sync):
        """The call's slices: [(slot, rows, bytes)], and which of them land on a slot an earlier call still holds:
        [(slice index, slot, (that call, its slice index, its slice bytes, owes))]."""
        step = slice_rows(call.nrows, call.row_bytes)
        out, meets = [], []
        for i, begin in enumerate(range(0, call.nrows, step)):
            rows = min(step, call.nrows - begin)
            slot = (self.next + i) % SLOTS
            if slot in self.held and self.held[slot][0] is not call:
                meets.append((i, slot, self.held[slot]))
            self.held[slot] = (call, i, rows * call.row_bytes, call.memory == "pageable")
            out.append((slot, rows, rows * call.row_bytes))
        self.next = (self.next + len(out)) % SLOTS
        if sync:
            self.held.clear()
        return out, meets


# ---- seeded images, the checker's outputs ----------------------------------------------------------------------------------

def hlg_f32(w, h):
    return abi.DecodeDesc(w, h, abi.COLORSPACE_YCBCR, abi.CHROMA_420, 10, abi.ALPHA_NONE, 32, cases.NCLX_2020_HLG(), 1, 1.2, 1000, 80)


def ycc_int(w, h):
    return abi.DecodeDesc(w, h, abi.COLORSPACE_YCBCR, abi.CHROMA_420, 10, abi.ALPHA_STRAIGHT, 16, cases.NCLX_709(0))


def pq_f32(w, h):
    return abi.EncodeDesc(w, h, 32, 3, abi.ALPHA_NONE, 12, abi.TRANSFER_PQ, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420,
                          abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, cases.NCLX_2020_PQ())


def rgba_int(w, h):
    return abi.EncodeDesc(w, h, 16, 4, abi.ALPHA_STRAIGHT, 10, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420,
                          abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, cases.NCLX_709())


# kind -> (description, reference_ok: the compiled reference has the path; the planar encodes are the restatement's)
KINDS = {"hlg_f32": (hlg_f32, True), "ycc_int": (ycc_int, True), "pq_f32": (pq_f32, False), "rgba_int": (rgba_int, False)}

# 4098 px: a right strip after the tuned kernels' 4- and 8-pixel groups.  RGB32f rows are 48 KiB, so a 2048-row call is
# four slices (682, 682, 682, 2 rows); RGBA16 rows make 1022-row slices.
BIG = (4098, 2048)
SMALL = (256, 64)  # one slice

_images = {}


def image(gpu, checker, port, kind, size):
    """(description, input -- host rows or code planes --, the checker's output for the whole image), drawn and converted
    once per session.  A plain call of the whole image on `gpu`, a context of its own, must give the checker's bits."""
    key = (kind, size)
    if key not in _images:
        make, reference_ok = KINDS[kind]
        desc = make(*size)
        rng = cases.rng_for(f"host_pipeline_{kind}_{size[0]}x{size[1]}")
        reference = pick(checker, port, reference_ok)
        if isinstance(desc, abi.EncodeDesc):
            data = (cases.float_host_rows(rng, size[1], size[0], 3, specials=True) if desc.host_depth == 32 else
                    cases.int_host_rows(rng, size[1], size[0], 4, 16, beyond=True))
            expected = reference.encode(desc, data, threads=THREADS)
            plain = gpu.encode(desc, data)
            for k, (e, g) in enumerate(zip(expected, plain)):
                assert (e is None) == (g is None) and (e is None or np.array_equal(e, g)), f"{kind}: plain call, plane {k} differs from the checker"
        else:
            data = cases.code_planes(rng, desc, overshoot=desc.host_depth == 16)
            expected = reference.decode(desc, data, threads=THREADS)
            assert bits(gpu.decode(desc, data)).tobytes() == bits(expected).tobytes(), f"{kind}: plain call differs from the checker"
        _images[key] = (desc, data, expected)
    return _images[key]


def bits(a):
    return a.view(np.uint32) if a.dtype == np.float32 else a


# ---- host memory -------------------------------------------------------------------------------------------------------------

_pinned = {}


class HostBuffer:
    """rows x payload bytes of host memory seen as `dtype`, on a row stride of payload + pad bytes; every byte starts as
    SENTINEL.  Pinned memory is allocated once per session for each (tag, shape) through `gpu` and refilled."""

    def __init__(self, gpu, memory, tag, rows, payload, pad, dtype):
        shape = (max(rows, 1), payload + pad)
        if memory == "pinned":
            if (tag, shape) not in _pinned:
                _pinned[(tag, shape)] = gpu.pinned_array(shape, np.uint8)
            self.backing = _pinned[(tag, shape)]
        else:
            self.backing = np.empty(shape, np.uint8)
        self.backing[...] = SENTINEL
        self.payload = payload
        self.view = self.backing[:rows, :payload].view(dtype)

    def padding_intact(self):
        return bool((self.backing[:, self.payload:] == SENTINEL).all())


class Call:
    """One host-pointer call of image rows [y0, y0 + nrows): its input copied into fresh host buffers, its output buffers
    filled with SENTINEL (with `pad` bytes of row padding: libheif's planes on the encode side, the host's row stride on
    the decode side); the buffers of both sides are pageable or pinned (`memory`)."""

    def __init__(self, gpu, checker, port, kind, size, memory, tag, y0=0, nrows=None, pad=0):
        self.desc, data, self.expected = image(gpu, checker, port, kind, size)
        self.kind, self.memory, self.y0 = kind, memory, y0
        self.nrows = size[1] - y0 if nrows is None else nrows
        self.encode = isinstance(self.desc, abi.EncodeDesc)
        if self.encode:
            self.row_bytes = size[0] * self.desc.host_channels * self.desc.host_depth // 8
            self.rows = HostBuffer(gpu, memory, tag + "_rows", self.nrows, self.row_bytes, 0, data.dtype)
            self.rows.view[...] = data[y0:y0 + self.nrows]
            dtype = abi.code_dtype(self.desc.image_bit_depth)
            self.planes = [None if s is None else HostBuffer(gpu, memory, f"{tag}_plane{k}", s[0], s[1] * np.dtype(dtype).itemsize, pad, dtype)
                           for k, s in enumerate(abi.encode_plane_shapes(self.desc))]
        else:
            dtype = abi.host_dtype(self.desc.host_depth)
            self.row_bytes = size[0] * abi.decode_host_channels(self.desc) * np.dtype(dtype).itemsize
            self.planes = []
            for k, p in enumerate(data):
                if p is None:
                    self.planes.append(None)
                    continue
                b = HostBuffer(gpu, memory, f"{tag}_plane{k}", p.shape[0], p.shape[1] * p.itemsize, 0, p.dtype)
                b.view[...] = p
                self.planes.append(b)
            self.out = HostBuffer(gpu, memory, tag + "_out", self.nrows, self.row_bytes, pad, dtype)

    def issue(self, ctx, sync, nrows=None):
        """The call (sync: the blocking entry point; otherwise the _async one, whose ticket is returned)."""
        nrows = self.nrows if nrows is None else nrows
        planes = [None if p is None else p.view for p in self.planes]
        if self.encode:
            if sync:
                ctx.encode(self.desc, self.rows.view, y0=self.y0, nrows=nrows, planes=planes)
                return None
            return ctx.encode_async(self.desc, self.rows.view, planes, y0=self.y0, nrows=nrows)
        if sync:
            ctx.decode(self.desc, planes, y0=self.y0, nrows=nrows, out=self.out.view)
            return None
        return ctx.decode_async(self.desc, planes, self.out.view, y0=self.y0, nrows=nrows)

    def check(self, what):
        """The converted rows equal the checker's, the rest of every output buffer (rows outside the block, row padding)
        still holds SENTINEL.  A difference names the first image row (plane row, on the encode side) that differs."""
        if self.encode:
            for k, (b, e) in enumerate(zip(self.planes, self.expected)):
                if b is None:
                    continue
                ys = 1 if k in (1, 2) and self.desc.chroma == abi.CHROMA_420 else 0
                first, last = self.y0 >> ys, (self.y0 + self.nrows + ys) >> ys
                assert_rows(b.view[first:last], e[first:last], first, f"{what}: plane {k}")
                outside = np.concatenate([b.backing[:first], b.backing[last:]])
                assert (outside == SENTINEL).all(), f"{what}: plane {k} written outside rows [{first}, {last})"
                assert b.padding_intact(), f"{what}: plane {k} written into its row padding"
        else:
            assert_rows(self.out.view, self.expected[self.y0:self.y0 + self.nrows], self.y0, f"{what}: rows")
            assert self.out.padding_intact(), f"{what}: rows written into their padding"


def assert_rows(got, want, first, what):
    differ = np.flatnonzero((bits(got) != bits(want)).any(axis=1))
    if differ.size:
        run = np.argmax(np.append(np.diff(differ) != 1, True))  # the end of the first run of differing rows
        raise AssertionError(f"{what}: row {first + differ[0]} is the first that differs from the checker "
                             f"(rows {first + differ[0]}..{first + differ[run]} in a row, {differ.size} of {got.shape[0]} in all)")


@pytest.fixture
def make(gpu, checker, port):
    return lambda *args, **kwargs: Call(gpu, checker, port, *args, **kwargs)


# ---- reuse across directions -------------------------------------------------------------------------------------------------

FIRST = [("decode", "pageable"), ("decode", "pinned"), ("encode", "pageable"), ("encode", "pinned")]
SECOND = [(direction, form, memory) for direction in ("encode", "decode") for form in ("sync", "async") for memory in ("pageable", "pinned")]


def first_kind(direction):
    return "hlg_f32" if direction == "decode" else "pq_f32"


def assert_meets(meets, first):
    """The first slice of the second call on a slot the first call's slice still holds -- owing its copy when the first
    call's memory is pageable: (its index, the slot, the bytes of the first call's slice there)."""
    assert meets, "no slice of the second call lands on a slot the first call still holds"
    index, slot, (call, their_index, their_bytes, owes) = meets[0]
    assert call is first and owes == (first.memory == "pageable"), (index, slot, their_index, owes)
    return index, slot, their_bytes


@pytest.mark.parametrize("direction,form,memory", SECOND, ids=["-".join(s) for s in SECOND])
@pytest.mark.parametrize("first_direction,first_memory", FIRST, ids=["-".join(f) for f in FIRST])
def test_second_call_reuses_a_slot_the_first_still_owes(ctx, make, first_direction, first_memory, direction, form, memory):
    """An asynchronous call of a 4098 x 2048 image -- four slices on slots 0, 1, 2, 0, of which the last three are not
    retired -- then a one-slice call of a 256 x 64 image on slot 1, whose buffers already hold more than it needs.  A
    decode into pageable rows owes slot 1's rows (682..1363) until the slot retires: an encode from pageable rows must
    not stage its own rows over them first."""
    pipeline = Pipeline()
    first = make(first_kind(first_direction), BIG, first_memory, "first")
    slices, _ = pipeline.issue(first, sync=False)
    assert [s for s, _, _ in slices] == [0, 1, 2, 0] and [r for _, r, _ in slices] == [682, 682, 682, 2], slices
    second = make(first_kind(direction), SMALL, memory, "second")
    second_slices, meets = pipeline.issue(second, sync=form == "sync")
    index, slot, their_bytes = assert_meets(meets, first)
    assert (index, slot) == (0, 1) and second_slices[0][2] <= their_bytes, (second_slices, their_bytes)

    first.issue(ctx, sync=False)
    second.issue(ctx, sync=form == "sync")
    ctx.wait()
    first.check("first call")
    second.check("second call")


@pytest.mark.parametrize("direction,form,memory", SECOND, ids=["-".join(s) for s in SECOND])
@pytest.mark.parametrize("first_direction,first_memory", FIRST, ids=["-".join(f) for f in FIRST])
def test_second_call_grows_a_slot_the_first_still_owes(ctx, make, first_direction, first_memory, direction, form, memory):
    """An asynchronous one-slice call of a 256 x 64 image on slot 0, then a call of a 4098 x 2048 image on slots 1, 2, 0,
    1: its third slice (682 rows, 32 MiB) needs larger device and pinned buffers than slot 0 holds while slot 0 still
    holds -- and, with pageable memory, owes -- the first call's slice.  Regrowing a pinned buffer frees it: what the
    slot owes must have left it before."""
    pipeline = Pipeline()
    first = make(first_kind(first_direction), SMALL, first_memory, "first")
    slices, _ = pipeline.issue(first, sync=False)
    assert [s for s, _, _ in slices] == [0], slices
    second = make(first_kind(direction), BIG, memory, "second")
    second_slices, meets = pipeline.issue(second, sync=form == "sync")
    index, slot, their_bytes = assert_meets(meets, first)
    assert (index, slot) == (2, 0) and second_slices[2][2] > their_bytes, (second_slices, their_bytes)

    first.issue(ctx, sync=False)
    second.issue(ctx, sync=form == "sync")
    ctx.wait()
    first.check("first call")
    second.check("second call")


# ---- release of the previous call's rows -------------------------------------------------------------------------------------

def overwrite_backwards(rows):
    """NaN into every row, a few rows at a time from the last: the copies still queued or on the wire read them last."""
    for end in range(rows.shape[0], 0, -8):
        rows[max(end - 8, 0):end] = np.nan


NEXT = [(direction, form) for direction in ("encode", "decode") for form in ("sync", "async", "empty-sync", "empty-async")]


@pytest.mark.parametrize("direction,form", NEXT, ids=["-".join(n) for n in NEXT])
def test_next_call_releases_the_previous_async_encodes_rows(ctx, make, direction, form):
    """encode_rows_async from page-locked rows A (four slices: the last H2D is queued behind three others), then one
    host-pointer call X of either direction, synchronous, asynchronous or of an empty row block.  Once X has returned, A
    is the caller's again (avifgpu.h): overwriting it with NaN must not reach the planes."""
    pipeline = Pipeline()
    a = make("pq_f32", BIG, "pinned", "A")
    slices, _ = pipeline.issue(a, sync=False)
    assert len(slices) >= 4, slices
    x = make(first_kind(direction), SMALL, "pageable", "X")
    empty = form.startswith("empty")

    a.issue(ctx, sync=False)
    x.issue(ctx, sync=form in ("sync", "empty-sync"), nrows=0 if empty else None)
    overwrite_backwards(a.rows.view)
    ctx.wait()
    a.check("A's planes")
    if not empty:
        x.check("X")


# ---- tickets, and a refused call in the middle -------------------------------------------------------------------------------

def test_waiting_for_the_second_of_three_mixed_calls(ctx, make):
    """An encode into pageable planes (slots 0, 1, 2, 0), a decode into pageable rows (slots 1, 2, 0, 1) and an encode
    from page-locked rows (slot 2, which holds the decode's second slice): wait(second ticket) completes the first two
    calls while the third may still run; wait(0) completes the third."""
    pipeline = Pipeline()
    calls = [make("pq_f32", BIG, "pageable", "first"), make("hlg_f32", BIG, "pageable", "second"), make("pq_f32", SMALL, "pinned", "third")]
    placed = [pipeline.issue(call, sync=False) for call in calls]
    assert [s for s, _, _ in placed[2][0]] == [2] and placed[2][1][0][2][0] is calls[1], placed[2]
    tickets = [call.issue(ctx, sync=False) for call in calls]
    assert tickets == [tickets[0], tickets[0] + 1, tickets[0] + 2], tickets
    ctx.wait(tickets[1])
    calls[0].check("first call")
    calls[1].check("second call")
    ctx.wait(0)
    calls[2].check("third call")


def test_refused_call_takes_no_ticket_and_releases_nothing(ctx, make):
    """A decode into pageable rows, an encode from page-locked rows A, then two calls refused for their row block -- an
    encode starting on an odd 4:2:0 row and a decode past the image: ERR_BAD_PARAM, no ticket, the pending outputs
    intact and A not released by them.  The next call takes the following ticket and releases A."""
    import avifgpu
    pending = make("hlg_f32", BIG, "pageable", "pending")
    a = make("pq_f32", BIG, "pinned", "A")
    x = make("pq_f32", SMALL, "pageable", "X")
    bad_encode = make("pq_f32", SMALL, "pageable", "refused_encode", y0=1, nrows=2)
    bad_decode = make("hlg_f32", SMALL, "pageable", "refused_decode", y0=SMALL[1] - 1, nrows=2)
    pending.issue(ctx, sync=False)
    ticket = a.issue(ctx, sync=False)
    for refused in (bad_encode, bad_decode):
        for sync in (True, False):
            with pytest.raises(avifgpu.AvifGpuError) as error:
                refused.issue(ctx, sync=sync)
            assert error.value.status == BAD, error.value
    assert x.issue(ctx, sync=False) == ticket + 1
    overwrite_backwards(a.rows.view)
    ctx.wait()
    pending.check("pending decode")
    a.check("A's planes")
    x.check("X")
    assert (bad_encode.planes[0].backing == SENTINEL).all() and (bad_decode.out.backing == SENTINEL).all(), "a refused call wrote"


# ---- blocks as the shuttle sends them ----------------------------------------------------------------------------------------

GROUP = {"hlg_f32": 4, "ycc_int": 8, "pq_f32": 4, "rgba_int": 8}  # the tuned kernel's pixel group (DecodeYccF32BlockInterior, ...)
BLOCKS = [("hlg_f32", 1), ("hlg_f32", 2), ("ycc_int", 1), ("ycc_int", 2), ("pq_f32", 2), ("rgba_int", 2)]


@pytest.mark.parametrize("memory", ["pageable", "pinned"])
@pytest.mark.parametrize("kind,y0", BLOCKS, ids=[f"{k}-y{y}" for k, y in BLOCKS])
def test_block_over_several_slices(ctx, make, kind, y0, memory):
    """Rows [y0, y0 + 2046) of a 4098 x 2048 image in one call of three slices, the host rows (decode) or planes (encode) on
    a row stride 72 bytes longer than the payload, SENTINEL in the padding.  A block starting on a 4:2:0 row pair gives
    every slice to the tuned kernel with its right strip: 1 + 1 launches per slice.  One starting on the pair's second
    row (decode only: an encode block must start on a pair) has no tuned route -- the tuned YCbCr decodes take a
    block on a row pair (DecodeYccF32BlockInterior, DecodeYccIntBlockInterior) -- so every slice is one launch of the
    generic kernel with the odd phase."""
    call = make(kind, BIG, memory, "block", y0=y0, nrows=2046, pad=72)
    slices, _ = Pipeline().issue(call, sync=True)
    assert len(slices) == 3 and all(rows % 2 == 0 for _, rows, _ in slices), slices
    assert BIG[0] % GROUP[kind] != 0
    if call.encode:
        ctx.prepare_encode(call.desc)  # the step table of the float encode, built before the count
    else:
        ctx.prepare_decode(call.desc)  # the verified divisions of the decodes
    before = ctx.launch_count()
    call.issue(ctx, sync=False)
    ctx.wait()
    launches = ctx.launch_count() - before
    per_slice = 1 if y0 & 1 else 1 + 1
    assert launches == len(slices) * per_slice, f"{launches} launches for {len(slices)} slices, expected {per_slice} each"
    call.check("block")
