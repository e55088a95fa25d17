"""CUDA graph capture of the device-pointer entry points (include/avifgpu.h, "CUDA graph capture").

Every case runs on a fresh context -- the session contexts' first-use state is shared by the whole suite -- and
captures with torch.cuda.graph in its default global mode, where an allocation or a synchronisation anywhere in the
process during the capture invalidates it.

  * Prepared capture, one case per tuned route: prepare, capture one call, then replay on two seeded inputs copied into
    the captured buffers.  Each replay equals a direct call and the CPU checker bit for bit; the capture counts the
    launches a direct call counts (the same route was recorded); a replay counts none.
  * Unprepared capture: a call of each kind of first-use state (Gray16 LUT, premultiply check, HLG / PQ / green
    divisions, step table) is first made inside a capture.  The capture ends cleanly, the replay is exact, and a later
    direct call still does the first-use work (it launches more kernels than the steady state).
  * A graph outlives later preparation on its context.

test_first_launches_inside_a_capture repeats the prepared cases in a fresh process, where each tuned kernel's first
launch -- with its one-off cudaFuncSetAttribute / occupancy query -- happens inside the capture."""
import os
import subprocess
import sys

import numpy as np
import pytest

import cases
from avifgpu import abi
from gpu_harness import ctx  # noqa: F401
from gpu_harness import SENTINEL, capture, pick

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H = 261, 9  # a right strip for every tuned launcher (4- and 8-pixel groups) and an odd last 4:2:0 row


# ---- the routes ---------------------------------------------------------------------------------------------------------

class Case:
    """One configuration: its description, seeded inputs, whether the compiled reference has the path, and what prepares
    the context for it."""

    def __init__(self, name, desc, reference_ok, prepare):
        self.name, self.desc, self.reference_ok, self.prepare_kind = name, desc, reference_ok, prepare
        self.encode = isinstance(desc, abi.EncodeDesc)

    def inputs(self, seed):
        d, rng = self.desc, cases.rng_for(f"graph_{self.name}_{seed}")
        if not self.encode:
            # planar RGB float: codes above the maximum are outside the reference's contract (test_gpu_parity.py)
            return cases.code_planes(rng, d, overshoot=not (d.colorspace == abi.COLORSPACE_RGB and d.host_depth == 32))
        if d.host_depth == 32:
            return cases.float_host_rows(rng, d.height, d.width, d.host_channels)
        return cases.int_host_rows(rng, d.height, d.width, d.host_channels, d.host_depth)

    def prepare(self, ctx, io):
        if self.prepare_kind == "encode":
            ctx.prepare_encode(self.desc)
        elif self.prepare_kind == "decode":
            ctx.prepare_decode(self.desc)
        elif self.prepare_kind == "direct":  # the premultiply check: one direct call outside the capture
            io.call(ctx, 0)
        import torch
        torch.cuda.synchronize()

    def expected(self, checker, port, inputs):
        reference = pick(checker, port, self.reference_ok)
        if self.encode:
            return reference.encode(self.desc, inputs, threads=os.cpu_count())
        return [reference.decode(self.desc, inputs, threads=os.cpu_count())]


def planar(host_depth, channels, alpha, depth, transfer, chroma, nclx):
    return abi.EncodeDesc(W, H, host_depth, channels, alpha, depth, transfer, 80, abi.LAYOUT_PLANAR_YCBCR, chroma, abi.DOWN_FILTER_BOX,
                          abi.GRAY16_LUT, nclx)


def rgb32_nclx(make):
    nclx = make()
    nclx.matrix_coefficients = abi.MATRIX_GBR
    return nclx


CASES = {c.name: c for c in [
    Case("flat_pq_420", planar(32, 3, abi.ALPHA_NONE, 12, abi.TRANSFER_PQ, abi.CHROMA_420, cases.NCLX_2020_PQ()), False, "encode"),
    Case("rgba_pq", planar(32, 4, abi.ALPHA_STRAIGHT, 12, abi.TRANSFER_PQ, abi.CHROMA_420, cases.NCLX_2020_PQ()), False, "encode"),
    Case("clip", planar(32, 3, abi.ALPHA_NONE, 10, abi.TRANSFER_CLIP, abi.CHROMA_444, cases.NCLX_2020_PQ()), False, "encode"),
    Case("gray32_pq", abi.EncodeDesc(W, H, 32, 1, abi.ALPHA_NONE, 12, abi.TRANSFER_PQ, 80), True, "encode"),
    Case("gray16_lut", abi.EncodeDesc(W, H, 16, 1, abi.ALPHA_NONE, 12), True, "encode"),
    Case("gray16_smpte428", abi.EncodeDesc(W, H, 16, 1, abi.ALPHA_NONE, 12, gray16_curve=abi.GRAY16_SMPTE428), False, "encode"),
    Case("rgba16_premultiplied_422", planar(16, 4, abi.ALPHA_PREMULTIPLIED, 10, abi.TRANSFER_CLIP, abi.CHROMA_422, cases.NCLX_709()), False, "direct"),
    Case("gray_int", abi.EncodeDesc(W, H, 8, 2, abi.ALPHA_STRAIGHT, 10), True, None),
    Case("hlg_ootf_decode", abi.DecodeDesc(W, H, abi.COLORSPACE_YCBCR, abi.CHROMA_420, 10, abi.ALPHA_NONE, 32, cases.NCLX_2020_HLG(),
                                           hlg_apply_ootf=1, hlg_display_gamma=1.2, hlg_peak_nits=1000), True, "decode"),
    Case("pq_ycbcr_decode", abi.DecodeDesc(W, H, abi.COLORSPACE_YCBCR, abi.CHROMA_420, 10, abi.ALPHA_NONE, 32, cases.NCLX_2020_PQ(),
                                           pq_peak_nits=80), True, "decode"),
    Case("planar_rgb_table_decode", abi.DecodeDesc(W, H, abi.COLORSPACE_RGB, abi.CHROMA_444, 12, abi.ALPHA_NONE, 32,
                                                   rgb32_nclx(cases.NCLX_2020_PQ), pq_peak_nits=1000), True, "decode"),
    Case("ycbcr_int_decode", abi.DecodeDesc(W, H, abi.COLORSPACE_YCBCR, abi.CHROMA_422, 10, abi.ALPHA_STRAIGHT, 16, cases.NCLX_709(0)),
         True, "decode"),
    Case("stream_mono_decode", abi.DecodeDesc(W, H, abi.COLORSPACE_MONOCHROME, abi.CHROMA_MONOCHROME, 12, abi.ALPHA_NONE, 16,
                                              cases.NCLX_2020_PQ(0)), True, "decode"),
]}


# ---- device buffers: 256-byte row strides, a sentinel in the padding ---------------------------------------------------------

class Padded:
    def __init__(self, rows, cols, dtype):
        import torch
        self.dtype = np.dtype(dtype)
        self.shape = (rows, cols)
        self.payload = cols * self.dtype.itemsize
        self.stride = -(-self.payload // 256) * 256
        self.bytes = torch.full((rows, self.stride), SENTINEL, dtype=torch.uint8, device="cuda:0")

    def load(self, array):
        import torch
        assert array.shape == self.shape and array.dtype == self.dtype
        host = torch.from_numpy(np.ascontiguousarray(array).view(np.uint8).reshape(self.shape[0], self.payload))
        self.bytes[:, :self.payload].copy_(host)

    def clear(self):
        self.bytes.fill_(SENTINEL)

    def host(self):
        return self.bytes[:, :self.payload].contiguous().cpu().numpy().view(self.dtype).reshape(self.shape)

    def padding_intact(self):
        return self.payload == self.stride or bool((self.bytes[:, self.payload:] == SENTINEL).all().item())


def planes_struct(padded):
    planes = abi.Planes()
    for k, p in enumerate(padded):
        planes.data[k] = None if p is None else p.bytes.data_ptr()
        planes.stride[k] = 0 if p is None else p.stride
    return planes


class DeviceIO:
    """The captured buffers of one case: inputs the caller refills between replays, outputs it reads."""

    def __init__(self, case):
        d = case.desc
        self.case = case
        if case.encode:
            self.src = [Padded(d.height, d.width * d.host_channels, abi.host_dtype(d.host_depth))]
            self.dst = [None if s is None else Padded(s[0], s[1], abi.code_dtype(d.image_bit_depth)) for s in abi.encode_plane_shapes(d)]
        else:
            self.src = [None if s is None else Padded(s[0], s[1], abi.code_dtype(d.bit_depth)) for s in abi.decode_plane_shapes(d)]
            self.dst = [Padded(d.height, d.width * abi.decode_host_channels(d), abi.host_dtype(d.host_depth))]
        self.src_planes = planes_struct(self.src)
        self.dst_planes = planes_struct(self.dst)

    def load(self, inputs):
        for buffer, array in zip(self.src, inputs if not self.case.encode else [inputs]):
            assert (buffer is None) == (array is None)
            if buffer is not None:
                buffer.load(array)
        for buffer in self.dst:
            if buffer is not None:
                buffer.clear()

    def call(self, ctx, stream):
        d = self.case.desc
        if self.case.encode:
            ctx.encode_device(d, self.src[0].bytes.data_ptr(), self.src[0].stride, self.dst_planes, stream=stream)
        else:
            ctx.decode_device(d, self.src_planes, self.dst[0].bytes.data_ptr(), self.dst[0].stride, stream=stream)

    def outputs(self):
        for buffer in self.dst:
            assert buffer is None or buffer.padding_intact(), "wrote into the row padding"
        return [None if b is None else b.host() for b in self.dst]


def same(expected, got):
    assert len(expected) == len(got)
    for k, (e, g) in enumerate(zip(expected, got)):
        assert (e is None) == (g is None), k
        if e is not None:
            differ = (e.view(np.uint32) != g.view(np.uint32)) if e.dtype == np.float32 else (e != g)
            assert not differ.any(), f"output {k}: {int(differ.sum())} of {e.size} values differ; first at {np.argwhere(differ)[0]}"


def replay(ctx, graph):
    import torch
    before = ctx.launch_count()
    graph.replay()
    torch.cuda.synchronize()
    assert ctx.launch_count() == before, "a replay must not count launches"


def direct(ctx, io, stream):
    """A direct (uncaptured) call; returns its launches."""
    import torch
    before = ctx.launch_count()
    io.call(ctx, stream)
    torch.cuda.synchronize()
    return ctx.launch_count() - before


# ---- 1. prepared capture ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(CASES))
def test_prepared_capture(ctx, checker, port, name):
    import torch
    case = CASES[name]
    io = DeviceIO(case)
    io.load(case.inputs("capture"))
    case.prepare(ctx, io)
    graph, captured = capture(ctx, lambda stream: io.call(ctx, stream))
    assert captured >= 2, f"{captured} launch(es) captured: the tuned kernel leaves a right strip to the generic one"
    if name == "flat_pq_420":
        assert captured == 3, "tuned kernel, right strip, odd last row"
    stream = torch.cuda.Stream()
    for seed in ("first", "second"):
        inputs = case.inputs(seed)
        io.load(inputs)
        replay(ctx, graph)
        replayed = io.outputs()
        same(case.expected(checker, port, inputs), replayed)
        io.load(inputs)
        assert direct(ctx, io, stream.cuda_stream) == captured, "the capture recorded another route than a direct call takes"
        same(replayed, io.outputs())
    del graph


# ---- 2. unprepared capture ---------------------------------------------------------------------------------------------------

UNPREPARED = {
    "gray16_lut": "gray16_lut",
    "premultiply": "rgba16_premultiplied_422",
    "hlg_divisions": "hlg_ootf_decode",
    "pq_ratio": "pq_ycbcr_decode",
    "green_division": "ycbcr_int_decode",
    "step_table": "flat_pq_420",
}


@pytest.mark.parametrize("kind", list(UNPREPARED))
def test_unprepared_capture(ctx, checker, port, kind):
    """The first call of the configuration is captured: it takes the path that needs no preparation, caches nothing, and
    the first direct call afterwards still does the first-use work."""
    import torch
    case = CASES[UNPREPARED[kind]]
    if kind == "step_table":
        ctx.set_table_autobuild(0)  # a direct call would build the table at once
    io = DeviceIO(case)
    io.load(case.inputs("capture"))
    graph, captured = capture(ctx, lambda stream: io.call(ctx, stream))
    assert captured >= 1
    inputs = case.inputs("first")
    io.load(inputs)
    replay(ctx, graph)
    replayed = io.outputs()
    same(case.expected(checker, port, inputs), replayed)

    stream = torch.cuda.Stream()
    io.load(inputs)
    first = direct(ctx, io, stream.cuda_stream)
    same(replayed, io.outputs())
    io.load(inputs)
    steady = direct(ctx, io, stream.cuda_stream)
    same(replayed, io.outputs())
    assert first > steady, f"the first direct call launched {first}, the next {steady}: the capture cached the first-use state"
    del graph


# ---- 3. a graph outlives later preparation ----------------------------------------------------------------------------------

def test_graph_outlives_later_preparation(ctx, checker, port):
    case = CASES["flat_pq_420"]
    io = DeviceIO(case)
    io.load(case.inputs("capture"))
    case.prepare(ctx, io)
    graph, _ = capture(ctx, lambda stream: io.call(ctx, stream))
    inputs = case.inputs("first")
    io.load(inputs)
    replay(ctx, graph)
    before = io.outputs()
    same(case.expected(checker, port, inputs), before)

    for other in ("rgba_pq", "gray32_pq", "gray16_lut", "gray16_smpte428"):
        ctx.prepare_encode(CASES[other].desc)
    for depth, transfer, peak in ((10, abi.TRANSFER_PQ, 1000), (12, abi.TRANSFER_SMPTE428, 80), (12, abi.TRANSFER_PQ, 10000)):
        ctx.prepare_encode(case.desc.copy(image_bit_depth=depth, transfer=transfer, pq_peak_nits=peak))
    for other in ("hlg_ootf_decode", "pq_ycbcr_decode", "ycbcr_int_decode"):
        ctx.prepare_decode(CASES[other].desc)

    io.load(inputs)
    replay(ctx, graph)
    same(before, io.outputs())
    del graph


# ---- the prepared cases in a process of their own ------------------------------------------------------------------------------

def test_first_launches_inside_a_capture():
    """In a fresh process the prepared cases capture each tuned kernel's very first launch: AllowDynamicShared's
    cudaFuncSetAttribute and the table decode's occupancy query then run inside the capture, and must not invalidate it."""
    out = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-k", "test_prepared_capture",
                          "-p", "no:cacheprovider"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-6000:] + out.stderr[-3000:]
    assert f"{len(CASES)} passed" in out.stdout, out.stdout[-2000:]
