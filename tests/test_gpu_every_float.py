"""Every float through every encode route that reads a step table, and the exact curve itself, against the compiled
reference -- not against another GPU route.

The step tables (curve_tables.cu) are verified by the builder against ExactCurveCode, the DEVICE evaluation, and the
other whole-domain tests compare one GPU route with another, so a mistake in ExactCurveCode or the device libm under it
would be copied into every table and agreed with everywhere.  Here the expected code of every bit pattern from +0 through
the positive NaNs is the reference's own: oracle/_ref/libavifref.so's transfer function of the float, quantised the way
its encoder quantises (trunc(clamp(v * max, 0, max)) in float32, NaN -> 0; the CPU test below pins that composition to
the reference's encoder).  +inf and NaN, where the reference's cast is undefined, take the project's definition: the
restatement (oracle/liboracle.so).  The expected codes are built once per curve on host threads, chunk by chunk, and
kept on the device; alongside, avifgpu_transfer_f32 must give the reference's float bit for bit on every finite input.

Each (curve, route) case runs 10- and 12-bit where the route serves that depth, and proves its route by launch count.
The image is 4094 pixels wide on 256-byte aligned rows: a tuned launcher covers 4092 columns with its kernel and hands
the last two to the generic kernel (2 launches, the strip's samples compared like the rest), the generic kernel alone
makes 1, so a launcher that quietly declines shows up as a wrong count:

  flat_interleaved   EncodeRgbF32FlatKernel, reference layout (RGB32f, no alpha)
  flat_planar        EncodeRgbF32FlatKernel, planar 4:4:4 with the identity matrix: each plane holds per-sample codes
  rgba_planar        EncodeRgbaF32FlatKernel, identity matrix, straight alpha 1.0 (no colour clamp)
  gray_alpha         EncodeGrayF32Kernel, Gray + straight alpha 1.0 (no clamp)
  rgba_reference     generic kernel, compact table read from global memory (RGBA32f, reference layout)
  hlg_generic        generic kernel, compact table read from global memory (RGB32f, HLG OETF save path)
  exact              generic kernel on a context that never builds tables: its own evaluation of the curve (the same
                     device transfer function and libm that ExactCurveCode, and so every table, is built on)

A negative slice (-0, the smallest and largest negatives, 2^24 patterns around -1.0, -inf and the negative NaNs) runs
through the same routes.  Last, the 12-bit float decodes: every (Y, Cr) and every (Y, Cb) pair through the tuned YCbCr
kernel, and every code through the per-code table kernel (planar RGB, monochrome), bit for bit against the reference,
each at a width that leaves the tuned kernel a generic right strip (2 launches)."""
import collections
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import cases
import encode_spec
import oracle
from avifgpu import abi
from gpu_harness import aligned_rows, assert_same_floats, decode_counted

THREADS = max(1, min(32, len(os.sched_getaffinity(0))))
CHUNK = 1 << 22             # bit patterns per host work item
SLAB = 1 << 26              # samples per device fill / compare step
DOMAIN = 1 << 31            # +0 .. 0x7fffffff: every non-negative finite float, +inf and the positive NaNs
FINITE_END = 0x7f800000     # the bits of +inf
ALPHA_ONE = 0x3f800000      # the bits of 1.0
W = 4094                    # encode width: 4 - 2, so a tuned launcher leaves a two-column strip to the generic kernel
TUNED, GENERIC = 2, 1       # launches of a tuned launcher at that width (kernel + right strip), and of the generic kernel

PQ, SMPTE428, HLG = abi.TRANSFER_PQ, abi.TRANSFER_SMPTE428, abi.TRANSFER_HLG
FUNCTION = {PQ: abi.FN_LINEAR_TO_PQ, SMPTE428: abi.FN_LINEAR_TO_SMPTE428, HLG: abi.FN_LINEAR_TO_HLG}
CURVES = {"pq80": (PQ, 80), "pq1000": (PQ, 1000), "pq10000": (PQ, 10000), "smpte428": (SMPTE428, 80), "hlg": (HLG, 80)}


def transfer_param(transfer, peak):
    return float(peak) if transfer == PQ else 0.0


# ---- the CPU ground truth ------------------------------------------------------------------------------------------------

def reference_values(ref, port, transfer, peak, bits):
    """The curve's float for uint32 bit patterns: the reference's for finite inputs, the restatement's for +-inf / NaN."""
    x = np.ascontiguousarray(bits, np.uint32).view(np.float32)
    fn, param = FUNCTION[transfer], transfer_param(transfer, peak)
    finite = np.isfinite(x)
    if finite.all():
        return ref.transfer(fn, x, param)
    out = np.empty_like(x)
    out[finite] = ref.transfer(fn, x[finite], param)
    out[~finite] = port.transfer(fn, x[~finite], param)
    return out


def quantise(values, depth):
    """The reference encoder's float quantiser (encode_spec._quantise) as uint16 codes."""
    return encode_spec._quantise(values, (1 << depth) - 1).astype(np.uint16)


def reference_thresholds(ref, transfer, peak, depth, count):
    """The smallest input bits of `count` codes spread over the range, located by bisection on the reference."""
    top = (1 << depth) - 1
    ks = np.unique(np.linspace(1, top, count).astype(np.int64))
    lo = np.zeros(ks.size, np.uint32)
    hi = np.full(ks.size, FINITE_END - 1, np.uint32)
    fn, param = FUNCTION[transfer], transfer_param(transfer, peak)
    for _ in range(32):
        mid = ((lo.astype(np.uint64) + hi.astype(np.uint64)) // 2).astype(np.uint32)
        below = quantise(ref.transfer(fn, mid.view(np.float32), param), depth) < ks
        lo = np.where(below, mid, lo)
        hi = np.where(below, hi, mid)
    return hi


def bounded_map(pool, work, items, window):
    """pool.map with at most `window` results in flight, in order."""
    pending = collections.deque()
    for item in items:
        pending.append(pool.submit(work, item))
        if len(pending) >= window:
            yield pending.popleft().result()
    while pending:
        yield pending.popleft().result()


@pytest.mark.parametrize("curve", ["pq80", "pq1000", "pq10000", "smpte428"])
@pytest.mark.parametrize("depth", [10, 12])
def test_quantised_reference_transfer_is_the_reference_encoder(ref, port, curve, depth):
    """The ground truth's composition (reference transfer function, then the float quantiser) equals the reference's own
    RGB32f encoder in its interleaved layout, on every 4093rd finite pattern of both signs and on +-64 patterns around
    200 thresholds located on the reference.  HLG has no reference encoder: there the composition is the definition."""
    transfer, peak = CURVES[curve]
    positive = np.arange(0, FINITE_END, 4093, dtype=np.uint32)
    negative = positive[::16] | np.uint32(0x80000000)
    around = reference_thresholds(ref, transfer, peak, depth, 200).astype(np.int64)[:, None] + np.arange(-64, 65)
    bits = np.concatenate([positive, negative, around.clip(0, FINITE_END - 1).astype(np.uint32).ravel()])
    bits = np.concatenate([bits, np.zeros(-bits.size % (3 * 1024), np.uint32)])
    rows = bits.view(np.float32).reshape(-1, 3 * 1024)
    desc = abi.EncodeDesc(1024, rows.shape[0], 32, 3, abi.ALPHA_NONE, depth, transfer, peak, abi.LAYOUT_REFERENCE)
    encoded = ref.encode(desc, rows, threads=THREADS)[0].ravel()
    composed = quantise(reference_values(ref, port, transfer, peak, bits), depth)
    differing = np.flatnonzero(encoded != composed)
    assert differing.size == 0, (f"{differing.size} codes differ, first (bits, encoder, composed): "
                                 + ", ".join(f"(0x{bits[i]:08x}, {encoded[i]}, {composed[i]})" for i in differing[:8]))


# ---- the GPU side ------------------------------------------------------------------------------------------------------------

class Truth:
    """The expected 10- and 12-bit codes of every pattern +0 .. 0x7fffffff for one curve, as device int16 vectors, and
    what avifgpu_transfer_f32 got wrong on the way (count, first few (bits, reference, device) floats)."""

    def __init__(self, gpu, ref, port, transfer, peak):
        import torch
        dev = torch.device("cuda", gpu.device)
        self.codes = {depth: torch.empty(DOMAIN, dtype=torch.int16, device=dev) for depth in (10, 12)}
        self.transfer_mismatches = 0
        self.transfer_examples = []
        fn, param = FUNCTION[transfer], transfer_param(transfer, peak)

        def work(start):
            bits = np.arange(start, start + CHUNK, dtype=np.uint32)
            curved = reference_values(ref, port, transfer, peak, bits)
            return start, bits, curved, quantise(curved, 10), quantise(curved, 12)

        with ThreadPoolExecutor(THREADS) as pool:
            for start, bits, curved, c10, c12 in bounded_map(pool, work, range(0, DOMAIN, CHUNK), 2 * THREADS):
                if start < FINITE_END:  # CHUNK divides FINITE_END: a chunk is all finite or all +inf / NaN
                    self._check_transfer(bits, curved, gpu.transfer(fn, bits.view(np.float32), param))
                self.codes[10][start:start + CHUNK].copy_(torch.from_numpy(c10.view(np.int16)))
                self.codes[12][start:start + CHUNK].copy_(torch.from_numpy(c12.view(np.int16)))
        torch.cuda.synchronize(dev)

    def _check_transfer(self, bits, expected, got):
        nan_e, nan_g = np.isnan(expected), np.isnan(got)
        bad = (nan_e != nan_g) | (~nan_e & (expected.view(np.uint32) != got.view(np.uint32)))
        count = int(bad.sum())
        if count:
            self.transfer_mismatches += count
            for i in np.flatnonzero(bad)[:8 - len(self.transfer_examples)]:
                self.transfer_examples.append(f"(0x{bits[i]:08x}, {expected[i]!r}, {got[i]!r})")


@pytest.fixture(scope="module")
def reference():
    checker = oracle.load_reference()
    if checker is None:
        pytest.fail("oracle/_ref/libavifref.so is not loaded: the expected codes are the compiled reference's -- build it "
                    "where the reference tree is mounted (make -C oracle); it ships with the tree")
    return checker


@pytest.fixture(scope="module")
def truths(gpu, reference, port):
    """truths(curve) -> Truth.  One curve at a time stays resident (8 GB of device memory); the cases are ordered by curve."""
    import torch
    held = {}

    def get(curve):
        if curve not in held:
            held.clear()
            torch.cuda.empty_cache()
            held[curve] = Truth(gpu, reference, port, *CURVES[curve])
        return held[curve]
    yield get
    held.clear()
    torch.cuda.empty_cache()


def require_memory(dev, gigabytes):
    import torch
    if torch.cuda.get_device_properties(dev).total_memory < gigabytes * 2**30:
        pytest.skip(f"needs ~{gigabytes} GB of device memory")


class Samples:
    """The input samples of one case, in order: `pattern(start, count)` gives their bits as a device int32 vector,
    `bits_of(i)` the bits of sample i (for messages), `want[depth]` the expected codes (device int16)."""

    def __init__(self, n, pattern, bits_of, want):
        self.n, self.pattern, self.bits_of, self.want = n, pattern, bits_of, want


def whole_domain(dev, truth):
    import torch

    def pattern(start, count):
        return torch.arange(start, start + count, dtype=torch.int64, device=dev).to(torch.int32)
    return Samples(DOMAIN, pattern, lambda i: i, truth.codes)


def assert_codes(got, samples, depth, what):
    """Every code of `got` (device int16, input-sample order) against the expected ones; the message names how many differ,
    the range of input bits they span and the first few (bits, expected, got)."""
    import torch
    want = samples.want[depth]
    assert got.numel() == samples.n == want.numel()
    count, first, last, examples = 0, None, None, []
    for s in range(0, samples.n, SLAB):
        bad = got[s:s + SLAB] != want[s:s + SLAB]
        n = int(bad.sum().item())
        if n == 0:
            continue
        count += n
        where = torch.nonzero(bad).view(-1)
        first = s + int(where[0].item()) if first is None else first
        last = s + int(where[-1].item())
        for i in where[:8 - len(examples)].tolist():
            examples.append((samples.bits_of(s + i), int(want[s + i].item()), int(got[s + i].item())))
    assert count == 0, (f"{what}, {depth}-bit: {count} of {samples.n} codes differ, input bits 0x{samples.bits_of(first):08x} .. "
                        f"0x{samples.bits_of(last):08x}; first (bits, expected, got): "
                        + ", ".join(f"(0x{b:08x}, {e}, {g})" for b, e, g in examples))


def fill_rows(dev, samples, channels, colours):
    """(h, W * channels) float rows: the samples in order over the first `colours` channels of each pixel, the rest 1.0
    (straight alpha), trailing pixels 0."""
    import torch
    per_row = W * colours
    h = -(-samples.n // per_row)
    rows = aligned_rows(dev, h, W * channels, torch.float32, 0.0)
    px = rows.view(torch.int32).view(h, W, channels)
    if channels > colours:
        px[:, :, colours:] = ALPHA_ONE
    band = max(1, SLAB // per_row)
    for r0 in range(0, h, band):
        r1 = min(h, r0 + band)
        part = torch.zeros((r1 - r0) * per_row, dtype=torch.int32, device=dev)
        count = min(part.numel(), samples.n - r0 * per_row)
        part[:count] = samples.pattern(r0 * per_row, count)
        px[r0:r1, :, :colours] = part.view(r1 - r0, W, colours)
    return rows


def run(ctx, desc, rows, launches, what):
    """Encodes device `rows` into fresh planes (filled with -1) and asserts the launch count; returns the planes."""
    import torch
    import avifgpu
    dev = rows.device
    planes = [None if s is None else aligned_rows(dev, s[0], s[1], torch.int16, -1) for s in abi.encode_plane_shapes(desc)]
    before = ctx.launch_count()
    ctx.encode_device(desc, rows.data_ptr(), rows.stride(0) * 4, avifgpu.planes_from_tensors(planes))
    torch.cuda.synchronize(dev)
    made = ctx.launch_count() - before
    if launches == TUNED:
        assert made == TUNED, f"{made} launches: {what} and its right strip make {TUNED}, the generic kernel alone 1"
    else:
        assert made == GENERIC, f"{made} launches: {what} alone makes 1, a tuned launcher {TUNED}"
    return planes


def prepared(gpu, desc):
    """Builds (or finds) the step table `desc` reads and asserts it verified."""
    stats = gpu.prepare_encode(desc).as_dict()
    assert stats["applicable"] == 1 and stats["valid"] == 1 and stats["verify_mismatches"] == 0, stats
    return stats


IDENTITY = lambda: abi.Nclx(1, abi.PRIMARIES_BT2020, abi.TRANSFER_CHAR_PQ, abi.MATRIX_GBR, 1)  # noqa: E731


def rgb_desc(h, depth, transfer, peak, channels=3, planar=False):
    alpha = abi.ALPHA_STRAIGHT if channels in (2, 4) else abi.ALPHA_NONE
    if planar:
        return abi.EncodeDesc(W, h, 32, channels, alpha, depth, transfer, peak, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_444,
                              abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, IDENTITY())
    nclx = cases.NCLX_2020_HLG() if transfer == HLG else None
    return abi.EncodeDesc(W, h, 32, channels, alpha, depth, transfer, peak, abi.LAYOUT_REFERENCE, abi.CHROMA_444,
                          abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, nclx, hlg_extension=abi.HLG_OETF if transfer == HLG else 0)


def planar_codes(planes, n):
    """Identity matrix: Y = G, Cb = B, Cr = R; back into input-sample order."""
    import torch
    return torch.stack([planes[2], planes[0], planes[1]], -1).view(-1)[:n]


def assert_alpha_is_top(plane, depth, what):
    top = (1 << depth) - 1
    wrong = int((plane != top).sum().item())
    assert wrong == 0, f"{what}, {depth}-bit: {wrong} alpha codes are not {top}"


# Each route: (env, samples, depth) -> None.  env = (gpu, gpu_exact, transfer, peak).

def route_flat_interleaved(env, samples, depth):
    gpu, _, transfer, peak = env
    rows = fill_rows(samples.want[depth].device, samples, 3, 3)
    desc = rgb_desc(rows.shape[0], depth, transfer, peak)
    prepared(gpu, desc)
    what = "EncodeRgbF32FlatKernel, interleaved"
    planes = run(gpu, desc, rows, TUNED, what)
    del rows
    assert_codes(planes[0].reshape(-1)[:samples.n], samples, depth, what)


def route_flat_planar(env, samples, depth):
    gpu, _, transfer, peak = env
    rows = fill_rows(samples.want[depth].device, samples, 3, 3)
    desc = rgb_desc(rows.shape[0], depth, transfer, peak, planar=True)
    prepared(gpu, desc)
    what = "EncodeRgbF32FlatKernel, planar"
    planes = run(gpu, desc, rows, TUNED, what)
    del rows
    assert_codes(planar_codes(planes, samples.n), samples, depth, what)


def route_rgba_planar(env, samples, depth):
    gpu, _, transfer, peak = env
    rows = fill_rows(samples.want[depth].device, samples, 4, 3)
    desc = rgb_desc(rows.shape[0], depth, transfer, peak, channels=4, planar=True)
    prepared(gpu, desc)
    what = "EncodeRgbaF32FlatKernel"
    planes = run(gpu, desc, rows, TUNED, what)
    del rows
    assert_alpha_is_top(planes[3], depth, what)
    assert_codes(planar_codes(planes, samples.n), samples, depth, what)


def route_gray_alpha(env, samples, depth):
    gpu, _, transfer, peak = env
    rows = fill_rows(samples.want[depth].device, samples, 2, 1)
    desc = abi.EncodeDesc(W, rows.shape[0], 32, 2, abi.ALPHA_STRAIGHT, depth, transfer, peak)
    prepared(gpu, desc)
    what = "EncodeGrayF32Kernel"
    planes = run(gpu, desc, rows, TUNED, what)
    del rows
    assert_alpha_is_top(planes[3], depth, what)
    assert_codes(planes[0].reshape(-1)[:samples.n], samples, depth, what)


def route_rgba_reference(env, samples, depth):
    gpu, _, transfer, peak = env
    rows = fill_rows(samples.want[depth].device, samples, 4, 3)
    desc = rgb_desc(rows.shape[0], depth, transfer, peak, channels=4)
    prepared(gpu, desc)
    what = "generic kernel, compact table, RGBA reference layout"
    planes = run(gpu, desc, rows, GENERIC, what)
    del rows
    codes = planes[0].view(-1, W, 4)
    assert_alpha_is_top(codes[:, :, 3], depth, what)
    assert_codes(codes[:, :, :3].reshape(-1)[:samples.n], samples, depth, what)


def route_hlg_generic(env, samples, depth):
    gpu, _, transfer, peak = env
    rows = fill_rows(samples.want[depth].device, samples, 3, 3)
    desc = rgb_desc(rows.shape[0], depth, transfer, peak)
    prepared(gpu, desc)
    what = "generic kernel, compact HLG table"
    planes = run(gpu, desc, rows, GENERIC, what)
    del rows
    assert_codes(planes[0].reshape(-1)[:samples.n], samples, depth, what)


def route_exact(env, samples, depth):
    _, gpu_exact, transfer, peak = env
    rows = fill_rows(samples.want[depth].device, samples, 3, 3)
    desc = rgb_desc(rows.shape[0], depth, transfer, peak)
    what = "generic exact kernel (no table)"
    planes = run(gpu_exact, desc, rows, GENERIC, what)
    del rows
    assert_codes(planes[0].reshape(-1)[:samples.n], samples, depth, what)


# route: (function, device memory the whole domain needs with the expected codes resident, in GB, {curve: depths})
PQ_BOTH = {"pq80": (10, 12), "pq1000": (10, 12), "pq10000": (10, 12)}
ROUTES = {
    "flat_interleaved": (route_flat_interleaved, 24, {**PQ_BOTH, "smpte428": (10, 12)}),
    "flat_planar": (route_flat_planar, 28, {**PQ_BOTH, "smpte428": (10, 12)}),
    "rgba_planar": (route_rgba_planar, 30, {**PQ_BOTH, "smpte428": (10,)}),
    "gray_alpha": (route_gray_alpha, 36, {"pq80": (10, 12), "pq10000": (10, 12)}),
    "rgba_reference": (route_rgba_reference, 30, PQ_BOTH),
    "hlg_generic": (route_hlg_generic, 24, {"hlg": (10, 12)}),
    "exact": (route_exact, 24, {curve: (10, 12) for curve in CURVES}),
}
# Ordered by curve, so that each curve's expected codes are built once; "device_transfer" is the float check made while
# building them.
CASES = [(curve, route) for curve in CURVES for route in ["device_transfer", *ROUTES] if route == "device_transfer" or curve in ROUTES[route][2]]


@pytest.mark.gpu
@pytest.mark.parametrize("curve,route", CASES)
def test_every_float_through(gpu, gpu_exact, truths, curve, route):
    import torch
    dev = torch.device("cuda", gpu.device)
    if route == "device_transfer":
        # avifgpu_transfer_f32 against the reference's transfer function over every non-negative finite float: bit for
        # bit, NaN results NaN on both sides (test_gpu_primitives.py's rule: the payload is the FPU's)
        truth = truths(curve)
        assert truth.transfer_mismatches == 0, (f"{truth.transfer_mismatches} floats differ, first (bits, reference, device): "
                                                + ", ".join(truth.transfer_examples))
        return
    function, gigabytes, served = ROUTES[route]
    require_memory(dev, gigabytes)
    samples = whole_domain(dev, truths(curve))
    try:
        for depth in served[curve]:
            function((gpu, gpu_exact, *CURVES[curve]), samples, depth)
    finally:
        torch.cuda.empty_cache()


def negative_slice():
    """-0 and the 2^24 smallest negatives, 2^24 patterns around -1.0, the 2^24 largest finite negatives, -inf and the
    negative NaNs, as uint32 bits."""
    return np.concatenate([np.arange(0x80000000, 0x81000000, dtype=np.uint32),
                           np.arange(0xbf800000 - (1 << 23), 0xbf800000 + (1 << 23), dtype=np.uint32),
                           np.arange(0xff800000 - (1 << 24), 0xff800000, dtype=np.uint32),
                           np.arange(0xff800000, 1 << 32, dtype=np.uint64).astype(np.uint32)])


@pytest.mark.gpu
@pytest.mark.parametrize("curve", list(CURVES))
def test_negative_slice_through_every_route(gpu, gpu_exact, reference, port, curve):
    import torch
    dev = torch.device("cuda", gpu.device)
    transfer, peak = CURVES[curve]
    bits = negative_slice()
    curved = reference_values(reference, port, transfer, peak, bits)
    want = {depth: torch.from_numpy(quantise(curved, depth).view(np.int16)).to(dev) for depth in (10, 12)}
    device_bits = torch.from_numpy(bits.view(np.int32)).to(dev)
    samples = Samples(bits.size, lambda s, c: device_bits[s:s + c], lambda i: int(bits[i]), want)
    for route, (function, _, served) in ROUTES.items():
        for depth in served.get(curve, ()):
            function((gpu, gpu_exact, transfer, peak), samples, depth)


# ---- 12-bit float decodes --------------------------------------------------------------------------------------------------

DECODES = {
    "pq1000": (cases.NCLX_2020_PQ, dict(pq_peak_nits=1000)),
    "hlg_ootf": (cases.NCLX_2020_HLG, dict(hlg_apply_ootf=1, hlg_display_gamma=1.2, hlg_peak_nits=1000)),
    "smpte428": (cases.NCLX_2020_428, dict()),
}


@pytest.mark.gpu
@pytest.mark.parametrize("curve", list(DECODES))
@pytest.mark.parametrize("pair", ["y_cr", "y_cb"])
def test_every_12bit_luma_chroma_pair_through_the_float_decode_kernel(gpu, reference, curve, pair):
    """4:4:4, full range, BT.2020, 4096 rows: in the first 4096 columns one image holds every (Y, Cr) pair (R sees them
    all), the other every (Y, Cb) pair (B sees them all); the third plane is seeded noise, so G sees 2^24 random triples
    per image.  Two more columns of noise (width 4098, the kernel takes groups of 4) are the generic kernel's right strip."""
    n = 1 << 12
    nclx_fn, kwargs = DECODES[curve]
    desc = abi.DecodeDesc(n + 2, n, abi.COLORSPACE_YCBCR, abi.CHROMA_444, 12, abi.ALPHA_NONE, 32, nclx_fn(1), **kwargs)
    luma, paired, noise = cases.rng_for(f"every_pair_{curve}_{pair}").integers(0, n, (3, n, n + 2)).astype(np.uint16)
    luma[:, :n] = np.arange(n, dtype=np.uint16)[None, :]
    paired[:, :n] = np.arange(n, dtype=np.uint16)[:, None]
    planes = [luma, noise, paired, None] if pair == "y_cr" else [luma, paired, noise, None]
    expected = reference.decode(desc, planes, threads=THREADS)
    got = decode_counted(gpu, desc, planes, "the tuned YCbCr decode kernel")
    assert_same_floats(expected, got, planes, f"{curve}, every {pair} pair")


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [10, 12])
@pytest.mark.parametrize("curve", list(DECODES))
def test_every_code_through_the_planar_rgb_table_decode_kernel(gpu, reference, depth, curve):
    """Planar RGB (identity matrix) into RGB32f: each plane holds every code 0 .. 2^depth - 1 in every row (three
    different permutations, so the HLG OOTF's luma mixes them).  Width 4100: the kernel takes groups of 8, the last four
    columns are the generic kernel's right strip."""
    top = (1 << depth) - 1
    h = 8
    nclx_fn, kwargs = DECODES[curve]
    nclx = nclx_fn(1)
    nclx.matrix_coefficients = abi.MATRIX_GBR
    w = 4100
    desc = abi.DecodeDesc(w, h, abi.COLORSPACE_RGB, abi.CHROMA_444, depth, abi.ALPHA_NONE, 32, nclx, **kwargs)
    x = np.arange(w, dtype=np.int64)[None, :]
    y = np.arange(h, dtype=np.int64)[:, None]
    planes = [((x + y) & top).astype(np.uint16), ((x * 1027 + 7 * y) & top).astype(np.uint16),
              ((x * 389 + 11 * y + 5) & top).astype(np.uint16), None]
    expected = reference.decode(desc, planes, threads=THREADS)
    got = decode_counted(gpu, desc, planes, "the table decode kernel")
    assert_same_floats(expected, got, planes, f"{curve}, planar RGB, {depth}-bit")


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [10, 12])
@pytest.mark.parametrize("full_range", [1, 0])
def test_every_container_value_through_the_monochrome_table_decode_kernel(gpu, reference, depth, full_range):
    """Monochrome PQ into Gray32f: every 16-bit container value (codes above 2^depth - 1 included, which the reference
    clamps), full and limited range.  Width 4100, 16 rows: the last four columns are the generic kernel's right strip."""
    w, h = 4100, 16
    values = (np.arange(w * h, dtype=np.uint32) & 0xffff).astype(np.uint16).reshape(h, w)
    desc = abi.DecodeDesc(w, h, abi.COLORSPACE_MONOCHROME, abi.CHROMA_MONOCHROME, depth, abi.ALPHA_NONE, 32,
                          cases.NCLX_2020_PQ(full_range), pq_peak_nits=1000)
    planes = [values, None, None, None]
    expected = reference.decode(desc, planes, threads=THREADS)
    got = decode_counted(gpu, desc, planes, "the table decode kernel")
    assert_same_floats(expected, got, planes, f"monochrome PQ, {depth}-bit, full range {full_range}")
