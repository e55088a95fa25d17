"""The tuned YCbCr decoders over whole code domains, one configuration at a time.

DecodeYccToRgbIntKernel and DecodeYccToRgbF32Kernel (and their batched forms) compute from state chosen per
configuration: the unorm tables of the (depth, range), the inverse-matrix constants of a preset or of the primaries
(MATRIX_CHROMA_DERIVED_NCL), the green division -- the 3-instruction DivideByConstant once VerifyGreenDivisionKernel has
accepted it for that (matrix, range, maxCode), else the IEEE division -- and for PQ the FASTDIV = 1 quotient once
VerifyPqRatio has accepted it.  Each case below holds one configuration, 4:4:4, over a domain that covers every value its
per-pixel arithmetic can see, and compares three things: the tuned kernel, the generic kernel (reached through a row
pointer that is only 4-byte aligned) and, on every domain of at most 2^24 pixels, the compiled reference, bit for bit
(floats as bit patterns, NaN equal to NaN).  The domains:

  triples  every (Y, Cb, Cr) triple: 2^24 at 8 bits (against the reference too), 2^30 at 10 bits (tuned vs generic)
  pairs    every (Y, Cr) and every (Y, Cb) pair, the third plane seeded noise: R and B see every code pair
  g_slab   every (Cb, Cr) pair at Y = 0, limited black, mid and top: G, the channel of the verified division, sees them all

Every image is 2 columns wider than its domain (width = 2 mod 4), so the tuned launcher makes 2 launches (its kernel and
the generic right strip, whose two noise columns are compared like the rest) and the generic kernel alone 1.  Each case
runs on a fresh context, whose first use of the configuration must launch its green-division check (and PQ's ratio or
HLG's divisions): the tuned kernel under test is the one the verification chose.

A capture made before avifgpu_prepare_decode runs the unverified variants instead -- the IEEE green division, the
FASTDIV = 0 PQ quotient -- which the captures below replay over the whole domain against a prepared context.  The 12-bit
pair image also goes through both batch APIs as 64 bands."""
import dataclasses
import os

import numpy as np
import pytest

import cases
from avifgpu import abi
from gpu_harness import aligned_rows, capture, differing_samples, host_or_device, launches_of

THREADS = max(1, min(32, len(os.sched_getaffinity(0))))
TUNED, GENERIC = 2, 1     # launches at width = 2 mod 4: the tuned kernel + its right strip; the generic kernel alone
REFERENCE_LIMIT = 1 << 24  # the largest domain held to the compiled reference
SLAB_ROWS = 2048          # rows per device comparison step of the 2^30 domains

# ---- the configurations ------------------------------------------------------------------------------------------------

CURVES = {
    "": ({}, abi.TRANSFER_CHAR_SRGB),
    "pq1000": (dict(pq_peak_nits=1000), abi.TRANSFER_CHAR_PQ),
    "hlg_ootf": (dict(hlg_apply_ootf=1, hlg_display_gamma=1.2, hlg_peak_nits=1000), abi.TRANSFER_CHAR_HLG),
    "hlg": (dict(hlg_apply_ootf=0), abi.TRANSFER_CHAR_HLG),
    "smpte428": ({}, abi.TRANSFER_CHAR_SMPTE428),
}
# matrix kind: (colour primaries, matrix coefficients); "absent" is no nclx, "absent_flag0" an nclx that is not present
# but carries a limited-range flag, which must be ignored (no nclx: full range and BT.601, YuvLookupTables.cpp:143-144)
MATRICES = {
    "bt601": (abi.PRIMARIES_BT601, abi.MATRIX_BT601),
    "bt709": (abi.PRIMARIES_BT709, abi.MATRIX_BT709),
    "bt2020": (abi.PRIMARIES_BT2020, abi.MATRIX_BT2020_NCL),
    "derived": (abi.PRIMARIES_BT601, abi.MATRIX_CHROMA_DERIVED_NCL),
    "gbr": (abi.PRIMARIES_BT709, abi.MATRIX_GBR),
    "absent": None,
    "absent_flag0": None,
}
# what each tuned family accepts: (code depth, host depth) pairs and matrix kinds (a float host needs an nclx)
FAMILIES = {
    "int": ({(8, 8), (10, 16), (12, 16)}, {"bt601", "bt709", "bt2020", "derived", "gbr", "absent"}),
    "f32": ({(10, 32), (12, 32)}, {"bt601", "bt709", "bt2020", "derived", "gbr"}),
}


@dataclasses.dataclass(frozen=True)
class Config:
    name: str
    family: str    # "int": DecodeYccToRgbIntKernel, "f32": DecodeYccToRgbF32Kernel
    depth: int
    matrix: str
    full: int
    curve: str = ""
    domains: tuple = ("pairs", "g_slab")
    alpha: bool = False

    @property
    def host_depth(self):
        return 32 if self.family == "f32" else 8 if self.depth == 8 else 16

    @property
    def limited(self):
        return not self.full and self.matrix != "absent_flag0"

    def nclx(self):
        transfer = CURVES[self.curve][1]
        if self.matrix == "absent":
            return None
        if self.matrix == "absent_flag0":
            return abi.Nclx(0, abi.PRIMARIES_BT2020, transfer, abi.MATRIX_BT2020_NCL, 0)
        primaries, matrix = MATRICES[self.matrix]
        return abi.Nclx(1, primaries, transfer, matrix, self.full)

    def desc(self, w, h):
        alpha = abi.ALPHA_STRAIGHT if self.alpha else abi.ALPHA_NONE
        return abi.DecodeDesc(w, h, abi.COLORSPACE_YCBCR, abi.CHROMA_444, self.depth, alpha, self.host_depth, self.nclx(),
                              **CURVES[self.curve][0])

    def verifications(self):
        """The launches of the first-use checks on a fresh context: the green division, plus PQ's ratio or HLG's divisions."""
        return 1 + (self.family == "f32" and self.curve != "smpte428")


def int8(matrix, full, alpha=False):
    return Config(f"int8_{matrix}_{'full' if full else 'limited'}{'_alpha' if alpha else ''}", "int", 8, matrix, full,
                  domains=("triples",), alpha=alpha)


def config(family, depth, curve, matrix, full, domains=("pairs", "g_slab")):
    label = f"{'int' if family == 'int' else 'float'}{depth}_{curve + '_' if curve else ''}{matrix}_{'full' if full else 'limited'}"
    return Config(label, family, depth, matrix, full, curve, domains)


WHOLE = ("triples", "pairs", "g_slab")
CONFIGS = [
    *(int8(m, full) for m in ("bt601", "bt709", "bt2020", "derived") for full in (1, 0)),
    int8("absent", 1), int8("absent_flag0", 0), int8("gbr", 1), int8("bt709", 0, alpha=True),
    config("int", 10, "", "bt2020", 0, WHOLE), config("int", 10, "", "bt709", 1, WHOLE),
    config("int", 12, "", "bt2020", 1), config("int", 12, "", "bt2020", 0), config("int", 12, "", "bt709", 0),
    config("f32", 10, "pq1000", "bt2020", 0, WHOLE), config("f32", 10, "hlg_ootf", "bt2020", 0, WHOLE),
    config("f32", 10, "hlg", "bt2020", 1, WHOLE), config("f32", 10, "smpte428", "bt2020", 1, WHOLE),
    config("f32", 10, "pq1000", "bt709", 1), config("f32", 10, "smpte428", "derived", 0),
    config("f32", 10, "hlg_ootf", "bt601", 0), config("f32", 10, "pq1000", "gbr", 1),
    config("f32", 12, "pq1000", "bt2020", 0), config("f32", 12, "hlg_ootf", "bt2020", 0),
    *(config("f32", 12, curve, "bt2020", 1, ("g_slab",)) for curve in ("pq1000", "hlg_ootf", "smpte428")),
]
BY_NAME = {c.name: c for c in CONFIGS}


def test_the_table_covers_every_family_depth_range_and_matrix():
    """Per tuned YCbCr family: at every depth pair it accepts a full-range and a limited-range configuration, and every
    matrix kind it accepts at least once; every 2^30 domain is a 10-bit one, and every configuration has a domain."""
    assert len(BY_NAME) == len(CONFIGS), "configuration names repeat"
    for family, (pairs, matrices) in FAMILIES.items():
        mine = [c for c in CONFIGS if c.family == family]
        for depth, host in sorted(pairs):
            here = [c for c in mine if (c.depth, c.host_depth) == (depth, host)]
            assert any(not c.limited for c in here), f"{family} {depth} -> {host}: no full-range configuration"
            assert any(c.limited for c in here), f"{family} {depth} -> {host}: no limited-range configuration"
        seen = {c.matrix.replace("_flag0", "") for c in mine}
        assert matrices <= seen, f"{family}: matrix kinds {sorted(matrices - seen)} are missing"
        assert {(c.depth, c.host_depth) for c in mine} <= pairs, f"{family}: a depth pair the family does not take"
    for c in CONFIGS:
        assert c.domains and set(c.domains) <= set(WHOLE), c.name
        assert "triples" not in c.domains or c.depth in (8, 10), f"{c.name}: no triple domain at {c.depth} bits"
        assert c.depth == 8 or "pairs" in c.domains or "g_slab" in c.domains, f"{c.name}: nothing against the reference"
    assert any(c.alpha for c in CONFIGS), "no straight-alpha configuration"


# ---- the domain images ---------------------------------------------------------------------------------------------------

def black(depth):
    return 16 << (depth - 8)


def host_images(c):
    """(label, [Y, Cb, Cr, A]) numpy code planes of every domain of `c` of at most 2^24 pixels: n rows of n + 2 columns
    (n x n + 2 for the 8-bit triples, n = 4096), the last two columns noise."""
    n = 1 << c.depth
    top = n - 1
    dtype = abi.code_dtype(c.depth)
    out = []
    if "triples" in c.domains and c.depth == 8:
        rng = cases.rng_for(f"domains_{c.name}_triples")
        y, x = np.mgrid[0:4096, 0:4098]
        index = (y * 4096 + x).astype(np.int64)
        planes = [index & 255, (index >> 8) & 255, index >> 16]
        planes = [np.where(x < 4096, p, rng.integers(0, 256, p.shape)).astype(dtype) for p in planes]
        alpha = ((x + 3 * y) & 255).astype(dtype) if c.alpha else None  # every code in every row
        out.append(("every triple", planes + [alpha]))
    if "pairs" in c.domains:
        for pair in ("y_cr", "y_cb"):
            luma, paired, noise = cases.rng_for(f"domains_{c.name}_{pair}").integers(0, n, (3, n, n + 2)).astype(dtype)
            luma[:, :n] = np.arange(n, dtype=dtype)[None, :]
            paired[:, :n] = np.arange(n, dtype=dtype)[:, None]
            planes = [luma, noise, paired] if pair == "y_cr" else [luma, paired, noise]
            out.append((f"every {pair} pair", planes + [None]))
    if "g_slab" in c.domains:
        for code in (0, black(c.depth), n // 2, top):
            luma, cb, cr = cases.rng_for(f"domains_{c.name}_g{code}").integers(0, n, (3, n, n + 2)).astype(dtype)
            luma[:, :n] = code
            cb[:, :n] = np.arange(n, dtype=dtype)[None, :]
            cr[:, :n] = np.arange(n, dtype=dtype)[:, None]
            out.append((f"every (Cb, Cr) pair at Y = {code}", [luma, cb, cr, None]))
    assert all(p[0].shape[0] * (p[0].shape[1] - 2) <= REFERENCE_LIMIT for _, p in out), "a domain too large for the reference"
    return out


def device_triples(dev, c):
    """Every 10-bit (Y, Cb, Cr) triple as a 32768 x 32770 image on the device: pixel (x, y) of the first 32768 columns
    holds index i = 32768 y + x as Y = i & 1023, Cb = (i >> 10) & 1023, Cr = i >> 20; the last two columns noise."""
    import torch
    n = 1 << 15
    x = torch.arange(n, dtype=torch.int32, device=dev)[None, :]
    y = torch.arange(n, dtype=torch.int32, device=dev)[:, None]
    generator = torch.Generator(device=dev)
    generator.manual_seed(int(cases.rng_for(f"domains_{c.name}_triples").integers(1 << 31)))
    planes = []
    for values in (x & 1023, ((y & 31) << 5) | (x >> 10), y >> 5):
        plane = aligned_rows(dev, n, n + 2, torch.int16, 0)
        plane[:, :n] = values.to(torch.int16)
        plane[:, n:] = torch.randint(0, 1024, (n, 2), dtype=torch.int16, device=dev, generator=generator)
        planes.append(plane)
    return planes + [None]


def upload(dev, planes):
    import torch
    out = []
    for p in planes:
        if p is None:
            out.append(None)
            continue
        wide = p.dtype != np.uint8
        plane = aligned_rows(dev, p.shape[0], p.shape[1], torch.int16 if wide else torch.uint8, 0)
        plane.copy_(torch.from_numpy(p.view(np.int16) if wide else p))
        out.append(plane)
    return out


@pytest.fixture(scope="module")
def reference():
    """The compiled reference.  Missing, it is a failure, not a skip: the launch-count and tuned-vs-generic checks of
    every case run beside the reference comparisons."""
    import oracle
    checker = oracle.load_reference()
    if checker is None:
        pytest.fail("oracle/_ref/libavifref.so is not loaded: the expected samples are the compiled reference's -- build it "
                    "where the reference tree is mounted (make -C oracle); it ships with the tree")
    return checker


# ---- running and comparing ------------------------------------------------------------------------------------------------

def output_rows(dev, desc, offset=0):
    """Destination rows as a byte view: 256-byte aligned, or `offset` bytes past that (4: only 4-byte aligned, which
    sends the call to the generic kernel)."""
    import torch
    row_bytes = desc.width * abi.decode_host_channels(desc) * desc.host_depth // 8
    return aligned_rows(dev, desc.height, row_bytes + offset, torch.uint8, 0xCD)[:, offset:]


def decode_into(ctx, desc, planes, rows, launches, what, stream=0):
    import torch
    import avifgpu
    before = ctx.launch_count()
    ctx.decode_device(desc, avifgpu.planes_from_tensors(planes), rows.data_ptr(), rows.stride(0), stream=stream)
    torch.cuda.synchronize()
    made = ctx.launch_count() - before
    assert made == launches, f"{what}: {made} launches, the tuned launcher and its strip make {TUNED}, the generic kernel {GENERIC}"
    return rows


def host_values(rows, desc):
    return rows.contiguous().cpu().numpy().view(abi.host_dtype(desc.host_depth))


def assert_agree(results, planes, desc, what):
    """results: {"tuned" / "generic" / "reference": host rows}.  Every pair must agree; otherwise the message names
    which pairs disagree and, for the first few differing samples, the pixel's codes and all three values."""
    channels = abi.decode_host_channels(desc)
    names = list(results)
    failures = []
    for i, a in enumerate(names):
        for b in names[i + 1:]:
            bad = differing_samples(results[a], results[b])
            if bad.any():
                shown = []
                for y, x in np.argwhere(bad)[:4]:
                    codes = tuple(int(p[y, x // channels]) for p in planes if p is not None)
                    values = ", ".join(f"{k} {results[k][y, x].item()!r}" for k in names)
                    shown.append(f"codes {codes} channel {x % channels}: {values}")
                failures.append(f"{a} and {b} differ in {int(bad.sum())} of {bad.size} samples; " + "; ".join(shown))
    if failures:
        pytest.fail(f"{what}: " + " | ".join(failures))


def check_host_image(ctx, reference, c, label, planes):
    """One domain image of at most 2^24 pixels: tuned, generic and the compiled reference."""
    import torch
    dev = torch.device("cuda", ctx.device)
    h, w = planes[0].shape
    desc = c.desc(w, h)
    device_planes = upload(dev, planes)
    what = f"{c.name}, {label}"
    tuned = host_values(decode_into(ctx, desc, device_planes, output_rows(dev, desc), TUNED, what + " (tuned)"), desc)
    generic = host_values(decode_into(ctx, desc, device_planes, output_rows(dev, desc, 4), GENERIC, what + " (generic)"), desc)
    expected = reference.decode(desc, planes, threads=THREADS)
    assert_agree({"tuned": tuned, "generic": generic, "reference": expected}, planes, desc, what)


def require_memory(dev, gigabytes=60):
    import torch
    if torch.cuda.get_device_properties(dev).total_memory < gigabytes * 2**30:
        pytest.skip(f"the 2^30 domains need {gigabytes} GB of device memory")


def assert_same_rows(a, b, desc, planes, what, names=("tuned", "generic")):
    """Two device byte views of the same rows, slab by slab; the message names the first differing samples by their
    codes (read back from the device planes)."""
    import torch
    floats = desc.host_depth == 32
    count, examples = 0, []
    channels = abi.decode_host_channels(desc)
    sample_bytes = desc.host_depth // 8
    for y0 in range(0, desc.height, SLAB_ROWS):
        sa, sb = a[y0:y0 + SLAB_ROWS], b[y0:y0 + SLAB_ROWS]
        if floats:
            fa, fb = sa.view(torch.float32), sb.view(torch.float32)
            bad = (fa.view(torch.int32) != fb.view(torch.int32)) & ~(torch.isnan(fa) & torch.isnan(fb))
        else:
            bad = sa != sb
            fa, fb = sa, sb
        n = int(bad.sum().item())
        if n == 0:
            continue
        count += n
        for y, x in torch.nonzero(bad)[:4 - len(examples)].tolist():
            pixel = x // channels if floats else x // (channels * sample_bytes)
            codes = tuple(int(p[y0 + y, pixel].item()) & 0xffff for p in planes if p is not None)
            if floats:
                va, vb = float(fa[y, x].item()), float(fb[y, x].item())
            else:
                k = x - x % sample_bytes
                va = int.from_bytes(bytes(sa[y, k:k + sample_bytes].tolist()), "little")
                vb = int.from_bytes(bytes(sb[y, k:k + sample_bytes].tolist()), "little")
            examples.append(f"row {y0 + y} pixel {pixel} codes {codes} channel {(x // (1 if floats else sample_bytes)) % channels}: "
                            f"{names[0]} {va!r}, {names[1]} {vb!r}")
    assert count == 0, f"{what}: {names[0]} and {names[1]} differ in {count} samples; " + "; ".join(examples)


def check_device_triples(ctx, c):
    """Every 10-bit triple: tuned vs generic on the device."""
    import torch
    dev = torch.device("cuda", ctx.device)
    require_memory(dev)
    planes = device_triples(dev, c)
    desc = c.desc(planes[0].shape[1], planes[0].shape[0])
    what = f"{c.name}, every 10-bit triple"
    try:
        tuned = decode_into(ctx, desc, planes, output_rows(dev, desc), TUNED, what + " (tuned)")
        generic = decode_into(ctx, desc, planes, output_rows(dev, desc, 4), GENERIC, what + " (generic)")
        assert_same_rows(tuned, generic, desc, planes, what)
    finally:
        del planes
        tuned = generic = None
        torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BY_NAME))
def test_every_code_of_the_domain(reference, name):
    """One configuration on a fresh context: its first use launches its checks, then every domain image runs through the
    tuned kernel (2 launches) and the generic kernel (1), compared with each other and, up to 2^24 pixels, with the
    compiled reference."""
    import avifgpu
    c = BY_NAME[name]
    with avifgpu.Context(0) as ctx:
        first = c.desc(4098, 2)
        checks = launches_of(ctx, lambda: ctx.prepare_decode(first))
        assert checks == c.verifications(), f"{name}: {checks} launches at first use, its checks make {c.verifications()}"
        assert launches_of(ctx, lambda: ctx.prepare_decode(first)) == 0, "the checks ran again"
        for label, planes in host_images(c):
            check_host_image(ctx, reference, c, label, planes)
        if "triples" in c.domains and c.depth == 10:
            check_device_triples(ctx, c)


# ---- captures before prepare: the unverified variants --------------------------------------------------------------------

CAPTURES = ["int10_bt2020_limited", "float10_pq1000_bt2020_limited", "float12_smpte428_bt2020_full"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CAPTURES)
def test_unprepared_capture_over_the_domain(case):
    """A fresh context that has verified nothing captures one call: the tuned route (2 launches) with no check launched,
    so the graph holds the IEEE green division (and for PQ the FASTDIV = 0 quotient).  Replayed over every domain image
    copied into the captured planes, it must equal a prepared context's direct call."""
    import torch
    import avifgpu
    c = BY_NAME[case]
    dev = torch.device("cuda", 0)
    if c.depth == 10:
        require_memory(dev)
        images = [("every 10-bit triple", None)]
    else:
        images = host_images(dataclasses.replace(c, domains=("pairs", "g_slab")))
    with avifgpu.Context(0) as fresh, avifgpu.Context(0) as prepared:
        planes = device_triples(dev, c) if c.depth == 10 else upload(dev, images[0][1])
        desc = c.desc(planes[0].shape[1], planes[0].shape[0])
        prepared.prepare_decode(desc)
        rows = output_rows(dev, desc)
        struct = avifgpu.planes_from_tensors(planes)
        stream = torch.cuda.Stream()
        stream.wait_stream(torch.cuda.current_stream())
        graph, launches = capture(fresh, lambda s: fresh.decode_device(desc, struct, rows.data_ptr(), rows.stride(0), stream=s), stream)
        assert launches == TUNED, f"{launches} launches captured: the tuned route makes {TUNED}, and no check may run inside a capture"
        try:
            direct = output_rows(dev, desc)
            for label, host in images:
                with torch.cuda.stream(stream):  # the copies and the replay in one stream order
                    if host is not None:
                        for plane, p in zip(planes, host):
                            if p is not None:
                                plane.copy_(torch.from_numpy(p.view(np.int16)))
                    graph.replay()
                torch.cuda.synchronize()
                decode_into(prepared, desc, planes, direct, TUNED, f"{case}, prepared")
                assert_same_rows(rows, direct, desc, planes, f"{case}, {label}", ("captured", "prepared"))
            assert fresh.launch_count() == launches, "the fresh context launched something after the capture"
        finally:
            del graph
            planes = rows = direct = None
            torch.cuda.empty_cache()


# ---- both batch APIs on the 12-bit pair image ----------------------------------------------------------------------------

class Band:
    """64 rows of the pair image: its planes and destination rows as views into the whole image's."""

    def __init__(self, w, h, rows, planes):
        self.w, self.h, self.rows, self.planes = w, h, rows, planes

    def record(self):
        return (self.w, self.h, self.rows, self.planes)


@pytest.mark.gpu
@pytest.mark.parametrize("api", ["host", "device"])
@pytest.mark.parametrize("name", ["int12_bt2020_limited", "float12_pq1000_bt2020_limited"])
def test_the_pair_image_as_a_batch(reference, name, api):
    """The 12-bit (Y, Cr) pair image cut into 64 bands of 64 rows, one batch of 64 images (DecodeYccToRgbIntBatchKernel
    or DecodeYccToRgbF32BatchKernel and the edge kernel): the rows equal a direct call's, which equal the reference's."""
    import torch
    import avifgpu
    c = BY_NAME[name]
    dev = torch.device("cuda", 0)
    label, host = host_images(c)[0]
    h, w = host[0].shape
    desc = c.desc(w, h)
    band_desc = c.desc(0, 0)
    with avifgpu.Context(0) as ctx:
        ctx.prepare_decode(desc)
        planes = upload(dev, host)
        direct = decode_into(ctx, desc, planes, output_rows(dev, desc), TUNED, f"{name}, direct")
        assert_agree({"direct": host_values(direct, desc), "reference": reference.decode(desc, host, threads=THREADS)}, host, desc, f"{name}, {label}")
        rows = output_rows(dev, desc)
        step = h // 64
        bands = [Band(w, step, rows[y:y + step], [None if p is None else p[y:y + step] for p in planes]) for y in range(0, h, step)]

        def check(images):
            assert_same_rows(rows, direct, desc, planes, f"{name}, {label}, {api}-described batch", ("batch", "direct"))

        host_or_device(ctx, band_desc, "decode", api, bands, check)
