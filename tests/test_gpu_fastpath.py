"""The tuned float-host encode kernel (kernels_fast.cu) and its exact step tables (curve_tables.cu) on an H100:
table self-verification over every float, inputs aimed at the step thresholds and fuzzy bands, queue overflow,
edge strips, strides -- all bit-exact against the CPU checker."""
import numpy as np
import pytest

import cases
from avifgpu import abi

pytestmark = pytest.mark.gpu


def planar_desc(w, h, depth=12, transfer=abi.TRANSFER_PQ, peak=80, chroma=abi.CHROMA_420, down=abi.DOWN_FILTER_BOX, nclx=None):
    return abi.EncodeDesc(w, h, 32, 3, abi.ALPHA_NONE, depth, transfer, peak, abi.LAYOUT_PLANAR_YCBCR, chroma, down, abi.GRAY16_LUT,
                          nclx if nclx is not None else cases.NCLX_2020_PQ())


@pytest.mark.parametrize("transfer,peak,depth", [(abi.TRANSFER_PQ, 80, 12), (abi.TRANSFER_PQ, 80, 10), (abi.TRANSFER_PQ, 1000, 12),
                                                 (abi.TRANSFER_PQ, 10000, 12), (abi.TRANSFER_PQ, 1, 10), (abi.TRANSFER_SMPTE428, 80, 12),
                                                 (abi.TRANSFER_SMPTE428, 80, 10), (abi.TRANSFER_HLG, 80, 10), (abi.TRANSFER_HLG, 80, 12)])
def test_step_tables_verify_against_every_float(gpu, transfer, peak, depth):
    desc = planar_desc(8, 8, depth, transfer, peak)
    if transfer == abi.TRANSFER_HLG:
        desc.hlg_extension = abi.HLG_OETF  # the HLG save path: its table serves the generic kernel
    stats = gpu.prepare_encode(desc).as_dict()
    print(stats)
    assert stats["applicable"] == 1 and stats["valid"] == 1, stats
    assert stats["verify_mismatches"] == 0
    assert stats["swept_inputs"] == 0x7f800000
    assert stats["steps"] == (1 << depth) - 1
    if transfer == abi.TRANSFER_SMPTE428:
        assert stats["bands"] == 0  # a single powf is monotone: SURVEY.md 7.3
    assert stats["in_band_inputs"] < 0.02 * stats["swept_inputs"]


def threshold_inputs(port, transfer, peak, depth, rng, count_codes=400, window=2600, per_code=48):
    """Floats around the step thresholds of the quantised curve, located by bisection on the CPU checker."""
    fn = abi.FN_LINEAR_TO_PQ if transfer == abi.TRANSFER_PQ else abi.FN_LINEAR_TO_SMPTE428
    maxv = np.float32((1 << depth) - 1)

    def codes(x):
        v = port.transfer(fn, x, float(peak)) * maxv
        v = np.where(v < 0, np.float32(0), np.where(v > maxv, maxv, v))
        return np.nan_to_num(v, nan=0.0).astype(np.uint32)

    ks = np.unique(np.concatenate([rng.integers(1, 1 << depth, count_codes), [1, 2, (1 << depth) - 2, (1 << depth) - 1]]))
    lo = np.zeros(ks.size, np.uint32)
    hi = np.full(ks.size, np.float32(3.0e38).view(np.uint32), np.uint32)
    for _ in range(33):
        mid = ((lo.astype(np.uint64) + hi.astype(np.uint64)) // 2).astype(np.uint32)
        c = codes(mid.view(np.float32))
        below = c < ks
        lo = np.where(below, mid, lo)
        hi = np.where(below, hi, mid)
    offsets = rng.integers(-window, window + 1, (ks.size, per_code))
    bits = (hi.astype(np.int64)[:, None] + offsets).clip(0, 0x7f7fffff).astype(np.uint32)
    return bits.reshape(-1).view(np.float32)


@pytest.mark.parametrize("transfer,peak,depth", [(abi.TRANSFER_PQ, 80, 12), (abi.TRANSFER_PQ, 1000, 10), (abi.TRANSFER_SMPTE428, 80, 12)])
def test_inputs_at_the_thresholds(gpu, port, transfer, peak, depth):
    rng = np.random.default_rng(depth * 1000 + peak)
    values = threshold_inputs(port, transfer, peak, depth, rng)
    w = 256
    h = (values.size // (3 * w)) & ~1
    rows = np.ascontiguousarray(values[:h * w * 3].reshape(h, w * 3))
    for chroma in (abi.CHROMA_420, abi.CHROMA_444):
        desc = planar_desc(w, h, depth, transfer, peak, chroma)
        assert cases.same_planes(port.encode(desc, rows, threads=8), gpu.encode(desc, rows))


def test_all_samples_in_a_band_overflow_the_queue(gpu, port):
    """A flat image whose value sits inside a fuzzy band sends every sample down the exact path (768 per warp tile,
    queue capacity 128): the flush-and-continue logic must still give the exact result."""
    rng = np.random.default_rng(7)
    near = threshold_inputs(port, abi.TRANSFER_PQ, 80, 12, rng, count_codes=8, window=300, per_code=8)
    w, h = 512, 8
    for value in near[:6]:
        rows = np.full((h, w * 3), value, np.float32)
        rows[::2, ::7] = np.nextafter(value, np.float32(2.0))
        desc = planar_desc(w, h)
        assert cases.same_planes(port.encode(desc, rows), gpu.encode(desc, rows))


SHAPES = [(4, 2), (5, 3), (7, 2), (128, 2), (129, 3), (130, 4), (131, 5), (257, 7), (1024, 33), (4, 1)]


@pytest.mark.parametrize("w,h", SHAPES)
@pytest.mark.parametrize("chroma", [abi.CHROMA_420, abi.CHROMA_422, abi.CHROMA_444])
def test_edges_and_chroma_modes(gpu, port, w, h, chroma):
    rng = cases.rng_for(f"fast_{w}x{h}_{chroma}")
    rows = cases.float_host_rows(rng, h, w, 3, specials=True)
    for transfer, depth, down, nclx in ((abi.TRANSFER_PQ, 12, abi.DOWN_FILTER_BOX, cases.NCLX_2020_PQ()),
                                        (abi.TRANSFER_PQ, 10, abi.DOWN_FILTER_TOP_LEFT, None),
                                        (abi.TRANSFER_SMPTE428, 12, abi.DOWN_FILTER_BOX, cases.NCLX_709()),
                                        (abi.TRANSFER_CLIP, 10, abi.DOWN_FILTER_BOX, cases.NCLX_DERIVED())):
        desc = planar_desc(w, h, depth, transfer, 80, chroma, down, nclx)
        got = gpu.encode(desc, rows, pad=5)
        assert cases.same_planes(port.encode(desc, rows), got), (transfer, depth, down)
        for g in got:
            if g is not None:
                assert (g.base[:, g.shape[1]:] == 0xCD).all(), "wrote into the row padding"


@pytest.mark.parametrize("w,h", [(4, 2), (5, 3), (128, 2), (131, 5), (260, 8), (1024, 33)])
@pytest.mark.parametrize("chroma", [abi.CHROMA_420, abi.CHROMA_422, abi.CHROMA_444])
@pytest.mark.parametrize("alpha", [abi.ALPHA_STRAIGHT, abi.ALPHA_PREMULTIPLIED])
def test_rgba32f_fast_kernel(gpu, gpu_exact, port, w, h, chroma, alpha):
    """Float RGBA hosts (kernels_fast_rgba.cu): clamp / premultiplication before the curve, alpha plane beside Y/Cb/Cr."""
    rng = cases.rng_for(f"rgba32_{w}x{h}_{chroma}_{alpha}")
    rows = cases.float_host_rows(rng, h, w, 4, specials=True)
    for depth, peak, nclx in ((12, 80, cases.NCLX_2020_PQ()), (10, 1000, None)):
        desc = abi.EncodeDesc(w, h, 32, 4, alpha, depth, abi.TRANSFER_PQ, peak, abi.LAYOUT_PLANAR_YCBCR, chroma, abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, nclx)
        expected = port.encode(desc, rows)
        for ctx in (gpu, gpu_exact):
            got = ctx.encode(desc, rows, pad=5)
            assert cases.same_planes(expected, got), (depth, peak)
            for g in got:
                if g is not None:
                    assert (g.base[:, g.shape[1]:] == 0xCD).all(), "wrote into the row padding"


def test_unaligned_device_buffers_fall_back_correctly(gpu, port):
    """Odd strides / offsets defeat the 128-bit loads: the launcher must route those calls to the generic kernel."""
    import torch
    import avifgpu
    dev = torch.device("cuda", gpu.device)
    w, h = 64, 6
    desc = planar_desc(w, h)
    rows = cases.float_host_rows(np.random.default_rng(11), h, w, 3)
    expected = port.encode(desc, rows)
    backing = torch.zeros((h, w * 3 + 1), dtype=torch.float32, device=dev)  # row stride not a multiple of 16 bytes
    backing[:, :w * 3] = torch.from_numpy(rows).to(dev)
    shapes = abi.encode_plane_shapes(desc)
    planes = [None if s is None else torch.zeros((s[0], s[1] + 1), dtype=torch.int16, device=dev) for s in shapes]
    views = [None if t is None else t[:, 1:] for t in planes]  # 2-byte aligned plane origins
    gpu.encode_device(desc, backing.data_ptr(), backing.stride(0) * 4, avifgpu.planes_from_tensors(views))
    torch.cuda.synchronize(dev)
    for e, v in zip(expected, views):
        if e is not None:
            assert np.array_equal(v.cpu().numpy().view(np.uint16), e)


# ---- 16-bit integer hosts (kernels_fast_int.cu) ------------------------------------------------------------------------

@pytest.mark.parametrize("w,h", [(8, 2), (9, 3), (16, 1), (67, 5), (256, 17), (1031, 6)])
@pytest.mark.parametrize("channels", [3, 4])
@pytest.mark.parametrize("chroma", [abi.CHROMA_420, abi.CHROMA_422, abi.CHROMA_444])
def test_rgb16_planar_fast_kernel(gpu, port, w, h, channels, chroma):
    rng = cases.rng_for(f"rgb16_{w}x{h}_{channels}_{chroma}")
    rows = cases.int_host_rows(rng, h, w, channels, 16, beyond=True)
    alpha = abi.ALPHA_NONE if channels == 3 else abi.ALPHA_STRAIGHT
    for depth, down, nclx in ((10, abi.DOWN_FILTER_BOX, None), (12, abi.DOWN_FILTER_TOP_LEFT, cases.NCLX_709()),
                              (10, abi.DOWN_FILTER_BOX, cases.NCLX_GBR() if chroma == abi.CHROMA_444 else cases.NCLX_2020_PQ())):
        desc = abi.EncodeDesc(w, h, 16, channels, alpha, depth, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, chroma, down, abi.GRAY16_LUT, nclx)
        got = gpu.encode(desc, rows, pad=8)
        assert cases.same_planes(port.encode(desc, rows), got), (depth, down)
        for g in got:
            if g is not None:
                assert (g.base[:, g.shape[1]:] == 0xCD).all(), "wrote into the row padding"


@pytest.mark.parametrize("w,h", [(8, 2), (9, 3), (16, 1), (67, 5), (256, 17), (1031, 6)])
@pytest.mark.parametrize("channels", [3, 4])
@pytest.mark.parametrize("chroma", [abi.CHROMA_420, abi.CHROMA_422, abi.CHROMA_444])
def test_rgb8_planar_fast_kernel(gpu, port, w, h, channels, chroma):
    """8-bit hosts (WriteHeifImage.cpp:629-806) into 8-bit planes (the sample is the code) and into 10 / 12-bit planes
    (the 256-entry depth table), plus 16-bit hosts into 8-bit planes: the same tuned kernel, other sample types."""
    rng = cases.rng_for(f"rgb8_{w}x{h}_{channels}_{chroma}")
    alpha = abi.ALPHA_NONE if channels == 3 else abi.ALPHA_STRAIGHT
    for host_depth, depth, down, nclx in ((8, 8, abi.DOWN_FILTER_BOX, cases.NCLX_601()), (8, 8, abi.DOWN_FILTER_TOP_LEFT, None),
                                          (8, 10, abi.DOWN_FILTER_BOX, cases.NCLX_709()), (8, 12, abi.DOWN_FILTER_BOX, cases.NCLX_2020_PQ()),
                                          (8, 8, abi.DOWN_FILTER_BOX, cases.NCLX_GBR() if chroma == abi.CHROMA_444 else cases.NCLX_601()),
                                          (16, 8, abi.DOWN_FILTER_BOX, cases.NCLX_601())):
        rows = cases.int_host_rows(rng, h, w, channels, host_depth, beyond=(host_depth == 16))
        desc = abi.EncodeDesc(w, h, host_depth, channels, alpha, depth, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, chroma, down, abi.GRAY16_LUT, nclx)
        got = gpu.encode(desc, rows, pad=8)
        assert cases.same_planes(port.encode(desc, rows), got), (host_depth, depth, down)
        for g in got:
            if g is not None:
                assert (g.base[:, g.shape[1]:] == 0xCD).all(), "wrote into the row padding"


def test_rgb8_every_triple_through_the_integer_encode_kernel(gpu):
    """All 2^24 RGB8 triples (4096 x 4096) into 8-bit and 10-bit 4:4:4 planes: tuned kernel == generic kernel (reached
    through a plane origin that is only 2-byte aligned)."""
    import torch
    import avifgpu
    dev = torch.device("cuda", gpu.device)
    w = h = 4096
    index = torch.arange(w * h, dtype=torch.int32, device=dev)
    rows = torch.stack([index & 255, (index >> 8) & 255, index >> 16], dim=1).to(torch.uint8).view(h, w * 3).contiguous()
    for depth in (8, 10):
        desc = abi.EncodeDesc(w, h, 8, 3, abi.ALPHA_NONE, depth, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_444,
                              abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, cases.NCLX_601())
        dt = torch.uint8 if depth == 8 else torch.int16
        shapes = abi.encode_plane_shapes(desc)
        fast = [None if s is None else torch.zeros(s, dtype=dt, device=dev) for s in shapes]
        gpu.encode_device(desc, rows.data_ptr(), rows.stride(0), avifgpu.planes_from_tensors(fast))
        backing = [None if s is None else torch.zeros((s[0], s[1] + 8), dtype=dt, device=dev) for s in shapes]
        exact = [None if t is None else t[:, 1:shapes[k][1] + 1] for k, t in enumerate(backing)]
        gpu.encode_device(desc, rows.data_ptr(), rows.stride(0), avifgpu.planes_from_tensors(exact))
        torch.cuda.synchronize(dev)
        for a, b in zip(fast, exact):
            if a is not None:
                assert int((a != b).sum().item()) == 0


@pytest.mark.parametrize("w,h", [(8, 1), (13, 3), (64, 9), (4096, 4)])
@pytest.mark.parametrize("curve", [abi.GRAY16_LUT, abi.GRAY16_SMPTE428])
@pytest.mark.parametrize("depth", [10, 12])
def test_gray16_lut_fast_kernel(gpu, port, w, h, curve, depth):
    rng = cases.rng_for(f"gray16_{w}x{h}_{curve}_{depth}")
    rows = cases.int_host_rows(rng, h, w, 1, 16, beyond=True)
    desc = abi.EncodeDesc(w, h, 16, 1, abi.ALPHA_NONE, depth, gray16_curve=curve)
    assert cases.same_planes(port.encode(desc, rows), gpu.encode(desc, rows, pad=8))


def test_gray16_lut_every_input(gpu, port):
    """All 65536 host samples through both Gray16 curves, against the CPU checker."""
    rows = np.arange(65536, dtype=np.uint32).astype(np.uint16).reshape(16, 4096)
    for curve in (abi.GRAY16_LUT, abi.GRAY16_SMPTE428):
        for depth in (10, 12):
            desc = abi.EncodeDesc(4096, 16, 16, 1, abi.ALPHA_NONE, depth, gray16_curve=curve)
            assert cases.same_planes(port.encode(desc, rows), gpu.encode(desc, rows))


# ---- float decode (kernels_fast_decode.cu) -------------------------------------------------------------------------------

@pytest.mark.parametrize("channels", [1, 2])
def test_every_float_through_the_gray_float_kernel(gpu, gpu_exact, channels):
    """kernels_fast_gray32.cu over every bit pattern from +0 through the NaNs into the first negative values, against the
    generic exact kernel of a context that never builds tables.  Gray alone is clamped to [0, 1] before the curve
    (WriteHeifImage.cpp:602), so that run pins the clamp and the table below 1.0; Gray + straight alpha (alpha = 1.0) is
    not clamped and takes every float through the table, the band bitmap and the +inf / NaN route."""
    import torch
    import avifgpu
    dev = torch.device("cuda", gpu.device)
    if torch.cuda.get_device_properties(dev).total_memory < 60 * 2**30:
        pytest.skip("needs ~40 GB of device memory")
    w = 4096
    h = ((1 << 31) // w + 2) & ~1
    alpha = abi.ALPHA_STRAIGHT if channels == 2 else abi.ALPHA_NONE
    desc = abi.EncodeDesc(w, h, 32, channels, alpha, 12, abi.TRANSFER_PQ, 80)
    rows = torch.empty((h, w * channels), dtype=torch.float32, device=dev)
    bits = rows.view(torch.int32).view(h * w, channels)
    chunk = 1 << 27
    for start in range(0, h * w, chunk):
        n = min(chunk, h * w - start)
        bits[start:start + n, 0] = torch.arange(start, start + n, dtype=torch.int64, device=dev).to(torch.int32)  # wraps past 2^31
        if channels == 2:
            bits[start:start + n, 1] = 0x3f800000
    shapes = abi.encode_plane_shapes(desc)
    fast = [None if s is None else torch.full(s, -1, dtype=torch.int16, device=dev) for s in shapes]
    assert gpu.prepare_encode(desc).as_dict()["valid"] == 1  # the step table, built and verified before the count below
    before_fast = gpu.launch_count()
    gpu.encode_device(desc, rows.data_ptr(), rows.stride(0) * 4, avifgpu.planes_from_tensors(fast))
    assert gpu.launch_count() - before_fast == 1  # the tuned kernel alone (width is a multiple of 4)
    backing = [None if s is None else torch.full((s[0], s[1] + 1), -1, dtype=torch.int16, device=dev) for s in shapes]
    exact = [None if t is None else t[:, 1:] for t in backing]  # 2-byte aligned origins: the launcher takes the generic kernel
    gpu_exact.encode_device(desc, rows.data_ptr(), rows.stride(0) * 4, avifgpu.planes_from_tensors(exact))
    torch.cuda.synchronize(dev)
    for k, plane in enumerate(fast):
        if plane is None:
            continue
        differing = int((plane != exact[k]).sum().item())
        assert differing == 0, f"plane {k}: {differing} of {plane.numel()} codes differ"
    codes = exact[0].reshape(-1)[:0x3f800000].to(torch.int32) & 0xffff  # +0 .. 1.0: monotone up to the one-code flips inside bands
    assert int(codes.min().item()) == 0 and bool((codes[1:] >= codes[:-1] - 1).all().item())
    assert 1900 < int((exact[0].reshape(-1)[0x3f800000].to(torch.int32) & 0xffff).item()) < 2050  # 1.0 at 80 nit: PQ 0.482


@pytest.mark.parametrize("w,h", [(4, 2), (5, 3), (128, 2), (131, 7), (260, 9), (1024, 16)])
@pytest.mark.parametrize("chroma", [abi.CHROMA_420, abi.CHROMA_422, abi.CHROMA_444])
def test_ycc_to_rgb32_fast_kernel(gpu, port, w, h, chroma):
    for bit_depth, nclx, kwargs in ((10, cases.NCLX_2020_HLG(1), dict(hlg_apply_ootf=1)),
                                    (10, cases.NCLX_2020_HLG(0), dict(hlg_apply_ootf=0)),
                                    (12, cases.NCLX_2020_PQ(1), dict(pq_peak_nits=1000)),
                                    (12, cases.NCLX_2020_428(0), dict()),
                                    (10, abi.Nclx(1, abi.PRIMARIES_BT709, abi.TRANSFER_CHAR_HLG, abi.MATRIX_BT709, 1), dict(hlg_display_gamma=1.4, hlg_peak_nits=400))):
        desc = abi.DecodeDesc(w, h, abi.COLORSPACE_YCBCR, chroma, bit_depth, abi.ALPHA_NONE, 32, nclx, **kwargs)
        planes = cases.code_planes(cases.rng_for(f"dec32_{w}x{h}_{chroma}_{bit_depth}"), desc, overshoot=True)
        expected = port.decode(desc, planes, threads=4)
        got = gpu.decode(desc, planes)
        assert cases.same_bits(expected, got), (bit_depth, kwargs, int((expected.view(np.uint32) != got.view(np.uint32)).sum()))
        for alpha in (abi.ALPHA_STRAIGHT, abi.ALPHA_PREMULTIPLIED):  # straight: the tuned kernel's RGBA variant; premultiplied: generic
            adesc = desc.copy(alpha_state=alpha)
            aplanes = cases.code_planes(cases.rng_for(f"dec32a_{w}x{h}_{chroma}_{bit_depth}_{alpha}"), adesc, overshoot=True)
            assert cases.same_bits(port.decode(adesc, aplanes, threads=4), gpu.decode(adesc, aplanes)), (bit_depth, kwargs, alpha)
        # odd first rows (4:2:0 blocks may start anywhere on decode) must still agree
        if h > 3:
            out = np.zeros_like(expected)
            gpu.decode(desc, planes, y0=0, nrows=1, out=out[0:1])
            gpu.decode(desc, planes, y0=1, nrows=h - 1, out=out[1:])
            assert cases.same_bits(expected, out)


@pytest.mark.parametrize("gamma,peak", [(1.2, 1000), (0.85, 100), (1.0, 334), (1.79, 25000), (1.8, 27000), (2.5, 100000)])
def test_hlg_ootf_exponents_on_both_sides_of_the_screen_free_powf(gpu, port, gamma, peak):
    """The tuned decode kernel's OOTF calls the branch-free powf when |gamma - 1| is in (0, 0.8) (device_math.cuh
    PowfStraightLineCovers / PowfStraightLineWide); gamma = 1 (exponent 0), 1.8 and 2.5 go to the generic kernel.  Either way the
    float samples are the reference's, bit for bit -- black pixels (luma 0) included."""
    w, h = 260, 8
    nclx = cases.NCLX_2020_HLG(1)
    for chroma, alpha in ((abi.CHROMA_420, abi.ALPHA_NONE), (abi.CHROMA_444, abi.ALPHA_STRAIGHT)):
        desc = abi.DecodeDesc(w, h, abi.COLORSPACE_YCBCR, chroma, 10, alpha, 32, nclx, hlg_apply_ootf=1, hlg_display_gamma=gamma, hlg_peak_nits=peak)
        planes = cases.code_planes(cases.rng_for(f"ootf_{gamma}_{chroma}"), desc, overshoot=True)
        planes[0][0, :8] = 0  # black: luma 0 under neutral chroma -> powf(0, gamma - 1), +inf for gamma < 1, then 0 * inf
        planes[1][0, :8 >> (0 if chroma == abi.CHROMA_444 else 1)] = 512
        planes[2][0, :8 >> (0 if chroma == abi.CHROMA_444 else 1)] = 512
        expected = port.decode(desc, planes, threads=4)
        got = gpu.decode(desc, planes)
        e, g = expected.view(np.uint32).ravel(), got.view(np.uint32).ravel()
        both_nan = np.isnan(expected.ravel()) & np.isnan(got.ravel())  # 0 * inf: a NaN on both sides, the payload is the FPU's
        assert np.array_equal(e[~both_nan], g[~both_nan]) and np.array_equal(np.isnan(expected), np.isnan(got)), (gamma, chroma, int((e != g).sum()))


# ---- every float through the production kernel ---------------------------------------------------------------------------

def test_every_float_through_the_production_encode_kernel(gpu, gpu_exact):
    """The step tables are verified against the exact curve by the builder's own sweep; this runs the PRODUCTION kernel
    (copy-engine staging, table look-up, band bitmap, +inf / NaN route) over an image that contains every bit pattern
    from +0 through the positive NaNs and on into the first negative values -- 2^31 + samples -- with the identity
    (GBR) matrix in 4:4:4, so the three planes ARE the per-sample codes.  The expected planes come from the generic
    exact kernel of a context that never builds tables (glibc-identical powf per sample), which test_gpu_parity.py pins
    to the CPU checker."""
    import torch
    import avifgpu
    dev = torch.device("cuda", gpu.device)
    if torch.cuda.get_device_properties(dev).total_memory < 40 * 2**30:
        pytest.skip("needs ~20 GB of device memory")
    w = 4096
    samples_per_row = w * 3
    h = ((1 << 31) // samples_per_row + 2) & ~1
    desc = abi.EncodeDesc(w, h, 32, 3, abi.ALPHA_NONE, 12, abi.TRANSFER_PQ, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_444,
                          abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, abi.Nclx(1, abi.PRIMARIES_BT2020, abi.TRANSFER_CHAR_PQ, 0, 1))
    rows = torch.empty((h, samples_per_row), dtype=torch.float32, device=dev)
    flat_bits = rows.view(torch.int32).view(-1)
    chunk = 1 << 27
    for start in range(0, flat_bits.numel(), chunk):
        n = min(chunk, flat_bits.numel() - start)
        flat_bits[start:start + n] = torch.arange(start, start + n, dtype=torch.int64, device=dev).to(torch.int32)  # wraps past 2^31
    shapes = abi.encode_plane_shapes(desc)
    fast = [None if s is None else torch.full(s, -1, dtype=torch.int16, device=dev) for s in shapes]
    gpu.encode_device(desc, rows.data_ptr(), rows.stride(0) * 4, avifgpu.planes_from_tensors(fast))
    backing = [None if s is None else torch.full((s[0], s[1] + 1), -1, dtype=torch.int16, device=dev) for s in shapes]
    exact = [None if t is None else t[:, 1:] for t in backing]  # 2-byte aligned origins: the launcher takes the generic kernel
    before = gpu_exact.launch_count()
    gpu_exact.encode_device(desc, rows.data_ptr(), rows.stride(0) * 4, avifgpu.planes_from_tensors(exact))  # and no tables at all
    torch.cuda.synchronize(dev)
    assert gpu_exact.launch_count() - before == 1
    for k in range(3):
        differing = int((fast[k] != exact[k]).sum().item())
        assert differing == 0, f"plane {k}: {differing} of {fast[k].numel()} codes differ"
    # and the planes are what the identity matrix promises: Y = G, Cb = B, Cr = R of monotone inputs
    codes = exact[2].reshape(-1)[: (0x7f800000 // 3)].to(torch.int32) & 0xffff  # Cr = R samples, bits 0, 3, 6, ... below +inf
    assert int(codes.max().item()) == 4095 and int(codes.min().item()) == 0
    assert bool((codes[1:] >= codes[:-1] - 1).all().item())  # non-decreasing up to the one-code flips inside fuzzy bands


def test_every_10bit_triple_through_the_production_decode_kernel(gpu):
    """Config 3's whole input domain: all 2^30 (Y, Cb, Cr) triples of 10-bit codes as one 32768 x 32768 4:4:4 image
    (what 4:2:0 feeds the per-pixel arithmetic is a subset of these), HLG + OOTF, through the tuned decode kernel and
    through the generic exact kernel (reached with a row pointer that is only 4-byte aligned); the float outputs must
    be bit-identical.  test_gpu_parity.py / test_gpu_fullsize.py pin the generic kernel to the reference's CPU loop."""
    import torch
    import avifgpu
    dev = torch.device("cuda", gpu.device)
    if torch.cuda.get_device_properties(dev).total_memory < 60 * 2**30:
        pytest.skip("needs ~45 GB of device memory")
    w = h = 1 << 15
    desc = abi.DecodeDesc(w, h, abi.COLORSPACE_YCBCR, abi.CHROMA_444, 10, abi.ALPHA_NONE, 32, cases.NCLX_2020_HLG(1), 1, 1.2, 1000, 80)
    index = torch.arange(w * h, dtype=torch.int32, device=dev).view(h, w)
    planes = [(index & 1023).to(torch.int16), ((index >> 10) & 1023).to(torch.int16), (index >> 20).to(torch.int16)]
    del index
    struct = avifgpu.planes_from_tensors(planes + [None])
    fast = torch.empty((h, w * 3), dtype=torch.float32, device=dev)
    before = gpu.launch_count()
    gpu.decode_device(desc, struct, fast.data_ptr(), fast.stride(0) * 4)
    fast_launches = gpu.launch_count() - before
    backing = torch.empty((h, w * 3 + 4), dtype=torch.float32, device=dev)
    exact = backing[:, 1:w * 3 + 1]  # 4-byte aligned rows: the launcher takes the generic kernel
    gpu.decode_device(desc, struct, exact.data_ptr(), exact.stride(0) * 4)
    torch.cuda.synchronize(dev)
    assert fast_launches >= 1
    differing = 0
    for y in range(0, h, 4096):  # compare in slabs to bound the temporaries
        differing += int((fast[y:y + 4096].view(torch.int32) != exact[y:y + 4096].view(torch.int32)).sum().item())
    assert differing == 0, f"{differing} of {fast.numel()} output samples differ"
    assert bool(torch.isfinite(fast[:4096]).all().item())


def test_every_10bit_triple_through_the_production_pq_decode_kernel(gpu):
    """The same whole-domain sweep for the PQ sibling of config 3: all 2^30 (Y, Cb, Cr) triples of 10-bit codes, PQ at 1000 nit,
    through the tuned kernel -- two branch-free powf per channel on the exponent-folded log2 table, the quotient between them by
    the verified reciprocal-seed division -- and through the generic exact kernel (full powf, IEEE division)."""
    import torch
    import avifgpu
    dev = torch.device("cuda", gpu.device)
    if torch.cuda.get_device_properties(dev).total_memory < 60 * 2**30:
        pytest.skip("needs ~45 GB of device memory")
    w = h = 1 << 15
    desc = abi.DecodeDesc(w, h, abi.COLORSPACE_YCBCR, abi.CHROMA_444, 10, abi.ALPHA_NONE, 32, cases.NCLX_2020_PQ(1), pq_peak_nits=1000)
    index = torch.arange(w * h, dtype=torch.int32, device=dev).view(h, w)
    planes = [(index & 1023).to(torch.int16), ((index >> 10) & 1023).to(torch.int16), (index >> 20).to(torch.int16)]
    del index
    struct = avifgpu.planes_from_tensors(planes + [None])
    fast = torch.empty((h, w * 3), dtype=torch.float32, device=dev)
    before = gpu.launch_count()
    gpu.decode_device(desc, struct, fast.data_ptr(), fast.stride(0) * 4)
    fast_launches = gpu.launch_count() - before
    backing = torch.empty((h, w * 3 + 4), dtype=torch.float32, device=dev)
    exact = backing[:, 1:w * 3 + 1]  # 4-byte aligned rows: the launcher takes the generic kernel
    gpu.decode_device(desc, struct, exact.data_ptr(), exact.stride(0) * 4)
    torch.cuda.synchronize(dev)
    assert fast_launches >= 1
    differing = 0
    for y in range(0, h, 4096):  # compare in slabs to bound the temporaries
        differing += int((fast[y:y + 4096].view(torch.int32) != exact[y:y + 4096].view(torch.int32)).sum().item())
    assert differing == 0, f"{differing} of {fast.numel()} output samples differ"
    assert bool(torch.isfinite(fast[:4096]).all().item())


# ---- integer hosts, decode (kernels_fast_decode_int.cu) -----------------------------------------------------------------

@pytest.mark.parametrize("w,h", [(8, 2), (9, 3), (24, 1), (67, 5), (256, 16), (263, 9), (1031, 6)])
@pytest.mark.parametrize("chroma", [abi.CHROMA_420, abi.CHROMA_422, abi.CHROMA_444])
@pytest.mark.parametrize("alpha", [abi.ALPHA_NONE, abi.ALPHA_STRAIGHT, abi.ALPHA_PREMULTIPLIED])
def test_ycc_to_rgb_integer_fast_kernel(gpu, checker, w, h, chroma, alpha):
    for bit_depth, host_depth, nclx in ((8, 8, cases.NCLX_601(1)), (8, 8, cases.NCLX_709(0)), (10, 16, cases.NCLX_601(1)),
                                        (12, 16, cases.NCLX_2020_PQ(0))):
        desc = abi.DecodeDesc(w, h, abi.COLORSPACE_YCBCR, chroma, bit_depth, alpha, host_depth, nclx)
        planes = cases.code_planes(cases.rng_for(f"decint_{w}x{h}_{chroma}_{alpha}_{bit_depth}"), desc, overshoot=True)
        expected = checker.decode(desc, planes, threads=4)
        got = gpu.decode(desc, planes)
        assert np.array_equal(expected, got), (bit_depth, host_depth, int((expected != got).sum()))
        if h > 3:  # a block that starts on an odd row (generic kernel) next to blocks that do not
            out = np.zeros_like(expected)
            gpu.decode(desc, planes, y0=0, nrows=1, out=out[0:1])
            gpu.decode(desc, planes, y0=1, nrows=h - 1, out=out[1:])
            assert np.array_equal(expected, out)


def test_every_8bit_triple_through_the_integer_decode_kernel(gpu):
    """All 2^24 (Y, Cb, Cr) triples of 8-bit codes (4096 x 4096, 4:4:4, BT.601 full and limited range) through the tuned
    kernel and through the generic kernel (reached with an unaligned row pointer): identical bytes."""
    import torch
    import avifgpu
    dev = torch.device("cuda", gpu.device)
    w = h = 4096
    index = torch.arange(w * h, dtype=torch.int32, device=dev).view(h, w)
    planes = [(index & 255).to(torch.uint8), ((index >> 8) & 255).to(torch.uint8), (index >> 16).to(torch.uint8)]
    struct = avifgpu.planes_from_tensors(planes + [None])
    for full_range in (1, 0):
        desc = abi.DecodeDesc(w, h, abi.COLORSPACE_YCBCR, abi.CHROMA_444, 8, abi.ALPHA_NONE, 8, cases.NCLX_601(full_range))
        fast = torch.zeros((h, w * 3), dtype=torch.uint8, device=dev)
        gpu.decode_device(desc, struct, fast.data_ptr(), fast.stride(0))
        backing = torch.zeros((h, w * 3 + 8), dtype=torch.uint8, device=dev)
        exact = backing[:, 1:w * 3 + 1]
        gpu.decode_device(desc, struct, exact.data_ptr(), exact.stride(0))
        torch.cuda.synchronize(dev)
        assert int((fast != exact).sum().item()) == 0


# ---- when the step tables get built ---------------------------------------------------------------------------------------

def test_step_tables_are_built_when_they_pay_off(port):
    """A fresh context converts with the exact kernel (one launch, no 40 ms table build) until one configuration has
    seen more pixels than the auto-build threshold, or until avifgpu_prepare_encode(); the planes never change."""
    import avifgpu
    w, h = 256, 64
    desc = planar_desc(w, h)
    rows = cases.float_host_rows(np.random.default_rng(99), h, w, 3)
    expected = port.encode(desc, rows)
    with avifgpu.Context(0) as ctx:
        assert cases.same_planes(expected, ctx.encode(desc, rows))
        per_call = ctx.launch_count()
        assert per_call == 1, "a single small image must not pay for table construction"
        ctx.set_table_autobuild(3 * w * h)  # pixels of this configuration before the tables are worth building
        assert cases.same_planes(expected, ctx.encode(desc, rows))
        assert cases.same_planes(expected, ctx.encode(desc, rows))
        assert ctx.launch_count() == 3 * per_call
        assert cases.same_planes(expected, ctx.encode(desc, rows))  # 4 * w * h > threshold: sweep + bitmap + verify + kernel
        assert ctx.launch_count() == 4 * per_call + 3
        assert cases.same_planes(expected, ctx.encode(desc, rows))
        assert ctx.launch_count() == 5 * per_call + 3
    with avifgpu.Context(0) as ctx:
        ctx.set_table_autobuild(-1)
        for _ in range(3):
            assert cases.same_planes(expected, ctx.encode(desc, rows))
        assert ctx.launch_count() == 3
        assert ctx.prepare_encode(desc).as_dict()["valid"] == 1  # explicit request still builds
        assert cases.same_planes(expected, ctx.encode(desc, rows))


def test_two_devices_in_one_process(port):
    """The C ABI lets one process drive several GPUs (avifgpu_create(device)); per-device kernel attributes and tables
    must follow.  Needs two visible GPUs."""
    import torch
    import avifgpu
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    w, h = 512, 32
    desc = planar_desc(w, h)
    rows = cases.float_host_rows(np.random.default_rng(5), h, w, 3)
    expected = port.encode(desc, rows)
    ddesc = abi.DecodeDesc(w, h, abi.COLORSPACE_YCBCR, abi.CHROMA_420, 10, abi.ALPHA_NONE, 32, cases.NCLX_2020_HLG())
    planes = cases.code_planes(np.random.default_rng(6), ddesc)
    decoded = port.decode(ddesc, planes)
    for device in (1, 0, 1):
        with avifgpu.Context(device) as ctx:
            ctx.set_table_autobuild(0)
            assert cases.same_planes(expected, ctx.encode(desc, rows))
            assert cases.same_bits(decoded, ctx.decode(ddesc, planes))


def test_every_10bit_triple_through_the_integer_decode_kernel(gpu):
    """All 2^30 (Y, Cb, Cr) triples of 10-bit codes (32768 x 32768, 4:4:4, BT.2020 full range) -> RGB16 through the tuned
    kernel and through the generic kernel (unaligned row pointer): identical samples.  Covers the fused-quantiser proof
    (tools/check_fused_quantiser.py) on the device for the 32768 scale; the 8-bit sibling above covers 255."""
    import torch
    import avifgpu
    dev = torch.device("cuda", gpu.device)
    if torch.cuda.get_device_properties(dev).total_memory < 60 * 2**30:
        pytest.skip("needs ~25 GB of device memory")
    w = h = 1 << 15
    desc = abi.DecodeDesc(w, h, abi.COLORSPACE_YCBCR, abi.CHROMA_444, 10, abi.ALPHA_NONE, 16, cases.NCLX_2020_PQ(1))
    index = torch.arange(w * h, dtype=torch.int32, device=dev).view(h, w)
    planes = [(index & 1023).to(torch.int16), ((index >> 10) & 1023).to(torch.int16), (index >> 20).to(torch.int16)]
    del index
    struct = avifgpu.planes_from_tensors(planes + [None])
    fast = torch.empty((h, w * 3), dtype=torch.int16, device=dev)
    gpu.decode_device(desc, struct, fast.data_ptr(), fast.stride(0) * 2)
    backing = torch.empty((h, w * 3 + 8), dtype=torch.int16, device=dev)
    exact = backing[:, 1:w * 3 + 1]
    gpu.decode_device(desc, struct, exact.data_ptr(), exact.stride(0) * 2)
    torch.cuda.synchronize(dev)
    differing = 0
    for y in range(0, h, 4096):
        differing += int((fast[y:y + 4096] != exact[y:y + 4096]).sum().item())
    assert differing == 0
