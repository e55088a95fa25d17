"""The content light level measured inside the device encode (avifgpu_encode_rows_device_light_level; DESIGN.md section 5).

Every case encodes the same rows twice, with the plain device call and with the light-level call, and checks:
  * the planes, row padding included, are bit-identical, and the launch counts are equal -- the light-level call takes
    the plain call's route (tuned kernel + generic strips, or the generic kernel alone);
  * the accumulator equals one computed on the CPU from the checker's own R'G'B' codes: the reference-layout encode of
    the same rows, by the restatement, gives them interleaved (light_level_spec.py).
CASES has one case per route: the flat kernel on the compact tables (12-bit PQ: compact-14, 10-bit PQ: compact) in every
chroma mode and destination layout and the reference interleaved layout; RGBA straight and premultiplied; Gray and
Gray+A; and the generic kernel (no table, row matrix, misaligned rows, right strips, odd 4:2:0 rows).  Inputs
are random, with NaN / +-inf / negatives / over-peak values, saturated, and one code everywhere; shapes where each tuned
grid walks the image at least twice; row blocks that add up; a captured call replayed on new rows after an in-graph
memset of the accumulator; and the refusals, which launch nothing."""
import ctypes as C

import numpy as np
import pytest

import cases
import light_level_spec as spec
from avifgpu import abi
from gpu_harness import SENTINEL, EncodeImage, launches_of, sm_count, whole

pytestmark = pytest.mark.gpu

C444, C422, C420 = abi.CHROMA_444, abi.CHROMA_422, abi.CHROMA_420
NONE, STRAIGHT, PREMUL = abi.ALPHA_NONE, abi.ALPHA_STRAIGHT, abi.ALPHA_PREMULTIPLIED
NV, MSB = abi.SOURCE_CHROMA_INTERLEAVED, abi.SOURCE_MSB_ALIGNED
LAYOUTS = {"planar": 0, "nv": NV, "msb": MSB, "nvmsb": NV | MSB}
CHROMAS = {"444": C444, "422": C422, "420": C420}
# threads of one CTA and CTAs per SM of each tuned kernel's persistent grid (kernel_params.h, kernels_fast_*.cu)
FLAT_WARPS, RGBA_WARPS, GRAY_THREADS = 28, 16, 1024


def desc_of(channels, alpha, depth, layout=abi.LAYOUT_PLANAR_YCBCR, chroma=C420, dest=0, transfer=abi.TRANSFER_PQ, peak=1000,
            row_matrix=None, down=abi.DOWN_FILTER_BOX):
    d = abi.EncodeDesc(0, 0, 32, channels, alpha, depth, transfer, peak, layout, chroma if layout == abi.LAYOUT_PLANAR_YCBCR else C444,
                       down, abi.GRAY16_LUT, cases.NCLX_2020_PQ(), dest_layout=dest)
    if row_matrix is not None:
        d.row_matrix_enabled = 1
        for i, v in enumerate(row_matrix):
            d.row_matrix[i] = v
    return d


# (name, desc, route): route "tuned" = the tuned kernel (prepared context), "generic" = the generic kernel alone
CASES = []
for depth in (12, 10):
    for cname, chroma in CHROMAS.items():
        for lname, dest in LAYOUTS.items():
            CASES.append((f"flat_d{depth}_{cname}_{lname}", desc_of(3, NONE, depth, chroma=chroma, dest=dest,
                                                                     down=abi.DOWN_FILTER_TOP_LEFT if lname == "nv" else abi.DOWN_FILTER_BOX), "tuned"))
    CASES.append((f"flat_d{depth}_interleaved", desc_of(3, NONE, depth, layout=abi.LAYOUT_REFERENCE), "tuned"))
for alpha, aname in ((STRAIGHT, "straight"), (PREMUL, "premul")):
    for cname, chroma in CHROMAS.items():
        CASES.append((f"rgba_{aname}_{cname}", desc_of(4, alpha, 12, chroma=chroma, dest=NV | MSB if chroma == C420 else 0), "tuned"))
CASES += [("gray", desc_of(1, NONE, 12, layout=abi.LAYOUT_REFERENCE), "tuned"),
          ("gray_alpha", desc_of(2, STRAIGHT, 12, layout=abi.LAYOUT_REFERENCE), "tuned"),
          ("gray_alpha_premul", desc_of(2, PREMUL, 10, layout=abi.LAYOUT_REFERENCE), "tuned"),
          ("generic_no_table_planar", desc_of(3, NONE, 12), "generic"),
          ("generic_no_table_rgba", desc_of(4, PREMUL, 10, chroma=C422), "generic"),
          ("generic_no_table_interleaved", desc_of(4, STRAIGHT, 12, layout=abi.LAYOUT_REFERENCE), "generic"),
          ("generic_no_table_gray", desc_of(1, NONE, 10, layout=abi.LAYOUT_REFERENCE), "generic"),
          ("generic_row_matrix", desc_of(3, NONE, 12, row_matrix=[0.6274, 0.3293, 0.0433, 0.0691, 0.9195, 0.0114, 0.0164, 0.0880, 0.8956]), "tuned"),
          ("generic_row_matrix_rgba", desc_of(4, STRAIGHT, 10, chroma=C444, row_matrix=[1.2, -0.1, -0.1, -0.05, 1.1, -0.05, 0.0, -0.2, 1.2]), "tuned")]


def test_case_table_covers_every_light_instantiation():
    flat = {(d.image_bit_depth, d.chroma, d.dest_layout) for n, d, _ in CASES if n.startswith("flat_") and d.layout == abi.LAYOUT_PLANAR_YCBCR}
    assert flat == {(b, c, l) for b in (10, 12) for c in CHROMAS.values() for l in LAYOUTS.values()}
    assert {(d.host_channels, d.alpha_state) for n, d, _ in CASES if n.startswith("gray")} == {(1, NONE), (2, STRAIGHT), (2, PREMUL)}
    assert len({n for n, _, _ in CASES}) == len(CASES)


@pytest.fixture(scope="module")
def contexts():
    import avifgpu
    tuned, generic = avifgpu.Context(0), avifgpu.Context(0)
    generic.set_table_autobuild(-1)
    yield {"tuned": tuned, "generic": generic}
    tuned.close()
    generic.close()


def reference_desc(desc):
    d = abi.EncodeDesc.from_buffer_copy(desc)
    d.layout, d.dest_layout, d.chroma = abi.LAYOUT_REFERENCE, 0, C444
    return d


def expected_acc(port, desc, host):
    """The accumulator of `host`'s rows from the restatement's reference-layout codes."""
    ref = reference_desc(desc)
    ref.width, ref.height = host.shape[1] // desc.host_channels, host.shape[0]
    codes = port.encode(ref, host, threads=8)[0]
    return spec.accumulate(codes, desc.host_channels if desc.host_channels >= 3 else 1, spec.levels(port, desc.image_bit_depth))


def acc_tensor():
    import torch
    return torch.zeros(3, dtype=torch.int64, device="cuda")


def acc_of(tensor):
    import torch
    torch.cuda.synchronize()
    raw = tensor.cpu().numpy().view(np.uint32)
    return {"max_code": int(raw[0]), "reserved": int(raw[1]), "level_sum": int(tensor[1].item()), "pixels": int(tensor[2].item())}


def light_call(ctx, im, acc, y0=0, nrows=None, stream=0):
    import avifgpu
    return lambda: ctx.encode_device_light_level(im.desc, im.rows.data_ptr() + y0 * im.rows.stride(0), im.rows.stride(0),
                                                 avifgpu.planes_from_tensors(im.planes), acc.data_ptr(), y0, nrows, stream)


def make_image(desc, w, h, seed, host=None, rows_misalign=0):
    im = EncodeImage(desc, w, h, seed, prefix="light_", rows_misalign=rows_misalign)
    if host is not None:
        import torch
        im.host = np.ascontiguousarray(host.reshape(h, w * desc.host_channels).astype(np.float32))
        im.rows.copy_(torch.from_numpy(im.host.view(np.uint8).reshape(h, im.row_bytes)).cuda())
    return im


def check(ctx, port, desc, w, h, seed, host=None, rows_misalign=0, prepare=True):
    """Plain call vs light-level call of one image: planes, launches, accumulator."""
    if prepare:
        ctx.prepare_encode(desc)
    im = make_image(desc, w, h, seed, host, rows_misalign)
    plain = im.fresh_planes()
    plain_launches = launches_of(ctx, lambda: im.direct(ctx, plain))
    acc = acc_tensor()
    light_launches = launches_of(ctx, light_call(ctx, im, acc))
    assert light_launches == plain_launches, (light_launches, plain_launches)
    for k, (got, want) in enumerate(zip(im.planes, plain)):
        if got is not None:
            assert np.array_equal(whole(got), whole(want)), ("planes differ from the plain call", w, h, k)
    got = acc_of(acc)
    want = expected_acc(port, im.desc, im.host)
    assert got == want, (got, want)
    return plain_launches, got


def shapes_for(name):
    if name.startswith("generic"):
        return [(37, 9), (64, 5)]
    return [(509, 66), (130, 7), (8, 2)]  # right strips and odd 4:2:0 rows around the tuned interior


@pytest.mark.parametrize("name, desc, route", CASES, ids=[c[0] for c in CASES])
def test_route(contexts, port, name, desc, route):
    ctx = contexts[route]
    rng = cases.rng_for(f"light_{name}")
    for i, (w, h) in enumerate(shapes_for(name)):
        d = abi.EncodeDesc.from_buffer_copy(desc)
        d.width, d.height = w, h
        host = cases.float_host_rows(rng, h, w, d.host_channels, specials=(i == 0))
        launches, acc = check(ctx, port, d, w, h, f"{name}_{i}", host, prepare=route == "tuned")
        assert acc["pixels"] == w * h
        if route == "generic":
            assert launches == 1


def degenerate_rows(rng, h, w, channels, kind):
    n = h * w * channels
    if kind == "specials":
        pool = np.array([np.nan, np.inf, -np.inf, -1.0, -0.0, 0.0, 1.0, 1e30, 7.5, 1e-38, 3.4e38], np.float32)
        v = rng.choice(pool, n)
    elif kind == "saturated":
        v = np.where(rng.random(n) < 0.5, np.float32(100.0), np.float32(1.0)).astype(np.float32)
    else:  # one code everywhere
        v = np.full(n, np.float32(0.25))
    v = v.astype(np.float32).reshape(h, w, channels)
    if channels in (2, 4):  # opaque for one code everywhere; else some half-transparent pixels
        v[..., -1] = np.where((rng.random((h, w)) < 0.3) & (kind != "uniform"), np.float32(0.5), np.float32(1.0))
    return v


@pytest.mark.parametrize("kind", ["specials", "saturated", "uniform"])
@pytest.mark.parametrize("name", ["flat_d12_420_planar", "rgba_premul_444", "gray_alpha", "generic_no_table_planar"])
def test_degenerate_inputs(contexts, port, name, kind):
    _, desc, route = next(c for c in CASES if c[0] == name)
    w, h = 261, 10
    d = abi.EncodeDesc.from_buffer_copy(desc)
    d.width, d.height = w, h
    host = degenerate_rows(cases.rng_for(f"light_{name}_{kind}"), h, w, d.host_channels, kind)
    _, acc = check(contexts[route], port, d, w, h, f"{name}_{kind}", host, prepare=route == "tuned")
    if kind == "uniform":
        level = int(spec.levels(port, d.image_bit_depth)[acc["max_code"]])
        assert acc["level_sum"] == level * w * h


def test_misaligned_rows_take_the_generic_kernel(contexts, port):
    d = desc_of(3, NONE, 12, chroma=C420)
    d.width, d.height = 96, 6
    launches, _ = check(contexts["tuned"], port, d, 96, 6, "misaligned", rows_misalign=4)
    assert launches == 1


@pytest.mark.parametrize("name", ["flat_d12_420_planar", "flat_d10_444_nvmsb", "flat_d12_interleaved", "rgba_straight_420", "gray_alpha"])
def test_grids_walk_the_image_at_least_twice(contexts, port, name):
    ctx = contexts["tuned"]
    sms = sm_count(ctx)
    _, desc, _ = next(c for c in CASES if c[0] == name)
    if name.startswith("gray"):
        w = 1024
        h = -(-2 * GRAY_THREADS * sms * 4 // w)  # groups of 4 pixels: at least two per thread of the grid
    else:
        warps = FLAT_WARPS if name.startswith("flat") else RGBA_WARPS
        w = 1024
        h = 2 * -(-2 * warps * sms // (w // 128))  # 2 x 128-pixel tiles: at least two per warp of the grid
    d = abi.EncodeDesc.from_buffer_copy(desc)
    d.width, d.height = w + 3, h + 1  # a right strip and an odd last row too
    host = cases.float_host_rows(cases.rng_for(f"light_walk_{name}"), d.height, d.width, d.host_channels)
    check(ctx, port, d, d.width, d.height, f"walk_{name}", host)


@pytest.mark.parametrize("name", ["flat_d12_420_nv", "rgba_premul_422", "gray", "generic_no_table_planar"])
def test_row_blocks_add_up(contexts, port, name):
    _, desc, route = next(c for c in CASES if c[0] == name)
    ctx = contexts[route]
    w, h = 300, 38
    d = abi.EncodeDesc.from_buffer_copy(desc)
    d.width, d.height = w, h
    if route == "tuned":
        ctx.prepare_encode(d)
    im = make_image(d, w, h, f"blocks_{name}")
    whole_acc, halves = acc_tensor(), acc_tensor()
    launches_of(ctx, light_call(ctx, im, whole_acc))
    first = [whole(p) for p in im.planes if p is not None]
    for p in im.planes:
        if p is not None:
            p.fill_(SENTINEL)
    for y0, n in ((0, 12), (12, 20), (32, 6)):
        launches_of(ctx, light_call(ctx, im, halves, y0, n))
    assert all(np.array_equal(a, whole(b)) for a, b in zip(first, [p for p in im.planes if p is not None])), "row blocks wrote other planes"
    assert acc_of(halves) == acc_of(whole_acc) == expected_acc(port, im.desc, im.host)


@pytest.mark.parametrize("prepared", [True, False], ids=["tuned", "before_tables"])
def test_captured_call_replays_on_new_rows(port, prepared):
    import avifgpu
    import torch
    ctx = avifgpu.Context(0)
    try:
        if not prepared:
            ctx.set_table_autobuild(-1)
        w, h = 517, 22
        d = desc_of(3, NONE, 12, chroma=C420, dest=NV | MSB)
        d.width, d.height = w, h
        if prepared:
            ctx.prepare_encode(d)
        im = make_image(d, w, h, "capture_0")
        acc = acc_tensor()
        stream = torch.cuda.Stream()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        before = ctx.launch_count()
        with torch.cuda.graph(graph, stream=stream):
            acc.zero_()  # an in-graph memset of the accumulator
            light_call(ctx, im, acc, stream=torch.cuda.current_stream().cuda_stream)()
        captured = ctx.launch_count() - before
        assert captured == (2 if prepared else 1)  # flat kernel + the odd 4:2:0 right strip, or the generic kernel
        for i in range(3):
            host = cases.float_host_rows(cases.rng_for(f"light_capture_{i}"), h, w, 3, specials=i == 1)
            im.rows.copy_(torch.from_numpy(host.reshape(h, -1).view(np.uint8)).cuda())
            im.host = host.reshape(h, -1)
            acc.fill_(12345)  # the memset inside the graph clears it
            graph.replay()
            assert acc_of(acc) == expected_acc(port, im.desc, im.host), i
            plain = im.fresh_planes()
            im.direct(ctx, plain)
            torch.cuda.synchronize()
            for got, want in zip(im.planes, plain):
                if got is not None:
                    assert np.array_equal(whole(got), whole(want)), i
        del graph
    finally:
        ctx.close()


@pytest.mark.parametrize("host_depth, transfer", [(8, abi.TRANSFER_CLIP), (16, abi.TRANSFER_CLIP), (32, abi.TRANSFER_SMPTE428),
                                                  (32, abi.TRANSFER_CLIP), (32, abi.TRANSFER_HLG)])
def test_refusals_launch_nothing(contexts, host_depth, transfer):
    import avifgpu
    ctx = contexts["tuned"]
    d = desc_of(3, NONE, 10, chroma=C420, transfer=transfer)
    d.host_depth = host_depth
    if transfer == abi.TRANSFER_HLG:
        d.hlg_extension = abi.HLG_OETF
        d.nclx = cases.NCLX_2020_HLG()
    d.width, d.height = 64, 4
    im = make_image(d, 64, 4, f"refuse_{host_depth}_{transfer}")
    acc = acc_tensor()
    with pytest.raises(avifgpu.AvifGpuError) as failure:
        launches_of(ctx, light_call(ctx, im, acc))
    assert failure.value.status == abi.ERR_UNSUPPORTED
    assert acc_of(acc) == {"max_code": 0, "reserved": 0, "level_sum": 0, "pixels": 0}
    assert im.untouched()


def test_null_accumulator_is_a_bad_parameter(contexts):
    import avifgpu
    ctx = contexts["tuned"]
    d = desc_of(3, NONE, 12)
    d.width, d.height = 64, 4
    im = make_image(d, 64, 4, "null_acc")
    before = ctx.launch_count()
    status = ctx.lib.avifgpu_encode_rows_device_light_level(ctx.handle, C.byref(im.desc), im.rows.data_ptr(), im.rows.stride(0), 0, 4,
                                                            C.byref(avifgpu.planes_from_tensors(im.planes)), None, None)
    assert status == abi.ERR_BAD_PARAM and ctx.launch_count() == before


def test_content_light_level_of_a_measured_frame(contexts, port):
    import avifgpu
    d = desc_of(3, NONE, 12)
    d.width, d.height = 256, 16
    _, acc = check(contexts["tuned"], port, d, 256, 16, "clli")
    assert avifgpu.content_light_level(acc, 12) == spec.content_light_level(acc, spec.levels(port, 12))
