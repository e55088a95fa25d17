"""The batched kernels (kernels_batch.cu) under their chunk record source held to the CPU checker: every instantiation,
and every grid-stride loop over several passes (test_gpu_batch_indirect.py does the same under the workspace source).

A chunk of avifgpu_{encode,decode}_batch_device launches the instantiation its description selects (host depth, plane
depth, channels / premultiply, chroma) and walks the chunk's concatenated units with a capped, persistent grid, finding
each unit's image as it goes.  test_gpu_batch.py checks the entry points' contract on a few configurations; here:

  * ENCODE_KERNELS and DECODE_KERNELS (gpu_harness.py) hold one case per instantiation of EncodeRgbIntBatchKernel (36) and
    DecodeYccToRgbIntBatchKernel (12); test_instantiation_tables_are_complete checks their keys without a GPU.  Each
    case's launch count proves that its eligible images reached the batched kernels;
  * the multi-pass cases make the loops of all four batched kernels run at least twice (asserted from the SM count and
    the launchers' grid caps, gpu_harness.BATCH_CAPS), and the edge kernels walk bottom strips of several units per row;
  * a batch led by an empty image, on a fresh context, still does its first-use checks.

Every image is compared bit for bit with the CPU checker -- the restatement for encode (the reference has no planar
YCbCr encoder), the compiled reference for decode -- and with a direct *_rows_device call, and the sentinel in the row
padding must survive.  16-bit hosts carry samples above 32768, 10 / 12-bit planes codes above the maximum."""
import collections
import itertools
import os

import pytest

import cases
from avifgpu import abi
from gpu_harness import ctx  # noqa: F401
from gpu_harness import (BOX, C420, C422, C444, CHUNK, DECODE_KERNELS, ENCODE_KERNELS, MIXED, N601, N709, N2020, NONE, PREMUL, STRAIGHT, TOP_LEFT,
                         DecodeImage, EncodeImage, Empty, assert_batched, assert_decode_same_as_direct, assert_passes,
                         assert_same_as_direct, bottom_units, edge_units, expected_launches, interior_units, launches_of, pick, planar,
                         run_batch, run_decode_batch, sm_count, ycc, ys_of)

# ---- the instantiation tables ------------------------------------------------------------------------------------------

CHANNELS = {(3, NONE): "c3", (4, STRAIGHT): "c4s", (4, PREMUL): "c4p"}


def encode_key(desc):
    """The template arguments WithRgbIntKey (launch_keys.h) picks for `desc`: host depth, plane bytes, channels /
    premultiply, chroma."""
    return desc.host_depth, 2 if desc.image_bit_depth > 8 else 1, CHANNELS[(desc.host_channels, desc.alpha_state)], desc.chroma


def decode_key(desc):
    """The template arguments WithYccIntKey (launch_keys.h) picks for `desc`: sample type, alpha, chroma."""
    assert desc.alpha_state != PREMUL and (desc.host_depth == 8) == (desc.bit_depth == 8)
    return desc.host_depth, desc.alpha_state == STRAIGHT, desc.chroma


def matrix_name(nclx):
    return "none" if not nclx.present else {abi.MATRIX_BT601: "601", abi.MATRIX_BT709: "709", abi.MATRIX_BT2020_NCL: "2020",
                                             abi.MATRIX_GBR: "gbr"}[nclx.matrix_coefficients]


def test_instantiation_tables_are_complete():
    """Each table has exactly one case per instantiation, and spreads every runtime parameter over at least two cases."""
    encode = [encode_key(d) for _, d in ENCODE_KERNELS]
    assert sorted(encode) == sorted(itertools.product((8, 16), (1, 2), ("c3", "c4s", "c4p"), (C444, C422, C420)))
    decode = [decode_key(d) for _, d in DECODE_KERNELS]
    assert sorted(decode) == sorted(itertools.product((8, 16), (False, True), (C444, C422, C420)))
    assert len({name for name, _ in ENCODE_KERNELS + DECODE_KERNELS}) == len(ENCODE_KERNELS) + len(DECODE_KERNELS)

    def at_least_twice(values, expected):
        counts = collections.Counter(values)
        assert set(counts) == set(expected) and min(counts.values()) >= 2, counts

    at_least_twice([matrix_name(d.nclx) for _, d in ENCODE_KERNELS], ("none", "601", "709", "2020", "gbr"))
    at_least_twice([matrix_name(d.nclx) for _, d in DECODE_KERNELS], ("none", "601", "709", "2020", "gbr"))
    assert all(d.chroma == C444 for _, d in ENCODE_KERNELS + DECODE_KERNELS if matrix_name(d.nclx) == "gbr")
    at_least_twice([d.down_filter for _, d in ENCODE_KERNELS if d.chroma != C444], (BOX, TOP_LEFT))
    at_least_twice([d.image_bit_depth for _, d in ENCODE_KERNELS if d.image_bit_depth > 8], (10, 12))
    at_least_twice([d.bit_depth for _, d in DECODE_KERNELS if d.bit_depth > 8], (10, 12))
    at_least_twice([(d.host_depth, bool(d.nclx.full_range_flag) or not d.nclx.present) for _, d in DECODE_KERNELS],
                   ((8, True), (8, False), (16, True), (16, False)))
    assert {d.chroma for _, d in DECODE_KERNELS if d.bit_depth == 12 and d.alpha_state == STRAIGHT} == {C444, C422, C420}


# ---- launches: proof that the eligible images reached the batched kernels (gpu_harness.assert_batched) -----------------

@pytest.mark.gpu
@pytest.mark.parametrize("name,desc", ENCODE_KERNELS, ids=[c[0] for c in ENCODE_KERNELS])
def test_encode_instantiation(ctx, port, name, desc):
    images = [EncodeImage(desc, w, h, f"kernels_{name}_{i}", beyond=True) for i, (w, h) in enumerate(MIXED)]
    assert_batched(ctx, lambda: run_batch(ctx, desc, images), images, ys_of(desc))
    assert_same_as_direct(ctx, images, port)


@pytest.mark.gpu
@pytest.mark.parametrize("name,desc", DECODE_KERNELS, ids=[c[0] for c in DECODE_KERNELS])
def test_decode_instantiation(ctx, checker, port, name, desc):
    images = [DecodeImage(desc, w, h, f"kernels_{name}_{i}", overshoot=True) for i, (w, h) in enumerate(MIXED)]
    assert_batched(ctx, lambda: run_decode_batch(ctx, desc, images), images, ys_of(desc))
    assert_decode_same_as_direct(ctx, images, pick(checker, port, True))


# ---- several passes of every loop -----------------------------------------------------------------------------------------

def run_multipass_encode(ctx, port, desc, n, w, h, seed):
    sms = sm_count(ctx)
    ys = ys_of(desc)
    assert_passes("encode_interior", n * interior_units(w, h, ys), sms)
    assert_passes("encode_edge", n * edge_units(w, h, desc.chroma, False), sms)
    images = [EncodeImage(desc, w, h, f"{seed}_{i}", beyond=True) for i in range(n)]
    assert_batched(ctx, lambda: run_batch(ctx, desc, images), images, ys)
    assert_same_as_direct(ctx, images, port, threads=os.cpu_count())


def run_multipass_decode(ctx, checker, desc, n, w, h, seed):
    sms = sm_count(ctx)
    ys = ys_of(desc)
    assert_passes("ycc_int_interior", n * interior_units(w, h, ys), sms)
    assert_passes("decode_edge", n * edge_units(w, h, desc.chroma, True), sms)
    images = [DecodeImage(desc, w, h, f"{seed}_{i}", overshoot=True) for i in range(n)]
    assert_batched(ctx, lambda: run_decode_batch(ctx, desc, images), images, ys)
    assert_decode_same_as_direct(ctx, images, checker, threads=os.cpu_count())


@pytest.mark.gpu
@pytest.mark.parametrize("chroma,h", [(C444, 264), (C420, 527)], ids=["444", "420"])
def test_encode_batch_multipass(ctx, port, chroma, h):
    """64 images of 527 px: three 256-px units per interior row (the last with one active lane) and a 7-px right strip.
    The interior walk takes about 3 passes of its grid, the edge walk about 8; in 4:2:0 the odd last rows' bottom strips
    join the edge walk."""
    desc = planar(16, 4, STRAIGHT, 10, chroma, N709 if chroma == C444 else N2020)
    run_multipass_encode(ctx, port, desc, CHUNK, 527, h, f"kernels_multipass_{chroma}")


@pytest.mark.gpu
@pytest.mark.parametrize("bit_depth,host_depth,nclx", [(8, 8, N601), (10, 16, cases.NCLX_2020_PQ(0))], ids=["8to8", "10to16"])
def test_decode_batch_multipass(ctx, checker, port, bit_depth, host_depth, nclx):
    """64 images of 527 x 263, 4:2:0 with alpha: 393 interior units (row pairs) and 266 edge units (263 right-strip rows,
    3 units of the last row) per image -- about 8 passes of both grids."""
    desc = ycc(host_depth, bit_depth, C420, STRAIGHT, nclx)
    run_multipass_decode(ctx, pick(checker, port, True), desc, CHUNK, 527, 263, f"kernels_multipass_{bit_depth}")


@pytest.mark.gpu
def test_encode_bottom_strip_of_several_units(ctx, port):
    """Odd 4:2:0 heights 1289 px wide: each bottom strip is 644 chroma sites, three edge units, the last one partial."""
    w = 1289
    desc = planar(8, 4, STRAIGHT, 8, C420, N601)
    assert bottom_units(w, C420, False) == 3
    images = [EncodeImage(desc, w, h, f"kernels_bottom_{i}") for i, h in enumerate((5, 3, 9, 2))]
    assert_batched(ctx, lambda: run_batch(ctx, desc, images), images, 1)
    assert_same_as_direct(ctx, images, port, threads=os.cpu_count())


@pytest.mark.gpu
def test_decode_bottom_strip_of_several_units(ctx, checker, port):
    """Odd 4:2:0 heights 1289 px wide: each bottom strip is 1288 pixels, six edge units, the last one partial."""
    w = 1289
    desc = ycc(16, 12, C420, STRAIGHT, N709)
    assert bottom_units(w, C420, True) == 6
    images = [DecodeImage(desc, w, h, f"kernels_bottom_{i}", overshoot=True) for i, h in enumerate((5, 3, 9, 2))]
    assert_batched(ctx, lambda: run_decode_batch(ctx, desc, images), images, 1)
    assert_decode_same_as_direct(ctx, images, pick(checker, port, True), threads=os.cpu_count())


# ---- the first image is empty ---------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_encode_batch_led_by_an_empty_image_on_a_fresh_context(port):
    """The first call of a premultiplied configuration verifies the fast premultiply (one launch) before it plans the
    batch; the first image converting nothing must not change that."""
    import avifgpu
    desc = planar(8, 4, PREMUL, 10, C422, N709, BOX)
    with avifgpu.Context(0) as fresh:
        images = [EncodeImage(desc, w, h, f"kernels_empty_first_{i}") for i, (w, h) in enumerate(MIXED)]
        launches = launches_of(fresh, lambda: run_batch(fresh, desc, [Empty()] + images))
        assert launches == 1 + expected_launches(fresh, images, 0)
        assert_same_as_direct(fresh, images, port)


@pytest.mark.gpu
def test_decode_batch_led_by_an_empty_image_on_a_fresh_context(checker, port):
    """The first decode call of a YCbCr configuration verifies the fast green-channel division (one launch) with the
    first image's parameters; a first image that converts nothing must still carry the description's matrix and range."""
    import avifgpu
    desc = ycc(16, 12, C420, STRAIGHT, cases.NCLX_2020_PQ(0))
    with avifgpu.Context(0) as fresh:
        images = [DecodeImage(desc, w, h, f"kernels_empty_first_{i}", overshoot=True) for i, (w, h) in enumerate(MIXED)]
        launches = launches_of(fresh, lambda: run_decode_batch(fresh, desc, [Empty()] + images))
        assert launches == 1 + expected_launches(fresh, images, 1)
        assert_decode_same_as_direct(fresh, images, pick(checker, port, True))
