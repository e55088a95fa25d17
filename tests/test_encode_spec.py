"""The encode model (encode_spec.py) against the C restatement, without a GPU.

Every family of cases.encode_cases() that the compiled reference cannot check directly (reference_ok = False: planar
YCbCr, the HLG save path, the row matrix, Gray16 -> SMPTE 428, non-finite floats, 16-bit samples above 32768) is held
to the model, once with the seeded random rows and once with extreme_rows().  Hand-computed answers pin the H.273
equations at the corners of the cube, and the model must reject planes with one code moved."""
import os
import subprocess
import sys

import numpy as np
import pytest

import cases
import encode_spec
from avifgpu import abi

SPEC_CASES = [(name, desc, rows) for name, desc, rows, reference_ok in cases.encode_cases(cases.SIZES, full=True) if not reference_ok]


def test_model_never_loads_the_restatement(ref):
    """Neither by name in its source nor at run time: a process that only builds the model's planes never maps
    liboracle.so."""
    here = os.path.dirname(os.path.abspath(__file__))
    with open(os.path.join(here, "encode_spec.py")) as f:
        source = f.read()
    for word in ("load_restatement", "best_checker", "liboracle", "CpuChecker("):
        assert word not in source, word
    script = ("import sys; sys.path[:0] = sys.argv[1:]\n"
              "import numpy as np, cases, encode_spec\n"
              "from avifgpu import abi\n"
              "d = abi.EncodeDesc(5, 3, 32, 4, abi.ALPHA_PREMULTIPLIED, 12, abi.TRANSFER_HLG, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420,"
              " abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, cases.NCLX_2020_HLG(), hlg_extension=abi.HLG_INVERSE_OOTF_THEN_OETF)\n"
              "encode_spec.Expected(encode_spec.load(), d, encode_spec.extreme_rows(d, 5, 3, 0))\n"
              "maps = open('/proc/self/maps').read()\n"
              "assert 'libavifref' in maps and 'liboracle' not in maps\n")
    root = os.path.dirname(here)
    paths = [here, os.path.join(root, "oracle"), os.path.join(root, "avif-format_b200", "python")]
    out = subprocess.run([sys.executable, "-c", script, *paths], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


def test_every_unpinned_family_is_covered():
    families = {name.split("_")[1] for name, _, _ in SPEC_CASES}
    assert families == {"ycc", "hlg", "rowmatrix", "gray16", "specials", "beyond"}, families


@pytest.mark.parametrize("name,desc,rows", SPEC_CASES, ids=[c[0] for c in SPEC_CASES])
def test_restatement_matches_model(ref, port, name, desc, rows):
    encode_spec.assert_matches(ref, desc, rows, port.encode(desc, rows), f"{name} random")
    extreme = encode_spec.extreme_rows(desc, desc.width, desc.height, name)
    encode_spec.assert_matches(ref, desc, extreme, port.encode(desc, extreme), f"{name} extreme")


FLOAT_COMPOSED = [(3, abi.ALPHA_NONE, abi.TRANSFER_PQ, 1000), (4, abi.ALPHA_STRAIGHT, abi.TRANSFER_SMPTE428, 80),
                  (4, abi.ALPHA_PREMULTIPLIED, abi.TRANSFER_PQ, 80), (4, abi.ALPHA_PREMULTIPLIED, abi.TRANSFER_CLIP, 80)]


@pytest.mark.parametrize("channels,alpha,transfer,peak", FLOAT_COMPOSED)
def test_composed_float_path_equals_the_reference_encoder(ref, channels, alpha, transfer, peak):
    """The scalar composition the model uses for the row matrix, HLG and non-finite samples is the reference's own
    encoder wherever both apply."""
    w, h = 37, 23
    desc = abi.EncodeDesc(w, h, 32, channels, alpha, 12, transfer, peak)
    for rows in (cases.float_host_rows(np.random.default_rng(channels + transfer), h, w, channels),
                 encode_spec.extreme_rows(desc, w, h, 5)):
        assert np.array_equal(encode_spec._composed_float_codes(ref, desc, rows), encode_spec._reference_codes(ref, desc, rows))


# ---- known answers ----------------------------------------------------------------------------------------------------------

def site_420(host, rgb):
    return np.array([[*rgb, *rgb], [*rgb, *rgb]], abi.host_dtype(host))


@pytest.mark.parametrize("host,top", [(16, 32768), (16, 65535), (32, 125.0)])
def test_known_answers_bt2020_12_bit_420(ref, port, host, top):
    """A 2x2 site of one colour, BT.2020, 12 bits, 4:2:0, full range: pure blue and pure red saturate their chroma (the
    float64 value is exactly 4095.5, clipped to 4095), neutral grey sits on the 2048 offset, white gives Y 4095."""
    transfer = abi.TRANSFER_PQ if host == 32 else abi.TRANSFER_CLIP
    desc = abi.EncodeDesc(2, 2, host, 3, abi.ALPHA_NONE, 12, transfer, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420,
                          abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, cases.NCLX_2020_PQ())
    grey = 16384 if host == 16 else 0.5  # any grey: R = G = B
    answers = {"blue": ((0, 0, top), {1: 4095}), "red": ((top, 0, 0), {2: 4095}), "grey": ((grey,) * 3, {1: 2048, 2: 2048}),
               "white": ((top,) * 3, {0: 4095, 1: 2048, 2: 2048}), "black": ((0, 0, 0), {0: 0, 1: 2048, 2: 2048})}
    for name, (rgb, want) in answers.items():
        rows = site_420(host, rgb)
        model = encode_spec.Expected(ref, desc, rows)
        got = port.encode(desc, rows)
        for k, code in want.items():
            assert int(model.codes[k].ravel()[0]) == code, (name, k)
            assert int(got[k].ravel()[0]) == code, (name, k)
        if name in ("blue", "red"):
            k = 1 if name == "blue" else 2
            assert model.exact[k].ravel()[0] == 4095.5  # on the clip: 2^12 before it
        assert not model.mismatches(got), name


def test_gray16_smpte428_is_near_st428(ref):
    """Every Gray16 input at 10 and 12 bits: the model's codes are within one code of a float64 SMPTE ST 428-1 curve,
    E' = (48 L / 52.37)^(1/2.6), with L = v / 32768 (above 32768 the curve continues until E' clamps to 1)."""
    rows = np.arange(65536, dtype=np.uint32).astype(np.uint16).reshape(256, 256)
    for depth in (10, 12):
        desc = abi.EncodeDesc(256, 256, 16, 1, abi.ALPHA_NONE, depth, gray16_curve=abi.GRAY16_SMPTE428)
        got = encode_spec.Expected(ref, desc, rows).codes[0]
        linear = rows.astype(np.float64) / 32768
        st428 = np.floor(np.clip((48 * linear / 52.37) ** (1 / 2.6), 0, 1) * ((1 << depth) - 1))
        assert np.abs(st428 - got).max() <= 1


# ---- teeth ---------------------------------------------------------------------------------------------------------------------

def test_model_rejects_one_moved_code(ref, port):
    desc = abi.EncodeDesc(37, 23, 32, 4, abi.ALPHA_PREMULTIPLIED, 12, abi.TRANSFER_PQ, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420,
                          abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, cases.NCLX_2020_PQ())
    rows = cases.float_host_rows(np.random.default_rng(11), 23, 37, 4)
    model = encode_spec.Expected(ref, desc, rows)
    planes = port.encode(desc, rows)
    assert not model.mismatches(planes)
    for k in range(4):
        if k < 3:
            v = model.exact[k] + 0.5
            frac = v - np.floor(v)
            far = (np.minimum(frac, 1 - frac) > 0.2) & (model.codes[k] > 0) & (model.codes[k] < model.top)
        else:
            far = (model.codes[k] > 0) & (model.codes[k] < model.top)
        at = tuple(np.argwhere(far)[-1])  # the last such sample: the odd bottom row / right column where there is one
        for step in (-1, 1):
            moved = [None if p is None else p.copy() for p in planes]
            moved[k][at] = int(moved[k][at]) + step
            assert model.mismatches(moved), (k, at, step)


def test_model_rejects_an_unclipped_saturated_site(ref, port):
    """A saturated blue site written as 2^depth is one code from the expected value and on a rounding boundary: only
    the range check rejects it."""
    desc = abi.EncodeDesc(2, 2, 16, 3, abi.ALPHA_NONE, 12, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420,
                          abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, cases.NCLX_2020_PQ())
    rows = site_420(16, (0, 0, 32768))
    model = encode_spec.Expected(ref, desc, rows)
    planes = port.encode(desc, rows)
    planes[1][0, 0] = 4096
    assert any("outside" in m for m in model.mismatches(planes))


def test_extreme_rows_cover_every_corner_in_every_region():
    """The right column and the bottom row of sites each see all eight corners, as does the interior."""
    desc = abi.EncodeDesc(37, 23, 8, 3, abi.ALPHA_NONE, 8, layout=abi.LAYOUT_PLANAR_YCBCR, chroma=abi.CHROMA_420)
    px = encode_spec.extreme_rows(desc, 37, 23, 1).reshape(23, 37, 3)
    corner = (px[..., 0] // 255) * 4 + (px[..., 1] // 255) * 2 + px[..., 2] // 255
    for region in (corner[:, -1], corner[-1, :], corner[:16, :32]):
        assert set(np.unique(region)) == set(range(8))
