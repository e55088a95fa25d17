"""The content light level's host half (include/avifgpu.h, avifgpu_content_light_level; DESIGN.md section 5), without a GPU:
MaxCLL / MaxFALL against the Python restatement, and the library's level(k) -- the arithmetic its level tables are built
with -- against the checker's PQToLinear for every code of every depth."""
import os
import subprocess

import numpy as np
import pytest

import avifgpu
import light_level_spec as spec
from avifgpu import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEPTHS = (8, 10, 12)


@pytest.fixture(scope="module")
def library_levels(tmp_path_factory):
    """level(k) of every code as the library computes it (light_level.cuh compiled for the CPU), per depth."""
    exe = tmp_path_factory.mktemp("light") / "light_level_dump"
    subprocess.run(["g++", "-std=c++17", "-O2", "-mfma", "-ffp-contract=off", "-I", os.path.join(ROOT, "avif-format_b200", "csrc"),
                    os.path.join(ROOT, "tests", "native", "light_level_dump.cpp"), "-o", str(exe)], check=True)
    out = {}
    for depth in DEPTHS:
        raw = subprocess.run([str(exe), str(depth)], check=True, capture_output=True).stdout
        out[depth] = np.frombuffer(raw, dtype=np.uint32)
    return out


@pytest.mark.parametrize("depth", DEPTHS)
def test_level_of_every_code_matches_the_checker(library_levels, checker, depth):
    expected = spec.levels(checker, depth)
    got = library_levels[depth]
    assert got.shape == expected.shape
    differ = np.flatnonzero(got != expected)
    assert differ.size == 0, f"{differ.size} codes differ, first {differ[0]}: {got[differ[0]]} != {expected[differ[0]]} ({checker.kind})"
    assert got[0] == 0 and got[-1] == spec.SCALE  # code 0 is black, the top code 10000 cd/m2
    assert (np.diff(got.astype(np.int64)) >= 0).all()


def test_no_pixels_gives_zeros():
    assert avifgpu.content_light_level({"max_code": 0, "level_sum": 0, "pixels": 0}, 12) == (0, 0)


@pytest.mark.parametrize("depth", DEPTHS)
def test_every_max_code(checker, depth):
    table = spec.levels(checker, depth)
    for k in range(1 << depth):
        # three pixels: two at code k, one black -- MaxFALL rounds up a third of the level
        acc = {"max_code": k, "level_sum": 2 * int(table[k]), "pixels": 3}
        assert avifgpu.content_light_level(acc, depth) == spec.content_light_level(acc, table), (depth, k)


def test_two_to_the_31_pixels_at_full_level(checker):
    table = spec.levels(checker, 12)
    pixels = 1 << 31
    acc = {"max_code": 4095, "level_sum": spec.SCALE * pixels, "pixels": pixels}
    assert avifgpu.content_light_level(acc, 12) == spec.content_light_level(acc, table) == (10000, 10000)
    acc["level_sum"] -= 1  # one unit short of the peak: MaxFALL still rounds up to 10000
    assert avifgpu.content_light_level(acc, 12) == spec.content_light_level(acc, table) == (10000, 10000)


def test_mixed_frame(checker):
    table = spec.levels(checker, 10)
    rng = np.random.default_rng(7)
    codes = rng.integers(0, 1024, size=(64, 3 * 100))
    acc = spec.accumulate(codes, 3, table)
    assert avifgpu.content_light_level(acc, 10) == spec.content_light_level(acc, table)


@pytest.mark.parametrize("acc, depth", [
    ({"max_code": 0, "level_sum": 0, "pixels": 0}, 9),                      # not an image depth
    ({"max_code": 1024, "level_sum": 0, "pixels": 1}, 10),                  # code above 2^10 - 1
    ({"max_code": 4095, "level_sum": spec.SCALE * 2 + 1, "pixels": 2}, 12),  # above the peak level of every pixel
    ({"max_code": 0, "level_sum": 1, "pixels": 0}, 12),
])
def test_impossible_accumulators_are_refused(acc, depth):
    with pytest.raises(avifgpu.AvifGpuError) as failure:
        avifgpu.content_light_level(acc, depth)
    assert failure.value.status == abi.ERR_BAD_PARAM


def test_struct_layout():
    import ctypes as C
    assert C.sizeof(abi.LightLevel) == 24
    assert [abi.LightLevel.max_code.offset, abi.LightLevel.level_sum.offset, abi.LightLevel.pixels.offset] == [0, 8, 16]
