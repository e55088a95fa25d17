"""The float decode kernels that read semi-planar and MSB-aligned sources (DecodeSourceYccF32Kernel,
DecodeSourceYccF32BatchKernel under both record sources) hold the planar kernels' per-pixel arithmetic: per pixel 44 FP64
instructions for HLG + OOTF and 102 for PQ, and no checked division (FCHK ... CALL) in the main loop of the PQ kernel with the
verified quotient beyond the green-term fallback -- for each of the three layouts.  Checked on the built library with
cuobjdump (no GPU needed)."""
import collections
import functools
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "avif-format_b200", "lib", "libavifgpu.so")


@functools.lru_cache(maxsize=None)
def main_loops(kernel):
    """{mangled name: Counter of opcodes inside the kernel's largest backward-branch span} of the kernels named `kernel`"""
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    loops = {}
    for block in sass.split("Function : ")[1:]:
        mangled = block.split("\n", 1)[0].strip()
        if kernel not in mangled:
            continue
        instructions = [(int(m.group(1), 16), m.group(2).strip()) for m in re.finditer(r"/\*([0-9a-f]{4,})\*/\s+(.*?);", block)]
        best = None
        for address, text in instructions:
            target = re.search(r"BRA\S*\s+.*?(0x[0-9a-f]+)", text)
            if target and int(target.group(1), 16) < address:
                span = address - int(target.group(1), 16)
                if best is None or span > best[0]:
                    best = (span, int(target.group(1), 16), address)
        counts = collections.Counter()
        for address, text in instructions:
            if best and best[1] <= address <= best[2]:
                words = text.split()
                if words[0].startswith("@"):
                    words = words[1:]
                counts[words[0].split(".")[0]] += 1
        loops[mangled] = counts
    return loops


@pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(LIB), reason="needs cuobjdump and the built library")
@pytest.mark.parametrize("kernel,source,count", [("DecodeSourceYccF32Kernel", "", 72),
                                                 ("DecodeSourceYccF32BatchKernel", "ChunkSource", 72),
                                                 ("DecodeSourceYccF32BatchKernel", "WorkspaceSource", 72)],
                         ids=["single", "chunk", "workspace"])
@pytest.mark.parametrize("layout", [1, 2, 3], ids=["interleaved", "msb", "interleaved_msb"])
def test_semiplanar_float_loops_hold_the_planar_fp64_sequences(kernel, source, count, layout):
    loops = {k: v for k, v in main_loops(kernel).items() if source in k}
    # 3 chroma modes x 4 curve kernels x alpha x 3 layouts
    assert len(loops) == count, sorted(loops)
    # template arguments <[Source,] XS, YS, TRANSFER, ALPHA, FASTDIV, SOURCE>: 4:2:0 without alpha; TRANSFER 1 = HLG, 0 = PQ
    hlg = next(v for k, v in loops.items() if f"Li1ELi1ELi1ELi0ELi0ELi{layout}EE" in k)
    pq = next(v for k, v in loops.items() if f"Li1ELi1ELi0ELi0ELi1ELi{layout}EE" in k)
    pq_ieee = next(v for k, v in loops.items() if f"Li1ELi1ELi0ELi0ELi0ELi{layout}EE" in k)
    fp64 = lambda c: c["DFMA"] + c["DMUL"] + c["DADD"]  # noqa: E731
    pixels_per_iteration = 8  # a lane's 4 pixels of each row of a row pair
    assert fp64(hlg) == 44 * pixels_per_iteration
    assert fp64(pq) == 102 * pixels_per_iteration
    assert fp64(pq_ieee) == 102 * pixels_per_iteration
    assert pq["MUFU"] >= 24 and pq_ieee["FCHK"] >= 24
    assert pq["FCHK"] <= 2 and pq["CALL"] <= 2
    assert hlg["FCHK"] <= 2 and hlg["CALL"] <= 2
    if layout & 1:
        assert pq["PRMT"] >= 2  # the pairs are split by byte permutation
