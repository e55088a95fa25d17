"""The content light level of PQ encodes (include/avifgpu.h, avifgpu_light_level; DESIGN.md section 5), restated in Python
from the checker's own numbers: level(k) from the checker's PQToLinear, the accumulator from R'G'B' codes, MaxCLL and
MaxFALL from an accumulator.  A plain module, imported like cases.py; it touches no GPU."""
import functools

import numpy as np

from avifgpu import abi

SCALE = 1 << 22  # level units per 10000 cd/m2


@functools.lru_cache(maxsize=None)
def _levels(checker_key, depth):
    import oracle
    checker = {"reference": oracle.load_reference, "port": oracle.load_restatement}[checker_key]()
    top = (1 << depth) - 1
    codes = np.arange(top + 1, dtype=np.float32) / np.float32(top)
    linear = checker.transfer(abi.FN_PQ_TO_LINEAR, codes, 10000.0).astype(np.float32)
    return (linear * np.float32(SCALE)).astype(np.uint32)  # the product is exact: a power-of-two scale


def levels(checker, depth):
    """level(k) for every code k of `depth`: trunc(PQToLinear(k / maxCode, multiplier 1) * 2^22) by `checker`."""
    return _levels(checker.kind, depth)


def accumulate(codes, channels, level_table):
    """The accumulator of pixels whose interleaved codes are `codes` (rows x width*channels): k = max of the colour codes
    (the first three of RGB(A), the first of Gray(+A))."""
    pixels = np.asarray(codes).reshape(-1, channels)
    k = pixels[:, :3].max(axis=1) if channels >= 3 else pixels[:, 0]
    k = k.astype(np.int64)
    return {"max_code": int(k.max()) if k.size else 0, "reserved": 0,
            "level_sum": int(level_table[k].astype(np.uint64).sum()), "pixels": int(k.size)}


def add(a, b):
    return {"max_code": max(a["max_code"], b["max_code"]), "reserved": 0, "level_sum": a["level_sum"] + b["level_sum"],
            "pixels": a["pixels"] + b["pixels"]}


def content_light_level(acc, level_table):
    """(MaxCLL, MaxFALL): ceil(10000 level(max_code) / 2^22), ceil(10000 level_sum / (2^22 pixels)); 0, 0 without pixels."""
    if acc["pixels"] == 0:
        return 0, 0
    peak = int(level_table[acc["max_code"]])
    return -(-10000 * peak // SCALE), -(-10000 * acc["level_sum"] // (SCALE * acc["pixels"]))
