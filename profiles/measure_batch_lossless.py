#!/usr/bin/env python3
"""Per-image device time of batched planar-RGB (lossless) decodes -- DecodePlanarRgbIntBatchKernel for 8/16-bit hosts,
TableDecodeF32BatchKernel for 32-bit hosts -- against the other ways to decode N images, for N = 1, 8, 64, 256, 1024:

  pq12     512 x 512 12-bit planar RGB, PQ -> RGB32f;
  hlg10a   512 x 512 10-bit planar RGBA, HLG + OOTF -> RGBA32f;
  rgba8    512 x 512 8-bit planar RGBA -> RGBA8;
  mixed16  10-bit planar RGB -> RGB16 at 197 x 131, 320 x 240, 517 x 389 and 64 x 63 (right strips).

Four ways per workload, as profiles/measure_batch_indirect.py measures them: N direct device calls, one host-described
batch call, one device-described call and one replay of a captured device-described call; CUDA-event time over at least
`--seconds` of back-to-back calls on one stream, the ways alternating for `--rounds` rounds, the median kept.  The four
ways' outputs are compared bit for bit, and every device-described status must be 0.  Prints one JSON line with the card's
name, power limit and maximum SM clock, read in the same run.

    python profiles/measure_batch_lossless.py [--seconds 1.0] [--rounds 3] [--counts 1,8,64,256,1024] [--out lossless.json]
"""
import harness
import torch

import avifgpu
from avifgpu import abi

COUNTS = (1, 8, 64, 256, 1024)


def nclx(transfer):
    return abi.Nclx(1, abi.PRIMARIES_BT2020, transfer, abi.MATRIX_GBR, 1)


GBR = abi.Nclx(1, abi.PRIMARIES_BT709, abi.TRANSFER_CHAR_SRGB, abi.MATRIX_GBR, 1)
WORKLOADS = {
    "pq12": (abi.DecodeDesc(0, 0, abi.COLORSPACE_RGB, abi.CHROMA_444, 12, abi.ALPHA_NONE, 32, nclx(abi.TRANSFER_CHAR_PQ), pq_peak_nits=1000),
             harness.size_512),
    "hlg10a": (abi.DecodeDesc(0, 0, abi.COLORSPACE_RGB, abi.CHROMA_444, 10, abi.ALPHA_STRAIGHT, 32, nclx(abi.TRANSFER_CHAR_HLG), hlg_apply_ootf=1),
               harness.size_512),
    "rgba8": (abi.DecodeDesc(0, 0, abi.COLORSPACE_RGB, abi.CHROMA_444, 8, abi.ALPHA_STRAIGHT, 8, GBR), harness.size_512),
    "mixed16": (abi.DecodeDesc(0, 0, abi.COLORSPACE_RGB, abi.CHROMA_444, 10, abi.ALPHA_NONE, 16, GBR), harness.mixed_size),
}


def main():
    ap = harness.arguments(rounds=3)
    ap.add_argument("--counts", default=",".join(map(str, COUNTS)))
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()
    harness.require_gpu()
    result = {"card": harness.card(), "workloads": []}
    g = torch.Generator(device="cuda")
    g.manual_seed(17)
    stream = torch.cuda.Stream()
    for name in args.workloads.split(","):
        desc, size_of = WORKLOADS[name]
        for n in (int(c) for c in args.counts.split(",")):
            ctx = avifgpu.Context(0)
            images = harness.decode_images(desc, size_of, n, g)
            ways = harness.BatchWays(ctx, desc, images, False, stream)
            result["workloads"].append(harness.measure_indirect(name, n, ways, args.seconds, args.rounds))
            del images, ways
            ctx.close()
            torch.cuda.empty_cache()
    harness.emit([result], args.out)


if __name__ == "__main__":
    main()
