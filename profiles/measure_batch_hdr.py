#!/usr/bin/env python3
"""Per-image device time of batched HDR decodes (YCbCr 10 / 12-bit -> RGB(A)32f through DecodeYccToRgbF32BatchKernel)
against the other ways to decode N images, for N = 1, 8, 64, 256, 1024:

  hlg420   512 x 512 10-bit YCbCr 4:2:0, HLG + OOTF -> RGB32f;
  pq422a   512 x 512 12-bit YCbCr 4:2:2 + alpha, PQ -> RGBA32f;
  mixed    10-bit 4:2:0 PQ -> RGB32f at 197 x 131, 320 x 240, 517 x 389 and 64 x 63 (right strips, odd rows).

Four ways per workload, as profiles/measure_batch_indirect.py measures them: N direct device calls, one host-described
batch call, one device-described call and one replay of a captured device-described call; CUDA-event time over at least
`--seconds` of back-to-back calls on one stream, the ways alternating for `--rounds` rounds, the median kept.  The four
ways' outputs are compared bit for bit.  Prints one JSON line with the card's name, power limit and maximum SM clock,
read in the same run.

    python profiles/measure_batch_hdr.py [--seconds 1.0] [--rounds 3] [--out hdr.json]
"""
import harness
import torch

import avifgpu
from avifgpu import abi

COUNTS = (1, 8, 64, 256, 1024)


def nclx(transfer):
    return abi.Nclx(1, abi.PRIMARIES_BT2020, transfer, abi.MATRIX_BT2020_NCL, 1)


WORKLOADS = {
    "hlg420": (abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, abi.CHROMA_420, 10, abi.ALPHA_NONE, 32, nclx(abi.TRANSFER_CHAR_HLG)),
               harness.size_512),
    "pq422a": (abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, abi.CHROMA_422, 12, abi.ALPHA_STRAIGHT, 32, nclx(abi.TRANSFER_CHAR_PQ),
                              pq_peak_nits=1000), harness.size_512),
    "mixed": (abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, abi.CHROMA_420, 10, abi.ALPHA_NONE, 32, nclx(abi.TRANSFER_CHAR_PQ),
                             pq_peak_nits=1000), harness.mixed_size),
}


def main():
    ap = harness.arguments(rounds=3)
    ap.add_argument("--counts", default=",".join(map(str, COUNTS)))
    args = ap.parse_args()
    harness.require_gpu()
    result = {"card": harness.card(), "workloads": []}
    g = torch.Generator(device="cuda")
    g.manual_seed(13)
    stream = torch.cuda.Stream()
    for name, (desc, size_of) in WORKLOADS.items():
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
