#!/usr/bin/env python3
"""Per-image device time of a device-described batch (avifgpu_{encode,decode}_batch_indirect) against the other ways to
convert N images, for N = 1, 8, 64, 256, 1024:

  c1      512 x 512 RGBA8 -> 8-bit YCbCr 4:4:4 + alpha;
  mixed   RGBA8 -> 8-bit 4:2:0 + alpha at 197 x 131, 320 x 240, 517 x 389 and 64 x 63 (right strips, odd rows);
  dec420  512 x 512 8-bit YCbCr 4:2:0 + alpha -> RGBA8.

Four ways per workload: N direct device calls, one host-described batch call (*_batch_device), one device-described call
(*_batch_indirect) and one replay of a captured device-described call.  Each figure is CUDA-event time over at least
`--seconds` of back-to-back calls on one stream, the ways alternating for `--rounds` rounds; the JSON keeps every round.
The four ways' outputs are compared bit for bit.  A torch.profiler pass over the device-described call splits its time
between the plan, interior and edge kernels (the plan's one CTA, and the persistent grids when they have little or no
work).  Prints one JSON line with the card's name, power limit and maximum SM clock, read in the same run.

    python profiles/measure_batch_indirect.py [--seconds 1.0] [--rounds 3] [--out indirect.json]
"""
import harness
import torch

import avifgpu

COUNTS = (1, 8, 64, 256, 1024)
WORKLOADS = {  # name: (desc, encode, size of image i)
    "c1": (harness.C1, True, harness.size_512),
    "mixed": (harness.MIXED, True, harness.mixed_size),
    "dec420": (harness.DEC420, False, harness.size_512),
}


def main():
    args = harness.arguments(rounds=3).parse_args()
    harness.require_gpu()
    result = {"card": harness.card(), "workloads": []}
    g = torch.Generator(device="cuda")
    g.manual_seed(11)
    stream = torch.cuda.Stream()
    for name, (desc, encode, size_of) in WORKLOADS.items():
        for n in COUNTS:
            ctx = avifgpu.Context(0)
            images = (harness.encode_images if encode else harness.decode_images)(desc, size_of, n, g)
            ways = harness.BatchWays(ctx, desc, images, encode, stream)
            result["workloads"].append(harness.measure_indirect(name, n, ways, args.seconds, args.rounds))
            del images, ways
            ctx.close()
            torch.cuda.empty_cache()
    harness.emit([result], args.out)


if __name__ == "__main__":
    main()
