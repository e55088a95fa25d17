#!/usr/bin/env python3
"""Per-image device time of N direct device calls, one avifgpu_encode_batch_device call and one replay of a captured
batch call, for N images of a workload:

  c1      BASELINE config 1's 512 x 512 RGBA8 -> 8-bit YCbCr 4:4:4 + alpha, N = 1, 8, 64, 256;
  mixed   RGBA8 -> 8-bit 4:2:0 + alpha at sizes with right strips and odd rows (edge launches), N = 8, 64, 256;
  large   one 4096 x 4096 RGBA16 -> 10-bit 4:2:2 + alpha, N = 1;
  dec420  the decode counterpart of c1: 512 x 512 8-bit YCbCr 4:2:0 + alpha -> RGBA8, N = 1, 8, 64, 256.

Also, in the same run, the per-frame time of a CUDA-graph replay of one direct config-1 call (profiles/
measure_graph_replay.py's figure).  Each figure is CUDA-event time over at least `--seconds` of back-to-back calls on
one stream; the ways alternate for `--rounds` rounds.  Each figure's share of 3.35 TB/s (H100 SXM data sheet) counts
the algorithmic bytes: host rows read plus planes written.  The three ways' outputs are compared bit for bit.  Prints one
JSON line with the card's name, power limit and maximum SM clock, read in the same run.

    python profiles/measure_batch.py [--seconds 1.0] [--rounds 3] [--out batch.json]
"""
import json
import statistics
import sys

import harness
import torch

import avifgpu
from avifgpu import abi

PEAK_BYTES_PER_S = 3.35e12

LARGE = abi.EncodeDesc(0, 0, 16, 4, abi.ALPHA_STRAIGHT, 10, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_422,
                       abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, harness.N601)
WORKLOADS = {  # name: (desc, encode, size of image i, counts)
    "c1": (harness.C1, True, harness.size_512, (1, 8, 64, 256)),
    "mixed": (harness.MIXED, True, harness.mixed_size, (8, 64, 256)),
    "large": (LARGE, True, lambda i: (4096, 4096), (1,)),
    "dec420": (harness.DEC420, False, harness.size_512, (1, 8, 64, 256)),
}


def measure(name, n, encode, ctx, desc, images, stream, args):
    nbytes = sum(rows.numel() + sum(p.numel() for p in planes if p is not None) for _, rows, planes in images)
    ways = harness.BatchWays(ctx, desc, images, encode, stream)
    with torch.cuda.stream(stream):
        ways.warm(ways.batch)
        before = ctx.launch_count()
        ways.batch()
        torch.cuda.synchronize()
        launches = ctx.launch_count() - before
        captured = ways.capture(ways.batch)
        identical = ways.identical([ways.batch, captured])
        timing = {"direct": ways.direct, "batch": ways.batch, "captured_batch": captured}
        if name == "c1" and n == 1:
            timing["captured_direct"] = ways.capture(ways.direct)
        times = harness.timed(timing, args.seconds, args.rounds, stream)
    entry = {"workload": name, "n": n, "bytes": nbytes, "batch_launches": launches, "outputs_identical": identical}
    for way, ms in times.items():
        med = statistics.median(ms)
        entry[way] = {"per_image_us": [t * 1e3 / n for t in ms], "median_per_image_us": med * 1e3 / n,
                      "hbm_share": nbytes / (med * 1e-3) / PEAK_BYTES_PER_S}
    print(json.dumps({k: entry[k] for k in ("workload", "n")} | {w: round(entry[w]["median_per_image_us"], 3) for w in times}), file=sys.stderr)
    return entry


def main():
    args = harness.arguments(rounds=3).parse_args()
    harness.require_gpu()
    result = {"card": harness.card(), "peak_bytes_per_s": PEAK_BYTES_PER_S, "workloads": []}
    g = torch.Generator(device="cuda")
    g.manual_seed(11)
    stream = torch.cuda.Stream()
    for name, (desc, encode, size_of, counts) in WORKLOADS.items():
        for n in counts:
            ctx = avifgpu.Context(0)
            images = (harness.encode_images if encode else harness.decode_images)(desc, size_of, n, g)
            result["workloads"].append(measure(name, n, encode, ctx, desc, images, stream, args))
            ctx.close()
    harness.emit([result], args.out)


if __name__ == "__main__":
    main()
