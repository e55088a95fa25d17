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
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import measure_batch_indirect  # noqa: E402
from measure_batch import card, padded  # noqa: E402

import torch  # noqa: E402

import avifgpu  # noqa: E402
from avifgpu import abi  # noqa: E402

COUNTS = (1, 8, 64, 256, 1024)


def nclx(transfer):
    return abi.Nclx(1, abi.PRIMARIES_BT2020, transfer, abi.MATRIX_BT2020_NCL, 1)


WORKLOADS = {
    "hlg420": (abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, abi.CHROMA_420, 10, abi.ALPHA_NONE, 32, nclx(abi.TRANSFER_CHAR_HLG)),
               lambda i: (512, 512)),
    "pq422a": (abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, abi.CHROMA_422, 12, abi.ALPHA_STRAIGHT, 32, nclx(abi.TRANSFER_CHAR_PQ),
                              pq_peak_nits=1000), lambda i: (512, 512)),
    "mixed": (abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, abi.CHROMA_420, 10, abi.ALPHA_NONE, 32, nclx(abi.TRANSFER_CHAR_PQ),
                             pq_peak_nits=1000), lambda i: ((197, 131), (320, 240), (517, 389), (64, 63))[i % 4]),
}


def decode_images(desc, size_of, n, generator):
    """(desc, rows, planes) per image: random codes (the top codes included) in 64-byte-padded 16-bit planes."""
    images = []
    for i in range(n):
        d = abi.DecodeDesc.from_buffer_copy(desc)
        d.width, d.height = size_of(i)
        planes = []
        for shape in abi.decode_plane_shapes(d):
            if shape is None:
                planes.append(None)
                continue
            codes = torch.randint(0, 1 << d.bit_depth, (shape[0], padded(shape[1] * 2) // 2), generator=generator, device="cuda", dtype=torch.int32)
            planes.append(codes.to(torch.int16).view(torch.uint8)[:, :shape[1] * 2])
        row_bytes = d.width * abi.decode_host_channels(d) * 4
        images.append((d, torch.empty((d.height, padded(row_bytes)), dtype=torch.uint8, device="cuda")[:, :row_bytes], planes))
    return images


def kernel_split(run, calls=50):
    """Mean device microseconds per call of the device-described call's plan, interior and edge kernels (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            run()
        torch.cuda.synchronize()
    out = {}
    for event in prof.key_averages():
        if "PlanIndirect" in event.key or "WorkspaceSource" in event.key:
            name = "plan" if "PlanIndirect" in event.key else "interior" if "F32Batch" in event.key else "edge"
            out[name] = out.get(name, 0.0) + event.device_time_total / calls
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--counts", default=",".join(map(str, COUNTS)))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    measure_batch_indirect.kernel_split = kernel_split  # the float interior kernel's name
    result = {"card": card(), "workloads": []}
    g = torch.Generator(device="cuda")
    g.manual_seed(13)
    stream = torch.cuda.Stream()
    for name, (desc, size_of) in WORKLOADS.items():
        for n in (int(c) for c in args.counts.split(",")):
            ctx = avifgpu.Context(0)
            images = decode_images(desc, size_of, n, g)
            result["workloads"].append(measure_batch_indirect.measure(name, n, False, images, ctx, desc, stream, args))
            del images
            ctx.close()
            torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
