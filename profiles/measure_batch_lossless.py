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
    return abi.Nclx(1, abi.PRIMARIES_BT2020, transfer, abi.MATRIX_GBR, 1)


GBR = abi.Nclx(1, abi.PRIMARIES_BT709, abi.TRANSFER_CHAR_SRGB, abi.MATRIX_GBR, 1)
WORKLOADS = {
    "pq12": (abi.DecodeDesc(0, 0, abi.COLORSPACE_RGB, abi.CHROMA_444, 12, abi.ALPHA_NONE, 32, nclx(abi.TRANSFER_CHAR_PQ), pq_peak_nits=1000),
             lambda i: (512, 512)),
    "hlg10a": (abi.DecodeDesc(0, 0, abi.COLORSPACE_RGB, abi.CHROMA_444, 10, abi.ALPHA_STRAIGHT, 32, nclx(abi.TRANSFER_CHAR_HLG), hlg_apply_ootf=1),
               lambda i: (512, 512)),
    "rgba8": (abi.DecodeDesc(0, 0, abi.COLORSPACE_RGB, abi.CHROMA_444, 8, abi.ALPHA_STRAIGHT, 8, GBR), lambda i: (512, 512)),
    "mixed16": (abi.DecodeDesc(0, 0, abi.COLORSPACE_RGB, abi.CHROMA_444, 10, abi.ALPHA_NONE, 16, GBR),
                lambda i: ((197, 131), (320, 240), (517, 389), (64, 63))[i % 4]),
}


def decode_images(desc, size_of, n, generator):
    """(desc, rows, planes) per image: random codes up to the depth's maximum in 64-byte-padded planes."""
    images = []
    for i in range(n):
        d = abi.DecodeDesc.from_buffer_copy(desc)
        d.width, d.height = size_of(i)
        sample_bytes = 2 if d.bit_depth > 8 else 1
        planes = []
        for shape in abi.decode_plane_shapes(d):
            if shape is None:
                planes.append(None)
                continue
            codes = torch.randint(0, 1 << d.bit_depth, (shape[0], padded(shape[1] * sample_bytes) // sample_bytes), generator=generator,
                                  device="cuda", dtype=torch.int32)
            wide = codes.to(torch.int16).view(torch.uint8) if sample_bytes == 2 else codes.to(torch.uint8)
            planes.append(wide[:, :shape[1] * sample_bytes])
        row_bytes = d.width * abi.decode_host_channels(d) * d.host_depth // 8
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
            name = "plan" if "PlanIndirect" in event.key else "interior" if ("PlanarRgb" in event.key or "TableDecode" in event.key) else "edge"
            out[name] = out.get(name, 0.0) + event.device_time_total / calls
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--counts", default=",".join(map(str, COUNTS)))
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    measure_batch_indirect.kernel_split = kernel_split  # the planar-RGB interior kernels' names
    result = {"card": card(), "workloads": []}
    g = torch.Generator(device="cuda")
    g.manual_seed(17)
    stream = torch.cuda.Stream()
    for name in args.workloads.split(","):
        desc, size_of = WORKLOADS[name]
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
