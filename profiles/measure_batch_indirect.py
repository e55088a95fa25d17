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
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from measure_batch import N601, WORKLOADS, card, make_images, padded, per_call_ms, timed  # noqa: E402

import torch  # noqa: E402

import avifgpu  # noqa: E402
from avifgpu import abi  # noqa: E402

COUNTS = (1, 8, 64, 256, 1024)
DECODE = abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, abi.CHROMA_420, 8, abi.ALPHA_STRAIGHT, 8, N601)


def decode_images(n, generator):
    images = []
    for _ in range(n):
        d = abi.DecodeDesc.from_buffer_copy(DECODE)
        d.width = d.height = 512
        planes = [None if sh is None else torch.randint(0, 256, (sh[0], padded(sh[1])), generator=generator, device="cuda", dtype=torch.int32)
                  .to(torch.uint8)[:, :sh[1]] for sh in abi.decode_plane_shapes(d)]
        images.append((d, torch.empty((512, 512 * 4), dtype=torch.uint8, device="cuda"), planes))
    return images


def kernel_split(run, calls=50):
    """Mean device microseconds per call of each kernel `run` launches, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            run()
        torch.cuda.synchronize()
    out = {}
    for event in prof.key_averages():
        if "PlanIndirect" in event.key or "WorkspaceSource" in event.key:
            name = ("plan" if "PlanIndirect" in event.key else "interior" if ("RgbInt" in event.key or "YccToRgbInt" in event.key) else "edge")
            out[name] = out.get(name, 0.0) + event.device_time_total / calls
    return out


def measure(name, n, encode, images, ctx, desc, stream, args):
    handle = stream.cuda_stream
    records = avifgpu.batch_images_from_tensors([(d.width, d.height, rows, planes) for d, rows, planes in images])
    device_records = avifgpu.pack_batch_images(records)
    count = torch.tensor([n], dtype=torch.int32, device="cuda")
    workspace = torch.empty(avifgpu.batch_workspace_bytes(n), dtype=torch.uint8, device="cuda")
    status = torch.empty(n, dtype=torch.int32, device="cuda")
    if encode:
        structs = [(d, rows.data_ptr(), rows.stride(0), avifgpu.planes_from_tensors(planes)) for d, rows, planes in images]

        def direct():
            for d, ptr, stride, planes in structs:
                ctx.encode_device(d, ptr, stride, planes, stream=handle)

        def batch():
            ctx.encode_batch_device(desc, records, stream=handle)

        def indirect():
            ctx.encode_batch_indirect(desc, device_records, count, n, workspace, status, stream=handle)

        def outputs():
            return [p.clone() for _, _, planes in images for p in planes if p is not None]

        def clear():
            for _, _, planes in images:
                for p in planes:
                    if p is not None:
                        p.zero_()
    else:
        structs = [(d, avifgpu.planes_from_tensors(planes), rows.data_ptr(), rows.stride(0)) for d, rows, planes in images]

        def direct():
            for d, planes, ptr, stride in structs:
                ctx.decode_device(d, planes, ptr, stride, stream=handle)

        def batch():
            ctx.decode_batch_device(desc, records, stream=handle)

        def indirect():
            ctx.decode_batch_indirect(desc, device_records, count, n, workspace, status, stream=handle)

        def outputs():
            return [rows.clone() for _, rows, _ in images]

        def clear():
            for _, rows, _ in images:
                rows.zero_()

    with torch.cuda.stream(stream):
        if not encode:
            ctx.prepare_decode(desc)
        batch()  # first-use work outside the capture
        indirect()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            indirect()
        direct()
        torch.cuda.synchronize()
        reference = outputs()
        identical = True
        for run in (batch, indirect, graph.replay):
            clear()
            run()
            torch.cuda.synchronize()
            identical = identical and all(torch.equal(a, b) for a, b in zip(reference, outputs()))
        identical = identical and bool((status == 0).all())
        times = timed({"direct": direct, "batch": batch, "indirect": indirect, "captured_indirect": graph.replay}, args.seconds, args.rounds, stream)
        split = kernel_split(indirect)
    entry = {"workload": name, "n": n, "outputs_identical": identical, "indirect_kernel_us": split}
    for way, ms in times.items():
        per_image = [t * 1e3 / n for t in ms]
        entry[way] = {"per_image_us": per_image, "median_per_image_us": statistics.median(per_image),
                      "spread_per_image_us": max(per_image) - min(per_image)}
    entry["captured_indirect_over_batch"] = entry["captured_indirect"]["median_per_image_us"] / entry["batch"]["median_per_image_us"]
    print(json.dumps({"workload": name, "n": n} | {w: round(entry[w]["median_per_image_us"], 3) for w in times} |
                     {"split_us": {k: round(v, 2) for k, v in split.items()}}), file=sys.stderr)
    del graph
    return entry


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    result = {"card": card(), "workloads": []}
    g = torch.Generator(device="cuda")
    g.manual_seed(11)
    stream = torch.cuda.Stream()
    for name in ("c1", "mixed", "dec420"):
        for n in COUNTS:
            ctx = avifgpu.Context(0)
            if name == "dec420":
                desc, images = DECODE, decode_images(n, g)
            else:
                desc, size_of, _ = WORKLOADS[name]
                images, _ = make_images(desc, size_of, n, g)
            result["workloads"].append(measure(name, n, name != "dec420", images, ctx, desc, stream, args))
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
