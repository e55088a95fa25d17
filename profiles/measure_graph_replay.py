#!/usr/bin/env python3
"""Per-frame device time of K direct device calls against K replays of a one-frame CUDA graph of the same call, for a
small frame (BASELINE config 1's 512 x 512 RGBA8 -> 8-bit YCbCr 4:4:4 + alpha) and a large one (config 2's 8K RGB32f ->
12-bit PQ 4:2:0).  Each figure is CUDA-event time over at least `--seconds` of back-to-back calls on one stream, divided
by K, each way's K sized from a 20-call probe; the two ways alternate for `--rounds` rounds.  Prints one JSON line with
the card's name, power limit and maximum SM clock, read in the same run.

    python profiles/measure_graph_replay.py [--seconds 1.0] [--rounds 3] [--out graph_replay.json]
"""
import statistics

import harness
import torch

import avifgpu
from avifgpu import abi
from bench import Workload


def frames():
    """(name, desc, input tensor, output planes) of the two frames."""
    g = torch.Generator(device="cuda")
    g.manual_seed(7)
    small = abi.EncodeDesc.from_buffer_copy(harness.C1)
    small.width = small.height = 512
    rows = torch.randint(0, 256, (512, 512 * 4), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
    planes = [None if s is None else torch.empty(s, dtype=torch.uint8, device="cuda") for s in abi.encode_plane_shapes(small)]
    yield "512x512 RGBA8 -> 8-bit YCbCr 4:4:4 + A (config 1)", small, rows, planes
    c2 = Workload("c2")
    yield c2.name + " (config 2)", c2.enc, c2.make_device_input(torch, torch.device("cuda"), 1)[0], c2.make_device_output(torch, torch.device("cuda"))


def main():
    args = harness.arguments(rounds=3).parse_args()
    harness.require_gpu()
    result = {"card": harness.card(), "frames": []}
    for name, desc, rows, planes in frames():
        ctx = avifgpu.Context(0)
        ctx.prepare_encode(desc)
        struct = avifgpu.planes_from_tensors(planes)
        stride = rows.stride(0) * rows.element_size()
        stream = torch.cuda.Stream()
        handle = stream.cuda_stream

        def call_direct():
            ctx.encode_device(desc, rows.data_ptr(), stride, struct, stream=handle)

        call_direct()  # warm-up outside the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            call_direct()
        direct_out = [None if p is None else p.clone() for p in planes]
        for p in planes:
            if p is not None:
                p.zero_()
        with torch.cuda.stream(stream):
            graph.replay()
        torch.cuda.synchronize()
        identical = all(a is None or torch.equal(a, b) for a, b in zip(direct_out, planes))

        k = {}
        with torch.cuda.stream(stream):
            times = harness.timed({"direct": call_direct, "graph": graph.replay}, args.seconds, args.rounds, stream, calls=k)
        d, r = statistics.median(times["direct"]), statistics.median(times["graph"])
        result["frames"].append({"frame": name, "k": k, "direct_ms": times["direct"], "graph_ms": times["graph"], "direct_median_ms": d,
                                 "graph_median_ms": r, "saved_us_per_frame": (d - r) * 1e3, "saved_share": (d - r) / d,
                                 "graph_output_identical": identical})
        del graph
        ctx.close()
    harness.emit([result], args.out)


if __name__ == "__main__":
    main()
