#!/usr/bin/env python3
"""Per-frame device time of K direct device calls against K replays of a one-frame CUDA graph of the same call, for a
small frame (BASELINE config 1's 512 x 512 RGBA8 -> 8-bit YCbCr 4:4:4 + alpha) and a large one (config 2's 8K RGB32f ->
12-bit PQ 4:2:0).  Each figure is CUDA-event time over at least one second of back-to-back calls on one stream, divided
by K; the two ways alternate for three rounds.  Prints one JSON line with the card's name, power limit and maximum SM
clock, read in the same run.

    python profiles/measure_graph_replay.py [--seconds 1.0] [--rounds 3] [--out graph_replay.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "avif-format_b200", "python"))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import avifgpu  # noqa: E402
from avifgpu import abi  # noqa: E402
from bench import Workload  # noqa: E402


def card():
    ident = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=10).stdout.strip().split(",")
        ident["power_limit_w"], ident["sm_max_mhz"] = float(out[0]), float(out[1])
    except Exception:
        ident["power_limit_w"] = ident["sm_max_mhz"] = None
    return ident


def frames():
    """(name, desc, input tensor, output planes) of the two frames."""
    g = torch.Generator(device="cuda")
    g.manual_seed(7)
    n601 = abi.Nclx(1, 1, 13, abi.MATRIX_BT601, 1)
    small = abi.EncodeDesc(512, 512, 8, 4, abi.ALPHA_STRAIGHT, 8, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_444,
                           abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, n601)
    rows = torch.randint(0, 256, (512, 512 * 4), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
    planes = [None if s is None else torch.empty(s, dtype=torch.uint8, device="cuda") for s in abi.encode_plane_shapes(small)]
    yield "512x512 RGBA8 -> 8-bit YCbCr 4:4:4 + A (config 1)", small, rows, planes
    c2 = Workload("c2")
    yield c2.name + " (config 2)", c2.enc, c2.make_device_input(torch, torch.device("cuda"), 1)[0], c2.make_device_output(torch, torch.device("cuda"))


def per_frame_ms(run, k, stream):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record(stream)
    for _ in range(k):
        run()
    end.record(stream)
    torch.cuda.synchronize()
    return start.elapsed_time(end) / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    result = {"card": card(), "frames": []}
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

        def call_graph():
            graph.replay()

        with torch.cuda.stream(stream):
            fastest = min(per_frame_ms(call_direct, 50, stream), per_frame_ms(call_graph, 50, stream))
            k = max(50, int(args.seconds / (fastest * 1e-3)) + 1)  # both windows last at least `seconds`
            direct, replayed = [], []
            for _ in range(args.rounds):
                direct.append(per_frame_ms(call_direct, k, stream))
                replayed.append(per_frame_ms(call_graph, k, stream))
        d, r = statistics.median(direct), statistics.median(replayed)
        result["frames"].append({"frame": name, "k": k, "direct_ms": direct, "graph_ms": replayed, "direct_median_ms": d,
                                 "graph_median_ms": r, "saved_us_per_frame": (d - r) * 1e3, "saved_share": (d - r) / d,
                                 "graph_output_identical": identical})
        del graph
        ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
