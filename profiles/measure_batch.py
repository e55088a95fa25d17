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
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "avif-format_b200", "python"))
import torch  # noqa: E402

import avifgpu  # noqa: E402
from avifgpu import abi  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12


def card():
    ident = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=10).stdout.strip().split(",")
        ident["power_limit_w"], ident["sm_max_mhz"] = float(out[0]), float(out[1])
    except Exception:
        ident["power_limit_w"] = ident["sm_max_mhz"] = None
    return ident


N601 = abi.Nclx(1, 1, 13, abi.MATRIX_BT601, 1)
WORKLOADS = {
    "c1": (abi.EncodeDesc(0, 0, 8, 4, abi.ALPHA_STRAIGHT, 8, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_444,
                          abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, N601), lambda i: (512, 512), (1, 8, 64, 256)),
    "mixed": (abi.EncodeDesc(0, 0, 8, 4, abi.ALPHA_STRAIGHT, 8, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420,
                             abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, N601), lambda i: ((197, 131), (320, 240), (517, 389), (64, 63))[i % 4],
              (8, 64, 256)),
    "large": (abi.EncodeDesc(0, 0, 16, 4, abi.ALPHA_STRAIGHT, 10, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_422,
                             abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, N601), lambda i: (4096, 4096), (1,)),
}


def padded(n):
    return (n + 63) // 64 * 64


def make_images(desc, size_of, n, generator):
    images, nbytes = [], 0
    for i in range(n):
        w, h = size_of(i)
        d = abi.EncodeDesc.from_buffer_copy(desc)
        d.width, d.height = w, h
        row_bytes = w * d.host_channels * d.host_depth // 8
        # rows and planes padded to 64-byte strides, as image buffers usually are: odd widths keep the tuned route
        rows = torch.randint(0, 256, (h, padded(row_bytes)), generator=generator, device="cuda", dtype=torch.int32).to(torch.uint8)
        if d.host_depth == 16:
            rows = rows.view(torch.int16).bitwise_and_(0x7fff).view(torch.uint8)
        rows = rows[:, :row_bytes]
        sample = 2 if d.image_bit_depth > 8 else 1
        planes = [None if s is None else torch.empty((s[0], padded(s[1] * sample)), dtype=torch.uint8, device="cuda")[:, :s[1] * sample]
                  for s in abi.encode_plane_shapes(d)]
        nbytes += rows.numel() + sum(p.numel() for p in planes if p is not None)
        images.append((d, rows, planes))
    return images, nbytes


def per_call_ms(run, k, stream):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record(stream)
    for _ in range(k):
        run()
    end.record(stream)
    torch.cuda.synchronize()
    return start.elapsed_time(end) / k


def timed(ways, seconds, rounds, stream):
    """{name: [ms per call] * rounds}, the ways alternating, each window at least `seconds` long."""
    k = {}
    for name, run in ways.items():
        run()
        fastest = per_call_ms(run, 20, stream)
        k[name] = max(20, int(seconds / (fastest * 1e-3)) + 1)
    out = {name: [] for name in ways}
    for _ in range(rounds):
        for name, run in ways.items():
            out[name].append(per_call_ms(run, k[name], stream))
    return out


def outputs(images):
    return [p.clone() for _, _, planes in images for p in planes if p is not None]  # the visible columns only


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    result = {"card": card(), "peak_bytes_per_s": PEAK_BYTES_PER_S, "workloads": []}
    g = torch.Generator(device="cuda")
    g.manual_seed(11)
    stream = torch.cuda.Stream()
    handle = stream.cuda_stream
    for name, (desc, size_of, counts) in WORKLOADS.items():
        for n in counts:
            ctx = avifgpu.Context(0)
            images, nbytes = make_images(desc, size_of, n, g)
            records = avifgpu.batch_images_from_tensors([(d.width, d.height, rows, planes) for d, rows, planes in images])
            structs = [(d, rows.data_ptr(), rows.stride(0), avifgpu.planes_from_tensors(planes)) for d, rows, planes in images]

            def direct():
                for d, ptr, stride, planes in structs:
                    ctx.encode_device(d, ptr, stride, planes, stream=handle)

            def batch():
                ctx.encode_batch_device(desc, records, stream=handle)

            with torch.cuda.stream(stream):
                batch()  # first-use work outside the capture
                torch.cuda.synchronize()
                before = ctx.launch_count()
                batch()
                torch.cuda.synchronize()
                launches = ctx.launch_count() - before
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, stream=stream):
                    batch()

                def captured():
                    graph.replay()

                direct()
                torch.cuda.synchronize()
                reference = outputs(images)
                identical = True
                for run in (batch, captured):
                    for _, _, planes in images:
                        for p in planes:
                            if p is not None:
                                p.zero_()
                    run()
                    torch.cuda.synchronize()
                    identical = identical and all(torch.equal(a, b) for a, b in zip(reference, outputs(images)))
                ways = {"direct": direct, "batch": batch, "captured_batch": captured}
                if name == "c1" and n == 1:
                    single = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(single, stream=stream):
                        direct()
                    ways["captured_direct"] = single.replay
                times = timed(ways, args.seconds, args.rounds, stream)
            entry = {"workload": name, "n": n, "bytes": nbytes, "batch_launches": launches, "outputs_identical": identical}
            for way, ms in times.items():
                per_image_us = [t * 1e3 / n for t in ms]
                med = statistics.median(ms)
                entry[way] = {"per_image_us": per_image_us, "median_per_image_us": med * 1e3 / n,
                              "hbm_share": nbytes / (med * 1e-3) / PEAK_BYTES_PER_S}
            result["workloads"].append(entry)
            print(json.dumps({k: entry[k] for k in ("workload", "n")} | {w: round(entry[w]["median_per_image_us"], 3) for w in times}), file=sys.stderr)
            del graph
            ctx.close()
    ddesc = abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, abi.CHROMA_420, 8, abi.ALPHA_STRAIGHT, 8, N601)
    for n in (1, 8, 64, 256):
        ctx = avifgpu.Context(0)
        images, nbytes = [], 0
        for _ in range(n):
            d = abi.DecodeDesc.from_buffer_copy(ddesc)
            d.width = d.height = 512
            planes = [None if sh is None else torch.randint(0, 256, (sh[0], padded(sh[1])), generator=g, device="cuda", dtype=torch.int32)
                      .to(torch.uint8)[:, :sh[1]] for sh in abi.decode_plane_shapes(d)]
            rows = torch.empty((512, 512 * 4), dtype=torch.uint8, device="cuda")
            nbytes += rows.numel() + sum(q.numel() for q in planes if q is not None)
            images.append((d, rows, planes))
        records = avifgpu.batch_images_from_tensors([(d.width, d.height, rows, planes) for d, rows, planes in images])
        structs = [(d, avifgpu.planes_from_tensors(planes), rows.data_ptr(), rows.stride(0)) for d, rows, planes in images]

        def direct():
            for d, planes, ptr, stride in structs:
                ctx.decode_device(d, planes, ptr, stride, stream=handle)

        def batch():
            ctx.decode_batch_device(ddesc, records, stream=handle)

        with torch.cuda.stream(stream):
            ctx.prepare_decode(ddesc)
            batch()
            torch.cuda.synchronize()
            before = ctx.launch_count()
            batch()
            torch.cuda.synchronize()
            launches = ctx.launch_count() - before
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=stream):
                batch()
            direct()
            torch.cuda.synchronize()
            reference = [rows.clone() for _, rows, _ in images]
            identical = True
            for run in (batch, graph.replay):
                for _, rows, _ in images:
                    rows.zero_()
                run()
                torch.cuda.synchronize()
                identical = identical and all(torch.equal(a, rows) for a, (_, rows, _) in zip(reference, images))
            times = timed({"direct": direct, "batch": batch, "captured_batch": graph.replay}, args.seconds, args.rounds, stream)
        entry = {"workload": "dec420", "n": n, "bytes": nbytes, "batch_launches": launches, "outputs_identical": identical}
        for way, ms in times.items():
            med = statistics.median(ms)
            entry[way] = {"per_image_us": [t * 1e3 / n for t in ms], "median_per_image_us": med * 1e3 / n,
                          "hbm_share": nbytes / (med * 1e-3) / PEAK_BYTES_PER_S}
        result["workloads"].append(entry)
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
