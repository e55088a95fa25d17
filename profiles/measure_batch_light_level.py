#!/usr/bin/env python3
"""Device time per image of HDR batches with each image's content light level, five ways:

  direct             N avifgpu_encode_rows_device_light_level calls, one per image, each into its own accumulator;
  batch              one avifgpu_encode_batch_device_light_level call;
  captured_batch     the replay of a CUDA graph of that call;
  indirect           one avifgpu_encode_batch_indirect_light_level call;
  captured_indirect  the replay of a CUDA graph of that call.

Workloads: N in {1, 8, 64, 256} images of 256 x 256, 512 x 512 and the harness's mixed sizes, for three descriptions --
12-bit PQ 4:2:0 from RGB32f, 10-bit PQ 4:4:4 from RGBA32f with straight alpha, and 10-bit PQ 4:2:0 into P010
(interleaved chroma, MSB-aligned codes).  Each way runs after a memset of the accumulators; the planes and accumulators of
every way are compared with the direct calls', bit for bit.  Ways alternate for `--rounds` rounds of at least `--seconds`
each (profiles/harness.py); the median per image is kept, and each batch way's ratio to the direct calls.  Prints one JSON
line per workload with the card's name, power limit and maximum SM clock, read in the same run.

    python profiles/measure_batch_light_level.py [--seconds 0.5] [--rounds 3] [--out batch_light_level.json]
"""
import statistics

import harness
import torch

import avifgpu
from avifgpu import abi

NV_MSB = abi.SOURCE_CHROMA_INTERLEAVED | abi.SOURCE_MSB_ALIGNED
NCLX_2020_PQ = abi.Nclx(1, 9, 16, 9, 1)  # BT.2020 primaries, PQ, BT.2020 NCL matrix, full range


def desc(channels, alpha, depth, chroma, dest=0):
    return abi.EncodeDesc(0, 0, 32, channels, alpha, depth, abi.TRANSFER_PQ, 1000, abi.LAYOUT_PLANAR_YCBCR, chroma, abi.DOWN_FILTER_BOX,
                          abi.GRAY16_LUT, NCLX_2020_PQ, dest_layout=dest)


DESCRIPTIONS = {
    "rgb_pq12_420": desc(3, abi.ALPHA_NONE, 12, abi.CHROMA_420),
    "rgba_pq10_444": desc(4, abi.ALPHA_STRAIGHT, 10, abi.CHROMA_444),
    "p010_pq10_420": desc(3, abi.ALPHA_NONE, 10, abi.CHROMA_420, NV_MSB),
}
SIZES = {"256": lambda i: (256, 256), "512": harness.size_512, "mixed": harness.mixed_size}


def float_images(d, size_of, n, generator):
    """(desc, rows, planes) per image: linear values in [0, 2) (up to 2000 cd/m2 at this peak) in 64-byte-padded rows."""
    images = []
    for i in range(n):
        w, h = size_of(i)
        di = abi.EncodeDesc.from_buffer_copy(d)
        di.width, di.height = w, h
        cols = w * d.host_channels
        rows = torch.rand((h, harness.padded(cols * 4) // 4), generator=generator, device="cuda") * 2.0
        if d.host_channels == 4:
            rows[:, 3:cols:4] = 1.0
        planes = [None if s is None else harness.plane(s[0], s[1], True) for s in abi.encode_plane_shapes(di)]
        images.append((di, rows.view(torch.uint8)[:, :cols * 4], planes))  # byte rows: strides in bytes
    return images


def measure(ctx, name, d, size_name, n, seconds, rounds, stream):
    images = float_images(d, SIZES[size_name], n, torch.Generator(device="cuda").manual_seed(n))
    handle = stream.cuda_stream
    records = avifgpu.batch_images_from_tensors([(di.width, di.height, rows, planes) for di, rows, planes in images])
    device_records = avifgpu.pack_batch_images(records)
    count = torch.tensor([n], dtype=torch.int32, device="cuda")
    workspace = torch.empty(avifgpu.batch_workspace_bytes(n), dtype=torch.uint8, device="cuda")
    status = torch.empty(n, dtype=torch.int32, device="cuda")
    acc = torch.zeros((n, 3), dtype=torch.int64, device="cuda")
    calls = [(di, rows.data_ptr(), rows.stride(0), avifgpu.planes_from_tensors(planes)) for di, rows, planes in images]
    written = [p for _, _, planes in images for p in planes if p is not None]

    def direct():
        acc.zero_()
        for i, call in enumerate(calls):
            ctx.encode_device_light_level(*call, acc.data_ptr() + 24 * i, stream=handle)

    def batch():
        acc.zero_()
        ctx.encode_batch_device_light_level(d, records, acc.data_ptr(), stream=handle)

    def indirect():
        acc.zero_()
        ctx.encode_batch_indirect_light_level(d, device_records, count, n, workspace, acc.data_ptr(), status, stream=handle)

    def capture(run):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            run()
        return graph  # kept alive by the caller

    with torch.cuda.stream(stream):
        for run in (direct, batch, indirect):
            run()
        torch.cuda.synchronize()
        graphs = {"captured_batch": capture(batch), "captured_indirect": capture(indirect)}
        ways = {"direct": direct, "batch": batch, "captured_batch": graphs["captured_batch"].replay, "indirect": indirect,
                "captured_indirect": graphs["captured_indirect"].replay}
        direct()
        torch.cuda.synchronize()
        reference = ([t.clone() for t in written], acc.clone())
        identical = {}
        for way, run in ways.items():
            for t in written:
                t.zero_()
            run()
            torch.cuda.synchronize()
            identical[way] = all(torch.equal(a, b) for a, b in zip(reference[0], written)) and torch.equal(reference[1], acc)
        times = harness.timed(ways, seconds, rounds, stream)
    entry = {"workload": f"{name}_{size_name}", "n": n, "outputs_identical": all(identical.values())}
    for way, ms in times.items():
        entry[way + "_us_per_image"] = round(statistics.median(ms) * 1e3 / n, 3)
    for way in ("batch", "captured_batch", "indirect", "captured_indirect"):
        entry[way + "_over_direct"] = round(entry[way + "_us_per_image"] / entry["direct_us_per_image"], 3)
    return entry


def main():
    args = harness.arguments(3).parse_args()
    harness.require_gpu()
    results = []
    stream = torch.cuda.Stream()
    with avifgpu.Context(0) as ctx:
        for name, d in DESCRIPTIONS.items():
            ctx.prepare_encode(d)
            for size_name in SIZES:
                for n in (1, 8, 64, 256):
                    results.append(measure(ctx, name, d, size_name, n, args.seconds, args.rounds, stream) | {"card": harness.card()})
    harness.emit(results, args.out)


if __name__ == "__main__":
    main()
