"""What the profile scripts share: the card's identity, one timer, padded buffers, the seeded batch images, the ways to
convert a batch, torch.profiler's kernel split of a device-described batch call, and the JSON output.

The scripts run as `python profiles/<script>.py`, which puts this directory on sys.path; importing this module puts the
package and the repository root there too.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "avif-format_b200", "python"))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import avifgpu  # noqa: E402
import bench  # noqa: E402
from avifgpu import abi  # noqa: E402

N601 = abi.Nclx(1, 1, 13, abi.MATRIX_BT601, 1)
# the batch scripts' shared workloads: config 1's encode, a 4:2:0 encode at sizes with right strips and odd rows, and
# config 1's decode counterpart
C1 = abi.EncodeDesc(0, 0, 8, 4, abi.ALPHA_STRAIGHT, 8, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_444,
                    abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, N601)
MIXED = abi.EncodeDesc(0, 0, 8, 4, abi.ALPHA_STRAIGHT, 8, abi.TRANSFER_CLIP, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420,
                       abi.DOWN_FILTER_BOX, abi.GRAY16_LUT, N601)
DEC420 = abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, abi.CHROMA_420, 8, abi.ALPHA_STRAIGHT, 8, N601)


def size_512(i):
    return 512, 512


def mixed_size(i):
    return ((197, 131), (320, 240), (517, 389), (64, 63))[i % 4]


def arguments(rounds):
    """The options every script takes; a script adds its own before parsing."""
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0, help="least length of each timed window")
    ap.add_argument("--rounds", type=int, default=rounds, help="rounds in which the ways alternate")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    return ap


def require_gpu():
    if not torch.cuda.is_available():
        sys.exit(f"{os.path.basename(sys.argv[0])} needs a CUDA device")


def card():
    """The card the numbers are measured on: name, power limit and maximum SM clock, read in the same run."""
    return bench.device_identity(torch, 0)


def emit(results, out):
    """Prints each result as one JSON line, and writes the lines to `out` too if it is given."""
    lines = "".join(json.dumps(r) + "\n" for r in results)
    print(lines, end="")
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            f.write(lines)


def padded(n):
    return (n + 63) // 64 * 64


def plane(rows, samples, wide):
    """An empty rows x samples plane of 8-bit (16-bit if `wide`) samples, its stride padded to 64 bytes."""
    t = torch.empty((rows, padded(samples * (2 if wide else 1))), dtype=torch.uint8, device="cuda")
    return t[:, :samples * (2 if wide else 1)]


def per_call_ms(run, calls, stream):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record(stream)
    for _ in range(calls):
        run()
    end.record(stream)
    torch.cuda.synchronize()
    return start.elapsed_time(end) / calls


def timed(ways, seconds, rounds, stream=None, calls=None):
    """{way: [ms per call] * rounds}, by CUDA events on `stream` (the current stream if None).  Each way is warmed by one
    call and its window sized from a 20-call probe to last at least `seconds`; then the ways alternate for `rounds`
    rounds.  `calls`, if given, receives each way's calls per window."""
    calls = {} if calls is None else calls
    for way, run in ways.items():
        run()
        calls[way] = max(20, int(seconds / (per_call_ms(run, 20, stream) * 1e-3)) + 1)
    out = {way: [] for way in ways}
    for _ in range(rounds):
        for way, run in ways.items():
            out[way].append(per_call_ms(run, calls[way], stream))
    return out


def median_us(ways, seconds, rounds, n=1):
    """{way: median microseconds per image}, for ways that convert `n` images per call on the current stream."""
    return {way: statistics.median(ms) * 1e3 / n for way, ms in timed(ways, seconds, rounds).items()}


def kernel_split(run, calls=50):
    """Mean device microseconds per call of a device-described batch call's kernels, from torch.profiler: `plan` is
    PlanIndirectKernel, `edge` the two edge kernels (EncodePlanarBatchKernel, DecodeBatchKernel) and `interior` every
    other kernel launched with a WorkspaceSource."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            run()
        torch.cuda.synchronize()
    out = {}
    for event in prof.key_averages():
        if "PlanIndirect" in event.key:
            part = "plan"
        elif "WorkspaceSource" in event.key:
            part = "edge" if "EncodePlanarBatchKernel" in event.key or "DecodeBatchKernel" in event.key else "interior"
        else:
            continue
        out[part] = out.get(part, 0.0) + event.device_time_total / calls
    return out


def encode_images(desc, size_of, n, generator):
    """(desc, rows, planes) per image: random rows (16-bit samples up to 0x7fff) and empty planes."""
    images = []
    for i in range(n):
        w, h = size_of(i)
        d = abi.EncodeDesc.from_buffer_copy(desc)
        d.width, d.height = w, h
        row_bytes = w * d.host_channels * d.host_depth // 8
        # rows and planes padded to 64-byte strides, as image buffers usually are: odd widths keep the tuned route
        rows = torch.randint(0, 256, (h, padded(row_bytes)), generator=generator, device="cuda", dtype=torch.int32).to(torch.uint8)
        if d.host_depth == 16:
            rows = rows.view(torch.int16).bitwise_and_(0x7fff).view(torch.uint8)
        planes = [None if s is None else plane(s[0], s[1], d.image_bit_depth > 8) for s in abi.encode_plane_shapes(d)]
        images.append((d, rows[:, :row_bytes], planes))
    return images


def decode_images(desc, size_of, n, generator):
    """(desc, rows, planes) per image: random codes up to the depth's maximum in 64-byte-padded planes, empty rows."""
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
        images.append((d, plane(d.height, d.width * abi.decode_host_channels(d) * d.host_depth // 8, False), planes))
    return images


class BatchWays:
    """The ways to convert one batch of (desc, rows, planes) images on `stream`: `direct` (one device call per image),
    `batch` (the host-described *_batch_device call) and `indirect` (the device-described *_batch_indirect call)."""

    def __init__(self, ctx, desc, images, encode, stream):
        self.ctx, self.desc, self.encode, self.stream = ctx, desc, encode, stream
        n, handle = len(images), stream.cuda_stream
        records = avifgpu.batch_images_from_tensors([(d.width, d.height, rows, planes) for d, rows, planes in images])
        device_records = avifgpu.pack_batch_images(records)
        count = torch.tensor([n], dtype=torch.int32, device="cuda")
        workspace = torch.empty(avifgpu.batch_workspace_bytes(n), dtype=torch.uint8, device="cuda")
        self.status = status = torch.empty(n, dtype=torch.int32, device="cuda")
        if encode:
            calls = [(d, rows.data_ptr(), rows.stride(0), avifgpu.planes_from_tensors(planes)) for d, rows, planes in images]
            one, batch, indirect = ctx.encode_device, ctx.encode_batch_device, ctx.encode_batch_indirect
            self.written = [p for _, _, planes in images for p in planes if p is not None]  # the visible columns only
        else:
            calls = [(d, avifgpu.planes_from_tensors(planes), rows.data_ptr(), rows.stride(0)) for d, rows, planes in images]
            one, batch, indirect = ctx.decode_device, ctx.decode_batch_device, ctx.decode_batch_indirect
            self.written = [rows for _, rows, _ in images]

        def direct():
            for call in calls:
                one(*call, stream=handle)

        self.direct = direct
        self.batch = lambda: batch(desc, records, stream=handle)
        self.indirect = lambda: indirect(desc, device_records, count, n, workspace, status, stream=handle)

    def outputs(self):
        return [t.clone() for t in self.written]

    def clear(self):
        for t in self.written:
            t.zero_()

    def warm(self, *runs):
        """First-use work outside any capture: the decode's preparation and one call of each of `runs`."""
        if not self.encode:
            self.ctx.prepare_decode(self.desc)
        for run in runs:
            run()
        torch.cuda.synchronize()

    def capture(self, run):
        """The replay of `run` captured into a CUDA graph on the batch's stream (the graph lives as long as the replay)."""
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=self.stream):
            run()
        return graph.replay

    def identical(self, runs):
        """Whether each of `runs`, into cleared outputs, writes what the direct calls write, bit for bit."""
        self.direct()
        torch.cuda.synchronize()
        reference = self.outputs()
        same = True
        for run in runs:
            self.clear()
            run()
            torch.cuda.synchronize()
            same = same and all(torch.equal(a, b) for a, b in zip(reference, self.outputs()))
        return same


def measure_indirect(name, n, ways, seconds, rounds):
    """One workload of the device-described batch scripts: N direct calls, one host-described call, one device-described
    call and one replay of a captured device-described call, their outputs compared bit for bit and every status 0,
    timed alternating, and torch.profiler's split of the device-described call."""
    with torch.cuda.stream(ways.stream):
        ways.warm(ways.batch, ways.indirect)
        captured = ways.capture(ways.indirect)
        identical = ways.identical([ways.batch, ways.indirect, captured]) and bool((ways.status == 0).all())
        times = timed({"direct": ways.direct, "batch": ways.batch, "indirect": ways.indirect, "captured_indirect": captured},
                      seconds, rounds, ways.stream)
        split = kernel_split(ways.indirect)
    entry = {"workload": name, "n": n, "outputs_identical": identical, "indirect_kernel_us": split}
    for way, ms in times.items():
        per_image = [t * 1e3 / n for t in ms]
        entry[way] = {"per_image_us": per_image, "median_per_image_us": statistics.median(per_image),
                      "spread_per_image_us": max(per_image) - min(per_image)}
    entry["captured_indirect_over_batch"] = entry["captured_indirect"]["median_per_image_us"] / entry["batch"]["median_per_image_us"]
    print(json.dumps({"workload": name, "n": n} | {w: round(entry[w]["median_per_image_us"], 3) for w in times} |
                     {"split_us": {k: round(v, 2) for k, v in split.items()}}), file=sys.stderr)
    return entry
