#!/usr/bin/env python3
"""Wall time of the content light level measured by the host-pointer encode (avifgpu_encode_rows_light_level) against
the plain host-pointer encode (avifgpu_encode_rows) on the 8K config-2 frame: 7680 x 4320 RGB32f -> 12-bit PQ 4:2:0,
rows and planes in page-locked host memory, so both calls stream the frame over PCIe through the three-slot pipeline.

Two cases, each on a context of its own:
  tables      step tables and level table prepared (avifgpu_prepare_encode): the tuned flat kernel;
  no_tables   a context that never builds tables: the generic kernel, which evaluates level(k) itself -- the route of a
              single save through the plug-in's row shuttle.

The two calls alternate for `--rounds` rounds, each timed by the host clock over at least `--seconds` of back-to-back
calls (a synchronous host call returns when its planes are in host memory); the median is kept.  The light-level call's
planes are compared bit for bit with the plain call's, launches counted, and its accumulator compared with the device
light-level call's over the same rows.  Prints one JSON line with the card's name, power limit and maximum SM clock,
read in the same run.

    python profiles/measure_host_light_level.py [--seconds 2.0] [--rounds 5] [--out host_light_level.json]
"""
import statistics
import time

import harness
import numpy as np
import torch

import avifgpu
from avifgpu import abi

W, H = 7680, 4320


def pinned_planes(ctx, desc):
    return [None if s is None else ctx.pinned_array(s, np.uint16) for s in abi.encode_plane_shapes(desc)]


def seconds_per_call(run, calls):
    start = time.perf_counter()
    for _ in range(calls):
        run()
    return (time.perf_counter() - start) / calls


def measure(ctx, desc, rows, seconds, rounds):
    plain_planes, light_planes = pinned_planes(ctx, desc), pinned_planes(ctx, desc)
    acc = abi.LightLevel()

    def plain():
        ctx.encode(desc, rows, planes=plain_planes)

    def light():
        acc.max_code, acc.level_sum, acc.pixels = 0, 0, 0
        ctx.encode_light_level(desc, rows, acc, planes=light_planes)

    ways = {"plain": plain, "light_level": light}
    calls = {}
    for way, run in ways.items():
        run()
        calls[way] = max(3, int(seconds / seconds_per_call(run, 3)) + 1)
    times = {way: [] for way in ways}
    for _ in range(rounds):
        for way, run in ways.items():
            times[way].append(seconds_per_call(run, calls[way]))
    out = {way: statistics.median(t) * 1e3 for way, t in times.items()}
    out["ratio_light_to_plain"] = out["light_level"] / out["plain"]
    out["spread_ms"] = {way: [round(min(t) * 1e3, 3), round(max(t) * 1e3, 3)] for way, t in times.items()}
    out["gb_per_s_host_to_device"] = {way: rows.nbytes / (out[way] * 1e-3) / 1e9 for way in ways}
    launches = {}
    for way, run in ways.items():
        before = ctx.launch_count()
        run()
        launches[way] = ctx.launch_count() - before
    out["launches"] = launches
    out["planes_identical"] = all(p is None or np.array_equal(p, q) for p, q in zip(plain_planes, light_planes))
    got = acc.as_dict()
    got.pop("reserved")
    out["accumulator"] = got
    dev = torch.from_numpy(rows.view(np.uint8)).cuda()
    planes = [None if s is None else torch.empty((s[0], s[1] * 2), dtype=torch.uint8, device="cuda") for s in abi.encode_plane_shapes(desc)]
    device_acc = torch.zeros(3, dtype=torch.int64, device="cuda")
    ctx.encode_device_light_level(desc, dev.data_ptr(), dev.stride(0), avifgpu.planes_from_tensors(planes), device_acc.data_ptr())
    raw = device_acc.cpu().numpy()
    out["accumulator_equals_device_call"] = got == {"max_code": int(raw.view(np.uint32)[0]), "level_sum": int(raw[1]), "pixels": int(raw[2])}
    out["max_cll_fall"] = avifgpu.content_light_level(acc, desc.image_bit_depth)
    return out


def main():
    ap = harness.arguments(rounds=5)
    ap.set_defaults(seconds=2.0)
    args = ap.parse_args()
    harness.require_gpu()
    pq = abi.Nclx(1, abi.PRIMARIES_BT2020, abi.TRANSFER_CHAR_PQ, abi.MATRIX_BT2020_NCL, 1)
    desc = abi.EncodeDesc(W, H, 32, 3, abi.ALPHA_NONE, 12, abi.TRANSFER_PQ, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420, nclx=pq)
    result = {"card": harness.card(), "unit": "milliseconds per 8K frame (host clock, median of rounds)", "frame": "7680x4320 RGB32f -> 12-bit PQ 4:2:0"}
    with avifgpu.Context(0) as tables, avifgpu.Context(0) as no_tables:
        no_tables.set_table_autobuild(-1)
        rows = tables.pinned_array((H, W * 3), np.float32)
        rows[:] = np.random.default_rng(20261019).random((H, W * 3), dtype=np.float32) * np.float32(1.05) - np.float32(0.02)
        result["table_valid"] = tables.prepare_encode(desc).as_dict()["valid"]
        result["tables"] = measure(tables, desc, rows, args.seconds, args.rounds)
        result["no_tables"] = measure(no_tables, desc, rows, args.seconds, args.rounds)
    harness.emit([result], args.out)


if __name__ == "__main__":
    main()
