#!/usr/bin/env python3
"""What measuring the content light level costs the sharded device-pointer encode on the 8K config-2 frame (7680 x 4320
RGB32f -> 12-bit PQ 4:2:0), rows resident on the members, planes on member 0:

  plain          avifgpu_encode_rows_sharded_device;
  light_level    avifgpu_encode_rows_sharded_device_light_level: on top of the light-level kernels, one memset, one
                 24-byte peer copy and an event per member, and a one-warp merge kernel on the owner.

A window is device time on the owner, from an event recorded before the window's first call to one recorded once
avifgpu_shard_group_synchronize has returned after its last; calls inside a window follow each other with no
synchronize.  Each window lasts at least `--seconds`, the two ways alternate for `--rounds` rounds and the median per
call is kept, with every round's value beside it.  In the same run: the light-level call's planes against the plain
call's, bit for bit; its accumulator against one avifgpu_encode_rows_device_light_level call over the whole frame on
device 0; the launches per member; and each member card's name, power limit and maximum SM clock.  The group of every
visible device is measured too when there are several; with one, the multi-member overhead is reported as not measured.

    python profiles/measure_sharded_device_light_level.py [--seconds 1.0] [--rounds 7] [--out sharded_light.json]
"""
import statistics

import harness
import numpy as np
import torch

import avifgpu
import bench
from avifgpu import abi
from harness import plane

W, H = 7680, 4320


def acc_dict(acc):
    raw = acc.cpu().numpy()
    return {"max_code": int(raw.view(np.uint32)[0]), "level_sum": int(raw[1]), "pixels": int(raw[2])}


def settle(devices):
    for device in devices:
        torch.cuda.synchronize(device)


class Sharded:
    """A prepared group with the frame's row blocks on their members and two sets of whole-image planes on member 0."""

    def __init__(self, devices, desc, values):
        self.devices, self.desc = devices, desc
        self.group = avifgpu.ShardGroup(devices)
        self.group.prepare_encode(desc)
        self.rows = []
        for member, (y0, count) in enumerate(avifgpu.shard_row_blocks(0, H, len(devices))):
            self.rows.append(values[y0:y0 + count].to(f"cuda:{devices[member]}").contiguous())
        self.pointers = [t.data_ptr() if t.shape[0] else None for t in self.rows]
        self.strides = [t.stride(0) * 4 for t in self.rows]
        shapes = abi.encode_plane_shapes(desc)
        self.plain_planes = [None if s is None else plane(s[0], s[1], True) for s in shapes]
        self.light_planes = [None if s is None else plane(s[0], s[1], True) for s in shapes]
        self.plain_struct = avifgpu.planes_from_tensors(self.plain_planes)
        self.light_struct = avifgpu.planes_from_tensors(self.light_planes)
        self.acc = torch.zeros(3, dtype=torch.int64, device="cuda")
        settle(devices)

    def plain(self):
        self.group.encode_device(self.desc, self.pointers, self.strides, self.plain_struct, owner=0)

    def light(self):
        self.group.encode_device_light_level(self.desc, self.pointers, self.strides, self.light_struct, self.acc.data_ptr(), owner=0)

    def launches(self):
        lib = self.group.lib
        return [int(lib.avifgpu_launch_count(lib.avifgpu_shard_group_context(self.group.handle, i))) for i in range(len(self.devices))]

    def window_ms(self, run, calls):
        """Device time on the owner per call, over `calls` back-to-back calls and the group's synchronize."""
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        settle(self.devices)
        start.record()
        for _ in range(calls):
            run()
        self.group.synchronize()
        end.record()
        torch.cuda.synchronize()
        return start.elapsed_time(end) / calls

    def checked(self):
        """One call of each way from a zeroed accumulator: (planes identical, accumulator, launches per member of each)."""
        self.acc.zero_()
        settle(self.devices)
        before = self.launches()
        self.plain()
        self.group.synchronize()
        middle = self.launches()
        self.light()
        self.group.synchronize()
        after = self.launches()
        identical = all(a is None or torch.equal(a, b) for a, b in zip(self.plain_planes, self.light_planes))
        return identical, acc_dict(self.acc), {"plain": [m - b for m, b in zip(middle, before)],
                                               "light_level": [a - m for a, m in zip(after, middle)]}

    def measure(self, seconds, rounds, reference):
        identical, acc, launches = self.checked()
        ways = {"plain": self.plain, "light_level": self.light}
        calls = {}
        for way, run in ways.items():
            run()
            calls[way] = max(20, int(seconds / (self.window_ms(run, 20) * 1e-3)) + 1)
        per_round = {way: [] for way in ways}
        for _ in range(rounds):
            for way, run in ways.items():
                per_round[way].append(self.window_ms(run, calls[way]) * 1e3)
        plain_us, light_us = statistics.median(per_round["plain"]), statistics.median(per_round["light_level"])
        return {
            "devices": self.devices,
            "cards": [bench.device_identity(torch, d) for d in self.devices],
            "plain_us": plain_us,
            "light_level_us": light_us,
            "overhead_us": light_us - plain_us,
            "overhead_relative": light_us / plain_us - 1.0,
            "rounds_us": per_round,
            "calls_per_window": calls,
            "planes_identical": identical,
            "accumulator": acc,
            "accumulator_identical_to_single_device": acc == reference,
            "launches": launches,
        }

    def close(self):
        self.group.close()


def single_device(desc, values):
    """The accumulator of one avifgpu_encode_rows_device_light_level call over the whole frame on device 0."""
    with avifgpu.Context(0) as ctx:
        ctx.prepare_encode(desc)
        planes = [None if s is None else plane(s[0], s[1], True) for s in abi.encode_plane_shapes(desc)]
        acc = torch.zeros(3, dtype=torch.int64, device="cuda")
        ctx.encode_device_light_level(desc, values.data_ptr(), values.stride(0) * 4, avifgpu.planes_from_tensors(planes), acc.data_ptr(), 0, H)
        torch.cuda.synchronize()
        return acc_dict(acc)


def main():
    args = harness.arguments(rounds=7).parse_args()
    harness.require_gpu()
    generator = torch.Generator(device="cuda")
    generator.manual_seed(20261019)
    pq = abi.Nclx(1, abi.PRIMARIES_BT2020, abi.TRANSFER_CHAR_PQ, abi.MATRIX_BT2020_NCL, 1)
    desc = abi.EncodeDesc(W, H, 32, 3, abi.ALPHA_NONE, 12, abi.TRANSFER_PQ, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420, nclx=pq)
    values = torch.rand((H, W * 3), generator=generator, device="cuda") * 1.05 - 0.02
    reference = single_device(desc, values)
    count = torch.cuda.device_count()
    result = {"workload": "7680x4320 RGB32f -> 12-bit PQ 4:2:0, rows resident on the members, planes on member 0",
              "unit": "microseconds per call (device time on the owner, median of rounds)",
              "single_device_accumulator": reference, "groups": []}
    for devices in [[0]] + ([list(range(count))] if count > 1 else []):
        sharded = Sharded(devices, desc, values)
        try:
            result["groups"].append(sharded.measure(args.seconds, args.rounds, reference))
        finally:
            sharded.close()
    if count == 1:
        result["multi_member_overhead"] = "not measured: one visible GPU"
    result["all_identical"] = all(g["planes_identical"] and g["accumulator_identical_to_single_device"] for g in result["groups"])
    harness.emit([result], args.out)


if __name__ == "__main__":
    main()
