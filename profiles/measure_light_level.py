#!/usr/bin/env python3
"""Device time of the content light level measured inside the encode (avifgpu_encode_rows_device_light_level) on the 8K
config-2 frame (7680 x 4320 RGB32f -> 12-bit PQ 4:2:0), into planar planes and into P016, three ways each:

  plain          avifgpu_encode_rows_device;
  light_level    avifgpu_encode_rows_device_light_level into a device accumulator (a memset of it first);
  plain_then_torch
                 the plain call, then a torch pass over the RGB32f frame computing the same statistic: PQ codes by torch's
                 float32 pow, max(R', G', B') per pixel, the level table gathered and summed.

Each way is timed with CUDA events over at least `--seconds` of back-to-back calls on one stream, the ways alternating
for `--rounds` rounds, the median kept.  The light-level call's planes are compared bit for bit with the plain call's,
its launches counted, and its accumulators of the planar and P016 encodes compared with each other.  The torch pass
evaluates the curve with torch's pow, not glibc's powf, so its accumulator may miss the encode's by a code on rare
samples; how far it is off is reported.  Prints one JSON line with the card's name, power limit and maximum SM clock,
read in the same run.

    python profiles/measure_light_level.py [--seconds 1.0] [--rounds 5] [--out light_level.json]
"""
import harness
import numpy as np
import torch

import avifgpu
from avifgpu import abi
from harness import median_us, padded, plane

NVMSB = abi.SOURCE_CHROMA_INTERLEAVED | abi.SOURCE_MSB_ALIGNED
W, H = 7680, 4320


def level_table(depth):
    """level(k) of every code (DESIGN.md section 5), from the library's PQToLinear primitive at peak 10000 (multiplier 1)."""
    with avifgpu.Context(0) as ctx:
        top = (1 << depth) - 1
        linear = ctx.transfer(abi.FN_PQ_TO_LINEAR, np.arange(top + 1, dtype=np.float32) / np.float32(top), 10000.0)
    return torch.from_numpy((linear.astype(np.float32) * np.float32(1 << 22)).astype(np.int64)).cuda()


class Frame:
    def __init__(self, desc, rows):
        self.desc = desc
        wide = True
        self.planes = [None if s is None else plane(s[0], s[1], wide) for s in abi.encode_plane_shapes(desc)]
        self.light_planes = [None if s is None else plane(s[0], s[1], wide) for s in abi.encode_plane_shapes(desc)]
        self.struct = avifgpu.planes_from_tensors(self.planes)
        self.light_struct = avifgpu.planes_from_tensors(self.light_planes)
        self.rows = rows
        self.acc = torch.zeros(3, dtype=torch.int64, device="cuda")

    def outputs(self, planes):
        return torch.cat([p.reshape(-1) for p in planes if p is not None])


def torch_statistic(values, levels, peak, max_code):
    """The statistic by torch: LinearToPQ's formula in float32, quantised as the encode does (trunc(clamp(c * max)))."""
    m1, m2 = 2610.0 / 16384.0, 2523.0 / 4096.0 * 128.0
    c1, c2, c3 = 3424.0 / 4096.0, 2413.0 / 4096.0 * 32.0, 2392.0 / 4096.0 * 32.0
    v = torch.clamp(values, min=0.0) * (peak / 10000.0)
    x = torch.pow(v, m1)
    pq = torch.pow((c1 + c2 * x) / (1.0 + c3 * x), m2)
    codes = torch.clamp(pq * max_code, 0.0, float(max_code)).to(torch.int64)
    k = codes.view(values.shape[0], -1, 3).amax(dim=2)
    return k.max(), levels[k].sum(), k.numel()


def measure(ctx, desc, rows, stride, values, levels, seconds, rounds):
    f = Frame(desc, rows)
    stats = ctx.prepare_encode(desc).as_dict()
    plain = lambda: ctx.encode_device(desc, rows.data_ptr(), stride, f.struct, 0, H)  # noqa: E731

    def light():
        f.acc.zero_()
        ctx.encode_device_light_level(desc, rows.data_ptr(), stride, f.light_struct, f.acc.data_ptr(), 0, H)

    result = {}

    def plain_then_torch():
        plain()
        result["torch"] = torch_statistic(values, levels, desc.pq_peak_nits, (1 << desc.image_bit_depth) - 1)

    plain()
    light()
    torch.cuda.synchronize()
    before = ctx.launch_count()
    plain()
    torch.cuda.synchronize()
    plain_launches = ctx.launch_count() - before
    before = ctx.launch_count()
    light()
    torch.cuda.synchronize()
    light_launches = ctx.launch_count() - before
    out = median_us({"plain": plain, "light_level": light, "plain_then_torch": plain_then_torch}, seconds, rounds)
    out["ratio_light_to_plain"] = out["light_level"] / out["plain"]
    out["launches"] = {"plain": plain_launches, "light_level": light_launches}
    out["planes_identical"] = torch.equal(f.outputs(f.planes), f.outputs(f.light_planes))
    out["table_valid"] = stats["valid"]
    acc = f.acc.cpu().numpy()
    out["accumulator"] = {"max_code": int(acc.view(np.uint32)[0]), "level_sum": int(acc[1]), "pixels": int(acc[2])}
    out["max_cll_fall"] = avifgpu.content_light_level(out["accumulator"], desc.image_bit_depth)
    k_max, level_sum, pixels = result["torch"]
    torch_acc = {"max_code": int(k_max), "level_sum": int(level_sum), "pixels": int(pixels)}
    out["torch_accumulator"] = torch_acc
    out["torch_identical"] = torch_acc == out["accumulator"]
    out["torch_level_sum_relative_error"] = abs(torch_acc["level_sum"] - out["accumulator"]["level_sum"]) / max(1, out["accumulator"]["level_sum"])
    return out


def main():
    args = harness.arguments(rounds=5).parse_args()
    harness.require_gpu()
    generator = torch.Generator(device="cuda")
    generator.manual_seed(20261018)
    pq = abi.Nclx(1, abi.PRIMARIES_BT2020, abi.TRANSFER_CHAR_PQ, abi.MATRIX_BT2020_NCL, 1)
    planar = abi.EncodeDesc(W, H, 32, 3, abi.ALPHA_NONE, 12, abi.TRANSFER_PQ, 80, abi.LAYOUT_PLANAR_YCBCR, abi.CHROMA_420, nclx=pq)
    p016 = abi.EncodeDesc.from_buffer_copy(planar)
    p016.dest_layout = NVMSB
    row_bytes = W * 12
    rows = torch.empty((H, padded(row_bytes)), dtype=torch.uint8, device="cuda")[:, :row_bytes]
    values = torch.rand((H, W * 3), generator=generator, device="cuda") * 1.05 - 0.02
    rows.copy_(values.view(torch.uint8))
    levels = level_table(12)
    result = {"card": harness.card(), "unit": "microseconds per frame (device events, median of rounds)"}
    with avifgpu.Context(0) as ctx:
        result["planar_8k"] = measure(ctx, planar, rows, rows.stride(0), values, levels, args.seconds, args.rounds)
        result["p016_8k"] = measure(ctx, p016, rows, rows.stride(0), values, levels, args.seconds, args.rounds)
    result["accumulators_identical"] = result["planar_8k"]["accumulator"] == result["p016_8k"]["accumulator"]
    harness.emit([result], args.out)


if __name__ == "__main__":
    main()
