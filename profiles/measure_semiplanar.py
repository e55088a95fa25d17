#!/usr/bin/env python3
"""Device time of decodes from semi-planar and MSB-aligned sources (avifgpu_decode_desc.source_layout) against the planar
decode of the same bytes and against a torch de-interleave (and shift) followed by the planar decode:

  p010_8k    7680 x 4320 P010 (10-bit, Cb / Cr pairs, codes in the top bits) 4:2:0 -> RGB32f, PQ, one direct device call;
  nv12_8k    7680 x 4320 NV12 4:2:0 + an 8-bit alpha plane -> RGBA8, one direct device call;
  nv12_b64   64 x 512 x 512 NV12 + alpha -> RGBA8 through the host-described and the device-described batch call;
  nv12_b256  the same with 256 images.

Each way is timed with CUDA events over at least `--seconds` of back-to-back calls on one stream, the ways alternating
for `--rounds` rounds, the median kept.  The semi-planar and planar outputs are compared bit for bit.  Prints one JSON
line with the card's name, power limit and maximum SM clock, read in the same run.

    python profiles/measure_semiplanar.py [--seconds 1.0] [--rounds 5] [--out semiplanar.json]
"""
import harness
import torch

import avifgpu
from avifgpu import abi
from harness import median_us, padded, plane

NV, NVMSB = abi.SOURCE_CHROMA_INTERLEAVED, abi.SOURCE_CHROMA_INTERLEAVED | abi.SOURCE_MSB_ALIGNED


class Frame:
    """One image in its semi-planar source, its planar equivalent (same codes) and the planar buffers a de-interleave fills."""

    def __init__(self, desc, w, h, generator):
        d = self.desc = abi.DecodeDesc.from_buffer_copy(desc)
        d.width, d.height = w, h
        self.planar_desc = abi.DecodeDesc.from_buffer_copy(d)
        self.planar_desc.source_layout = abi.SOURCE_PLANAR
        wide = d.bit_depth > 8
        self.wide = wide
        self.shift = 16 - d.bit_depth if d.source_layout & abi.SOURCE_MSB_ALIGNED else 0
        shapes = abi.decode_plane_shapes(self.planar_desc)
        self.planar = []
        for shape in shapes:
            if shape is None:
                self.planar.append(None)
                continue
            p = plane(shape[0], shape[1], wide)
            codes = torch.randint(0, 1 << d.bit_depth, shape, generator=generator, device="cuda", dtype=torch.int32)
            p.copy_((codes.to(torch.int16) if wide else codes.to(torch.uint8)).view(torch.uint8))
            self.planar.append(p)
        dtype = torch.int16 if wide else torch.uint8
        view = lambda t: t.view(dtype)  # noqa: E731
        self.source = [None] * 4
        for k in (0, 3):
            if self.planar[k] is not None:
                s = plane(self.planar[k].shape[0], self.planar[k].shape[1] // (2 if wide else 1), wide)
                s.view(dtype).copy_(view(self.planar[k]) << self.shift if self.shift else view(self.planar[k]))
                self.source[k] = s
        cb, cr = view(self.planar[1]), view(self.planar[2])
        pairs = plane(cb.shape[0], 2 * cb.shape[1], wide)
        pv = pairs.view(dtype)
        pv[:, 0::2] = cb << self.shift if self.shift else cb
        pv[:, 1::2] = cr << self.shift if self.shift else cr
        self.source[1] = pairs
        self.scratch = [None if p is None else torch.empty_like(p) for p in self.planar]
        row_bytes = w * abi.decode_host_channels(d) * d.host_depth // 8
        self.rows = torch.empty((h, padded(row_bytes)), dtype=torch.uint8, device="cuda")[:, :row_bytes]
        self.planes_semi = avifgpu.planes_from_tensors(self.source)
        self.planes_planar = avifgpu.planes_from_tensors(self.planar)
        self.planes_scratch = avifgpu.planes_from_tensors(self.scratch)

    def deinterleave(self):
        """What a pipeline without this feature runs first: split the pairs (and shift every plane) into planar buffers."""
        dtype = torch.int16 if self.wide else torch.uint8
        pairs = self.source[1].view(dtype)
        cb, cr = self.scratch[1].view(dtype), self.scratch[2].view(dtype)
        if self.shift:
            # logical shift of 16-bit samples: the sign bit of int16 must not spread
            torch.bitwise_and(torch.bitwise_right_shift(pairs[:, 0::2], self.shift), (1 << (16 - self.shift)) - 1, out=cb)
            torch.bitwise_and(torch.bitwise_right_shift(pairs[:, 1::2], self.shift), (1 << (16 - self.shift)) - 1, out=cr)
            for k in (0, 3):
                if self.source[k] is not None:
                    torch.bitwise_and(torch.bitwise_right_shift(self.source[k].view(dtype), self.shift), (1 << (16 - self.shift)) - 1,
                                      out=self.scratch[k].view(dtype))
        else:
            cb.copy_(pairs[:, 0::2])
            cr.copy_(pairs[:, 1::2])
            for k in (0, 3):
                if self.source[k] is not None:
                    self.scratch[k].copy_(self.source[k])


def single(ctx, desc, w, h, seconds, rounds, generator):
    f = Frame(desc, w, h, generator)
    ctx.prepare_decode(f.desc)
    stride = f.rows.stride(0)
    semi = lambda: ctx.decode_device(f.desc, f.planes_semi, f.rows.data_ptr(), stride, 0, h)  # noqa: E731
    planar = lambda: ctx.decode_device(f.planar_desc, f.planes_planar, f.rows.data_ptr(), stride, 0, h)  # noqa: E731

    def split_then_planar():
        f.deinterleave()
        ctx.decode_device(f.planar_desc, f.planes_scratch, f.rows.data_ptr(), stride, 0, h)

    semi()
    a = f.rows.clone()
    planar()
    b = f.rows.clone()
    split_then_planar()
    c = f.rows.clone()
    out = median_us({"semi_planar": semi, "planar": planar, "deinterleave_then_planar": split_then_planar}, seconds, rounds)
    out["identical"] = torch.equal(a, b) and torch.equal(a, c)
    source_bytes = sum(p.numel() for p in f.source if p is not None)
    out["bytes_moved"] = source_bytes + f.rows.numel()
    out["semi_planar_gbs"] = out["bytes_moved"] / out["semi_planar"] / 1e3
    return out


def batches(ctx, desc, n, w, h, seconds, rounds, generator):
    frames = [Frame(desc, w, h, generator) for _ in range(n)]
    ctx.prepare_decode(frames[0].desc)
    recs = lambda planes: avifgpu.batch_images_from_tensors([(w, h, f.rows, planes(f)) for f in frames])  # noqa: E731
    semi_recs, planar_recs, scratch_recs = recs(lambda f: f.source), recs(lambda f: f.planar), recs(lambda f: f.scratch)
    d_semi, d_planar = frames[0].desc, frames[0].planar_desc
    workspace = torch.empty(avifgpu.batch_workspace_bytes(n), dtype=torch.uint8, device="cuda")
    count = torch.full((1,), n, dtype=torch.int32, device="cuda")
    device_semi, device_planar = avifgpu.pack_batch_images(semi_recs), avifgpu.pack_batch_images(planar_recs)
    ways = {
        "host_semi_planar": lambda: ctx.decode_batch_device(d_semi, semi_recs),
        "host_planar": lambda: ctx.decode_batch_device(d_planar, planar_recs),
        "device_semi_planar": lambda: ctx.decode_batch_indirect(d_semi, device_semi, count, n, workspace),
        "device_planar": lambda: ctx.decode_batch_indirect(d_planar, device_planar, count, n, workspace),
    }

    def split_then_host():
        for f in frames:
            f.deinterleave()
        ctx.decode_batch_device(d_planar, scratch_recs)

    ways["deinterleave_then_host_planar"] = split_then_host
    outputs = {}
    for name, run in ways.items():
        run()
        torch.cuda.synchronize()
        outputs[name] = torch.cat([f.rows.reshape(-1) for f in frames]).clone()
    out = median_us(ways, seconds, rounds, n)
    first = next(iter(outputs.values()))
    out["identical"] = all(torch.equal(first, o) for o in outputs.values())
    return out


def main():
    args = harness.arguments(rounds=5).parse_args()
    harness.require_gpu()
    generator = torch.Generator(device="cuda")
    generator.manual_seed(20261016)
    pq = abi.Nclx(1, abi.PRIMARIES_BT2020, abi.TRANSFER_CHAR_PQ, abi.MATRIX_BT2020_NCL, 0)
    bt709 = abi.Nclx(1, abi.PRIMARIES_BT709, abi.TRANSFER_CHAR_SRGB, abi.MATRIX_BT709, 0)
    p010 = abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, abi.CHROMA_420, 10, abi.ALPHA_NONE, 32, pq, pq_peak_nits=1000, source_layout=NVMSB)
    nv12 = abi.DecodeDesc(0, 0, abi.COLORSPACE_YCBCR, abi.CHROMA_420, 8, abi.ALPHA_STRAIGHT, 8, bt709, source_layout=NV)
    result = {"card": harness.card(), "unit": "microseconds per image (device events, median of rounds)"}
    with avifgpu.Context(0) as ctx:
        result["p010_8k"] = single(ctx, p010, 7680, 4320, args.seconds, args.rounds, generator)
        result["nv12_8k"] = single(ctx, nv12, 7680, 4320, args.seconds, args.rounds, generator)
        result["nv12_b64"] = batches(ctx, nv12, 64, 512, 512, args.seconds, args.rounds, generator)
        result["nv12_b256"] = batches(ctx, nv12, 256, 512, 512, args.seconds, args.rounds, generator)
    harness.emit([result], args.out)


if __name__ == "__main__":
    main()
