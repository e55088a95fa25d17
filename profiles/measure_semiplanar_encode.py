#!/usr/bin/env python3
"""Device time of encodes into semi-planar and MSB-aligned planes (avifgpu_encode_desc.dest_layout) against the planar
encode of the same rows and against the planar encode followed by a torch interleave (and shift) into the same surfaces:

  p016_4k    3840 x 2160 RGB32f -> 12-bit PQ 4:2:0 in P016 (Cb / Cr pairs, codes in the top bits), one direct device call;
  p016_8k    7680 x 4320, the same;
  p010a_4k   3840 x 2160 RGBA16 -> 10-bit 4:2:0 in P010 + an MSB-aligned alpha plane, one direct device call;
  nv12_b64   64 x 512 x 512 RGB8 -> NV12 through the host-described and the device-described batch call;
  nv12_b256  the same with 256 images.

Each way is timed with CUDA events over at least `--seconds` of back-to-back calls on one stream, the ways alternating
for `--rounds` rounds, the median kept.  The semi-planar output and the interleaved planar output are compared bit for
bit.  Prints one JSON line with the card's name, power limit and maximum SM clock, read in the same run.

    python profiles/measure_semiplanar_encode.py [--seconds 1.0] [--rounds 5] [--out semiplanar_encode.json]
"""
import harness
import torch

import avifgpu
from avifgpu import abi
from harness import median_us, padded, plane

NV, NVMSB = abi.SOURCE_CHROMA_INTERLEAVED, abi.SOURCE_CHROMA_INTERLEAVED | abi.SOURCE_MSB_ALIGNED


class Frame:
    """One image's host rows, its planes in the semi-planar layout, the planar planes of the same description, and the
    semi-planar planes an interleave pass fills from those."""

    def __init__(self, desc, w, h, generator):
        d = self.desc = abi.EncodeDesc.from_buffer_copy(desc)
        d.width, d.height = w, h
        self.planar_desc = abi.EncodeDesc.from_buffer_copy(d)
        self.planar_desc.dest_layout = abi.SOURCE_PLANAR
        self.wide = d.image_bit_depth > 8
        self.shift = 16 - d.image_bit_depth if d.dest_layout & abi.SOURCE_MSB_ALIGNED else 0
        row_bytes = w * d.host_channels * d.host_depth // 8
        self.rows = torch.empty((h, padded(row_bytes)), dtype=torch.uint8, device="cuda")[:, :row_bytes]
        if d.host_depth == 32:
            values = torch.rand((h, w * d.host_channels), generator=generator, device="cuda") * 1.05 - 0.02
            self.rows.copy_(values.view(torch.uint8))
        else:
            top = 32768 if d.host_depth == 16 else 255
            values = torch.randint(0, top + 1, (h, w * d.host_channels), generator=generator, device="cuda", dtype=torch.int32)
            self.rows.copy_((values.to(torch.int16) if d.host_depth == 16 else values.to(torch.uint8)).view(torch.uint8))
        alloc = lambda shapes: [None if s is None else plane(s[0], s[1], self.wide) for s in shapes]  # noqa: E731
        self.semi = alloc(abi.encode_plane_shapes(d))
        self.planar = alloc(abi.encode_plane_shapes(self.planar_desc))
        self.relaid = alloc(abi.encode_plane_shapes(d))
        self.planes_semi = avifgpu.planes_from_tensors(self.semi)
        self.planes_planar = avifgpu.planes_from_tensors(self.planar)

    def interleave(self):
        """What a pipeline without this feature runs after the planar encode: pair Cb and Cr (and shift every plane)."""
        dtype = torch.int16 if self.wide else torch.uint8
        view = lambda t: t.view(dtype)  # noqa: E731
        moved = lambda t: view(t) << self.shift if self.shift else view(t)  # noqa: E731
        pairs = view(self.relaid[1])
        pairs[:, 0::2] = moved(self.planar[1])
        pairs[:, 1::2] = moved(self.planar[2])
        for k in (0, 3):
            if self.planar[k] is not None:
                view(self.relaid[k]).copy_(moved(self.planar[k]))

    def outputs(self, planes):
        return torch.cat([p.reshape(-1) for p in planes if p is not None]).clone()


def single(ctx, desc, w, h, seconds, rounds, generator):
    f = Frame(desc, w, h, generator)
    stats = ctx.prepare_encode(f.desc).as_dict()
    stride = f.rows.stride(0)
    semi = lambda: ctx.encode_device(f.desc, f.rows.data_ptr(), stride, f.planes_semi, 0, h)  # noqa: E731
    planar = lambda: ctx.encode_device(f.planar_desc, f.rows.data_ptr(), stride, f.planes_planar, 0, h)  # noqa: E731

    def planar_then_interleave():
        planar()
        f.interleave()

    semi()
    planar_then_interleave()
    torch.cuda.synchronize()
    before = ctx.launch_count()
    semi()
    torch.cuda.synchronize()
    launches = ctx.launch_count() - before  # one call, before the timing
    out = median_us({"semi_planar": semi, "planar": planar, "planar_then_interleave": planar_then_interleave}, seconds, rounds)
    out["semi_planar_launches"] = launches
    out["identical"] = torch.equal(f.outputs(f.semi), f.outputs(f.relaid))
    out["table_valid"] = stats["valid"]
    out["bytes_moved"] = f.rows.numel() + sum(p.numel() for p in f.semi if p is not None)
    out["semi_planar_gbs"] = out["bytes_moved"] / out["semi_planar"] / 1e3
    return out


def batches(ctx, desc, n, w, h, seconds, rounds, generator):
    frames = [Frame(desc, w, h, generator) for _ in range(n)]
    recs = lambda planes: avifgpu.batch_images_from_tensors([(w, h, f.rows, planes(f)) for f in frames])  # noqa: E731
    semi_recs, planar_recs = recs(lambda f: f.semi), recs(lambda f: f.planar)
    d_semi, d_planar = frames[0].desc, frames[0].planar_desc
    workspace = torch.empty(avifgpu.batch_workspace_bytes(n), dtype=torch.uint8, device="cuda")
    count = torch.full((1,), n, dtype=torch.int32, device="cuda")
    device_semi, device_planar = avifgpu.pack_batch_images(semi_recs), avifgpu.pack_batch_images(planar_recs)

    def host_planar_then_interleave():
        ctx.encode_batch_device(d_planar, planar_recs)
        for f in frames:
            f.interleave()

    def device_planar_then_interleave():
        ctx.encode_batch_indirect(d_planar, device_planar, count, n, workspace)
        for f in frames:
            f.interleave()

    ways = {
        "host_semi_planar": lambda: ctx.encode_batch_device(d_semi, semi_recs),
        "host_planar": lambda: ctx.encode_batch_device(d_planar, planar_recs),
        "host_planar_then_interleave": host_planar_then_interleave,
        "device_semi_planar": lambda: ctx.encode_batch_indirect(d_semi, device_semi, count, n, workspace),
        "device_planar": lambda: ctx.encode_batch_indirect(d_planar, device_planar, count, n, workspace),
        "device_planar_then_interleave": device_planar_then_interleave,
    }
    identical = True
    for semi_way, relaid_way in (("host_semi_planar", "host_planar_then_interleave"), ("device_semi_planar", "device_planar_then_interleave")):
        for f in frames:
            for p in f.semi + f.relaid:
                if p is not None:
                    p.zero_()
        ways[semi_way]()
        ways[relaid_way]()
        torch.cuda.synchronize()
        identical = identical and all(torch.equal(f.outputs(f.semi), f.outputs(f.relaid)) for f in frames)
    out = median_us(ways, seconds, rounds, n)
    out["identical"] = identical
    return out


def main():
    args = harness.arguments(rounds=5).parse_args()
    harness.require_gpu()
    generator = torch.Generator(device="cuda")
    generator.manual_seed(20261018)
    pq = abi.Nclx(1, abi.PRIMARIES_BT2020, abi.TRANSFER_CHAR_PQ, abi.MATRIX_BT2020_NCL, 1)
    bt709 = abi.Nclx(1, abi.PRIMARIES_BT709, abi.TRANSFER_CHAR_SRGB, abi.MATRIX_BT709, 1)
    planar = abi.LAYOUT_PLANAR_YCBCR
    p016 = abi.EncodeDesc(0, 0, 32, 3, abi.ALPHA_NONE, 12, abi.TRANSFER_PQ, 80, planar, abi.CHROMA_420, nclx=pq, dest_layout=NVMSB)
    p010a = abi.EncodeDesc(0, 0, 16, 4, abi.ALPHA_STRAIGHT, 10, abi.TRANSFER_CLIP, 80, planar, abi.CHROMA_420, nclx=pq, dest_layout=NVMSB)
    nv12 = abi.EncodeDesc(0, 0, 8, 3, abi.ALPHA_NONE, 8, abi.TRANSFER_CLIP, 80, planar, abi.CHROMA_420, nclx=bt709, dest_layout=NV)
    result = {"card": harness.card(), "unit": "microseconds per image (device events, median of rounds)"}
    with avifgpu.Context(0) as ctx:
        result["p016_4k"] = single(ctx, p016, 3840, 2160, args.seconds, args.rounds, generator)
        result["p016_8k"] = single(ctx, p016, 7680, 4320, args.seconds, args.rounds, generator)
        result["p010a_4k"] = single(ctx, p010a, 3840, 2160, args.seconds, args.rounds, generator)
        result["nv12_b64"] = batches(ctx, nv12, 64, 512, 512, args.seconds, args.rounds, generator)
        result["nv12_b256"] = batches(ctx, nv12, 256, 512, 512, args.seconds, args.rounds, generator)
    harness.emit([result], args.out)


if __name__ == "__main__":
    main()
