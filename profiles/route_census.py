"""Route census: which kernels every direct device call launches, for a grid of descriptions, context states and blocks.

For each encode (avifgpu_encode_rows_device) and decode (avifgpu_decode_rows_device) description of the grid below that
the library accepts, in a fresh context and in one whose tables and verified shortcuts were prepared first, and for a few
blocks of a 130 x 6 image (aligned; rows misaligned by 4 bytes; plane 0 misaligned by 2 bytes; an odd first row), it
records the call's status, the CUDA kernels it ran in order (torch.profiler), the library's launch count and a hash of
the bytes it wrote; a refused description is one record of its status.  Two libraries that route alike give identical records:

    AVIFGPU_LIBRARY=old/libavifgpu.so python profiles/route_census.py --out old1.json   (twice: old1, old2)
    python profiles/route_census.py --out new1.json                                     (twice: new1, new2)
    python profiles/route_census.py --compare old1.json,old2.json new1.json,new2.json

torch.profiler now and then loses every kernel record of a short session, so each library is recorded twice and a call's
kernels are those of the run that captured them.

The inputs are seeded: float hosts get values in [-0.1, 1.2], 16-bit hosts values in [0, 32768], planes codes of their
depth (MSB-aligned where the layout says so)."""
import argparse
import hashlib
import itertools
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "avif-format_b200", "python"))

WIDTH, HEIGHT = 130, 6
ROW_BYTES, PLANE_BYTES, SLACK = 4096, 2048, 256  # strides generous for every layout, and room for the offsets


def nclx(abi, primaries, transfer, matrix, full=1):
    return abi.Nclx(1, primaries, transfer, matrix, full)


def encode_grid(abi):
    for host, channels, alpha, depth in itertools.product((8, 16, 32), (1, 2, 3, 4), (0, 1, 2), (8, 10, 12)):
        transfers = (abi.TRANSFER_PQ, abi.TRANSFER_SMPTE428, abi.TRANSFER_CLIP, abi.TRANSFER_HLG) if host == 32 else (abi.TRANSFER_CLIP,)
        for transfer, layout in itertools.product(transfers, (abi.LAYOUT_REFERENCE, abi.LAYOUT_PLANAR_YCBCR)):
            chromas = (abi.CHROMA_420, abi.CHROMA_444) if layout == abi.LAYOUT_PLANAR_YCBCR else (abi.CHROMA_444,)
            dests = (0, 1, 3) if layout == abi.LAYOUT_PLANAR_YCBCR else (0,)
            for chroma, dest in itertools.product(chromas, dests):
                for gray16 in ((0, 1) if host == 16 and channels == 1 else (0,)):
                    hlg = 1 if transfer == abi.TRANSFER_HLG else 0
                    yield abi.EncodeDesc(WIDTH, HEIGHT, host, channels, alpha, depth, transfer, 1000, layout, chroma, 0, gray16,
                                         nclx(abi, 9, 16, 9), hlg, dest_layout=dest)


def decode_grid(abi):
    curves = ((9, 16, 9), (9, 18, 9), (1, 17, 1), (1, 1, 1))
    for host, colorspace, depth, alpha in itertools.product((8, 16, 32), (0, 1, 2), (8, 10, 12, 16), (0, 1, 2)):
        chromas = (abi.CHROMA_420, abi.CHROMA_444) if colorspace == abi.COLORSPACE_YCBCR else (abi.CHROMA_444,)
        sources = (0, 1, 3) if colorspace == abi.COLORSPACE_YCBCR else (0,)
        for chroma, source, curve in itertools.product(chromas, sources, curves if host == 32 else curves[:1]):
            yield abi.DecodeDesc(WIDTH, HEIGHT, colorspace, chroma, depth, alpha, host, nclx(abi, *curve), 1, 1.2, 1000, 1000, source)


BLOCKS = {"aligned": (0, HEIGHT, 0, 0), "rows+4": (0, HEIGHT, 4, 0), "plane0+2": (0, HEIGHT, 0, 2), "odd-first-row": (1, HEIGHT - 1, 0, 0)}


def describe(desc):
    fields = [f"{n}={getattr(desc, n)}" for n, _ in desc._fields_ if n not in ("nclx", "row_matrix", "struct_size")]
    return ",".join(fields + [f"nclx.{n}={getattr(desc.nclx, n)}" for n, _ in desc.nclx._fields_])


def host_values(torch, g, host, count):
    if host == 32:
        return (torch.rand(count, generator=g, device="cuda") * 1.3 - 0.1).view(torch.uint8)
    if host == 16:
        return torch.randint(0, 32769, (count,), generator=g, device="cuda", dtype=torch.int32).to(torch.int16).view(torch.uint8)
    return torch.randint(0, 256, (count,), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)


def plane_codes(torch, g, depth, msb, count):
    if depth == 8:
        return torch.randint(0, 256, (count,), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
    codes = torch.randint(0, 1 << depth, (count,), generator=g, device="cuda", dtype=torch.int32)
    return (codes << (16 - depth) if msb else codes).to(torch.int16).view(torch.uint8)


def census(args):
    import torch
    from torch.profiler import ProfilerActivity, profile

    import avifgpu
    from avifgpu import abi

    g = torch.Generator(device="cuda")
    records = []

    def run(kind, key, ctx, call, outputs):
        before = ctx.launch_count()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            try:
                call()
                status = "ok"
            except Exception as error:  # the library's status, recorded as it is
                status = str(error)
            torch.cuda.synchronize()
        kernels = [e.name for e in sorted(prof.events(), key=lambda e: e.time_range.start) if e.device_type == torch.autograd.DeviceType.CUDA]
        digest = hashlib.sha256(b"".join(t.cpu().numpy().tobytes() for t in outputs)).hexdigest()[:16]
        records.append({"kind": kind, "call": key, "status": status, "kernels": kernels, "launches": ctx.launch_count() - before,
                        "output": digest})

    kinds = ("encode", "decode") if args.kind == "both" else (args.kind,)
    probe = avifgpu.Context(0)  # tells accepted descriptions from refused ones; its own first-use state is not recorded
    for kind in kinds:
        for index, desc in enumerate(encode_grid(abi) if kind == "encode" else decode_grid(abi)):
            probeRows = torch.zeros(HEIGHT * ROW_BYTES, dtype=torch.uint8, device="cuda")
            scratch = [torch.zeros(HEIGHT * PLANE_BYTES, dtype=torch.uint8, device="cuda") for _ in range(4)]
            try:
                if kind == "encode":
                    probe.encode_device(desc, probeRows.data_ptr(), ROW_BYTES, avifgpu.planes_from_tensors([t.view(HEIGHT, -1) for t in scratch]))
                else:
                    probe.decode_device(desc, avifgpu.planes_from_tensors([t.view(HEIGHT, -1) for t in scratch]), probeRows.data_ptr(), ROW_BYTES)
                torch.cuda.synchronize()
            except Exception as error:
                records.append({"kind": kind, "call": f"refused:{describe(desc)}", "status": str(error)})
                continue
            depth = desc.image_bit_depth if kind == "encode" else desc.bit_depth
            msb = kind == "decode" and (desc.source_layout & abi.SOURCE_MSB_ALIGNED) != 0
            hostBytes = 4 if desc.host_depth == 32 else 2 if desc.host_depth == 16 else 1
            for state in ("fresh", "prepared"):
                with avifgpu.Context(0) as ctx:
                    if state == "prepared":
                        try:
                            (ctx.prepare_encode if kind == "encode" else ctx.prepare_decode)(desc)
                        except Exception:
                            pass
                        torch.cuda.synchronize()
                    for block, (y0, rows, rowOffset, planeOffset) in BLOCKS.items():
                        g.manual_seed(index * 7919 + 17)
                        zeros = torch.zeros(SLACK, dtype=torch.uint8, device="cuda")
                        host = torch.cat([host_values(torch, g, desc.host_depth, HEIGHT * ROW_BYTES // hostBytes), zeros])
                        planes = [torch.cat([plane_codes(torch, g, depth, msb, HEIGHT * PLANE_BYTES // (1 if depth == 8 else 2)), zeros]) for _ in range(4)]
                        for t in (planes if kind == "encode" else [host]):
                            t.zero_()  # the destination
                        struct = abi.Planes()
                        for k, p in enumerate(planes):
                            struct.data[k] = p.data_ptr() + (planeOffset if k == 0 else 0)
                            struct.stride[k] = PLANE_BYTES
                        rowsPtr = host.data_ptr() + rowOffset
                        key = f"{state}:{block}:{describe(desc)}"
                        if kind == "encode":
                            run(kind, key, ctx, lambda: ctx.encode_device(desc, rowsPtr, ROW_BYTES, struct, y0, rows), planes)
                        else:
                            run(kind, key, ctx, lambda: ctx.decode_device(desc, struct, rowsPtr, ROW_BYTES, y0, rows), [host])
    with open(args.out, "w") as f:
        json.dump(records, f)
    generic = ("EncodeReferenceLayoutKernel<", "EncodePlanarKernel<", "::DecodeKernel<")
    tuned = sum(1 for r in records if any("Kernel" in k and not any(n in k for n in generic) for k in r.get("kernels", [])))
    refused = sum(r["call"].startswith("refused:") for r in records)
    print(f"route census: {len(records) - refused} calls, {tuned} with a tuned kernel, {refused} descriptions refused -> {args.out}")


def merged(paths):
    """One library's records from several runs: torch.profiler now and then loses the kernel records of a short session
    (never a part of them), so a call's kernels are those of a run that captured any; everything else must agree."""
    runs = [json.load(open(p)) for p in paths]
    out = []
    for records in zip(*runs):
        base = dict(records[0])
        for r in records[1:]:
            if {k: v for k, v in r.items() if k != "kernels"} != {k: v for k, v in base.items() if k != "kernels"}:
                raise SystemExit(f"runs of one library disagree: {json.dumps(r)[:300]}")
            captured = [x.get("kernels") for x in (base, r) if x.get("kernels")]
            if len({tuple(k) for k in captured}) > 1:
                raise SystemExit(f"runs of one library launched different kernels: {json.dumps(r)[:300]}")
            base["kernels"] = captured[0] if captured else base.get("kernels")
        out.append(base)
    return out


def compare(a_paths, b_paths):
    a, b = merged(a_paths.split(",")), merged(b_paths.split(","))
    if len(a) != len(b):
        print(f"different call counts: {len(a)} vs {len(b)}")
        return 1
    differ = [(x, y) for x, y in zip(a, b) if x != y]
    for x, y in differ[:10]:
        print("differ:", json.dumps(x)[:400], "\n    vs:", json.dumps(y)[:400])
    lost = sum(1 for r in a + b if r.get("launches") and not r.get("kernels"))
    print(f"{len(a)} calls compared, {len(differ)} differ, {lost} records whose kernels no run captured")
    return 1 if differ else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--kind", choices=("encode", "decode", "both"), default="both")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"), help="comma-separated runs of each library")
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    if not args.out:
        ap.error("--out is required")
    census(args)


if __name__ == "__main__":
    main()
