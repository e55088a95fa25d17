// kernel_params.h -- plain parameter blocks handed to the CUDA kernels (device pointers, block-relative).
//
// "Block" = the row block [y0, y0 + rows) one launch converts.  All pointers already point at the first row of
// the block in their buffer (for sub-sampled chroma planes: at chroma row y0 >> ys), so kernels index rows from
// zero and never see y0 -- except `yPhase`, the parity of y0 for 4:2:0 decode, where an odd first row shares its
// chroma row with the row above it (ReadHeifImage.cpp:359 uvJ = y >> yChromaShift).
#ifndef AVIF_KERNEL_PARAMS_H
#define AVIF_KERNEL_PARAMS_H

#include <stddef.h>
#include <stdint.h>

#include <atomic>
#include <vector>

#include <driver_types.h>

#include "../../include/avifgpu.h"
#include "curve_tables.h"
#include "light_level.cuh"
#include "pixel_math.cuh"

// The routing and window arithmetic below is plain C++ that the plan kernel of the device-described batch
// (kernels_batch.cu) runs on the device too; the attribute is empty for the host compiler (host_params.cpp,
// tests/native).
#if defined(__CUDACC__)
#define AVIFGPU_HD __host__ __device__
#else
#define AVIFGPU_HD
#endif

namespace avifgpu
{

#if defined(__CUDACC__)
// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device setting; `configuredDevices` (one static per kernel
// instantiation) remembers the devices it has been made on, so a process that drives several GPUs configures each.
// It enqueues nothing, so a first launch inside a CUDA graph capture may make it (as may the table decode's occupancy
// query): tests/test_gpu_graph_capture.py captures every tuned kernel's first launch in a fresh process.
template <typename Kernel>
inline cudaError_t AllowDynamicShared(Kernel kernel, int bytes, std::atomic<uint64_t>& configuredDevices)
{
    int device = 0;
    cudaError_t e = cudaGetDevice(&device);
    if (e != cudaSuccess)
    {
        return e;
    }
    const uint64_t bit = 1ull << (device & 63);
    if (configuredDevices.load(std::memory_order_acquire) & bit)
    {
        return cudaSuccess;
    }
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess)
    {
        configuredDevices.fetch_or(bit, std::memory_order_release);
    }
    return e;
}

// One exhaustive device check of an arithmetic shortcut: `launch(counter, stream)` enqueues the kernel that adds its
// disagreements to the cleared device counter.  Returns their number (0 = verified) or -1 on a CUDA error.  Synchronous.
template <typename Launch>
inline long long CountDisagreements(cudaStream_t stream, Launch&& launch)
{
    unsigned long long* counter = nullptr;
    if (cudaMalloc(&counter, sizeof(unsigned long long)) != cudaSuccess)
    {
        return -1;
    }
    cudaMemsetAsync(counter, 0, sizeof(unsigned long long), stream);
    launch(counter, stream);
    unsigned long long bad = 0;
    const bool ok = cudaMemcpyAsync(&bad, counter, sizeof(bad), cudaMemcpyDeviceToHost, stream) == cudaSuccess &&
                    cudaStreamSynchronize(stream) == cudaSuccess;
    cudaFree(counter);
    return ok ? static_cast<long long>(bad) : -1;
}
#endif

struct EncodeParams
{
    const void* rows;      // interleaved host pixels (formatRecord->data layout), device memory
    int64_t rowStride;     // bytes
    void* plane[4];        // REFERENCE layout: [0] interleaved or Y, [3] alpha (gray); PLANAR: Y, Cb, Cr, A
    int64_t planeStride[4];
    int32_t width;
    int32_t rowCount;      // rows in this block
    int32_t channels;      // 1..4
    int32_t hasAlpha;
    int32_t premultiply;
    int32_t imageDepth;    // 8, 10, 12
    uint32_t maxCode;
    float maxCodeFloat;
    int32_t transfer;      // avifgpu_transfer (float hosts)
    float pqMultiplier;    // peak / 10000.0f
    int32_t gray16Smpte428;
    int32_t planar;        // AVIFGPU_LAYOUT_PLANAR_YCBCR
    int32_t xs, ys;        // chroma shifts
    int32_t topLeft;       // AVIFGPU_DOWN_FILTER_TOP_LEFT
    avifpix::ForwardMatrix matrix;
    float chromaOffset;
    int32_t hlgInverseOotf; // AVIFGPU_HLG_INVERSE_OOTF_THEN_OETF: ApplyInverseHLGOOTF on the pixel before LinearToHLG
    float hlgLuma[3];
    float hlgDisplayGamma;
    float hlgPeak;
    int32_t rowMatrixEnabled; // avifgpu_encode_desc.row_matrix: the colour-profile 3x3 ahead of everything else (float colour hosts)
    float rowMatrix[9];
    // Float hosts with a transfer curve: the compact step table + band bitmap in global memory (a by-value copy of
    // *curveTable made by the generic launcher), or useCurveView = 0 -> every sample takes the exact powf.
    CurveTableView curveView;
    int32_t useCurveView;
    // Host-side extras for the launcher (ignored by the kernels):
    const CurveTableView* curveTable; // verified exact step table for `transfer`, or nullptr
    const uint16_t* gray16Lut;        // 65536-entry code table for Gray16 hosts (device memory), or nullptr
    int32_t smCount;
    int32_t verifiedPremultiply;      // 1 once the context has verified FastPremultiplyBiased for this image depth on this device
    int32_t destLayout;               // avifgpu_source_layout bits of the planes written (planar YCbCr only): Cb, Cr pairs in plane 1; codes in the top bits
};

struct DecodeParams
{
    const void* plane[4];  // YCbCr: Y, Cb, Cr, A; mono: Y, -, -, A; planar RGB: R, G, B, A
    int64_t planeStride[4];
    void* rows;            // interleaved host pixels, device memory
    int64_t rowStride;
    int32_t width;
    int32_t rowCount;
    int32_t yPhase;        // y0 & ys
    int32_t colorspace;    // avifgpu_colorspace
    int32_t xs, ys;
    int32_t hasAlpha;
    int32_t premultiplied;
    int32_t bitDepth;
    uint32_t maxCode;
    avifpix::RangeParams range;
    avifpix::InverseMatrix matrix;
    int32_t hostDepth;     // 8, 16, 32
    int32_t transfer;      // avifgpu_transfer (host depth 32)
    float pqMultiplier;    // 10000.0f / peak
    int32_t applyOotf;
    float lumaR, lumaG, lumaB;
    float gammaMinusOne;
    float hlgPeak;
    int32_t smCount;              // host-side extra for the launcher
    int32_t verifiedHlgDivisions; // 1 once the context has verified HLGToLinearUnit's fast divisions on this device
    int32_t verifiedGreenDivision; // 1 once the context has verified the fast `/ kg` of YuvDecode.cpp:308 for this matrix, depth, range
    int32_t verifiedPqRatio;       // 1 once the context has verified the branch-free division inside PQToLinear on this device
    int32_t sourceLayout;          // avifgpu_source_layout bits (YCbCr only): Cb, Cr pairs in plane 1; codes in the top bits
};

// The source layout of a decode or the destination layout of an encode, as the tuned kernels take it: a template argument
// (SOURCE, DEST) whose bits are these, 0 being libheif's planar, low-bit layout.
AVIFGPU_HD constexpr bool SourceInterleaved(int source) { return (source & AVIFGPU_SOURCE_CHROMA_INTERLEAVED) != 0; }
AVIFGPU_HD constexpr bool SourceMsbAligned(int source) { return (source & AVIFGPU_SOURCE_MSB_ALIGNED) != 0; }

// The block restricted to its sub-rectangle [x0, x0 + width) x [y0, y0 + rows), for the edge strips the tuned
// launchers leave to the generic kernel.  Plane k moves by (y0 >> ys_k) rows and (x0 >> xs_k) sites of
// samplesPerPixel_k samples, as EncodePlaneGeometry / DecodePlaneGeometry lay the planes out: only planes 1 and 2 are
// sub-sampled (FillEncodeParams / FillDecodeParams leave xs = ys = 0 for every other layout), and only plane 0 of the
// reference layout with three or more channels interleaves `channels` samples per pixel.  A null plane stays null.
// Blocks carry no column phase, so x0 starts a chroma site (a multiple of 1 << xs); an encode block has no row phase
// either, so y0 is a multiple of 1 << ys (tests/native/launch_window_check.cpp).  Interleaved chroma (plane 1 only) moves
// by two samples per site.
AVIFGPU_HD inline EncodeParams EncodeWindow(const EncodeParams& p, int hostDepth, int x0, int y0, int width, int rows)
{
    EncodeParams w = p;
    w.rows = static_cast<const uint8_t*>(p.rows) + static_cast<int64_t>(y0) * p.rowStride + static_cast<int64_t>(x0) * p.channels * (hostDepth / 8);
    const int sampleBytes = p.imageDepth > 8 ? 2 : 1;
    for (int k = 0; k < 4; ++k)
    {
        if (p.plane[k] == nullptr)
        {
            continue;
        }
        const bool chroma = k == 1 || k == 2;
        const int samplesPerPixel = (!p.planar && k == 0 && p.channels >= 3) ? p.channels : (k == 1 && SourceInterleaved(p.destLayout)) ? 2 : 1;
        w.plane[k] = static_cast<uint8_t*>(p.plane[k]) + static_cast<int64_t>(y0 >> (chroma ? p.ys : 0)) * p.planeStride[k] +
                     static_cast<int64_t>(x0 >> (chroma ? p.xs : 0)) * samplesPerPixel * sampleBytes;
    }
    w.width = width;
    w.rowCount = rows;
    return w;
}

// The same for a decode block, whose first row may be the second of a 4:2:0 row pair (yPhase = 1): the chroma planes
// move by the chroma rows between the two first rows, and the window's phase is that of its own first row, so y0 may
// be odd.  Interleaved chroma (plane 1 only) moves by two samples per site.
AVIFGPU_HD inline DecodeParams DecodeWindow(const DecodeParams& p, int x0, int y0, int width, int rows)
{
    DecodeParams w = p;
    const int channels = (p.colorspace == AVIFGPU_COLORSPACE_MONOCHROME ? 1 : 3) + (p.hasAlpha ? 1 : 0);
    w.rows = static_cast<uint8_t*>(p.rows) + static_cast<int64_t>(y0) * p.rowStride + static_cast<int64_t>(x0) * channels * (p.hostDepth / 8);
    const int sampleBytes = p.bitDepth > 8 ? 2 : 1;
    for (int k = 0; k < 4; ++k)
    {
        if (p.plane[k] == nullptr)
        {
            continue;
        }
        const bool chroma = k == 1 || k == 2;
        const int planeRows = chroma ? (p.yPhase + y0) >> p.ys : y0;
        const int samplesPerSite = (k == 1 && SourceInterleaved(p.sourceLayout)) ? 2 : 1;
        w.plane[k] = static_cast<const uint8_t*>(p.plane[k]) + static_cast<int64_t>(planeRows) * p.planeStride[k] +
                     static_cast<int64_t>(x0 >> (chroma ? p.xs : 0)) * samplesPerSite * sampleBytes;
    }
    w.width = width;
    w.rowCount = rows;
    w.yPhase = (p.yPhase + y0) & p.ys;
    return w;
}

// True when `p` and every row `stride` bytes after it start on an `alignment`-byte boundary.
AVIFGPU_HD inline bool Aligned(const void* p, int64_t stride, int alignment)
{
    return (reinterpret_cast<uintptr_t>(p) % alignment) == 0 && (stride % alignment) == 0;
}

// The SM count the tuned launchers size their grids by: the context's, or H100's 132 when it is unknown.
inline int SmCountOrDefault(int32_t smCount)
{
    return smCount > 0 ? smCount : 132;
}

// The grid of a persistent kernel: one CTA per `blocks` of work, at most `cap` (CTAs per SM x SMs) and at least one.
inline unsigned GridFor(long long blocks, long long cap)
{
    return static_cast<unsigned>(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

struct Interior
{
    int32_t width;
    int32_t rows;
};

// ---- routing: which tuned kernel family converts a direct call's block, and on which aligned interior -----------------
//
// A route has two halves.  The description's (EncodeFamilyOf / DecodeFamilyOf, host_params.cpp; host only, once per call)
// names the one tuned family whose conditions the description and the context's first-use state meet (step table, Gray16
// LUT, verified shortcuts), or generic.  The block's (EncodeBlockInterior / DecodeBlockInterior; also run by the batch plan
// kernel) gives the interior [0, width) x [0, rows) that family's kernel converts for this block: buffer alignment, enough
// pixels, a 4:2:0 block starting on a row pair.  An empty interior (width 0) leaves the whole block to the generic kernel;
// no other tuned family is tried.  LaunchEncode / LaunchDecode launch the family's kernel on the interior and hand the
// strips around it to the generic kernel (CompleteEncode / CompleteDecode).
enum class EncodeFamily : int32_t
{
    Generic,
    RgbF32Interleaved, // RGB32f in the reference's interleaved layout through a step table (EncodeRgbF32FlatKernel, INTERLEAVED = 1)
    RgbF32Flat,        // RGB32f -> planar YCbCr through a step table (EncodeRgbF32FlatKernel)
    RgbaF32Flat,       // RGBA32f -> planar YCbCr + alpha through the compact table (EncodeRgbaF32FlatKernel)
    RgbF32Clip,        // RGB32f -> planar YCbCr with no transfer curve (EncodeRgbF32ClipKernel)
    Gray16Lut,         // Gray16 -> 10/12-bit Y through the context's code table (EncodeGray16LutKernel)
    GrayInt,           // Gray(+A) 8/16-bit -> Y (+A) (EncodeGrayIntKernel)
    RgbInt,            // RGB(A) 8/16-bit -> planar YCbCr (EncodeRgbIntPlanarKernel; batched)
    GrayF32,           // Gray(+A)32f -> Y (+A), PQ through the compact table or clip (EncodeGrayF32Kernel)
};

enum class DecodeFamily : int32_t
{
    Generic,
    YccF32,       // 10/12-bit YCbCr -> 32-bit hosts (DecodeYccToRgbF32Kernel; batched)
    YccInt,       // YCbCr -> 8/16-bit hosts (DecodeYccToRgbIntKernel; batched)
    MonoInt,      // monochrome -> 8/16-bit hosts (StreamDecodeKernel)
    PlanarRgbInt, // planar RGB -> 8/16-bit hosts (StreamDecodeKernel; batched)
    MonoF32,      // 10/12-bit monochrome PQ -> 32-bit hosts (TableDecodeF32Kernel)
    PlanarRgbF32, // 10/12-bit planar RGB -> 32-bit hosts (TableDecodeF32Kernel; batched without premultiplied alpha)
};

EncodeFamily EncodeFamilyOf(const EncodeParams& p, int hostDepth);
DecodeFamily DecodeFamilyOf(const DecodeParams& p);

// Shared-memory layouts of the tuned float encode kernels: what the kernels carve their dynamic shared memory into, and
// what the description's half checks a step table against.  kSharedLimit is the opt-in maximum per CTA on sm_90.
constexpr int kSharedLimit = 227 * 1024;
constexpr int kSharedLibm = 768; // avifmath::StageLibmTables' 96 words, first in every float encode kernel's shared memory
// EncodeRgbF32FlatKernel: libm tables, the warps' barriers (the last slot the table's), a two-row staging buffer per
// warp, then the step table (compact entries + first_k, or 256 octave entries + the bucket words).
constexpr int kFlatWarps = 28;
constexpr int kFlatSharedBarriers = 256;
constexpr int kFlatStageBytesPerWarp = 2 * 128 * 12; // both rows of a 128-pixel RGB32f tile
constexpr int kFlatOctaveBytes = 256 * 8;
AVIFGPU_HD constexpr int FlatFixedBytes() { return kSharedLibm + kFlatSharedBarriers + kFlatWarps * kFlatStageBytesPerWarp; }
inline size_t FlatTableBytes(const CurveTableView& t, bool twoLevel)
{
    return twoLevel ? kFlatOctaveBytes + static_cast<size_t>(t.bucketCount) * sizeof(uint32_t) : t.compactImageBytes;
}
inline bool FlatCompactFits(const CurveTableView& t)
{
    return t.compact != nullptr && t.firstBits != nullptr && t.bandBits != nullptr &&
           static_cast<size_t>(FlatFixedBytes()) + FlatTableBytes(t, false) <= static_cast<size_t>(kSharedLimit);
}
inline bool FlatTwoLevelFits(const CurveTableView& t)
{
    return t.buckets != nullptr && t.octaves != nullptr && static_cast<size_t>(FlatFixedBytes()) + FlatTableBytes(t, true) <= static_cast<size_t>(kSharedLimit);
}
// EncodeRgbaF32FlatKernel: libm tables, the table's barrier (padded), 28 words per lane of staged colour samples, the table.
constexpr int kRgbaWarps = 16;
constexpr int kRgbaTableBarrierBytes = 16;
constexpr int kRgbaLaneStrideWords = 28; // 24 colour samples + padding: 16-byte aligned, conflict-free for STS.128
constexpr int kRgbaStagePerWarp = 32 * kRgbaLaneStrideWords * 4;
AVIFGPU_HD constexpr int RgbaFixedBytes() { return kSharedLibm + kRgbaTableBarrierBytes + kRgbaWarps * kRgbaStagePerWarp; }
// EncodeLightF32BatchKernel (kernels_batch.cu): the RGBA kernel's layout with its own warp count -- libm tables, the table's
// barrier, 28 words per lane of staged colour samples, the compact table; one CTA per SM for the whole launch.
constexpr int kLightBatchWarps = 16;
AVIFGPU_HD constexpr int LightBatchFixedBytes() { return kSharedLibm + kRgbaTableBarrierBytes + kLightBatchWarps * kRgbaStagePerWarp; }
// EncodeGrayF32Kernel: libm tables, the table's barrier (padded), the compact table (PQ only), within 100 KiB.
constexpr int kGrayF32FixedBytes = kSharedLibm + 16;
constexpr int kGrayF32SharedLimit = 100 * 1024;

// The block halves.  8/16-bit RGB(A) hosts into planar YCbCr (EncodeRgbIntPlanarKernel): 8-pixel-aligned buffers and at
// least 8 x (1 << ys) pixels; width a multiple of 8, rows of 1 << ys.  Interleaved chroma is one plane of Cb, Cr pairs a
// thread writes in one store of twice the planar chroma's bytes (two 128-bit stores for 16-bit 4:4:4), so it is aligned to
// that store, at most 16 bytes.
AVIFGPU_HD inline Interior EncodeRgbIntBlockInterior(const EncodeParams& p, int hostDepth)
{
    const Interior none = { 0, 0 };
    const int hostBytes = hostDepth / 8;
    const int planeBytes = p.imageDepth > 8 ? 2 : 1;
    const int rowAlign = (8 * p.channels * hostBytes) % 16 == 0 ? 16 : 8; // a thread's 8-pixel chunk: 128-bit or 64-bit loads
    const int lumaAlign = 8 * planeBytes;
    const int chromaAlign = (p.xs ? 4 : 8) * planeBytes;
    const bool chromaAligned = SourceInterleaved(p.destLayout)
                                   ? Aligned(p.plane[1], p.planeStride[1], 2 * chromaAlign > 16 ? 16 : 2 * chromaAlign)
                                   : Aligned(p.plane[1], p.planeStride[1], chromaAlign) && Aligned(p.plane[2], p.planeStride[2], chromaAlign);
    if (p.width < 8 || !Aligned(p.rows, p.rowStride, rowAlign) || !Aligned(p.plane[0], p.planeStride[0], lumaAlign) || !chromaAligned ||
        (p.channels == 4 && !Aligned(p.plane[3], p.planeStride[3], lumaAlign)))
    {
        return none;
    }
    const int evenRows = p.ys ? (p.rowCount & ~1) : p.rowCount;
    if (evenRows < 1)
    {
        return none;
    }
    return Interior{ p.width & ~7, evenRows };
}

// The tuned float planar encodes (RgbF32Flat, RgbaF32Flat, RgbF32Clip): 10/12-bit planes, a lane on 4 pixels of each of 2
// rows, 128-bit row loads, 64-bit luma and alpha stores, 32-bit (4:2:0, 4:2:2) or 64-bit (4:4:4) planar chroma stores --
// or, into interleaved chroma, one store of twice those bytes -- and at least 4 x (1 << ys) pixels.  width is a multiple
// of 4, rows of 1 << ys.
AVIFGPU_HD inline Interior EncodeRgbF32BlockInterior(const EncodeParams& p)
{
    const Interior none = { 0, 0 };
    const int chromaAlign = p.xs ? 4 : 8;
    const bool chromaAligned = SourceInterleaved(p.destLayout)
                                   ? Aligned(p.plane[1], p.planeStride[1], 2 * chromaAlign)
                                   : Aligned(p.plane[1], p.planeStride[1], chromaAlign) && Aligned(p.plane[2], p.planeStride[2], chromaAlign);
    if (!Aligned(p.rows, p.rowStride, 16) || !Aligned(p.plane[0], p.planeStride[0], 8) || !chromaAligned ||
        (p.channels == 4 && p.hasAlpha && !Aligned(p.plane[3], p.planeStride[3], 8)))
    {
        return none;
    }
    const int width4 = p.width & ~3;
    const int evenRows = p.ys ? (p.rowCount & ~1) : p.rowCount;
    if (width4 < 4 || evenRows < 1)
    {
        return none;
    }
    return Interior{ width4, evenRows };
}

// The float kernels that read `rows` with 128-bit loads and write one or two 16-bit planes with 64-bit stores, 4 pixels
// a thread, no sub-sampling: the interleaved RGB32f encode (plane 0 only) and the gray float one (plane 3 too, with alpha).
AVIFGPU_HD inline Interior EncodeFourPixelInterior(const EncodeParams& p, bool alphaPlane)
{
    const Interior none = { 0, 0 };
    const int width4 = p.width & ~3;
    if (width4 < 4 || p.rowCount < 1 || !Aligned(p.rows, p.rowStride, 16) || !Aligned(p.plane[0], p.planeStride[0], 8) ||
        (alphaPlane && !Aligned(p.plane[3], p.planeStride[3], 8)))
    {
        return none;
    }
    return Interior{ width4, p.rowCount };
}

// Gray16 through the code table: a thread looks up 8 samples of one 128-bit load and stores them with one 128-bit store.
AVIFGPU_HD inline Interior EncodeGray16LutBlockInterior(const EncodeParams& p)
{
    const Interior none = { 0, 0 };
    if (p.width < 8 || !Aligned(p.rows, p.rowStride, 16) || !Aligned(p.plane[0], p.planeStride[0], 16))
    {
        return none;
    }
    return Interior{ p.width & ~7, p.rowCount };
}

// Gray(+A) 8/16-bit hosts: a thread's 8 pixels, 64- or 128-bit row loads, 8-sample plane stores.
AVIFGPU_HD inline Interior EncodeGrayIntBlockInterior(const EncodeParams& p, int hostDepth)
{
    const Interior none = { 0, 0 };
    const int planeBytes = p.imageDepth > 8 ? 2 : 1;
    const int rowAlign = (8 * p.channels * (hostDepth / 8)) % 16 == 0 ? 16 : 8;
    if (p.width < 8 || p.rowCount < 1 || !Aligned(p.rows, p.rowStride, rowAlign) || !Aligned(p.plane[0], p.planeStride[0], 8 * planeBytes) ||
        (p.channels == 2 && !Aligned(p.plane[3], p.planeStride[3], 8 * planeBytes)))
    {
        return none;
    }
    return Interior{ p.width & ~7, p.rowCount };
}

AVIFGPU_HD inline Interior EncodeBlockInterior(EncodeFamily family, const EncodeParams& p, int hostDepth)
{
    switch (family)
    {
    case EncodeFamily::RgbF32Interleaved: return EncodeFourPixelInterior(p, false);
    case EncodeFamily::RgbF32Flat:
    case EncodeFamily::RgbF32Clip: return EncodeRgbF32BlockInterior(p);
    case EncodeFamily::RgbaF32Flat: return p.plane[3] != nullptr ? EncodeRgbF32BlockInterior(p) : Interior{ 0, 0 };
    case EncodeFamily::Gray16Lut: return EncodeGray16LutBlockInterior(p);
    case EncodeFamily::GrayInt: return EncodeGrayIntBlockInterior(p, hostDepth);
    case EncodeFamily::RgbInt: return EncodeRgbIntBlockInterior(p, hostDepth);
    case EncodeFamily::GrayF32: return EncodeFourPixelInterior(p, p.channels == 2);
    default: return Interior{ 0, 0 };
    }
}

// The integer YCbCr decode (DecodeYccToRgbIntKernel): 8/16-bit hosts, a block starting on a 4:2:0 row pair, aligned
// buffers, at least 8 x (1 << ys) pixels.  Interleaved chroma is one plane of Cb, Cr pairs a lane reads in one load of
// twice the planar chroma's bytes (two 128-bit loads for 16-bit 4:4:4), so it is aligned to that load, at most 16 bytes.
AVIFGPU_HD inline Interior DecodeYccIntBlockInterior(const DecodeParams& p)
{
    const Interior none = { 0, 0 };
    const int sampleBytes = p.hostDepth == 8 ? 1 : 2;
    const int channels = p.hasAlpha ? 4 : 3;
    const int lumaAlign = 8 * sampleBytes;
    const int chromaAlign = (p.xs ? 4 : 8) * sampleBytes;
    const int rowAlign = channels == 4 ? 16 : 8 * sampleBytes; // RGB8: 64-bit stores, everything else 128-bit
    const bool interleaved = SourceInterleaved(p.sourceLayout);
    const bool chromaAligned = interleaved ? Aligned(p.plane[1], p.planeStride[1], 2 * chromaAlign > 16 ? 16 : 2 * chromaAlign)
                                           : Aligned(p.plane[1], p.planeStride[1], chromaAlign) && Aligned(p.plane[2], p.planeStride[2], chromaAlign);
    if (p.yPhase != 0 || !Aligned(p.plane[0], p.planeStride[0], lumaAlign) || !chromaAligned ||
        (p.hasAlpha && !Aligned(p.plane[3], p.planeStride[3], lumaAlign)) || !Aligned(p.rows, p.rowStride, rowAlign))
    {
        return none;
    }
    const int width8 = p.width & ~7;
    const int evenRows = p.ys ? (p.rowCount & ~1) : p.rowCount;
    if (width8 < 8 || evenRows < 1)
    {
        return none;
    }
    return Interior{ width8, evenRows };
}

// The float YCbCr decode (DecodeYccToRgbF32Kernel): a block starting on a 4:2:0 row pair, aligned buffers, equal Cb and Cr
// strides, at least 4 x (1 << ys) pixels.  width is a multiple of 4, rows of 1 << ys.  Interleaved chroma is one plane of
// Cb, Cr pairs read in one load of twice the planar chroma's bytes, aligned to it.
AVIFGPU_HD inline Interior DecodeYccF32BlockInterior(const DecodeParams& p)
{
    const Interior none = { 0, 0 };
    const int chromaAlign = p.xs ? 4 : 8;
    const bool interleaved = SourceInterleaved(p.sourceLayout);
    const bool chromaAligned = interleaved ? Aligned(p.plane[1], p.planeStride[1], 2 * chromaAlign)
                                           : Aligned(p.plane[1], p.planeStride[1], chromaAlign) && Aligned(p.plane[2], p.planeStride[2], chromaAlign);
    if (p.yPhase != 0 || !Aligned(p.plane[0], p.planeStride[0], 8) || !chromaAligned || !Aligned(p.rows, p.rowStride, 16) ||
        (p.hasAlpha && !Aligned(p.plane[3], p.planeStride[3], 8)))
    {
        return none;
    }
    if (!interleaved && p.planeStride[1] != p.planeStride[2])
    {
        return none; // the single-image kernel walks Cb and Cr with one offset
    }
    const int width4 = p.width & ~3;
    const int evenRows = p.ys ? (p.rowCount & ~1) : p.rowCount;
    if (width4 < 4 || evenRows < 1)
    {
        return none;
    }
    return Interior{ width4, evenRows };
}

// The planar-RGB decodes (StreamDecodeKernel for 8/16-bit hosts, TableDecodeF32Kernel for 32-bit hosts): planes aligned to
// a thread's 8 samples, rows to its stores, at least 8 pixels and one row.  width is a multiple of 8 and rows is the
// block's: the interior only ever leaves a right strip.
AVIFGPU_HD inline Interior DecodePlanarRgbBlockInterior(const DecodeParams& p)
{
    const Interior none = { 0, 0 };
    const int planeAlign = 8 * (p.hostDepth == 8 ? 1 : 2); // 8-bit hosts read 8-bit planes, the others 10/12-bit ones
    const int groupBytes = 8 * (p.hasAlpha ? 4 : 3) * (p.hostDepth / 8);
    const int rowAlign = groupBytes % 16 == 0 ? 16 : 8; // RGB8: 64-bit stores, everything else 128-bit
    for (int c = 0; c < 3; ++c)
    {
        if (!Aligned(p.plane[c], p.planeStride[c], planeAlign))
        {
            return none;
        }
    }
    if ((p.hasAlpha && !Aligned(p.plane[3], p.planeStride[3], planeAlign)) || !Aligned(p.rows, p.rowStride, rowAlign))
    {
        return none;
    }
    const int width8 = p.width & ~7;
    if (width8 < 8 || p.rowCount < 1)
    {
        return none;
    }
    return Interior{ width8, p.rowCount };
}

// The monochrome decodes: a thread's 8 samples of plane 0 (and 3), one or two host stores.  Integer hosts align the
// planes to 8 samples and the rows to the group's stores; float hosts both to 16 bytes.
AVIFGPU_HD inline Interior DecodeMonoBlockInterior(const DecodeParams& p)
{
    const Interior none = { 0, 0 };
    const bool f32 = p.hostDepth == 32;
    const int sampleBytes = p.hostDepth == 8 ? 1 : 2;
    const int planeAlign = f32 ? 16 : 8 * sampleBytes;
    const int rowAlign = f32 || (8 * (p.hasAlpha ? 2 : 1) * sampleBytes) % 16 == 0 ? 16 : 8;
    if (!Aligned(p.plane[0], p.planeStride[0], planeAlign) || (p.hasAlpha && !Aligned(p.plane[3], p.planeStride[3], planeAlign)) ||
        !Aligned(p.rows, p.rowStride, rowAlign))
    {
        return none;
    }
    const int width8 = p.width & ~7;
    if (width8 < 8 || p.rowCount < 1)
    {
        return none;
    }
    return Interior{ width8, p.rowCount };
}

AVIFGPU_HD inline Interior DecodeBlockInterior(DecodeFamily family, const DecodeParams& p)
{
    switch (family)
    {
    case DecodeFamily::YccF32: return DecodeYccF32BlockInterior(p);
    case DecodeFamily::YccInt: return DecodeYccIntBlockInterior(p);
    case DecodeFamily::MonoInt:
    case DecodeFamily::MonoF32: return DecodeMonoBlockInterior(p);
    case DecodeFamily::PlanarRgbInt:
    case DecodeFamily::PlanarRgbF32: return DecodePlanarRgbBlockInterior(p);
    default: return Interior{ 0, 0 };
    }
}

// The family a batch of images of this description runs its interiors on: integer RGB(A) into planar YCbCr for encodes;
// generic otherwise.
inline EncodeFamily EncodeBatchFamilyOf(const EncodeParams& p, int hostDepth)
{
    return EncodeFamilyOf(p, hostDepth) == EncodeFamily::RgbInt ? EncodeFamily::RgbInt : EncodeFamily::Generic;
}
// For the light-level batches (avifgpu_encode_batch_device_light_level / _indirect_light_level): float planar RGB through
// the PQ step table and float planar RGBA through the compact table, when the single-image light route takes them (it
// has the compact table only: FlatCompactFits) and the compact table fits EncodeLightF32BatchKernel; generic otherwise.
// A batch thus tunes exactly the images a direct light-level call tunes.  The caller leaves curveTable null when the
// context has no level table for the depth, as the direct call does.
inline EncodeFamily EncodeLightBatchFamilyOf(const EncodeParams& p, int hostDepth)
{
    const EncodeFamily family = EncodeFamilyOf(p, hostDepth);
    if (hostDepth != 32 || p.transfer != AVIFGPU_TRANSFER_PQ || (family != EncodeFamily::RgbF32Flat && family != EncodeFamily::RgbaF32Flat))
    {
        return EncodeFamily::Generic;
    }
    const CurveTableView& t = *p.curveTable; // a tuned family has its verified table
    const bool fits = FlatCompactFits(t) && static_cast<size_t>(LightBatchFixedBytes()) + t.compactImageBytes <= static_cast<size_t>(kSharedLimit);
    return fits ? family : EncodeFamily::Generic;
}
// For decodes: YCbCr and planar RGB into every host depth,
// except premultiplied alpha, which only the single-image table kernel un-premultiplies; generic otherwise.
inline DecodeFamily DecodeBatchFamilyOf(const DecodeParams& p)
{
    const DecodeFamily family = DecodeFamilyOf(p);
    const bool batched = family == DecodeFamily::YccF32 || family == DecodeFamily::YccInt || family == DecodeFamily::PlanarRgbInt ||
                         family == DecodeFamily::PlanarRgbF32;
    return batched && !(p.hasAlpha && p.premultiplied) ? family : DecodeFamily::Generic;
}

// The pixel-independent factors of the float decode's channel sums, YuvDecode.cpp:555-557 and :308 -- the reference's
// float expressions, evaluated once on the host without contraction (host_params.cpp).
struct F32DecodeFactors
{
    float rGain, bGain, gCr, gCb, kgReciprocal;
};
F32DecodeFactors F32DecodeFactorsOf(const avifpix::InverseMatrix& matrix);

// The strips CompleteEncode / CompleteDecode hand to the generic kernel around a block's interior, in their order: the
// right strip [inner.width, width) x [0, rows), then the bottom strip [0, inner.width) x [inner.rows, rows).  Returns how
// many of the two are non-empty; those come first in `strip`.
struct Strip
{
    int32_t x0, y0, width, rows;
};
AVIFGPU_HD inline int InteriorStrips(int width, int rows, Interior inner, Strip strip[2])
{
    const Strip candidate[2] = { { inner.width, 0, width - inner.width, rows }, { 0, inner.rows, inner.width, rows - inner.rows } };
    int count = 0;
    for (int k = 0; k < 2; ++k)
    {
        if (candidate[k].width > 0 && candidate[k].rows > 0)
        {
            strip[count++] = candidate[k];
        }
    }
    return count;
}

// ---- batches of whole images (avifgpu_encode_batch_device, avifgpu_decode_batch_device) -----------------------------------------------------------
//
// What differs between the images of a batched launch; the launch carries these records by value as a kernel parameter
// (no allocation, no copy, legal while capturing), so a chunk holds at most kBatchChunkImages images.  A launch walks one
// unit space made by concatenating its records' units: record i owns [firstUnit_i, firstUnit_{i+1}).
struct BatchRecord
{
    const void* rows;       // host-layout rows (encode source, decode destination) at the record's first row
    int64_t rowStride;
    void* plane[4];         // the same row in each plane (encode destination, decode source), as Encode/DecodeWindow place it
    int64_t planeStride[4];
    int32_t width;          // pixels
    int32_t rowCount;
    int64_t firstUnit;
};

constexpr int kBatchChunkImages = 64;
constexpr int kBatchUnitPixels = 256; // interior unit: 256 pixels of one row (row pair for 4:2:0), one warp
constexpr int kF32BatchUnitPixels = 128; // the float YCbCr decode's interior unit: its single-image kernel's 128-pixel tile
// The light-level float encode's interior unit (EncodeLightBatchFamilyOf): the single-image float kernels' 128-pixel tile of
// one row, or of a 4:2:0 row pair, one warp, a lane on 4 pixels of each row.
constexpr int kLightBatchUnitPixels = 128;
constexpr int kBatchEdgeThreads = 256; // edge unit: one CTA-sized run of chroma sites (encode) or pixels (decode) of one row (pair)

// Units of an interior of `width` x `rows` pixels, and of an edge window.
AVIFGPU_HD inline int64_t BatchInteriorUnits(int width, int rows, int ys, int unitPixels = kBatchUnitPixels)
{
    return static_cast<int64_t>((width + unitPixels - 1) / unitPixels) * ((rows + ys) >> ys);
}
// The interior unit width of a batched decode family: 128 pixels for the float YCbCr one, 256 for the others.
AVIFGPU_HD inline int DecodeBatchUnitPixels(DecodeFamily family)
{
    return family == DecodeFamily::YccF32 ? kF32BatchUnitPixels : kBatchUnitPixels;
}
AVIFGPU_HD inline int64_t BatchEdgeUnits(int width, int rows, int xs, int ys)
{
    return static_cast<int64_t>((((width + xs) >> xs) + kBatchEdgeThreads - 1) / kBatchEdgeThreads) * ((rows + ys) >> ys);
}

// The record of a block (an EncodeWindow / DecodeWindow), first unit 0.
template <typename Params>
AVIFGPU_HD inline BatchRecord RecordOf(const Params& w)
{
    BatchRecord r{};
    r.rows = w.rows;
    r.rowStride = w.rowStride;
    for (int k = 0; k < 4; ++k)
    {
        r.plane[k] = const_cast<void*>(static_cast<const void*>(w.plane[k]));
        r.planeStride[k] = w.planeStride[k];
    }
    r.width = w.width;
    r.rowCount = w.rowCount;
    return r;
}

// One chunk: at most two launches -- the batched tuned kernel over every image's interior, then the batched generic
// kernel over every image's right strip and odd last 4:2:0 row (none when no image has one).
struct BatchChunk
{
    int32_t images = 0;                       // interiors in this chunk
    int32_t imageIndex[kBatchChunkImages];    // their positions in the caller's array, increasing
    BatchRecord interior[kBatchChunkImages];
    int64_t interiorUnits = 0;
    int32_t windows = 0;
    int32_t windowImage[2 * kBatchChunkImages]; // position in the caller's array of each window's image
    BatchRecord window[2 * kBatchChunkImages];
    int64_t windowUnits = 0;
};

struct BatchPlan
{
    std::vector<BatchChunk> chunks;
    std::vector<int32_t> fallback; // positions of the images that take one direct call each (LaunchEncode), in order
};

// Launches of one chunk: 1 + (1 when it has edge windows).
inline int BatchChunkLaunches(const BatchChunk& chunk) { return 1 + (chunk.windows > 0 ? 1 : 0); }

// A launcher that sees a CUDA error has already consumed it (cudaGetLastError clears the slot), so it leaves the code
// here -- a thread-local slot in avifgpu_api.cu -- and returns AVIFGPU_ERR_CUDA; the API reports it from there instead
// of asking CUDA a second time (which would answer cudaSuccess and turn a failed launch into AVIFGPU_OK).
int ReportLaunchFailure(int cudaErrorCode);

// LaunchEncode / LaunchDecode (avifgpu_api.cu) route a direct call (EncodeFamilyOf / DecodeFamilyOf, then the block half),
// launch the family's kernel on the interior and complete the block.  They only enqueue work on `stream` and return the
// number of kernels launched (>= 1; 0 for an empty block) or a negative avifgpu_status.
// `light` (the light-level call, light_level.cuh): the same route through the LIGHT instantiations, which add the block's
// content light level into light->acc.
int LaunchEncode(const EncodeParams& params, int hostDepth, void* stream, const LightSink* light = nullptr);
int LaunchDecode(const DecodeParams& params, void* stream);
int LaunchEncodeGeneric(const EncodeParams& params, int hostDepth, void* stream, const LightSink* light = nullptr);
int LaunchDecodeGeneric(const DecodeParams& params, void* stream);
int LaunchTransfer(int function, float param, const float* in, float* out, size_t count, void* stream);
int LaunchHlgOotf(int inverse, const float luma[3], float displayGamma, float peak, const float* in, float* out, size_t pixels, void* stream);
// One warp adding the partials parts[r] whose bit r is set in `members` into *acc (the sharded device light-level call's
// merge, kernels_generic.cu).  Returns 1, or a negative status.
int LaunchMergeLightPartials(const avifgpu_light_level* parts, uint64_t members, avifgpu_light_level* acc, void* stream);

// The tuned launchers (kernels_fast*.cu): each fills its kernel's parameters for the interior `inner` of the block `p`
// that the route gave its family, enqueues the kernel and returns the launch's status.
cudaError_t LaunchEncodeRgbF32Interleaved(const EncodeParams& p, Interior inner, void* stream, const LightSink* light = nullptr);
cudaError_t LaunchEncodeRgbF32Planar(EncodeFamily family, const EncodeParams& p, Interior inner, void* stream,
                                     const LightSink* light = nullptr); // RgbF32Flat, RgbaF32Flat, RgbF32Clip
cudaError_t LaunchEncodeGray16Lut(const EncodeParams& p, Interior inner, void* stream);
cudaError_t LaunchEncodeGrayInt(const EncodeParams& p, int hostDepth, Interior inner, void* stream);
cudaError_t LaunchEncodeRgbInt(const EncodeParams& p, int hostDepth, Interior inner, void* stream);
cudaError_t LaunchEncodeGrayF32(const EncodeParams& p, Interior inner, void* stream, const LightSink* light = nullptr);
cudaError_t LaunchDecodeYccF32(const DecodeParams& p, Interior inner, void* stream);
cudaError_t LaunchDecodeYccInt(const DecodeParams& p, Interior inner, void* stream);
cudaError_t LaunchDecodeStream(const DecodeParams& p, Interior inner, void* stream); // MonoInt, PlanarRgbInt
cudaError_t LaunchDecodeTable(const DecodeParams& p, Interior inner, void* stream);  // MonoF32, PlanarRgbF32

// The end of every tuned launch.  The tuned kernel converts the block's interior [0, coveredWidth) x [0, coveredRows);
// `tuned` is its launch status.  On success the generic kernel converts the right strip [coveredWidth, width) x
// [0, rowCount), then the bottom strip [0, coveredWidth) x [coveredRows, rowCount); an empty strip launches nothing.
// Returns 1 + the strip launches, or a negative status.
int CompleteEncode(cudaError_t tuned, const EncodeParams& p, int hostDepth, int coveredWidth, int coveredRows, void* stream,
                   const LightSink* light = nullptr);
int CompleteDecode(cudaError_t tuned, const DecodeParams& p, int coveredWidth, int coveredRows, void* stream);

// The launches of one planned chunk (PlanEncodeBatch / PlanDecodeBatch, batch_plan.h; kernels_batch.cu); `shared` is the
// description's block (its pointers, strides and sizes are unused).  Returns BatchChunkLaunches(chunk) or a negative status.
int LaunchEncodeBatchChunk(const EncodeParams& shared, int hostDepth, const BatchChunk& chunk, void* stream);
int LaunchDecodeBatchChunk(const DecodeParams& shared, const BatchChunk& chunk, void* stream);
// The same for a chunk of a light-level batch (PlanEncodeLightBatch; float hosts): image chunk.imageIndex[j] /
// chunk.windowImage[j] adds its content light level into light.acc[that index].
int LaunchEncodeLightBatchChunk(const EncodeParams& shared, const BatchChunk& chunk, const LightSink& light, void* stream);

// The block the generic encode kernels read (LaunchEncodeGeneric): a float host with a verified compact table gets its
// by-value view.
EncodeParams GenericEncodeView(const EncodeParams& params, int hostDepth);

cudaError_t BuildGray16Lut(uint16_t* deviceLut, int smpte428, uint32_t maxCode, void* stream);

// Exhaustive device checks of the arithmetic shortcuts (kernels_fast_decode.cu, kernels_fast_int.cu).
long long VerifyHlgDivisions(void* stream);
long long VerifyPqRatio(void* stream);
long long VerifyFastPremultiply(uint32_t maxCode, void* stream);
long long VerifyGreenDivision(const DecodeParams& params, void* stream);

} // namespace avifgpu

#endif
