// kernel_params.h -- plain parameter blocks handed to the CUDA kernels (device pointers, block-relative).
//
// "Block" = the row block [y0, y0 + rows) one launch converts.  All pointers already point at the first row of
// the block in their buffer (for sub-sampled chroma planes: at chroma row y0 >> ys), so kernels index rows from
// zero and never see y0 -- except `yPhase`, the parity of y0 for 4:2:0 decode, where an odd first row shares its
// chroma row with the row above it (ReadHeifImage.cpp:359 uvJ = y >> yChromaShift).
#ifndef AVIF_KERNEL_PARAMS_H
#define AVIF_KERNEL_PARAMS_H

#include <stdint.h>

#include <atomic>
#include <vector>

#include <driver_types.h>

#include "../../include/avifgpu.h"
#include "curve_tables.h"
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

// The aligned interior [0, width) x [0, rows) the tuned integer planar encode kernel (EncodeRgbIntPlanarKernel)
// converts for this block, or {0, 0} when a direct call of the block takes another route: 8/16-bit RGB(A) hosts into
// planar YCbCr of at most 12 bits, no alpha, straight alpha or a verified premultiply, a matrix the biased truncation
// handles, 8-pixel-aligned buffers and at least 8 x (1 << ys) pixels.  width is a multiple of 8, rows of 1 << ys.
struct Interior
{
    int32_t width;
    int32_t rows;
};
// EncodeRgbIntInterior in two halves: the description's (host depth, layout, channels, premultiply, depth, matrix --
// the same for every block of one description, host only) and the block's (buffer alignment, at least 8 pixels and one
// 4:2:0 row pair).  Interleaved chroma is one plane of Cb, Cr pairs a thread writes in one store of twice the planar
// chroma's bytes (two 128-bit stores for 16-bit 4:4:4), so it is aligned to that store, at most 16 bytes; the
// destination layout is the block's business only, so the description's half does not read it.
bool EncodeRgbIntTuned(const EncodeParams& p, int hostDepth);
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
Interior EncodeRgbIntInterior(const EncodeParams& p, int hostDepth); // EncodeRgbIntTuned ? EncodeRgbIntBlockInterior : none

// The block's half of the tuned float planar encodes (EncodeRgbF32FlatKernel, EncodeRgbaF32FlatKernel,
// EncodeRgbF32ClipKernel; LaunchEncodeFast has the description's): 10/12-bit planes, a lane on 4 pixels of each of 2 rows,
// 128-bit row loads, 64-bit luma and alpha stores, 32-bit (4:2:0, 4:2:2) or 64-bit (4:4:4) planar chroma stores -- or,
// into interleaved chroma, one store of twice those bytes -- and at least 4 x (1 << ys) pixels.  width is a multiple of
// 4, rows of 1 << ys.
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

// The same for the tuned integer YCbCr decode kernel (DecodeYccToRgbIntKernel): 8/16-bit hosts reading 8-bit / 10-12-bit
// YCbCr (+ straight alpha), a block starting on a 4:2:0 row pair, aligned buffers, at least 8 x (1 << ys) pixels.
// Interleaved chroma is one plane of Cb, Cr pairs a lane reads in one load of twice the planar chroma's bytes (two 128-bit
// loads for 16-bit 4:4:4), so it is aligned to that load, at most 16 bytes.
bool DecodeYccIntTuned(const DecodeParams& p);
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
    if (!Aligned(p.plane[0], p.planeStride[0], lumaAlign) || !chromaAligned || (p.hasAlpha && !Aligned(p.plane[3], p.planeStride[3], lumaAlign)) ||
        !Aligned(p.rows, p.rowStride, rowAlign))
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
Interior DecodeYccIntInterior(const DecodeParams& p); // DecodeYccIntTuned ? DecodeYccIntBlockInterior : none

// The same for the tuned float YCbCr decode kernel (DecodeYccToRgbF32Kernel), split the same way.  The description's half:
// 10/12-bit YCbCr (+ straight alpha) into 32-bit hosts with the PQ, HLG or SMPTE 428 curve; for HLG the context's verified
// divisions, and with the OOTF an exponent and luma coefficients the branch-free powf covers; for PQ and SMPTE 428 a matrix
// whose channel sums are never subnormal.  The block's half: a block starting on a 4:2:0 row pair, aligned buffers, equal
// Cb and Cr strides, at least 4 x (1 << ys) pixels.  width is a multiple of 4, rows of 1 << ys.  Interleaved chroma is one
// plane of Cb, Cr pairs read in one load of twice the planar chroma's bytes, aligned to it.
bool DecodeYccF32Tuned(const DecodeParams& p);
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
Interior DecodeYccF32Interior(const DecodeParams& p); // DecodeYccF32Tuned ? DecodeYccF32BlockInterior : none

// The same for the tuned planar-RGB decode kernels (StreamDecodeKernel for 8/16-bit hosts, TableDecodeF32Kernel for 32-bit
// hosts), split the same way.  The description's half: colour space RGB with no or straight alpha; for 8/16-bit hosts at
// most 12 bits, 8-bit planes into 8-bit hosts and 10/12-bit planes into 16-bit hosts; for 32-bit hosts 10/12-bit planes
// with the PQ, HLG or SMPTE 428 curve.  The block's half: planes aligned to a thread's 8 samples, rows to its stores, at
// least 8 pixels and one row.  width is a multiple of 8 and rows is the block's: the interior only ever leaves a right strip.
bool DecodePlanarRgbTuned(const DecodeParams& p);
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
Interior DecodePlanarRgbInterior(const DecodeParams& p); // DecodePlanarRgbTuned ? DecodePlanarRgbBlockInterior : none

// The description half of whichever tuned decode kernel serves the description: the planar-RGB one for colour space RGB,
// otherwise the float YCbCr one for 32-bit hosts and the integer one for the others.  Both batch APIs route by it.
bool DecodeBatchTuned(const DecodeParams& p);

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
constexpr int kBatchEdgeThreads = 256; // edge unit: one CTA-sized run of chroma sites (encode) or pixels (decode) of one row (pair)

// Units of an interior of `width` x `rows` pixels, and of an edge window.
AVIFGPU_HD inline int64_t BatchInteriorUnits(int width, int rows, int ys, int unitPixels = kBatchUnitPixels)
{
    return static_cast<int64_t>((width + unitPixels - 1) / unitPixels) * ((rows + ys) >> ys);
}
// The interior unit width of a decode of `colorspace` into `hostDepth`-bit hosts: 128 pixels for YCbCr into 32-bit hosts,
// 256 for everything else (planar RGB into every host depth).
AVIFGPU_HD inline int DecodeBatchUnitPixels(int hostDepth, int colorspace)
{
    return hostDepth == 32 && colorspace != AVIFGPU_COLORSPACE_RGB ? kF32BatchUnitPixels : kBatchUnitPixels;
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

// Launchers implemented in kernels_*.cu.  They only enqueue work on `stream` and return the number of kernels
// launched (>= 1) or a negative avifgpu_status; the tuned ones (LaunchEncodeFast*, LaunchDecodeFast*) return 0 for a
// configuration they do not cover.
int LaunchEncode(const EncodeParams& params, int hostDepth, void* stream);
int LaunchDecode(const DecodeParams& params, void* stream);
int LaunchEncodeGeneric(const EncodeParams& params, int hostDepth, void* stream);
int LaunchDecodeGeneric(const DecodeParams& params, void* stream);
int LaunchEncodeFast(const EncodeParams& params, int hostDepth, void* stream);
int LaunchEncodeFastInteger(const EncodeParams& params, int hostDepth, void* stream);
int LaunchEncodeFastGray32(const EncodeParams& params, int hostDepth, void* stream);
int LaunchDecodeFast(const DecodeParams& params, void* stream);
int LaunchDecodeFastInteger(const DecodeParams& params, void* stream);
int LaunchDecodeFastTable(const DecodeParams& params, void* stream);
int LaunchTransfer(int function, float param, const float* in, float* out, size_t count, void* stream);
int LaunchHlgOotf(int inverse, const float luma[3], float displayGamma, float peak, const float* in, float* out, size_t pixels, void* stream);

// The end of every tuned launch site.  A tuned kernel converts the block's aligned interior [0, coveredWidth) x
// [0, coveredRows); `tuned` is its launch status.  On success the generic kernel converts the right strip
// [coveredWidth, width) x [0, rowCount), then the bottom strip [0, coveredWidth) x [coveredRows, rowCount); an empty
// strip launches nothing.  Returns 1 + the strip launches, or a negative status.
int CompleteEncode(cudaError_t tuned, const EncodeParams& p, int hostDepth, int coveredWidth, int coveredRows, void* stream);
int CompleteDecode(cudaError_t tuned, const DecodeParams& p, int coveredWidth, int coveredRows, void* stream);

// The launches of one planned chunk (PlanEncodeBatch / PlanDecodeBatch, batch_plan.h; kernels_batch.cu); `shared` is the
// description's block (its pointers, strides and sizes are unused).  Returns BatchChunkLaunches(chunk) or a negative status.
int LaunchEncodeBatchChunk(const EncodeParams& shared, int hostDepth, const BatchChunk& chunk, void* stream);
int LaunchDecodeBatchChunk(const DecodeParams& shared, const BatchChunk& chunk, void* stream);

cudaError_t BuildGray16Lut(uint16_t* deviceLut, int smpte428, uint32_t maxCode, void* stream);

// Exhaustive device checks of the arithmetic shortcuts (kernels_fast_decode.cu, kernels_fast_int.cu).
long long VerifyHlgDivisions(void* stream);
long long VerifyPqRatio(void* stream);
long long VerifyFastPremultiply(uint32_t maxCode, void* stream);
long long VerifyGreenDivision(const DecodeParams& params, void* stream);

} // namespace avifgpu

#endif
