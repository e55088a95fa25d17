// kernels_fast_rgba.cu -- float RGBA hosts -> planar YCbCr + alpha plane through the compact step table (one-word entries
// + first_k in shared memory, brought in by the copy engine; curve_tables.h) and the band bitmap
// (CreateHeifImageRGBThirtyTwoBit's alpha branch, WriteHeifImage.cpp:1039-1077, fused with the libheif stage).
//
// Same warp tile as kernels_fast_flat.cu (2 rows x 128 pixels, a lane owns 4 adjacent pixels in both rows), but 16 bytes
// per pixel do not lay out conflict-free in a linear staging buffer, so the loads are per-lane 128-bit loads (one pixel
// each, issued one tile ahead) and only the 24 colour samples of a lane -- after the clamp / premultiplication, the
// values the curve actually sees -- are parked in shared memory for the band-bitmap probes.  One CTA of 16 warps per SM.
#include "kernels_fast_common.cuh"
#include "launch_keys.h"
#include "table_staging.cuh"
#include "../../include/avifgpu.h"

namespace avifgpu
{

using namespace avifpix;
using namespace fastenc;
using avifmath::LibmTables;

namespace
{

// The shared-memory layout's sizes (kRgbaWarps, RgbaFixedBytes, ...) are in kernel_params.h, where the route reads them.
constexpr int kRgbaThreads = kRgbaWarps * 32;

// The compact table + first_k array in shared memory (kernels_fast_flat.cu has the commentary).  DEST: the
// avifgpu_source_layout bits of the planes written (StoreTile; the alpha plane is shifted like the others).  The body of
// EncodeRgbaF32FlatKernel (DEST 0) and of EncodeDestRgbaF32FlatKernel (the other layouts).  LIGHT = 1: also the content
// light level of the colour codes (light_level.cuh), the body of EncodeLightRgbaF32FlatKernel.
template <int CURVE, int XS, int YS, int DEST, int LIGHT = 0>
__device__ __forceinline__ void EncodeRgbaF32FlatBody(const FastEncodeParams& p, const LightSink& light = {})
{
    extern __shared__ __align__(16) uint8_t sharedBytes[];
    uint64_t* libmStorage = reinterpret_cast<uint64_t*>(sharedBytes);
    uint64_t* tableBarrier = reinterpret_cast<uint64_t*>(sharedBytes + kSharedLibm);
    uint32_t* stageAll = reinterpret_cast<uint32_t*>(sharedBytes + kSharedLibm + kRgbaTableBarrierBytes);
    uint32_t* compactEntries = reinterpret_cast<uint32_t*>(sharedBytes + RgbaFixedBytes());

    if (threadIdx.x == 0)
    {
        staging::BeginTableImageCopy(p.table, compactEntries, tableBarrier); // table_staging.cuh
    }
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads(); // the libm tables, the table barrier's initialisation

    const int lane = threadIdx.x & 31;
    const int warpInBlock = threadIdx.x >> 5;
    uint32_t* myStage = stageAll + warpInBlock * (32 * kRgbaLaneStrideWords) + lane * kRgbaLaneStrideWords;
    const CompactTable compact = CompactTableOf(p.table, compactEntries);

    const int tilesX = (p.width + kTilePixels - 1) / kTilePixels;
    const int tileRows = (p.rowCount + 1) / 2;
    const int tileCount = tilesX * tileRows;
    const int warpCount = static_cast<int>(gridDim.x) * kRgbaWarps;
    const int firstTile = static_cast<int>(blockIdx.x) * kRgbaWarps + warpInBlock;
    const int stepRows = warpCount / tilesX;
    const int stepX = warpCount - stepRows * tilesX;
    int tileRow = firstTile / tilesX;
    int tileX = firstTile - tileRow * tilesX;
    LightTally tally{ 0u, 0ull };

    uint4 raw[8]; // pixel i of row r = raw[4 * r + i] = { R, G, B, A }
    auto loadTile = [&](int row, int column, bool valid)
    {
        const int x = column * kTilePixels + lane * 4;
        const int y = row * 2;
        const bool active = valid && x < p.width;
        const bool second = active && (y + 1) < p.rowCount;
        const uint8_t* r0 = p.rows + static_cast<int64_t>(y) * p.rowStride + static_cast<int64_t>(x) * 16;
        const uint8_t* r1 = r0 + p.rowStride;
        const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int q = 0; q < 4; ++q)
        {
            raw[q] = active ? __ldg(reinterpret_cast<const uint4*>(r0 + 16 * q)) : zero;
            raw[4 + q] = second ? __ldg(reinterpret_cast<const uint4*>(r1 + 16 * q)) : zero;
        }
    };
    loadTile(tileRow, tileX, firstTile < tileCount); // in flight while the table image lands
    staging::WaitTableImage(tableBarrier);

#pragma unroll 1
    for (int tile = firstTile; tile < tileCount; tile += warpCount)
    {
        const int x0 = tileX * kTilePixels + lane * 4;
        const int y0 = tileRow * 2;
        const bool laneActive = x0 < p.width;
        const bool secondRow = (y0 + 1) < p.rowCount;
        int nextRow = tileRow + stepRows;
        int nextX = tileX + stepX;
        if (nextX >= tilesX)
        {
            nextX -= tilesX;
            ++nextRow;
        }

        uint32_t alphaCode[8];
        uint32_t colourBits[kValuesPerLane];
        PrepareRgbaSamples(p, raw, alphaCode, colourBits);
        float codeF[kValuesPerLane];
        uint32_t bandMask;
        int32_t largest;
        LookUpLaneCodes(compact, colourBits, myStage, codeF, bandMask, largest);
        loadTile(nextRow, nextX, tile + warpCount < tileCount); // raw is free: the rest of the tile reads the staged samples
        ResolveLaneCodes<CURVE, kValuesPerLane>(p, t, compact, myStage, bandMask, largest, codeF);

        if (LIGHT && laneActive)
        {
            TallyLaneCodes<8>(tally, codeF, light.levels, secondRow);
        }

        if (laneActive)
        {
            const int64_t chromaRow = YS ? tileRow : y0;
            const int64_t chromaColumn = static_cast<int64_t>(XS ? (x0 >> 1) : x0) * 2;
            StoreTile<XS, YS, DEST>(p, codeF, p.planeY + static_cast<int64_t>(y0) * p.strideY + static_cast<int64_t>(x0) * 2,
                                    p.planeCb + chromaRow * p.strideCb + chromaColumn * (SourceInterleaved(DEST) ? 2 : 1),
                                    p.planeCr + chromaRow * p.strideCr + chromaColumn, secondRow);
            uint8_t* alphaRow = p.planeA + static_cast<int64_t>(y0) * p.strideA + static_cast<int64_t>(x0) * 2;
            StoreAlphaRow<DEST>(p, alphaRow, alphaCode, 0);
            if (secondRow)
            {
                StoreAlphaRow<DEST>(p, alphaRow + p.strideA, alphaCode, 4);
            }
        }
        tileRow = nextRow;
        tileX = nextX;
    }
    if (LIGHT)
    {
        FlushLightTally(tally, LaunchPixelsForFirstWarp(static_cast<uint64_t>(p.width) * p.rowCount), light.acc);
    }
}

template <int CURVE, int XS, int YS>
__global__ void __launch_bounds__(kRgbaThreads, 1) EncodeRgbaF32FlatKernel(const FastEncodeParams p)
{
    EncodeRgbaF32FlatBody<CURVE, XS, YS, AVIFGPU_SOURCE_PLANAR>(p);
}

// The same into semi-planar and MSB-aligned planes (DEST != 0).
template <int CURVE, int XS, int YS, int DEST>
__global__ void __launch_bounds__(kRgbaThreads, 1) EncodeDestRgbaF32FlatKernel(const FastEncodeParams p)
{
    EncodeRgbaF32FlatBody<CURVE, XS, YS, DEST>(p);
}

// The same with the content light level (every layout; PQ only).
template <int CURVE, int XS, int YS, int DEST>
__global__ void __launch_bounds__(kRgbaThreads, 1) EncodeLightRgbaF32FlatKernel(const FastEncodeParams p, const LightSink light)
{
    EncodeRgbaF32FlatBody<CURVE, XS, YS, DEST, 1>(p, light);
}

template <int CURVE, int XS, int YS, int DEST, int LIGHT>
constexpr auto RgbaKernelFor()
{
    if constexpr (LIGHT)
    {
        return EncodeLightRgbaF32FlatKernel<CURVE, XS, YS, DEST>;
    }
    else if constexpr (DEST == AVIFGPU_SOURCE_PLANAR)
    {
        return EncodeRgbaF32FlatKernel<CURVE, XS, YS>;
    }
    else
    {
        return EncodeDestRgbaF32FlatKernel<CURVE, XS, YS, DEST>;
    }
}

template <int CURVE, int XS, int YS, int DEST, int LIGHT = 0>
cudaError_t LaunchRgbaKernel(const FastEncodeParams& fp, int smCount, cudaStream_t stream, const LightSink* light = nullptr)
{
    const size_t shared = static_cast<size_t>(RgbaFixedBytes()) + fp.table.compactImageBytes;
    static std::atomic<uint64_t> configuredDevices{ 0 }; // per instantiation
    {
        const cudaError_t e = AllowDynamicShared(RgbaKernelFor<CURVE, XS, YS, DEST, LIGHT>(), kSharedLimit, configuredDevices);
        if (e != cudaSuccess)
        {
            return e;
        }
    }
    const long long tiles = static_cast<long long>((fp.width + kTilePixels - 1) / kTilePixels) * ((fp.rowCount + 1) / 2);
    if (tiles > 0x7fffffffll || shared > static_cast<size_t>(kSharedLimit))
    {
        return cudaErrorInvalidValue;
    }
    long long blocks = (tiles + kRgbaWarps - 1) / kRgbaWarps;
    if (blocks > smCount)
    {
        blocks = smCount;
    }
    if constexpr (LIGHT)
    {
        RgbaKernelFor<CURVE, XS, YS, DEST, LIGHT>()<<<static_cast<unsigned>(blocks), kRgbaThreads, shared, stream>>>(fp, *light);
    }
    else
    {
        RgbaKernelFor<CURVE, XS, YS, DEST, LIGHT>()<<<static_cast<unsigned>(blocks), kRgbaThreads, shared, stream>>>(fp);
    }
    return cudaGetLastError();
}

} // namespace

cudaError_t LaunchFastEncodeRgba(const FastEncodeParams& fp, int curve, int xs, int ys, int dest, int smCount, cudaStream_t stream, const LightSink* light)
{
    return WithChroma(xs, ys, [&](auto XS, auto YS) {
        return WithLayout(dest, [&](auto DEST) {
            if (light != nullptr)
            {
                return curve == kCurveLinearToPQ ? LaunchRgbaKernel<kCurveLinearToPQ, XS(), YS(), DEST(), 1>(fp, smCount, stream, light) : cudaErrorInvalidValue;
            }
            return curve == kCurveLinearToPQ ? LaunchRgbaKernel<kCurveLinearToPQ, XS(), YS(), DEST()>(fp, smCount, stream)
                                             : LaunchRgbaKernel<kCurveLinearToSMPTE428, XS(), YS(), DEST()>(fp, smCount, stream);
        });
    });
}

} // namespace avifgpu
