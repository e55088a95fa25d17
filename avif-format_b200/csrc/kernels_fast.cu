// kernels_fast.cu -- launchers of the tuned float-RGB(A) encode kernels, and the kernel for "no transfer curve".
// EncodeFamilyOf (host_params.cpp) decides which description they serve; anything else takes kernels_generic.cu.  The
// arithmetic is the same pixel_math.cuh; what changes is the work decomposition and where the transcendental work goes:
//   curve with a verified step table (PQ, SMPTE 428)   kernels_fast_flat.cu (RGB), kernels_fast_rgba.cu (RGBA)
//   no curve (clip)                                     EncodeRgbF32ClipKernel below: warp tile = 2 rows x 128 pixels, a lane
//                                                       owns 4 adjacent pixels in both rows (two 2x2 chroma sites, the box
//                                                       filter needs no cross-lane traffic), 3 x LDG.128 per row per lane
//                                                       one tile ahead, persistent grid of 3 CTAs x 8 warps per SM.
#include "kernels_fast_common.cuh"
#include "launch_keys.h"
#include "../../include/avifgpu.h"

#include <cuda_runtime.h>

namespace avifgpu
{

using namespace avifpix;
using namespace fastenc;
using avifmath::LibmTables;

namespace
{

constexpr int kClipThreads = 256;
constexpr int kClipWarps = kClipThreads / 32;
constexpr int kClipBlocksPerSm = 3;

// No transfer curve (AVIFGPU_TRANSFER_CLIP): code = trunc(clamp(v * max)) per sample (WriteHeifImage.cpp:1128-1130), then
// the forward matrix.  No tables, no shared memory; the loads of tile i+1 are issued before tile i's arithmetic.  DEST:
// the avifgpu_source_layout bits of the planes written (StoreTile).  The body of EncodeRgbF32ClipKernel (DEST 0) and of
// EncodeDestRgbF32ClipKernel (the other layouts).
template <int XS, int YS, int DEST>
__device__ __forceinline__ void EncodeRgbF32ClipBody(const FastEncodeParams& p)
{
    const int lane = threadIdx.x & 31;
    const int warpInBlock = threadIdx.x >> 5;
    const int tilesX = (p.width + kTilePixels - 1) / kTilePixels;
    const int tileRows = (p.rowCount + 1) / 2;
    const int tileCount = tilesX * tileRows;
    const int warpCount = static_cast<int>(gridDim.x) * kClipWarps;

    // Tile coordinates advance incrementally (an integer division per tile costs ~24 instructions).
    const int firstTile = static_cast<int>(blockIdx.x) * kClipWarps + warpInBlock;
    const int stepRows = warpCount / tilesX;
    const int stepX = warpCount - stepRows * tilesX;
    int tileRow = firstTile / tilesX;
    int tileX = firstTile - tileRow * tilesX;
    uint4 raw[6];
    auto loadTile = [&](int row, int column, bool valid)
    {
        const int x = column * kTilePixels + lane * 4;
        const int y = row * 2;
        const bool active = valid && x < p.width;
        const bool second = active && (y + 1) < p.rowCount;
        const uint8_t* r0 = p.rows + static_cast<int64_t>(y) * p.rowStride + static_cast<int64_t>(x) * 12;
        const uint8_t* r1 = r0 + p.rowStride;
        const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int q = 0; q < 3; ++q)
        {
            raw[q] = active ? __ldg(reinterpret_cast<const uint4*>(r0 + 16 * q)) : zero;
        }
#pragma unroll
        for (int q = 0; q < 3; ++q)
        {
            raw[3 + q] = second ? __ldg(reinterpret_cast<const uint4*>(r1 + 16 * q)) : zero;
        }
    };
    loadTile(tileRow, tileX, firstTile < tileCount);

    for (int tile = firstTile; tile < tileCount; tile += warpCount)
    {
        const int x0 = tileX * kTilePixels + lane * 4;
        const int y0 = tileRow * 2;
        const bool laneActive = x0 < p.width;
        const bool secondRow = (y0 + 1) < p.rowCount;
        const int currentRow = tileRow;

        float codeF[kValuesPerLane]; // the codes, as the floats the forward matrix consumes
#pragma unroll
        for (int q = 0; q < 6; ++q)
        {
            codeF[4 * q + 0] = CodeToFloat(FloatToCode(__uint_as_float(raw[q].x), p.maxCodeFloat));
            codeF[4 * q + 1] = CodeToFloat(FloatToCode(__uint_as_float(raw[q].y), p.maxCodeFloat));
            codeF[4 * q + 2] = CodeToFloat(FloatToCode(__uint_as_float(raw[q].z), p.maxCodeFloat));
            codeF[4 * q + 3] = CodeToFloat(FloatToCode(__uint_as_float(raw[q].w), p.maxCodeFloat));
        }
        tileRow += stepRows;
        tileX += stepX;
        if (tileX >= tilesX)
        {
            tileX -= tilesX;
            ++tileRow;
        }
        loadTile(tileRow, tileX, tile + warpCount < tileCount);

        if (laneActive)
        {
            const int64_t chromaRow = YS ? currentRow : y0;
            const int64_t chromaColumn = static_cast<int64_t>(XS ? (x0 >> 1) : x0) * 2;
            StoreTile<XS, YS, DEST>(p, codeF, p.planeY + static_cast<int64_t>(y0) * p.strideY + static_cast<int64_t>(x0) * 2,
                                    p.planeCb + chromaRow * p.strideCb + chromaColumn * (SourceInterleaved(DEST) ? 2 : 1),
                                    p.planeCr + chromaRow * p.strideCr + chromaColumn, secondRow);
        }
    }
}

template <int XS, int YS>
__global__ void __launch_bounds__(kClipThreads, kClipBlocksPerSm) EncodeRgbF32ClipKernel(const FastEncodeParams p)
{
    EncodeRgbF32ClipBody<XS, YS, AVIFGPU_SOURCE_PLANAR>(p);
}

// The same into semi-planar and MSB-aligned planes (DEST != 0).
template <int XS, int YS, int DEST>
__global__ void __launch_bounds__(kClipThreads, kClipBlocksPerSm) EncodeDestRgbF32ClipKernel(const FastEncodeParams p)
{
    EncodeRgbF32ClipBody<XS, YS, DEST>(p);
}

template <int XS, int YS, int DEST>
cudaError_t LaunchClipKernel(const FastEncodeParams& fp, int smCount, cudaStream_t stream)
{
    const long long tiles = static_cast<long long>((fp.width + kTilePixels - 1) / kTilePixels) * ((fp.rowCount + 1) / 2);
    if (tiles > 0x7fffffffll)
    {
        return cudaErrorInvalidValue;
    }
    const unsigned grid = GridFor((tiles + kClipWarps - 1) / kClipWarps, static_cast<long long>(smCount) * kClipBlocksPerSm);
    if constexpr (DEST == AVIFGPU_SOURCE_PLANAR)
    {
        EncodeRgbF32ClipKernel<XS, YS><<<grid, kClipThreads, 0, stream>>>(fp);
    }
    else
    {
        EncodeDestRgbF32ClipKernel<XS, YS, DEST><<<grid, kClipThreads, 0, stream>>>(fp);
    }
    return cudaGetLastError();
}

} // namespace

cudaError_t LaunchEncodeRgbF32Interleaved(const EncodeParams& p, Interior inner, void* streamHandle, const LightSink* light)
{
    // The reference's own layout: interleaved RGB codes (WriteHeifImage.cpp:1098-1130), same kernel without the matrix.
    FastEncodeParams fp{};
    fp.rows = static_cast<const uint8_t*>(p.rows);
    fp.rowStride = p.rowStride;
    fp.planeY = static_cast<uint8_t*>(p.plane[0]);
    fp.strideY = p.planeStride[0];
    fp.width = inner.width;
    fp.rowCount = inner.rows;
    fp.pqMultiplier = p.pqMultiplier;
    fp.maxCodeFloat = p.maxCodeFloat;
    fp.maxCode = static_cast<int32_t>(p.maxCode);
    fp.table = *p.curveTable;
    const int curve = p.transfer == AVIFGPU_TRANSFER_PQ ? kCurveLinearToPQ : kCurveLinearToSMPTE428;
    return LaunchFastEncodeFlatInterleaved(fp, curve, SmCountOrDefault(p.smCount), static_cast<cudaStream_t>(streamHandle), light);
}

cudaError_t LaunchEncodeRgbF32Planar(EncodeFamily family, const EncodeParams& p, Interior inner, void* streamHandle, const LightSink* light)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const int curve = p.transfer == AVIFGPU_TRANSFER_PQ ? kCurveLinearToPQ : p.transfer == AVIFGPU_TRANSFER_SMPTE428 ? kCurveLinearToSMPTE428 : kCurveClip;
    FastEncodeParams fp{};
    fp.rows = static_cast<const uint8_t*>(p.rows);
    fp.rowStride = p.rowStride;
    fp.planeY = static_cast<uint8_t*>(p.plane[0]);
    fp.strideY = p.planeStride[0];
    fp.planeCb = static_cast<uint8_t*>(p.plane[1]);
    fp.strideCb = p.planeStride[1];
    fp.planeCr = static_cast<uint8_t*>(p.plane[2]);
    fp.strideCr = p.planeStride[2];
    fp.width = inner.width;
    fp.rowCount = inner.rows;
    fp.pqMultiplier = p.pqMultiplier;
    fp.maxCodeFloat = p.maxCodeFloat;
    fp.maxCode = static_cast<int32_t>(p.maxCode);
    fp.matrix = p.matrix;
    fp.chromaOffset = p.chromaOffset;
    fp.topLeft = p.topLeft;
    if (family != EncodeFamily::RgbF32Clip)
    {
        fp.table = *p.curveTable;
    }
    const int smCount = SmCountOrDefault(p.smCount);
    switch (family)
    {
    case EncodeFamily::RgbaF32Flat:
        fp.planeA = static_cast<uint8_t*>(p.plane[3]);
        fp.strideA = p.planeStride[3];
        fp.premultiply = p.premultiply;
        return LaunchFastEncodeRgba(fp, curve, p.xs, p.ys, p.destLayout, smCount, stream, light);
    case EncodeFamily::RgbF32Flat: return LaunchFastEncodeFlat(fp, curve, p.xs, p.ys, p.destLayout, smCount, stream, light);
    default:
        return WithChroma(p.xs, p.ys, [&](auto xs, auto ys) {
            return WithLayout(p.destLayout, [&](auto dest) { return LaunchClipKernel<xs(), ys(), dest()>(fp, smCount, stream); });
        });
    }
}

} // namespace avifgpu
