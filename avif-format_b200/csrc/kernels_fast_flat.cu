// kernels_fast_flat.cu -- the float RGB -> planar YCbCr encode kernel for curves with a step table in shared memory
// (curve_tables.h): BASELINE config 2, 7680x4320 RGB32f -> 12-bit PQ 4:2:0.
//
//   * one CTA per SM, kFlatWarps warps; the step table (compact one-word entries + first_k, 67 KB at 12 bits; or the
//     two-level table where the compact form does not apply) sits in shared memory next to one 3 KB staging buffer per
//     warp.  The compact table's image is brought in by the copy engine (table_staging.cuh).
//     Measured on the 8K PQ frame (Gpx/s, round 1): 16 warps 238 | 20: 251 | 24: 273 | 28: 278 | 30: 267 (30 leaves 64
//     registers); the kernel is bound by instruction issue and shared-memory wavefronts, so resident warps matter, and
//     the copy engine keeps the per-warp register cost of a fetch at zero;
//   * a warp converts tiles of 2 rows x 128 pixels, walking straight down one tile column (FlatSchedule).  The two
//     1536-byte row segments of a tile are fetched by the copy engine (cp.async.bulk, completion on the warp's own
//     mbarrier) straight into the staging buffer, so the fetch of tile i+1 costs the warp two instructions and no
//     registers and overlaps the matrix and the stores of tile i; the lanes then read their 48 bytes per row with three
//     conflict-free LDS.128;
//   * float -> code: one table look-up per sample (LookupCurveCompact: a 32-bit gather, 12 instructions); samples the
//     look-up flags as possibly inside a fuzzy band (~1.5 %) are resolved by first_k and one bit of the L2-resident band
//     bitmap, up to two samples of a lane at a time; +inf / NaN take the exact glibc-identical evaluation;
//   * forward matrix, quantisation, chroma down-filter and stores: StoreTile (kernels_fast_common.cuh, packed FP32).
#include "kernels_fast_common.cuh"
#include "launch_keys.h"
#include "table_staging.cuh"
#include "../../include/avifgpu.h"

namespace avifgpu
{

using namespace avifpix;
using namespace fastenc;
using namespace staging;
using avifmath::LibmTables;

namespace
{

// The shared-memory layout's sizes (kFlatWarps, FlatFixedBytes, ...) are in kernel_params.h, where the route reads them.
constexpr int kFlatThreads = kFlatWarps * 32;
constexpr int kRowSegmentBytes = kTilePixels * 12; // one tile row of RGB32f; a warp stages both rows, linear
static_assert(kFlatStageBytesPerWarp == 2 * kRowSegmentBytes, "a warp's staging buffer holds both rows of its tile");
constexpr int kRowSegmentWords = kRowSegmentBytes / 4;
constexpr int kTableBarrierSlot = kFlatSharedBarriers / 8 - 1; // kFlatWarps x 8 bytes, padded; the last slot is the table's barrier
static_assert(kFlatWarps <= kTableBarrierSlot, "the warps' barriers and the table's share kFlatSharedBarriers");

// How the persistent warps share the tiles, worked out once on the host (the grid is known at launch).  The image is cut
// into `items` = tilesX columns x `segments` runs of consecutive tile rows (run lengths differ by at most one), one item
// per warp when the grid has at least tilesX warps -- so a warp walks straight down one tile column and its per-tile
// bookkeeping is four pointer increments by launch constants: no column wrap, no division, no per-tile schedule state.
struct FlatSchedule
{
    int32_t tilesX, tileRows, warpCount;
    int32_t segments, items;          // items = tilesX * segments
    int32_t segmentRows, longSegments; // segment s holds segmentRows (+ 1 if s < longSegments) tile rows
    int32_t lastColumnBytes;          // row-segment bytes of the last tile column (width need not be a multiple of 128)
    int32_t unpairedTileRow;          // tile row whose second image row does not exist (odd row count), or -1
};

// One lane of the (converged) warp.
__device__ __forceinline__ bool ElectOne()
{
    uint32_t elected;
    asm volatile("{ .reg .pred p; elect.sync _|p, 0xffffffff; selp.u32 %0, 1, 0, p; }" : "=r"(elected));
    return elected != 0;
}

// Which step table a kernel stages.  kTableTwoLevel: the per-binade two-level table (curves whose steps are too dense
// for one bucket size, e.g. 12-bit SMPTE 428); its rare in-band samples take the exact evaluation in place.
// kTableCompact: the compact one-word entries (curve_tables.h "Compact entries") + the first_k array + band bitmap.
// kTableCompact14: the same with flatShift = 14 known at compile time (12-bit PQ).
constexpr int kTableTwoLevel = 1;
constexpr int kTableCompact = 2;
constexpr int kTableCompact14 = 3;

// INTERLEAVED = 1: the reference's own output layout (heif_channel_interleaved RGB, WriteHeifImage.cpp:1098-1130) -- the
// codes are stored as they are, 3 x uint16 per pixel into plane Y's buffer, no matrix (XS = YS = 0 then).
// DEST: the avifgpu_source_layout bits of the YCbCr planes written (StoreTile); with interleaved chroma the lane's chroma
// pointer walks plane 1 in steps of twice the bytes.  The body of EncodeRgbF32FlatKernel (DEST 0) and of
// EncodeDestRgbF32FlatKernel (the other layouts).
// LIGHT = 1: also the content light level of the tile's codes (light_level.cuh), the body of EncodeLightRgbF32FlatKernel.
template <int CURVE, int XS, int YS, int TABLE, int INTERLEAVED, int DEST, int LIGHT = 0>
__device__ __forceinline__ void EncodeRgbF32FlatBody(const FastEncodeParams& p, const FlatSchedule& schedule, const LightSink& light = {})
{
    constexpr bool kCompact = TABLE != kTableTwoLevel;
    constexpr int kCompactShift = TABLE == kTableCompact14 ? 14 : 0;
    extern __shared__ __align__(128) uint8_t sharedBytes[];
    uint64_t* libmStorage = reinterpret_cast<uint64_t*>(sharedBytes);
    uint64_t* barriers = reinterpret_cast<uint64_t*>(sharedBytes + kSharedLibm);
    uint8_t* stageAll = sharedBytes + kSharedLibm + kFlatSharedBarriers;
    uint32_t* compactEntries = reinterpret_cast<uint32_t*>(sharedBytes + FlatFixedBytes());  // compact: the entries ...
    const uint32_t* firstBits = compactEntries + ((p.table.flatCount + 3) & ~3);             // ... then first_k per code
    uint2* octaves = reinterpret_cast<uint2*>(sharedBytes + FlatFixedBytes());               // two-level: 256 entries ...
    uint32_t* bucketWords = reinterpret_cast<uint32_t*>(sharedBytes + FlatFixedBytes() + kFlatOctaveBytes); // ... then the bucket words

    const int lane = threadIdx.x & 31;
    // Read through a shuffle so the compiler knows the warp index (and everything derived from it: tile coordinates,
    // copy addresses) is warp-uniform and keeps it in the uniform datapath, which the bulk-copy instruction needs.
    const int warpInBlock = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
    const uint32_t barrier = SharedAddress(barriers + warpInBlock);
    uint32_t* stage = reinterpret_cast<uint32_t*>(stageAll + warpInBlock * kFlatStageBytesPerWarp);
    const uint32_t stageAddress = SharedAddress(stage);
    const uint32_t* myStage = stage + lane * 12; // row 0; row 1 is kRowSegmentWords further

    const int tilesX = schedule.tilesX;
    const int warpCount = schedule.warpCount;
    // Run lengths differ by one tile row.  The items are dealt round-robin over the CTAs (item = warp * CTAs + CTA), so every
    // CTA gets the same mix of long and short runs and the extra round is spread over every SM rather than run by a
    // fraction of them.
    const int firstItem = warpInBlock * static_cast<int>(gridDim.x) + static_cast<int>(blockIdx.x);
    constexpr int kChromaRowsPerTile = YS ? 1 : 2;
    constexpr int kChromaPairs = SourceInterleaved(DEST) ? 2 : 1; // interleaved: Cb, Cr pairs in plane 1
    constexpr int kChromaTileBytes = (XS ? kTilePixels : 2 * kTilePixels) * kChromaPairs;

    // An item's tile column and its run of tile rows [rowBegin, rowEnd).
    auto itemRows = [&](int item, int& column, int& rowBegin, int& rowEnd)
    {
        const int segment = item / tilesX;
        column = item - segment * tilesX;
        rowBegin = segment * schedule.segmentRows + min(segment, schedule.longSegments);
        rowEnd = rowBegin + schedule.segmentRows + (segment < schedule.longSegments ? 1 : 0);
    };
    // One elected lane asks the copy engine for a tile's row segments (warp-uniform arguments).
    auto fetchTile = [&](int row, uint32_t bytes, int64_t offset)
    {
        const bool second = row != schedule.unpairedTileRow;
        const uint8_t* source = p.rows + offset;
        BarrierExpect(barrier, second ? 2u * bytes : bytes);
        BulkCopyToShared(stageAddress, source, bytes, barrier);
        if (second)
        {
            BulkCopyToShared(stageAddress + kRowSegmentBytes, source + p.rowStride, bytes, barrier);
        }
    };
    auto columnBytes = [&](int column) { return column == tilesX - 1 ? static_cast<uint32_t>(schedule.lastColumnBytes) : static_cast<uint32_t>(kRowSegmentBytes); };
    auto sourceOffsetOf = [&](int row, int column) { return static_cast<int64_t>(row) * 2 * p.rowStride + static_cast<int64_t>(column) * kRowSegmentBytes; };

    if (kCompact && threadIdx.x == 0)
    {
        BeginTableImageCopy(p.table, compactEntries, barriers + kTableBarrierSlot); // table_staging.cuh
    }
    if (ElectOne())
    {
        BarrierInit(barrier, 1);
        BarrierInitFence();
        if (firstItem < schedule.items)
        {
            int column, rowBegin, rowEnd;
            itemRows(firstItem, column, rowBegin, rowEnd);
            if (rowBegin < rowEnd)
            {
                fetchTile(rowBegin, columnBytes(column), sourceOffsetOf(rowBegin, column)); // in flight while the table is staged
            }
        }
    }

    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    if (!kCompact) // the compact image is in flight (above)
    {
        for (int i = threadIdx.x; i < 256; i += blockDim.x)
        {
            octaves[i] = p.table.octaves[i];
        }
        for (int i = threadIdx.x; i < p.table.bucketCount; i += blockDim.x)
        {
            bucketWords[i] = p.table.buckets[i];
        }
    }
    __syncthreads(); // the libm tables, the barriers' initialisation
    if (kCompact)
    {
        WaitTableImage(barriers + kTableBarrierSlot);
    }

    const uint32_t flatShift = p.table.flatShift;
    const int32_t negativeLow = -static_cast<int32_t>(p.table.flatLow);
    const int32_t span = static_cast<int32_t>(p.table.flatHigh - p.table.flatLow);
    const uint32_t bandStrideLog2 = p.table.bandStrideLog2;
    const uint32_t* __restrict__ bandBits = p.table.bandBits;
    const uint32_t compactTopShift = 32u - flatShift;
    const uint32_t compactCodeMask = p.table.compactCodeMask;
    const uint32_t compactMagic = p.table.compactMagic;
    uint32_t parity = 0;
    LightTally tally{ 0u, 0ull };

#pragma unroll 1
    for (int item = firstItem; item < schedule.items; item += warpCount)
    {
        int column, rowBegin, rowEnd;
        itemRows(item, column, rowBegin, rowEnd);
        if (item != firstItem && rowBegin < rowEnd && ElectOne())
        {
            fetchTile(rowBegin, columnBytes(column), sourceOffsetOf(rowBegin, column)); // only grids smaller than tilesX warps get here
        }
        const uint32_t tileBytes = columnBytes(column);
        const bool laneActive = column * kTilePixels + lane * 4 < p.width;
        int64_t sourceOffset = sourceOffsetOf(rowBegin, column);
        uint8_t* yPointer = p.planeY + static_cast<int64_t>(rowBegin) * 2 * p.strideY +
                            (INTERLEAVED ? static_cast<int64_t>(column) * (6 * kTilePixels) + lane * 24 : static_cast<int64_t>(column) * (2 * kTilePixels) + lane * 8);
        uint8_t* cbPointer = p.planeCb + static_cast<int64_t>(rowBegin) * kChromaRowsPerTile * p.strideCb + static_cast<int64_t>(column) * kChromaTileBytes + lane * (XS ? 4 : 8) * kChromaPairs;
        uint8_t* crPointer = p.planeCr + static_cast<int64_t>(rowBegin) * kChromaRowsPerTile * p.strideCr + static_cast<int64_t>(column) * kChromaTileBytes + lane * (XS ? 4 : 8);

#pragma unroll 1
    for (int tileRow = rowBegin; tileRow < rowEnd; ++tileRow)
    {
        const bool secondRow = tileRow != schedule.unpairedTileRow;
        sourceOffset += 2 * p.rowStride; // the next tile of this column

        BarrierWait(barrier, parity);
        parity ^= 1u;

        // ---- float -> code through the exact step table ------------------------------------------------------------
        float codeF[kValuesPerLane]; // the codes, as the floats the forward matrix consumes
        uint32_t bandMask = 0;
        int32_t largest = 0; // max over the samples as signed integers: > 0x7f7fffff <=> a +inf / NaN is among them
#pragma unroll
        for (int q = 0; q < 6; ++q)
        {
            const uint4 w = *reinterpret_cast<const uint4*>(myStage + (q / 3) * kRowSegmentWords + (q % 3) * 4);
            const uint32_t bits[4] = { w.x, w.y, w.z, w.w };
#pragma unroll
            for (int e = 0; e < 4; ++e)
            {
                const int j = 4 * q + e;
                bool inBand;
                if (kCompact)
                {
                    uint32_t entry;
                    codeF[j] = LookupCurveCompact<kCompactShift>(bits[e], compactEntries, flatShift, negativeLow, span, compactTopShift, compactCodeMask,
                                                                 compactMagic, inBand, entry);
                }
                else
                {
                    codeF[j] = CodeToFloat(LookupCurveCode(bits[e], octaves, bucketWords, inBand)); // reports +inf / NaN in band itself
                }
                asm("{ .reg .pred p; setp.ne.u32 p, %1, 0; @p or.b32 %0, %0, %2; }" : "+r"(bandMask) : "r"(static_cast<uint32_t>(inBand)), "r"(1u << j));
            }
            if (kCompact)
            {
                largest = max(largest, __vimax3_s32(static_cast<int32_t>(w.x), static_cast<int32_t>(w.y), static_cast<int32_t>(w.z)));
                largest = max(largest, static_cast<int32_t>(w.w));
            }
        }

        // ---- in-band samples: one bit of the band bitmap each, two loads in flight per lane ---------------------------
        auto stagedBits = [&](int j) { return myStage[j + (j >= 12 ? kRowSegmentWords - 12 : 0)]; };
        uint32_t lowerMask = 0; // samples whose exact code is one below the table's
        if (kCompact)
        {
            // flagged samples: which step, how far above its first_k, one bit of the band bitmap -- two at a time
            uint32_t pending = bandMask;
            while (pending != 0)
            {
                uint32_t word[2] = { 0xffffffffu, 0xffffffffu }, index[2] = { 0u, 0u }, sampleBit[2] = { 0u, 0u };
#pragma unroll
                for (int u = 0; u < 2; ++u)
                {
                    if (pending != 0)
                    {
                        const int j = __ffs(static_cast<int>(pending)) - 1;
                        pending &= pending - 1;
                        const uint32_t bits = stagedBits(j);
                        const int32_t bucket = __viaddmin_s32_relu(static_cast<int32_t>(bits) >> flatShift, negativeLow, span);
                        const uint32_t entry = compactEntries[bucket];
                        const uint32_t k = ((entry & compactCodeMask) >> kCompactLenBits) + ((entry >> compactTopShift) != 0 ? 1u : 0u);
                        const uint32_t distance = bits - firstBits[k];
                        if (k != 0 && distance < (1u << bandStrideLog2)) // else flagged by the superset test only: the table's code stands
                        {
                            index[u] = (k << bandStrideLog2) + distance;
                            word[u] = __ldg(bandBits + (index[u] >> 5));
                            sampleBit[u] = 1u << j;
                        }
                    }
                }
#pragma unroll
                for (int u = 0; u < 2; ++u)
                {
                    if (((word[u] >> (index[u] & 31u)) & 1u) == 0)
                    {
                        lowerMask |= sampleBit[u];
                    }
                }
            }
        }

        // ---- +inf / NaN (never in real frames): the exact evaluation, lane by lane ------------------------------------
        if (__any_sync(0xffffffffu, kCompact ? largest > 0x7f7fffff : bandMask != 0))
        {
            for (int j = 0; j < kValuesPerLane; ++j)
            {
                const uint32_t bits = stagedBits(j);
                if (kCompact ? static_cast<int32_t>(bits) > 0x7f7fffff : ((bandMask >> j) & 1u) != 0)
                {
                    const float exact = CodeToFloat(ExactCurveCode<CURVE>(__uint_as_float(bits), p.pqMultiplier, p.maxCodeFloat, t));
#pragma unroll
                    for (int slot = 0; slot < kValuesPerLane; ++slot)
                    {
                        if (slot == j)
                        {
                            codeF[slot] = exact;
                        }
                    }
                }
            }
        }

        // The staging buffer is free: fetch the next tile while this one goes through the matrix and the stores.
        __syncwarp();
        if (tileRow + 1 < rowEnd && ElectOne())
        {
            fetchTile(tileRow + 1, tileBytes, sourceOffset);
        }

#pragma unroll
        for (int j = 0; j < kValuesPerLane; ++j)
        {
            if (lowerMask & (1u << j))
            {
                codeF[j] -= 1.0f;
            }
        }

        if (LIGHT && laneActive)
        {
#pragma unroll
            for (int pixel = 0; pixel < 8; ++pixel)
            {
                if (pixel < 4 || secondRow)
                {
                    const uint32_t k = __float2uint_rz(fmaxf(fmaxf(codeF[3 * pixel], codeF[3 * pixel + 1]), codeF[3 * pixel + 2]));
                    TallyCode(tally, k, __ldg(light.levels + k));
                }
            }
        }

        if (laneActive)
        {
            if (INTERLEAVED)
            {
                // 4 pixels x 3 codes per row = 24 bytes: three 64-bit stores
#pragma unroll
                for (int r = 0; r < 2; ++r)
                {
                    if (r == 1 && !secondRow) break;
                    uint32_t words[6];
#pragma unroll
                    for (int w = 0; w < 6; ++w)
                    {
                        words[w] = __float2uint_rz(codeF[12 * r + 2 * w]) | (__float2uint_rz(codeF[12 * r + 2 * w + 1]) << 16);
                    }
                    uint2* target = reinterpret_cast<uint2*>(yPointer + r * p.strideY);
                    __stcs(target, make_uint2(words[0], words[1]));
                    __stcs(target + 1, make_uint2(words[2], words[3]));
                    __stcs(target + 2, make_uint2(words[4], words[5]));
                }
            }
            else
            {
                StoreTile<XS, YS, DEST>(p, codeF, yPointer, cbPointer, crPointer, secondRow);
            }
        }
        yPointer += 2 * p.strideY;
        cbPointer += kChromaRowsPerTile * p.strideCb;
        crPointer += kChromaRowsPerTile * p.strideCr;
    }
    }
    if (LIGHT)
    {
        FlushLightTally(tally, LaunchPixelsForFirstWarp(static_cast<uint64_t>(p.width) * p.rowCount), light.acc);
    }
}

template <int CURVE, int XS, int YS, int TABLE, int INTERLEAVED>
__global__ void __launch_bounds__(kFlatThreads, 1) EncodeRgbF32FlatKernel(const FastEncodeParams p, const FlatSchedule schedule)
{
    EncodeRgbF32FlatBody<CURVE, XS, YS, TABLE, INTERLEAVED, AVIFGPU_SOURCE_PLANAR>(p, schedule);
}

// The same into semi-planar and MSB-aligned planes (DEST != 0).
template <int CURVE, int XS, int YS, int TABLE, int DEST>
__global__ void __launch_bounds__(kFlatThreads, 1) EncodeDestRgbF32FlatKernel(const FastEncodeParams p, const FlatSchedule schedule)
{
    EncodeRgbF32FlatBody<CURVE, XS, YS, TABLE, 0, DEST>(p, schedule);
}

// The same with the content light level (every layout; PQ only).
template <int CURVE, int XS, int YS, int TABLE, int INTERLEAVED, int DEST>
__global__ void __launch_bounds__(kFlatThreads, 1) EncodeLightRgbF32FlatKernel(const FastEncodeParams p, const FlatSchedule schedule, const LightSink light)
{
    EncodeRgbF32FlatBody<CURVE, XS, YS, TABLE, INTERLEAVED, DEST, 1>(p, schedule, light);
}

template <int CURVE, int XS, int YS, int TABLE, int INTERLEAVED, int DEST, int LIGHT>
constexpr auto FlatKernelFor()
{
    if constexpr (LIGHT)
    {
        return EncodeLightRgbF32FlatKernel<CURVE, XS, YS, TABLE, INTERLEAVED, DEST>;
    }
    else if constexpr (DEST == AVIFGPU_SOURCE_PLANAR)
    {
        return EncodeRgbF32FlatKernel<CURVE, XS, YS, TABLE, INTERLEAVED>;
    }
    else
    {
        return EncodeDestRgbF32FlatKernel<CURVE, XS, YS, TABLE, DEST>;
    }
}

template <int CURVE, int XS, int YS, int TABLE, int INTERLEAVED = 0, int DEST = AVIFGPU_SOURCE_PLANAR, int LIGHT = 0>
cudaError_t LaunchFlatKernel(const FastEncodeParams& fp, int smCount, cudaStream_t stream, const LightSink* light = nullptr)
{
    const size_t shared = static_cast<size_t>(FlatFixedBytes()) + FlatTableBytes(fp.table, TABLE == kTableTwoLevel);
    static std::atomic<uint64_t> configuredDevices{ 0 }; // per instantiation
    {
        const cudaError_t e = AllowDynamicShared(FlatKernelFor<CURVE, XS, YS, TABLE, INTERLEAVED, DEST, LIGHT>(), kSharedLimit, configuredDevices);
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
    long long blocks = (tiles + kFlatWarps - 1) / kFlatWarps;
    if (blocks > smCount)
    {
        blocks = smCount;
    }
    FlatSchedule schedule{};
    schedule.tilesX = (fp.width + kTilePixels - 1) / kTilePixels;
    schedule.tileRows = (fp.rowCount + 1) / 2;
    schedule.warpCount = static_cast<int32_t>(blocks) * kFlatWarps;
    schedule.segments = schedule.warpCount / schedule.tilesX;
    if (schedule.segments < 1) schedule.segments = 1;
    if (schedule.segments > schedule.tileRows) schedule.segments = schedule.tileRows;
    schedule.items = schedule.tilesX * schedule.segments;
    schedule.segmentRows = schedule.tileRows / schedule.segments;
    schedule.longSegments = schedule.tileRows % schedule.segments;
    schedule.lastColumnBytes = (fp.width - (schedule.tilesX - 1) * kTilePixels) * 12;
    schedule.unpairedTileRow = (fp.rowCount & 1) ? fp.rowCount / 2 : -1;
    if constexpr (LIGHT)
    {
        FlatKernelFor<CURVE, XS, YS, TABLE, INTERLEAVED, DEST, LIGHT>()<<<static_cast<unsigned>(blocks), kFlatThreads, shared, stream>>>(fp, schedule, *light);
    }
    else
    {
        FlatKernelFor<CURVE, XS, YS, TABLE, INTERLEAVED, DEST, LIGHT>()<<<static_cast<unsigned>(blocks), kFlatThreads, shared, stream>>>(fp, schedule);
    }
    return cudaGetLastError();
}

} // namespace

// The reference's interleaved RGB layout through the same kernel (fp.planeY / strideY = the interleaved buffer).
cudaError_t LaunchFastEncodeFlatInterleaved(const FastEncodeParams& fp, int curve, int smCount, cudaStream_t stream, const LightSink* light)
{
    if (FlatCompactFits(fp.table))
    {
        if (curve == kCurveLinearToPQ && light != nullptr)
        {
            return fp.table.flatShift == 14 ? LaunchFlatKernel<kCurveLinearToPQ, 0, 0, kTableCompact14, 1, AVIFGPU_SOURCE_PLANAR, 1>(fp, smCount, stream, light)
                                            : LaunchFlatKernel<kCurveLinearToPQ, 0, 0, kTableCompact, 1, AVIFGPU_SOURCE_PLANAR, 1>(fp, smCount, stream, light);
        }
        if (curve == kCurveLinearToPQ)
        {
            return fp.table.flatShift == 14 ? LaunchFlatKernel<kCurveLinearToPQ, 0, 0, kTableCompact14, 1>(fp, smCount, stream)
                                            : LaunchFlatKernel<kCurveLinearToPQ, 0, 0, kTableCompact, 1>(fp, smCount, stream);
        }
        return LaunchFlatKernel<kCurveLinearToSMPTE428, 0, 0, kTableCompact, 1>(fp, smCount, stream);
    }
    if (light != nullptr)
    {
        return cudaErrorInvalidValue; // LaunchEncode sends a light-level call without the compact table to the generic kernel
    }
    if (curve == kCurveLinearToPQ) return LaunchFlatKernel<kCurveLinearToPQ, 0, 0, kTableTwoLevel, 1>(fp, smCount, stream);
    return LaunchFlatKernel<kCurveLinearToSMPTE428, 0, 0, kTableTwoLevel, 1>(fp, smCount, stream);
}

// The table's form picks the instantiation: the compact form with its bitmap when it fits, else the two-level form.  The
// planar layout keeps every (curve, table) pair.  The other layouts (DEST != 0, picked by WithLayout) instantiate only the
// pairs the tables built for 10/12-bit encodes reach (DESIGN.md 4.2): PQ with the compact table (kTableCompact14 for
// flatShift 14, as at 12 bits, kTableCompact for any other shift), SMPTE 428 with the compact table (10 bits) or the
// two-level one (12 bits, the only form built there).  A PQ table without its compact form has not been built for any
// configuration so far; EncodeFamilyOf leaves such a description with another layout to the generic kernel, and LaunchEncode
// a light-level call (`light` set: the LIGHT = 1 instantiations, PQ with the compact table only) in any layout.
cudaError_t LaunchFastEncodeFlat(const FastEncodeParams& fp, int curve, int xs, int ys, int dest, int smCount, cudaStream_t stream, const LightSink* light)
{
    return WithChroma(xs, ys, [&](auto XS, auto YS) {
        return WithLayout(dest, [&](auto DEST) {
            if (light != nullptr)
            {
                if (curve != kCurveLinearToPQ || !FlatCompactFits(fp.table))
                {
                    return cudaErrorInvalidValue; // LaunchEncode said no: the launcher does not get here
                }
                return fp.table.flatShift == 14 ? LaunchFlatKernel<kCurveLinearToPQ, XS(), YS(), kTableCompact14, 0, DEST(), 1>(fp, smCount, stream, light)
                                                : LaunchFlatKernel<kCurveLinearToPQ, XS(), YS(), kTableCompact, 0, DEST(), 1>(fp, smCount, stream, light);
            }
            if (FlatCompactFits(fp.table))
            {
                if (curve == kCurveLinearToPQ)
                {
                    return fp.table.flatShift == 14 ? LaunchFlatKernel<kCurveLinearToPQ, XS(), YS(), kTableCompact14, 0, DEST()>(fp, smCount, stream)
                                                    : LaunchFlatKernel<kCurveLinearToPQ, XS(), YS(), kTableCompact, 0, DEST()>(fp, smCount, stream);
                }
                return LaunchFlatKernel<kCurveLinearToSMPTE428, XS(), YS(), kTableCompact, 0, DEST()>(fp, smCount, stream);
            }
            if constexpr (DEST() == AVIFGPU_SOURCE_PLANAR)
            {
                if (curve == kCurveLinearToPQ) return LaunchFlatKernel<kCurveLinearToPQ, XS(), YS(), kTableTwoLevel>(fp, smCount, stream);
            }
            else if (curve == kCurveLinearToPQ)
            {
                return cudaErrorInvalidValue; // EncodeFamilyOf said no: the launcher does not get here
            }
            return LaunchFlatKernel<kCurveLinearToSMPTE428, XS(), YS(), kTableTwoLevel, 0, DEST()>(fp, smCount, stream);
        });
    });
}

} // namespace avifgpu
