// kernels_batch.cu -- many small images per launch, for both batch APIs.  A 512 x 512 image is 2 MB of traffic, well
// under a microsecond of HBM time, so one launch per image is bound by the launch and the grid's ramp and drain.  Here
// one launch walks the units of every image of a batch:
//
//   EncodeRgbIntBatchKernel       the aligned interiors, with EncodeRgbIntGroup (int_units.cuh) -- the single-image
//                                 tuned kernel's own group code; a warp takes one unit (256 pixels of one row or 4:2:0 row
//                                 pair, 8 per lane) at a time, persistent over the concatenated unit space;
//   EncodePlanarBatchKernel       the windows -- right strips, odd last 4:2:0 rows, and whole images the tuned kernel does
//                                 not take -- with EncodePlanarSite (generic_units.cuh), the generic kernel's own site
//                                 code; a CTA takes one run of 256 chroma sites at a time;
//   DecodeYccToRgbIntBatchKernel  the decode interiors, with LoadYccUnit / ExpandYccUnit / StoreYccUnit (int_units.cuh);
//                                 the unorm -> float tables are staged once per CTA for the whole batch (one description);
//   DecodeYccToRgbF32BatchKernel  the float-host decode interiors, with LookUpLuma / ChromaSiteTerms / ConvertRows
//                                 (float_units.cuh); a warp takes one 128-pixel tile of a row (4:2:0 row pair) at a time,
//                                 and the libm, log2 and unorm tables are staged once per CTA for the whole batch;
//   DecodePlanarRgbIntBatchKernel the planar-RGB decode interiors into 8/16-bit hosts, with LoadStreamGroup /
//                                 ConvertRgbGroup (stream_units.cuh); a warp takes one unit (256 pixels of one row, 8 per
//                                 lane) at a time;
//   TableDecodeF32BatchKernel     the planar-RGB decode interiors into 32-bit hosts, with TableDecodeGroup
//                                 (float_units.cuh), in the same units; the libm tables and every code's curve (and alpha)
//                                 entry are staged once per CTA for the whole batch, not once per CTA per image;
//   DecodeBatchKernel             the decode windows, with DecodeChunkPixel (generic_units.cuh).
//   EncodeLightF32BatchKernel     the light-level float encode interiors (RGB(A)32f -> planar YCbCr through the PQ compact
//                                 step table, the content light level of every image on the side); a warp takes one
//                                 128-pixel tile of a row (4:2:0 row pair) at a time, and the libm tables and the step
//                                 table are staged once per CTA for the whole batch;
//   EncodeLightPlanarBatchKernel  the light-level encode windows, with EncodePlanarSite's light-level form.
//
// Each is a template on where its records come from:
//   ChunkSource      a host-described chunk (PlanEncodeBatch / PlanDecodeBatch): the records and their unit total travel
//                    in the kernel parameter (__grid_constant__) and the grid is sized to the units.  A worker's units
//                    increase, so it finds each unit's record by walking forward through the records' first units.
//   WorkspaceSource  a device-described batch: PlanIndirectKernel writes the records, their first units and the totals
//                    into the workspace when the work runs.  The host does not know how much work there is, so the grid
//                    is the chunk launchers' cap and a CTA with no unit returns before it stages anything; a worker finds
//                    its unit's record with a binary search (FindRecord), starting after the record of its previous unit.
// Either way the search is once per unit and warp- (CTA-) uniform, never per pixel.
// Which instantiation a description takes is the family's picker's decision (launch_keys.h), as in the single-image launchers.
#include "batch_plan.h"
#include "float_units.cuh"
#include "generic_units.cuh"
#include "int_units.cuh"
#include "kernel_params.h"
#include "kernels_fast_common.cuh"
#include "launch_keys.h"
#include "stream_units.cuh"
#include "table_staging.cuh"
#include "../../include/avifgpu.h"

#include <climits>

#include <cuda_runtime.h>

namespace avifgpu
{

namespace
{

constexpr int kWarps = kRgbThreads / 32;
constexpr int kPlanThreads = 1024;

// The record that owns `unit`, walking forward from `record` (units only increase along a worker's walk).
template <int N>
__device__ __forceinline__ int RecordOfUnit(const BatchRecord (&records)[N], int count, int record, long long unit)
{
    while (record + 1 < count && unit >= records[record + 1].firstUnit)
    {
        ++record;
    }
    return record;
}

// The records of one host-described chunk, by value.  `shared` carries the description (its pointers, strides and sizes
// are unused); N is kBatchChunkImages interiors or twice as many windows.
template <typename Shared, int N>
struct ChunkSource
{
    Shared shared;
    int32_t count;
    int64_t units;
    BatchRecord record[N];

    struct Walk
    {
        const ChunkSource& s;
        __device__ __forceinline__ explicit Walk(const ChunkSource& source) : s(source) {}
        __device__ __forceinline__ long long Units() const { return s.units; }
        __device__ __forceinline__ bool Idle(long long) const { return false; } // the grid is sized to the units
        __device__ __forceinline__ int Count() const { return s.count; }
        __device__ __forceinline__ int Find(int, int record, long long unit) const { return RecordOfUnit(s.record, s.count, record, unit); }
        __device__ __forceinline__ const BatchRecord& Record(int record) const { return s.record[record]; }
    };
};

// The workspace seen by the kernels.
struct IndirectView
{
    IndirectHeader* header;
    int64_t* interiorFirst;
    int64_t* windowFirst;
    BatchRecord* interior;
    BatchRecord* window;

    __device__ __forceinline__ IndirectView(void* workspace, int maxCount)
    {
        uint8_t* base = static_cast<uint8_t*>(workspace);
        const IndirectLayout l = IndirectWorkspaceLayout(maxCount);
        header = reinterpret_cast<IndirectHeader*>(base);
        interiorFirst = reinterpret_cast<int64_t*>(base + l.interiorFirst);
        windowFirst = reinterpret_cast<int64_t*>(base + l.windowFirst);
        interior = reinterpret_cast<BatchRecord*>(base + l.interior);
        window = reinterpret_cast<BatchRecord*>(base + l.window);
    }
};

// The interior (WINDOWS = 0) or window records of a device-described batch, in its workspace.
template <typename Shared, int WINDOWS>
struct WorkspaceSource
{
    Shared shared;
    void* workspace;
    int32_t maxCount;

    struct Walk
    {
        IndirectView w;
        long long units;
        __device__ __forceinline__ explicit Walk(const WorkspaceSource& source)
            : w(source.workspace, source.maxCount), units(WINDOWS ? w.header->windowUnits : w.header->interiorUnits)
        {
        }
        __device__ __forceinline__ long long Units() const { return units; }
        __device__ __forceinline__ bool Idle(long long firstUnit) const { return firstUnit >= units; } // no unit for this CTA
        __device__ __forceinline__ int Count() const { return WINDOWS ? 2 * w.header->count : w.header->count; }
        __device__ __forceinline__ int Find(int count, int record, long long unit) const
        {
            return FindRecord(WINDOWS ? w.windowFirst : w.interiorFirst, count, record, unit);
        }
        __device__ __forceinline__ const BatchRecord& Record(int record) const { return (WINDOWS ? w.window : w.interior)[record]; }
    };
};

// The records of a light-level launch, with the caller's image of each record and the sink its statistic goes to.  A host
// chunk carries its records' images (BatchChunk::imageIndex / windowImage); in the workspace, interior i and windows 2i,
// 2i + 1 are image i's.
template <typename Shared, int N>
struct LightChunkSource : ChunkSource<Shared, N>
{
    int32_t image[N];
    LightSink light;

    struct Walk : ChunkSource<Shared, N>::Walk
    {
        const int32_t* image;
        __device__ __forceinline__ explicit Walk(const LightChunkSource& source) : ChunkSource<Shared, N>::Walk(source), image(source.image) {}
        __device__ __forceinline__ int ImageOf(int record) const { return image[record]; }
    };
};

template <typename Shared, int WINDOWS>
struct LightWorkspaceSource : WorkspaceSource<Shared, WINDOWS>
{
    LightSink light;

    struct Walk : WorkspaceSource<Shared, WINDOWS>::Walk
    {
        __device__ __forceinline__ explicit Walk(const LightWorkspaceSource& source) : WorkspaceSource<Shared, WINDOWS>::Walk(source) {}
        __device__ __forceinline__ int ImageOf(int record) const { return WINDOWS ? record >> 1 : record; }
    };
};

// A light-level worker's statistic and the image it belongs to.  It goes into that image's accumulator (FlushLightTally,
// the whole warp converged) when the worker's next unit belongs to another image, and at exit.  `pixels` is the pixel
// count of the records whose first unit the worker converted: every record's first unit is converted by exactly one
// worker, and an image's records cover it exactly once, so each image's count is added once.
struct ImageTally
{
    int image = -1;
    LightTally tally{ 0u, 0ull };
    uint64_t pixels = 0;

    __device__ __forceinline__ void Flush(avifgpu_light_level* acc) const
    {
        if (image >= 0)
        {
            FlushLightTally(tally, pixels, acc + image);
        }
    }
    __device__ __forceinline__ void Switch(int owner, avifgpu_light_level* acc)
    {
        if (owner != image)
        {
            Flush(acc);
            image = owner;
            tally = LightTally{ 0u, 0ull };
            pixels = 0;
        }
    }
};

using RgbIntChunk = ChunkSource<Rgb16Params, kBatchChunkImages>;
using PlanarChunk = ChunkSource<EncodeParams, 2 * kBatchChunkImages>;
using YccIntChunk = ChunkSource<IntDecodeParams, kBatchChunkImages>;
using DecodeEdgeChunk = ChunkSource<DecodeParams, 2 * kBatchChunkImages>;
using YccF32Chunk = ChunkSource<FastDecodeParams, kBatchChunkImages>;
using PlanarRgbIntChunk = ChunkSource<StreamDecodeParams, kBatchChunkImages>;
using PlanarRgbF32Chunk = ChunkSource<TableDecodeParams, kBatchChunkImages>;

// CUDA 12.1+ on Volta and later: at most 32764 bytes of kernel parameters.
static_assert(sizeof(RgbIntChunk) <= 32764 && sizeof(PlanarChunk) <= 32764 && sizeof(YccIntChunk) <= 32764 && sizeof(DecodeEdgeChunk) <= 32764,
              "a chunk must fit one kernel parameter block");
static_assert(sizeof(YccF32Chunk) <= 32764, "a float decode chunk must fit one kernel parameter block");
static_assert(sizeof(PlanarRgbIntChunk) <= 32764 && sizeof(PlanarRgbF32Chunk) <= 32764, "a planar-RGB decode chunk must fit one kernel parameter block");
using LightF32Chunk = LightChunkSource<fastenc::FastEncodeParams, kBatchChunkImages>;
using LightEdgeChunk = LightChunkSource<EncodeParams, 2 * kBatchChunkImages>;
static_assert(sizeof(LightF32Chunk) <= 32764 && sizeof(LightEdgeChunk) <= 32764, "a light-level chunk must fit one kernel parameter block");
static_assert(kF32DecodeThreads == kRgbThreads && kStreamThreads == kRgbThreads && kTableThreads == kRgbThreads, "the batched kernels share kWarps");

// Block-wide exclusive scan of a pair of counts over kPlanThreads threads; every thread gets the block's totals too.
__device__ __forceinline__ void ScanPair(long long a, long long b, long long& beforeA, long long& beforeB, long long& totalA, long long& totalB)
{
    __shared__ long long warpA[kPlanThreads / 32], warpB[kPlanThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long sumA = a, sumB = b;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1)
    {
        const long long upA = __shfl_up_sync(0xffffffffu, sumA, d);
        const long long upB = __shfl_up_sync(0xffffffffu, sumB, d);
        if (lane >= d)
        {
            sumA += upA;
            sumB += upB;
        }
    }
    if (lane == 31)
    {
        warpA[warp] = sumA;
        warpB[warp] = sumB;
    }
    __syncthreads();
    if (warp == 0)
    {
        long long wA = warpA[lane], wB = warpB[lane]; // kPlanThreads / 32 == 32 warps
#pragma unroll
        for (int d = 1; d < 32; d <<= 1)
        {
            const long long upA = __shfl_up_sync(0xffffffffu, wA, d);
            const long long upB = __shfl_up_sync(0xffffffffu, wB, d);
            if (lane >= d)
            {
                wA += upA;
                wB += upB;
            }
        }
        warpA[lane] = wA;
        warpB[lane] = wB;
    }
    __syncthreads();
    beforeA = (warp ? warpA[warp - 1] : 0) + sumA - a;
    beforeB = (warp ? warpB[warp - 1] : 0) + sumB - b;
    totalA = warpA[kPlanThreads / 32 - 1];
    totalB = warpB[kPlanThreads / 32 - 1];
    __syncthreads(); // the next tile rewrites warpA / warpB
}
static_assert(kPlanThreads == 32 * 32, "ScanPair scans one value per warp in one warp");

struct EncodePlanner
{
    EncodeParams shared;
    int32_t hostDepth;
    EncodeFamily family;
    int32_t planeMask;
    __device__ __forceinline__ BatchImagePlan operator()(const avifgpu_batch_image& image) const
    {
        return PlanBatchEncodeImage(shared, hostDepth, family, planeMask, image);
    }
};

struct LightEncodePlanner
{
    EncodeParams shared;
    EncodeFamily family; // EncodeLightBatchFamilyOf
    int32_t planeMask;
    __device__ __forceinline__ BatchImagePlan operator()(const avifgpu_batch_image& image) const
    {
        return PlanBatchEncodeImage(shared, 32, family, planeMask, image, kLightBatchUnitPixels);
    }
};

struct DecodePlanner
{
    DecodeParams shared;
    DecodeFamily family;
    int32_t planeMask;
    __device__ __forceinline__ BatchImagePlan operator()(const avifgpu_batch_image& image) const
    {
        return PlanBatchDecodeImage(shared, family, planeMask, image);
    }
};

// Tiles of kPlanThreads images; the running sums carry across tiles.
template <typename Planner>
__global__ void __launch_bounds__(kPlanThreads) PlanIndirectKernel(const __grid_constant__ Planner planner, const avifgpu_batch_image* __restrict__ images,
                                                                   const int32_t* __restrict__ countPointer, int maxCount, void* workspace,
                                                                   int32_t* __restrict__ status)
{
    const IndirectView w(workspace, maxCount);
    const int n = *countPointer;
    if (n < 0 || n > maxCount)
    {
        for (int i = threadIdx.x; status != nullptr && i < maxCount; i += blockDim.x)
        {
            status[i] = AVIFGPU_ERR_BAD_PARAM;
        }
        if (threadIdx.x == 0)
        {
            *w.header = IndirectHeader{ 0, 0, 0, 0 };
        }
        return;
    }
    long long interiorCarry = 0, windowCarry = 0;
    for (int base = 0; base < n; base += kPlanThreads)
    {
        const int i = base + static_cast<int>(threadIdx.x);
        long long interiorUnits = 0, windowUnits[2] = { 0, 0 };
        if (i < n)
        {
            // the records go out now, their first units after the scan: only the unit counts stay in registers
            const BatchImagePlan plan = planner(images[i]);
            if (status != nullptr)
            {
                status[i] = plan.status;
            }
            w.interior[i] = plan.interior;
            w.window[2 * i] = plan.window[0];
            w.window[2 * i + 1] = plan.window[1];
            interiorUnits = plan.interiorUnits;
            windowUnits[0] = plan.windowUnits[0];
            windowUnits[1] = plan.windowUnits[1];
        }
        long long interiorBefore, windowBefore, interiorTotal, windowTotal;
        ScanPair(interiorUnits, windowUnits[0] + windowUnits[1], interiorBefore, windowBefore, interiorTotal, windowTotal);
        if (i < n)
        {
            const long long first = interiorCarry + interiorBefore;
            w.interiorFirst[i] = first;
            w.interior[i].firstUnit = first;
            long long windowFirst = windowCarry + windowBefore;
            for (int k = 0; k < 2; ++k)
            {
                w.windowFirst[2 * i + k] = windowFirst;
                w.window[2 * i + k].firstUnit = windowFirst;
                windowFirst += windowUnits[k];
            }
        }
        interiorCarry += interiorTotal;
        windowCarry += windowTotal;
    }
    if (threadIdx.x == 0)
    {
        *w.header = IndirectHeader{ interiorCarry, windowCarry, n, 0 };
    }
}

template <typename Source, typename HostT, typename PlaneT, int CHANNELS, int XS, int YS, int PREMULTIPLY, int DEST>
__global__ void __launch_bounds__(kRgbThreads) EncodeRgbIntBatchKernel(const __grid_constant__ Source s)
{
    const typename Source::Walk walk(s);
    if (walk.Idle(static_cast<long long>(blockIdx.x) * kWarps))
    {
        return;
    }
    const int count = walk.Count();
    __shared__ float hostLut[(sizeof(HostT) == 1 && sizeof(PlaneT) == 2) ? 256 : 1];
    StageHostLut<HostT, PlaneT>(hostLut, s.shared.maxCode);
    const int lane = threadIdx.x & 31;
    const long long warpCount = static_cast<long long>(gridDim.x) * kWarps;
    int record = 0;
    for (long long unit = static_cast<long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5); unit < walk.Units(); unit += warpCount)
    {
        record = walk.Find(count, record, unit);
        const BatchRecord& r = walk.Record(record);
        Rgb16Params p = s.shared;
        p.rows = static_cast<const uint8_t*>(r.rows);
        p.rowStride = r.rowStride;
        for (int k = 0; k < 4; ++k)
        {
            p.plane[k] = static_cast<uint8_t*>(r.plane[k]);
            p.stride[k] = r.planeStride[k];
        }
        p.groupsPerRow = r.width / 8;
        p.rowCount = r.rowCount;
        const int unitsX = (r.width + kBatchUnitPixels - 1) / kBatchUnitPixels;
        const int local = static_cast<int>(unit - r.firstUnit);
        const int rowPair = local / unitsX;
        const int column = (local - rowPair * unitsX) * 32 + lane;
        if (column < p.groupsPerRow)
        {
            EncodeRgbIntGroup<HostT, PlaneT, CHANNELS, XS, YS, PREMULTIPLY, DEST>(p, hostLut, rowPair, column);
        }
    }
}

template <typename Source, typename HostT>
__global__ void __launch_bounds__(kBatchEdgeThreads) EncodePlanarBatchKernel(const __grid_constant__ Source s)
{
    const typename Source::Walk walk(s);
    if (walk.Idle(blockIdx.x))
    {
        return;
    }
    const int count = walk.Count();
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();
    int record = 0;
    for (long long unit = blockIdx.x; unit < walk.Units(); unit += gridDim.x)
    {
        record = walk.Find(count, record, unit);
        const BatchRecord& r = walk.Record(record);
        EncodeParams p = s.shared;
        p.rows = r.rows;
        p.rowStride = r.rowStride;
        for (int k = 0; k < 4; ++k)
        {
            p.plane[k] = r.plane[k];
            p.planeStride[k] = r.planeStride[k];
        }
        p.width = r.width;
        p.rowCount = r.rowCount;
        EncodePlanarSite<HostT, kBatchEdgeThreads>(p, t, static_cast<unsigned>(unit - r.firstUnit));
    }
}

// The single-image RGBA kernel's per-lane work (kernels_fast_rgba.cu has the commentary) on one unit of kLightBatchUnitPixels
// pixels of a row, or of a 4:2:0 row pair, a lane on 4 pixels of each row, with the unit's record's pointers and no
// software pipelining: the next unit may belong to another image.  RGB hosts (CHANNELS 3) take the flat kernel's samples
// as they are, RGBA hosts the RGBA kernel's clamp / premultiplication and alpha plane.  An interior is 4-pixel aligned, so
// a lane is wholly inside its row or wholly past its end; a lane past it converts zeros and stores nothing.  Each pixel's
// max(R', G', B') code goes into the warp's tally with its level from the context's table.
template <typename Source, int CHANNELS, int XS, int YS, int DEST>
__global__ void __launch_bounds__(kLightBatchWarps * 32, 1) EncodeLightF32BatchKernel(const __grid_constant__ Source s)
{
    using namespace fastenc;
    const typename Source::Walk walk(s);
    if (walk.Idle(static_cast<long long>(blockIdx.x) * kLightBatchWarps))
    {
        return;
    }
    const int count = walk.Count();
    constexpr int kRows = YS ? 2 : 1;
    constexpr int kPixels = 4 * kRows;
    constexpr int kValues = 3 * kPixels;
    const FastEncodeParams& d = s.shared;
    extern __shared__ __align__(16) uint8_t sharedBytes[];
    uint64_t* libmStorage = reinterpret_cast<uint64_t*>(sharedBytes);
    uint64_t* tableBarrier = reinterpret_cast<uint64_t*>(sharedBytes + kSharedLibm);
    uint32_t* stageAll = reinterpret_cast<uint32_t*>(sharedBytes + kSharedLibm + kRgbaTableBarrierBytes);
    uint32_t* compactEntries = reinterpret_cast<uint32_t*>(sharedBytes + LightBatchFixedBytes());
    const uint32_t* firstBits = compactEntries + ((d.table.flatCount + 3) & ~3);
    if (threadIdx.x == 0)
    {
        staging::BeginTableImageCopy(d.table, compactEntries, tableBarrier);
    }
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads(); // the libm tables, the table barrier's initialisation
    staging::WaitTableImage(tableBarrier);

    const int lane = threadIdx.x & 31;
    const int warpInBlock = threadIdx.x >> 5;
    uint32_t* myStage = stageAll + warpInBlock * (32 * kRgbaLaneStrideWords) + lane * kRgbaLaneStrideWords;
    const uint32_t flatShift = d.table.flatShift;
    const int32_t negativeLow = -static_cast<int32_t>(d.table.flatLow);
    const int32_t span = static_cast<int32_t>(d.table.flatHigh - d.table.flatLow);
    const uint32_t bandStrideLog2 = d.table.bandStrideLog2;
    const uint32_t* __restrict__ bandBits = d.table.bandBits;
    const uint32_t compactTopShift = 32u - flatShift;
    const uint32_t compactCodeMask = d.table.compactCodeMask;
    const uint32_t compactMagic = d.table.compactMagic;
    const long long warpCount = static_cast<long long>(gridDim.x) * kLightBatchWarps;
    int record = 0;
    ImageTally light;
#pragma unroll 1
    for (long long unit = static_cast<long long>(blockIdx.x) * kLightBatchWarps + warpInBlock; unit < walk.Units(); unit += warpCount)
    {
        record = walk.Find(count, record, unit);
        const BatchRecord& r = walk.Record(record);
        light.Switch(walk.ImageOf(record), s.light.acc);
        const int local = static_cast<int>(unit - r.firstUnit);
        if (local == 0)
        {
            light.pixels += static_cast<uint64_t>(r.width) * static_cast<uint64_t>(r.rowCount);
        }
        const int tilesX = (r.width + kLightBatchUnitPixels - 1) / kLightBatchUnitPixels;
        const int unitRow = local / tilesX;
        const int x = (local - unitRow * tilesX) * kLightBatchUnitPixels + lane * 4;
        const bool laneActive = x < r.width;
        const int64_t y = static_cast<int64_t>(unitRow) * kRows;
        const uint8_t* source = static_cast<const uint8_t*>(r.rows) + y * r.rowStride + static_cast<int64_t>(x) * CHANNELS * 4;

        // ---- 128-bit row loads; RGBA: alpha, clamp / premultiplication; then the colour samples the curve sees ----------
        uint32_t colourBits[kValues];
        uint32_t alphaCode[kPixels];
        if constexpr (CHANNELS == 3)
        {
#pragma unroll
            for (int q = 0; q < 3 * kRows; ++q)
            {
                const uint4 w = laneActive ? __ldg(reinterpret_cast<const uint4*>(source + (q / 3) * r.rowStride + 16 * (q % 3))) : make_uint4(0u, 0u, 0u, 0u);
                colourBits[4 * q] = w.x;
                colourBits[4 * q + 1] = w.y;
                colourBits[4 * q + 2] = w.z;
                colourBits[4 * q + 3] = w.w;
            }
        }
        else
        {
            uint4 raw[kPixels]; // pixel i of row r = raw[4 * r + i] = { R, G, B, A }
#pragma unroll
            for (int k = 0; k < kPixels; ++k)
            {
                raw[k] = laneActive ? __ldg(reinterpret_cast<const uint4*>(source + (k / 4) * r.rowStride + 16 * (k % 4))) : make_uint4(0u, 0u, 0u, 0u);
            }
#pragma unroll
            for (int k = 0; k < kPixels; ++k)
            {
                const float alpha = ClampF(__uint_as_float(raw[k].w), 0.0f, 1.0f);
                float colour[3] = { __uint_as_float(raw[k].x), __uint_as_float(raw[k].y), __uint_as_float(raw[k].z) };
                if (d.premultiply && alpha < 1.0f)
                {
#pragma unroll
                    for (int c = 0; c < 3; ++c)
                    {
                        colour[c] = (alpha == 0) ? 0.0f : PremultiplyColor(ClampF(colour[c], 0.0f, 1.0f), alpha, 1.0f);
                    }
                }
                alphaCode[k] = FloatToCode(alpha, d.maxCodeFloat);
#pragma unroll
                for (int c = 0; c < 3; ++c)
                {
                    colourBits[3 * k + c] = __float_as_uint(colour[c]);
                }
            }
        }
#pragma unroll
        for (int q = 0; q < kValues / 4; ++q)
        {
            *reinterpret_cast<uint4*>(myStage + 4 * q) = make_uint4(colourBits[4 * q], colourBits[4 * q + 1], colourBits[4 * q + 2], colourBits[4 * q + 3]);
        }

        // ---- float -> code through the compact step table ----------------------------------------------------------
        float codeF[kValuesPerLane] = {}; // one row (YS 0): the second row's codes stay 0 and are not stored
        uint32_t bandMask = 0;
        int32_t largest = 0; // max over the samples as signed integers: > 0x7f7fffff <=> a +inf / NaN is among them
#pragma unroll
        for (int j = 0; j < kValues; ++j)
        {
            bool inBand;
            uint32_t entry;
            codeF[j] = LookupCurveCompact<0>(colourBits[j], compactEntries, flatShift, negativeLow, span, compactTopShift, compactCodeMask, compactMagic, inBand, entry);
            asm("{ .reg .pred q; setp.ne.u32 q, %1, 0; @q or.b32 %0, %0, %2; }" : "+r"(bandMask) : "r"(static_cast<uint32_t>(inBand)), "r"(1u << j));
            largest = max(largest, static_cast<int32_t>(colourBits[j]));
        }

        // ---- in-band samples: which step, how far above its first_k, one bit of the band bitmap ------------------------
        uint32_t lowerMask = 0;
        {
            uint32_t pending = bandMask;
            while (pending != 0)
            {
                const int j = __ffs(static_cast<int>(pending)) - 1;
                pending &= pending - 1;
                const uint32_t bits = myStage[j];
                const int32_t bucket = __viaddmin_s32_relu(static_cast<int32_t>(bits) >> flatShift, negativeLow, span);
                const uint32_t entry = compactEntries[bucket];
                const uint32_t k = ((entry & compactCodeMask) >> kCompactLenBits) + ((entry >> compactTopShift) != 0 ? 1u : 0u);
                const uint32_t distance = bits - firstBits[k];
                if (k != 0 && distance < (1u << bandStrideLog2)) // else flagged by the superset test only
                {
                    const uint32_t bitIndex = (k << bandStrideLog2) + distance;
                    const uint32_t word = __ldg(bandBits + (bitIndex >> 5));
                    lowerMask |= (((word >> (bitIndex & 31u)) & 1u) ^ 1u) << j;
                }
            }
        }
        // ---- +inf / NaN: the exact evaluation, lane by lane -------------------------------------------------------------
        if (__any_sync(0xffffffffu, largest > 0x7f7fffff))
        {
            for (int j = 0; j < kValues; ++j)
            {
                const uint32_t bits = myStage[j];
                if (static_cast<int32_t>(bits) > 0x7f7fffff)
                {
                    const float exact = CodeToFloat(ExactCurveCode<kCurveLinearToPQ>(__uint_as_float(bits), d.pqMultiplier, d.maxCodeFloat, t));
#pragma unroll
                    for (int slot = 0; slot < kValues; ++slot)
                    {
                        if (slot == j)
                        {
                            codeF[slot] = exact;
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int j = 0; j < kValues; ++j)
        {
            if (lowerMask & (1u << j))
            {
                codeF[j] -= 1.0f;
            }
        }
        if (!laneActive)
        {
            continue; // the next unit starts with the whole warp again (Switch)
        }
#pragma unroll
        for (int pixel = 0; pixel < kPixels; ++pixel)
        {
            const uint32_t k = __float2uint_rz(fmaxf(fmaxf(codeF[3 * pixel], codeF[3 * pixel + 1]), codeF[3 * pixel + 2]));
            TallyCode(light.tally, k, __ldg(s.light.levels + k));
        }
        FastEncodeParams p = d;
        p.strideY = r.planeStride[0];
        p.strideCb = r.planeStride[1];
        p.strideCr = r.planeStride[2];
        const int64_t chromaRow = YS ? unitRow : y;
        const int64_t chromaColumn = static_cast<int64_t>(XS ? (x >> 1) : x) * 2;
        StoreTile<XS, YS, DEST>(p, codeF, static_cast<uint8_t*>(r.plane[0]) + y * p.strideY + static_cast<int64_t>(x) * 2,
                                static_cast<uint8_t*>(r.plane[1]) + chromaRow * p.strideCb + chromaColumn * (SourceInterleaved(DEST) ? 2 : 1),
                                static_cast<uint8_t*>(r.plane[2]) + chromaRow * p.strideCr + chromaColumn, kRows == 2);
        if constexpr (CHANNELS == 4)
        {
#pragma unroll
            for (int row = 0; row < kRows; ++row)
            {
                uint8_t* alphaRow = static_cast<uint8_t*>(r.plane[3]) + (y + row) * r.planeStride[3] + static_cast<int64_t>(x) * 2;
                __stcs(reinterpret_cast<uint2*>(alphaRow), make_uint2(MsbWord<DEST>(alphaCode[4 * row] | (alphaCode[4 * row + 1] << 16), p),
                                                                      MsbWord<DEST>(alphaCode[4 * row + 2] | (alphaCode[4 * row + 3] << 16), p)));
            }
        }
    }
    light.Flush(s.light.acc);
}

// EncodePlanarBatchKernel's light-level form for float hosts: the generic kernel's own per-site code with its tally, the
// level read from the context's table or evaluated in place when there is none.
template <typename Source>
__global__ void __launch_bounds__(kBatchEdgeThreads, 1) EncodeLightPlanarBatchKernel(const __grid_constant__ Source s)
{
    const typename Source::Walk walk(s);
    if (walk.Idle(blockIdx.x))
    {
        return;
    }
    const int count = walk.Count();
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();
    int record = 0;
    ImageTally light;
#pragma unroll 1
    for (long long unit = blockIdx.x; unit < walk.Units(); unit += gridDim.x)
    {
        record = walk.Find(count, record, unit);
        const BatchRecord& r = walk.Record(record);
        light.Switch(walk.ImageOf(record), s.light.acc);
        if (unit == r.firstUnit && threadIdx.x < 32) // the CTA's first warp counts the record's pixels
        {
            light.pixels += static_cast<uint64_t>(r.width) * static_cast<uint64_t>(r.rowCount);
        }
        EncodeParams p = s.shared;
        p.rows = r.rows;
        p.rowStride = r.rowStride;
        for (int k = 0; k < 4; ++k)
        {
            p.plane[k] = r.plane[k];
            p.planeStride[k] = r.planeStride[k];
        }
        p.width = r.width;
        p.rowCount = r.rowCount;
        EncodePlanarSite<float, kBatchEdgeThreads, 1>(p, t, static_cast<unsigned>(unit - r.firstUnit), &light.tally, s.light.levels);
    }
    light.Flush(s.light.acc);
}

template <typename Source, typename SampleT, int XS, int YS, int ALPHA, int SOURCE>
__global__ void __launch_bounds__(kRgbThreads, kYccBlocksPerSm) DecodeYccToRgbIntBatchKernel(const __grid_constant__ Source s)
{
    const typename Source::Walk walk(s);
    if (walk.Idle(static_cast<long long>(blockIdx.x) * kWarps))
    {
        return;
    }
    const int count = walk.Count();
    constexpr int kRows = YS ? 2 : 1;
    extern __shared__ __align__(16) uint8_t sharedBytes[];
    const YccTables tables = StageYccTables<SampleT, ALPHA>(sharedBytes, s.shared);
    __syncthreads();
    const YccFactors factors = MakeYccFactors<SampleT>(s.shared.matrix);
    const int lane = threadIdx.x & 31;
    const long long warpCount = static_cast<long long>(gridDim.x) * kWarps;
    int record = 0;
    for (long long unit = static_cast<long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5); unit < walk.Units(); unit += warpCount)
    {
        record = walk.Find(count, record, unit);
        const BatchRecord& r = walk.Record(record);
        IntDecodeParams p = s.shared;
        for (int k = 0; k < 4; ++k)
        {
            p.plane[k] = static_cast<const uint8_t*>(r.plane[k]);
            p.planeStride[k] = r.planeStride[k];
        }
        p.rows = static_cast<uint8_t*>(const_cast<void*>(r.rows));
        p.rowStride = r.rowStride;
        p.width = r.width;
        p.rowCount = r.rowCount;
        const int unitsX = (r.width + kUnitPixels - 1) / kUnitPixels;
        const int local = static_cast<int>(unit - r.firstUnit);
        const int unitRow = local / unitsX;
        const int unitX = local - unitRow * unitsX;
        Raw8<SampleT> rawY[kRows] = {}, rawA[kRows] = {}, rawCb = {}, rawCr = {};
        LoadYccUnit<SampleT, XS, YS, ALPHA, SOURCE>(p, lane, unitRow, unitX, true, rawY, rawA, rawCb, rawCr);
        YccValues<XS, YS> values;
        ExpandYccUnit<SampleT, XS, YS, ALPHA>(p, tables, factors, rawY, rawA, rawCb, rawCr, values);
        const int x0 = unitX * kUnitPixels + lane * 8;
        const int y0 = unitRow * kRows;
        if (x0 < p.width)
        {
            StoreYccUnit<SampleT, XS, YS, ALPHA>(p, factors, values, x0, y0, kRows == 2 && (y0 + 1) < p.rowCount);
        }
    }
}

// The single-image kernel's unit -- 128 pixels of a row, or of a row pair for 4:2:0, a lane on 4 pixels of each row -- with
// 64-bit addresses from the unit's record instead of the 32-bit walk, and no software pipelining: the next unit may belong
// to another image.  An interior is 4-pixel aligned, so a lane is wholly inside its row or wholly past its end.  SOURCE as
// for the single-image kernel: the body of DecodeYccToRgbF32BatchKernel (SOURCE 0) and DecodeSourceYccF32BatchKernel.
template <typename Source, int XS, int YS, int TRANSFER, int ALPHA, int FASTDIV, int SOURCE>
__device__ __forceinline__ void DecodeYccF32BatchBody(const Source& s)
{
    const typename Source::Walk walk(s);
    if (walk.Idle(static_cast<long long>(blockIdx.x) * kWarps))
    {
        return;
    }
    const int count = walk.Count();
    constexpr int kRows = YS ? 2 : 1;
    constexpr int kChromaPerRow = XS ? 2 : 4;
    constexpr int kOutChannels = ALPHA ? 4 : 3;
    extern __shared__ __align__(16) uint8_t sharedBytes[];
    const F32Tables tables = StageF32Tables<TRANSFER, ALPHA>(sharedBytes, s.shared);
    const uint32_t maxCodePair = s.shared.maxCode * 0x10001u;
    const int lane = threadIdx.x & 31;
    const long long warpCount = static_cast<long long>(gridDim.x) * kWarps;
    int record = 0;
#pragma unroll 1
    for (long long unit = static_cast<long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5); unit < walk.Units(); unit += warpCount)
    {
        record = walk.Find(count, record, unit);
        const BatchRecord& r = walk.Record(record);
        const int tilesX = (r.width + kF32TilePixels - 1) / kF32TilePixels;
        const int local = static_cast<int>(unit - r.firstUnit);
        const int unitRow = local / tilesX;
        const int x = (local - unitRow * tilesX) * kF32TilePixels + lane * 4;
        if (x >= r.width)
        {
            continue;
        }
        const int64_t y = static_cast<int64_t>(unitRow) * kRows;
        uint2 yWords[kRows], aWords[kRows];
        const uint8_t* yAddress = static_cast<const uint8_t*>(r.plane[0]) + y * r.planeStride[0] + x * 2;
#pragma unroll
        for (int k = 0; k < kRows; ++k)
        {
            yWords[k] = __ldg(reinterpret_cast<const uint2*>(yAddress + k * r.planeStride[0]));
            aWords[k] = make_uint2(0u, 0u);
        }
        if (ALPHA)
        {
            const uint8_t* aAddress = static_cast<const uint8_t*>(r.plane[3]) + y * r.planeStride[3] + x * 2;
#pragma unroll
            for (int k = 0; k < kRows; ++k)
            {
                aWords[k] = __ldg(reinterpret_cast<const uint2*>(aAddress + k * r.planeStride[3]));
            }
        }
        // chroma row unitRow (one per row, or per 4:2:0 row pair), sites from x >> XS: 2 (XS) or 4 codes
        const int64_t chromaAt = static_cast<int64_t>(unitRow) * r.planeStride[1] + (x >> XS) * (SourceInterleaved(SOURCE) ? 4 : 2);
        uint2 cbWords = make_uint2(0u, 0u), crWords = make_uint2(0u, 0u);
        if constexpr (SourceInterleaved(SOURCE))
        {
            LoadInterleavedChromaWords<XS>(static_cast<const uint8_t*>(r.plane[1]) + chromaAt, cbWords, crWords);
        }
        else if (XS)
        {
            cbWords.x = __ldg(reinterpret_cast<const uint32_t*>(static_cast<const uint8_t*>(r.plane[1]) + chromaAt));
            crWords.x = __ldg(reinterpret_cast<const uint32_t*>(static_cast<const uint8_t*>(r.plane[2]) + chromaAt));
        }
        else
        {
            cbWords = __ldg(reinterpret_cast<const uint2*>(static_cast<const uint8_t*>(r.plane[1]) + chromaAt));
            crWords = __ldg(reinterpret_cast<const uint2*>(static_cast<const uint8_t*>(r.plane[2]) + chromaAt));
        }
        if constexpr (SourceMsbAligned(SOURCE))
        {
            const uint32_t shift = 16u - static_cast<uint32_t>(s.shared.bitDepth);
#pragma unroll
            for (int k = 0; k < kRows; ++k)
            {
                yWords[k] = MsbWordsToCodes(yWords[k], shift);
                aWords[k] = ALPHA ? MsbWordsToCodes(aWords[k], shift) : aWords[k];
            }
            cbWords = MsbWordsToCodes(cbWords, shift);
            crWords = MsbWordsToCodes(crWords, shift);
        }
        float Yf[kRows][4];
        uint2 aPairs[kRows];
        LookUpLuma<kRows>(yWords, aWords, maxCodePair, tables.sharedY, Yf, aPairs);
        float rOffset[kChromaPerRow], bOffset[kChromaPerRow], gOffset[kChromaPerRow];
        ChromaSiteTerms<XS>(s.shared, cbWords, crWords, maxCodePair, tables.sharedUV, rOffset, bOffset, gOffset);
        uint8_t* target = static_cast<uint8_t*>(const_cast<void*>(r.rows)) + y * r.rowStride + static_cast<int64_t>(x) * kOutChannels * 4;
        ConvertRows<XS, YS, TRANSFER, ALPHA, FASTDIV>(s.shared, Yf, aPairs, rOffset, bOffset, gOffset, target, r.rowStride, tables.sharedA, tables.t);
    }
}

template <typename Source, int XS, int YS, int TRANSFER, int ALPHA, int FASTDIV>
__global__ void __launch_bounds__(kF32DecodeThreads, kDecodeBlocksPerSm) DecodeYccToRgbF32BatchKernel(const __grid_constant__ Source s)
{
    DecodeYccF32BatchBody<Source, XS, YS, TRANSFER, ALPHA, FASTDIV, AVIFGPU_SOURCE_PLANAR>(s);
}

template <typename Source, int XS, int YS, int TRANSFER, int ALPHA, int FASTDIV, int SOURCE>
__global__ void __launch_bounds__(kF32DecodeThreads, kDecodeBlocksPerSm) DecodeSourceYccF32BatchKernel(const __grid_constant__ Source s)
{
    DecodeYccF32BatchBody<Source, XS, YS, TRANSFER, ALPHA, FASTDIV, SOURCE>(s);
}

// The pixel `column` (a multiple of 8) and row of a warp's lane in planar-RGB unit `unit` of record `r`: 256 pixels of one row.
__device__ __forceinline__ void PlanarRgbUnitPixel(const BatchRecord& r, long long unit, int lane, int& row, int& column)
{
    const int unitsX = (r.width + kBatchUnitPixels - 1) / kBatchUnitPixels;
    const int local = static_cast<int>(unit - r.firstUnit);
    row = local / unitsX;
    column = (local - row * unitsX) * kBatchUnitPixels + lane * 8;
}

// StreamDecodeKernel's planar-RGB group, one per lane, with the unit's record's pointers.  An interior is 8-pixel aligned, so
// a lane is wholly inside its row or wholly past its end.
template <typename Source, typename SampleT, int CHANNELS>
__global__ void __launch_bounds__(kStreamThreads) DecodePlanarRgbIntBatchKernel(const __grid_constant__ Source s)
{
    const typename Source::Walk walk(s);
    if (walk.Idle(static_cast<long long>(blockIdx.x) * kWarps))
    {
        return;
    }
    const int count = walk.Count();
    const int lane = threadIdx.x & 31;
    const long long warpCount = static_cast<long long>(gridDim.x) * kWarps;
    int record = 0;
    for (long long unit = static_cast<long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5); unit < walk.Units(); unit += warpCount)
    {
        record = walk.Find(count, record, unit);
        const BatchRecord& r = walk.Record(record);
        int row, column;
        PlanarRgbUnitPixel(r, unit, lane, row, column);
        if (column >= r.width)
        {
            continue;
        }
        StreamDecodeParams p = s.shared;
        for (int k = 0; k < 4; ++k)
        {
            p.plane[k] = static_cast<const uint8_t*>(r.plane[k]);
            p.planeStride[k] = r.planeStride[k];
        }
        Raw8<SampleT> raw[CHANNELS];
        LoadStreamGroup<SampleT, CHANNELS, false>(p, raw, row, column);
        uint8_t* target = static_cast<uint8_t*>(const_cast<void*>(r.rows)) + row * r.rowStride + static_cast<int64_t>(column) * CHANNELS * sizeof(SampleT);
        ConvertRgbGroup<SampleT, CHANNELS>(raw, p.maxCode, target);
    }
}

// TableDecodeF32Kernel's planar-RGB group, one per lane, with the unit's record's pointers; the tables are staged once per
// CTA for every image of the launch (one description).
template <typename Source, int ALPHA>
__global__ void __launch_bounds__(kTableThreads) TableDecodeF32BatchKernel(const __grid_constant__ Source s)
{
    const typename Source::Walk walk(s);
    if (walk.Idle(static_cast<long long>(blockIdx.x) * kWarps))
    {
        return;
    }
    const int count = walk.Count();
    extern __shared__ __align__(16) uint8_t sharedBytes[];
    const CodeTables tables = StageCodeTables<3, ALPHA>(sharedBytes, s.shared);
    const float maxCodeFloat = static_cast<float>(s.shared.maxCode);
    const int lane = threadIdx.x & 31;
    const long long warpCount = static_cast<long long>(gridDim.x) * kWarps;
    int record = 0;
    for (long long unit = static_cast<long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5); unit < walk.Units(); unit += warpCount)
    {
        record = walk.Find(count, record, unit);
        const BatchRecord& r = walk.Record(record);
        int row, column;
        PlanarRgbUnitPixel(r, unit, lane, row, column);
        if (column >= r.width)
        {
            continue;
        }
        TableDecodeParams p = s.shared;
        for (int k = 0; k < 4; ++k)
        {
            p.plane[k] = static_cast<const uint8_t*>(r.plane[k]);
            p.planeStride[k] = r.planeStride[k];
        }
        p.rows = static_cast<uint8_t*>(const_cast<void*>(r.rows));
        p.rowStride = r.rowStride;
        TableDecodeGroup<3, ALPHA>(p, tables, maxCodeFloat, row, column);
    }
}

template <typename Source, typename PlaneT, typename HostT>
__global__ void __launch_bounds__(kBatchEdgeThreads) DecodeBatchKernel(const __grid_constant__ Source s)
{
    const typename Source::Walk walk(s);
    if (walk.Idle(blockIdx.x))
    {
        return;
    }
    const int count = walk.Count();
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();
    int record = 0;
    for (long long unit = blockIdx.x; unit < walk.Units(); unit += gridDim.x)
    {
        record = walk.Find(count, record, unit);
        const BatchRecord& r = walk.Record(record);
        DecodeParams p = s.shared;
        for (int k = 0; k < 4; ++k)
        {
            p.plane[k] = r.plane[k];
            p.planeStride[k] = r.planeStride[k];
        }
        p.rows = const_cast<void*>(r.rows);
        p.rowStride = r.rowStride;
        p.width = r.width;
        p.rowCount = r.rowCount;
        p.yPhase = 0; // every window starts on a 4:2:0 row pair
        DecodeChunkPixel<PlaneT, HostT, kBatchEdgeThreads>(p, t, static_cast<unsigned>(unit - r.firstUnit));
    }
}

// ---- the launches, one per kernel family, for either source: the family's picker (launch_keys.h) chooses the instantiation ----

// The encode interiors.
template <typename Source>
void LaunchRgbInt(const Source& s, const EncodeParams& d, int hostDepth, unsigned grid, cudaStream_t stream)
{
    WithRgbIntKey(d, hostDepth, [&](auto host, auto plane, auto channels, auto premultiply, auto xs, auto ys, auto dest) {
        EncodeRgbIntBatchKernel<Source, TypeOf<decltype(host)>, TypeOf<decltype(plane)>, channels(), xs(), ys(), premultiply(), dest()><<<grid, kRgbThreads, 0, stream>>>(s);
    });
}

// The windows of an encode batch: its hosts are 8- or 16-bit.
template <typename Source>
void LaunchPlanar(const Source& s, int hostDepth, unsigned grid, cudaStream_t stream)
{
    WithIntHost(hostDepth, [&](auto host) { EncodePlanarBatchKernel<Source, TypeOf<decltype(host)>><<<grid, kBatchEdgeThreads, 0, stream>>>(s); });
}

// The light-level float encode interiors, with `bytes` of shared memory (0 for a launch that plans no interior unit).
template <typename Source>
void LaunchLightF32(const Source& s, const EncodeParams& d, unsigned grid, size_t bytes, cudaStream_t stream)
{
    WithLightF32Key(d, [&](auto channels, auto xs, auto ys, auto dest) {
        static std::atomic<uint64_t> configuredDevices{ 0 }; // per instantiation
        const auto kernel = EncodeLightF32BatchKernel<Source, channels(), xs(), ys(), dest()>;
        if (AllowDynamicShared(kernel, kSharedLimit, configuredDevices) == cudaSuccess)
        {
            kernel<<<grid, kLightBatchWarps * 32, bytes, stream>>>(s);
        } // else the failed attribute call is the error Launched() finds
    });
}

// The light-level interiors' description: the single-image float kernels' parameters without an image, and the compact
// step table when the description has one.
fastenc::FastEncodeParams LightF32Shared(const EncodeParams& d)
{
    fastenc::FastEncodeParams fp{};
    fp.premultiply = d.premultiply;
    fp.pqMultiplier = d.pqMultiplier;
    fp.maxCodeFloat = d.maxCodeFloat;
    fp.maxCode = static_cast<int32_t>(d.maxCode);
    fp.matrix = d.matrix;
    fp.chromaOffset = d.chromaOffset;
    fp.topLeft = d.topLeft;
    if (d.curveTable != nullptr)
    {
        fp.table = *d.curveTable;
    }
    return fp;
}

// The shared memory of EncodeLightF32BatchKernel over the description's step table.
size_t LightF32Bytes(const EncodeParams& d) { return static_cast<size_t>(LightBatchFixedBytes()) + d.curveTable->compactImageBytes; }

// The YCbCr decode interiors into 8/16-bit hosts, with `bytes` of staged tables.
template <typename Source>
void LaunchYccInt(const Source& s, const DecodeParams& d, unsigned grid, size_t bytes, cudaStream_t stream)
{
    WithYccIntKey(d, [&](auto sample, auto alpha, auto xs, auto ys, auto source) {
        DecodeYccToRgbIntBatchKernel<Source, TypeOf<decltype(sample)>, xs(), ys(), alpha(), source()><<<grid, kRgbThreads, bytes, stream>>>(s);
    });
}

template <typename Source, int XS, int YS, int TRANSFER, int ALPHA, int FASTDIV, int SOURCE>
void LaunchYccF32One(const Source& s, unsigned grid, size_t bytes, cudaStream_t stream)
{
    static std::atomic<uint64_t> configuredDevices{ 0 }; // per instantiation
    const auto kernel = [] {
        if constexpr (SOURCE == AVIFGPU_SOURCE_PLANAR)
        {
            return DecodeYccToRgbF32BatchKernel<Source, XS, YS, TRANSFER, ALPHA, FASTDIV>;
        }
        else
        {
            return DecodeSourceYccF32BatchKernel<Source, XS, YS, TRANSFER, ALPHA, FASTDIV, SOURCE>;
        }
    }();
    if (AllowDynamicShared(kernel, kF32MaxTableBytes, configuredDevices) == cudaSuccess)
    {
        kernel<<<grid, kF32DecodeThreads, bytes, stream>>>(s);
    } // else the failed attribute call is the error Launched() finds
}

// The YCbCr decode interiors into 32-bit hosts, with `bytes` of staged tables.
template <typename Source>
void LaunchYccF32(const Source& s, const DecodeParams& d, unsigned grid, size_t bytes, cudaStream_t stream)
{
    WithYccF32Key(d, [&](auto transfer, auto fastDiv, auto alpha, auto xs, auto ys, auto source) {
        LaunchYccF32One<Source, xs(), ys(), transfer(), alpha(), fastDiv(), source()>(s, grid, bytes, stream);
    });
}

// The float decode's tables for description `d`.
size_t F32TableBytesOf(const DecodeParams& d) { return F32TableBytes(d.transfer, d.bitDepth, d.hasAlpha != 0); }

// The planar-RGB decode interiors into 8/16-bit hosts.
template <typename Source>
void LaunchPlanarRgbInt(const Source& s, const DecodeParams& d, long long blocks, int smCount, cudaStream_t stream)
{
    const unsigned grid = GridFor(blocks, static_cast<long long>(smCount) * kStreamBlocksPerSm);
    WithIntDecodeKey(d, [&](auto sample, auto alpha) {
        DecodePlanarRgbIntBatchKernel<Source, TypeOf<decltype(sample)>, 3 + alpha()><<<grid, kStreamThreads, 0, stream>>>(s);
    });
}

// The planar-RGB decode interiors into 32-bit hosts, with `bytes` of staged tables, capped at the CTAs resident at once.
template <typename Source>
void LaunchPlanarRgbF32(const Source& s, const DecodeParams& d, long long blocks, int smCount, size_t bytes, cudaStream_t stream)
{
    WithTableF32Key(d, [&](auto alpha) {
        const long long cap = CodeTableGridCap(TableDecodeF32BatchKernel<Source, alpha()>, bytes, smCount);
        TableDecodeF32BatchKernel<Source, alpha()><<<GridFor(blocks, cap), kTableThreads, bytes, stream>>>(s);
    });
}

// The windows of a decode batch.
template <typename Source>
void LaunchDecodeEdge(const Source& s, int hostDepth, unsigned grid, cudaStream_t stream)
{
    WithHostDepth(hostDepth, [&](auto plane, auto host) {
        DecodeBatchKernel<Source, TypeOf<decltype(plane)>, TypeOf<decltype(host)>><<<grid, kBatchEdgeThreads, 0, stream>>>(s);
    });
}

// DecodeYccToRgbIntKernel's tables for description `d`.
size_t YccTableBytesOf(const DecodeParams& d) { return YccTableBytes(d.bitDepth, d.hasAlpha && d.hostDepth != 8); }

// The edge kernels' description: integer hosts have no transfer curve.
EncodeParams PlanarShared(const EncodeParams& shared)
{
    EncodeParams edge = shared;
    edge.useCurveView = 0;
    return edge;
}

template <typename Chunk>
Chunk ChunkOf(const decltype(Chunk::shared)& shared, const BatchRecord* records, int count, int64_t units)
{
    Chunk b{};
    b.shared = shared;
    b.count = count;
    b.units = units;
    for (int i = 0; i < count; ++i)
    {
        b.record[i] = records[i];
    }
    return b;
}

template <typename Chunk>
Chunk LightChunkOf(const decltype(Chunk::shared)& shared, const BatchRecord* records, const int32_t* images, int count, int64_t units, const LightSink& light)
{
    Chunk b = ChunkOf<Chunk>(shared, records, count, units);
    for (int i = 0; i < count; ++i)
    {
        b.image[i] = images[i];
    }
    b.light = light;
    return b;
}

// `launches` if the launches before it succeeded, else the failure's status.
int Launched(int launches)
{
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? launches : ReportLaunchFailure(static_cast<int>(e));
}

} // namespace

int LaunchEncodeBatchChunk(const EncodeParams& shared, int hostDepth, const BatchChunk& chunk, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const long long cap = static_cast<long long>(SmCountOrDefault(shared.smCount)) * kStreamBlocksPerSm;
    // one warp per unit
    LaunchRgbInt(ChunkOf<RgbIntChunk>(RgbIntShared(shared), chunk.interior, chunk.images, chunk.interiorUnits), shared, hostDepth,
                 GridFor((chunk.interiorUnits + kWarps - 1) / kWarps, cap), stream);
    const int interior = Launched(1);
    if (interior < 0 || chunk.windows == 0)
    {
        return interior;
    }
    LaunchPlanar(ChunkOf<PlanarChunk>(PlanarShared(shared), chunk.window, chunk.windows, chunk.windowUnits), hostDepth, GridFor(chunk.windowUnits, cap), stream);
    return Launched(2);
}

int LaunchEncodeLightBatchChunk(const EncodeParams& shared, const BatchChunk& chunk, const LightSink& light, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const int smCount = SmCountOrDefault(shared.smCount);
    // one warp per unit, one CTA per SM: the step table is staged once per CTA
    LaunchLightF32(LightChunkOf<LightF32Chunk>(LightF32Shared(shared), chunk.interior, chunk.imageIndex, chunk.images, chunk.interiorUnits, light), shared,
                   GridFor((chunk.interiorUnits + kLightBatchWarps - 1) / kLightBatchWarps, smCount), LightF32Bytes(shared), stream);
    const int interior = Launched(1);
    if (interior < 0 || chunk.windows == 0)
    {
        return interior;
    }
    EncodeLightPlanarBatchKernel<LightEdgeChunk><<<GridFor(chunk.windowUnits, static_cast<long long>(smCount) * kStreamBlocksPerSm), kBatchEdgeThreads, 0, stream>>>(
        LightChunkOf<LightEdgeChunk>(GenericEncodeView(shared, 32), chunk.window, chunk.windowImage, chunk.windows, chunk.windowUnits, light));
    return Launched(2);
}

int LaunchDecodeBatchChunk(const DecodeParams& shared, const BatchChunk& chunk, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const int smCount = SmCountOrDefault(shared.smCount);
    const long long warps = (chunk.interiorUnits + kWarps - 1) / kWarps; // one warp per unit
    switch (DecodeBatchFamilyOf(shared)) // a chunk has interiors: a batched family
    {
    case DecodeFamily::PlanarRgbF32:
        LaunchPlanarRgbF32(ChunkOf<PlanarRgbF32Chunk>(TableDecodeDescription(shared), chunk.interior, chunk.images, chunk.interiorUnits), shared, warps,
                           smCount, CodeTableBytes(shared.bitDepth, shared.hasAlpha != 0), stream);
        break;
    case DecodeFamily::PlanarRgbInt:
        LaunchPlanarRgbInt(ChunkOf<PlanarRgbIntChunk>(StreamDecodeDescription(shared), chunk.interior, chunk.images, chunk.interiorUnits), shared, warps,
                           smCount, stream);
        break;
    case DecodeFamily::YccF32:
        LaunchYccF32(ChunkOf<YccF32Chunk>(FillF32Description(shared), chunk.interior, chunk.images, chunk.interiorUnits), shared,
                     GridFor(warps, static_cast<long long>(smCount) * kDecodeBlocksPerSm), F32TableBytesOf(shared), stream);
        break;
    default:
        LaunchYccInt(ChunkOf<YccIntChunk>(IntDecodeShared(shared), chunk.interior, chunk.images, chunk.interiorUnits), shared,
                     GridFor(warps, static_cast<long long>(smCount) * kYccBlocksPerSm), YccTableBytesOf(shared), stream);
        break;
    }
    const int interior = Launched(1);
    if (interior < 0 || chunk.windows == 0)
    {
        return interior;
    }
    LaunchDecodeEdge(ChunkOf<DecodeEdgeChunk>(shared, chunk.window, chunk.windows, chunk.windowUnits), shared.hostDepth,
                     GridFor(chunk.windowUnits, static_cast<long long>(smCount) * kStreamBlocksPerSm), stream);
    return Launched(2);
}

int LaunchEncodeIndirect(const EncodeParams& shared, int hostDepth, EncodeFamily family, int planeMask, const avifgpu_batch_image* images,
                         const int32_t* count, int maxCount, void* workspace, int32_t* status, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const unsigned cap = static_cast<unsigned>(SmCountOrDefault(shared.smCount)) * kStreamBlocksPerSm; // the chunk launchers' caps
    EncodePlanner planner{};
    planner.shared = shared;
    planner.hostDepth = hostDepth;
    planner.family = family;
    planner.planeMask = planeMask;
    PlanIndirectKernel<EncodePlanner><<<1, kPlanThreads, 0, stream>>>(planner, images, count, maxCount, workspace, status);
    if (Launched(1) < 0)
    {
        return AVIFGPU_ERR_CUDA;
    }
    LaunchRgbInt(WorkspaceSource<Rgb16Params, 0>{ RgbIntShared(shared), workspace, maxCount }, shared, hostDepth, cap, stream);
    if (Launched(1) < 0)
    {
        return AVIFGPU_ERR_CUDA;
    }
    LaunchPlanar(WorkspaceSource<EncodeParams, 1>{ PlanarShared(shared), workspace, maxCount }, hostDepth, cap, stream);
    return Launched(3);
}

int LaunchEncodeLightIndirect(const EncodeParams& shared, int planeMask, const avifgpu_batch_image* images, const int32_t* count, int maxCount,
                              void* workspace, int32_t* status, const LightSink& light, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const int smCount = SmCountOrDefault(shared.smCount);
    LightEncodePlanner planner{};
    planner.shared = shared;
    planner.family = EncodeLightBatchFamilyOf(shared, 32);
    planner.planeMask = planeMask;
    PlanIndirectKernel<LightEncodePlanner><<<1, kPlanThreads, 0, stream>>>(planner, images, count, maxCount, workspace, status);
    if (Launched(1) < 0)
    {
        return AVIFGPU_ERR_CUDA;
    }
    // Without the tuned family (no step or level table, as in a capture before prepare) the plan has no interior unit and
    // the interior grid returns before staging anything, so it gets no shared memory.
    LightWorkspaceSource<fastenc::FastEncodeParams, 0> interior{};
    interior.shared = LightF32Shared(shared);
    interior.workspace = workspace;
    interior.maxCount = maxCount;
    interior.light = light;
    LaunchLightF32(interior, shared, static_cast<unsigned>(smCount), planner.family != EncodeFamily::Generic ? LightF32Bytes(shared) : 0, stream);
    if (Launched(1) < 0)
    {
        return AVIFGPU_ERR_CUDA;
    }
    LightWorkspaceSource<EncodeParams, 1> edge{};
    edge.shared = GenericEncodeView(shared, 32);
    edge.workspace = workspace;
    edge.maxCount = maxCount;
    edge.light = light;
    EncodeLightPlanarBatchKernel<LightWorkspaceSource<EncodeParams, 1>><<<static_cast<unsigned>(smCount * kStreamBlocksPerSm), kBatchEdgeThreads, 0, stream>>>(edge);
    return Launched(3);
}

int LaunchDecodeIndirect(const DecodeParams& shared, DecodeFamily family, int planeMask, const avifgpu_batch_image* images, const int32_t* count,
                         int maxCount, void* workspace, int32_t* status, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const int smCount = SmCountOrDefault(shared.smCount);
    DecodePlanner planner{};
    planner.shared = shared;
    planner.family = family;
    planner.planeMask = planeMask;
    PlanIndirectKernel<DecodePlanner><<<1, kPlanThreads, 0, stream>>>(planner, images, count, maxCount, workspace, status);
    if (Launched(1) < 0)
    {
        return AVIFGPU_ERR_CUDA;
    }
    // A description no batched family takes plans no interior unit; the call still makes its interior launch, on the batched
    // kernel of its colour space and host depth, whose grid returns before staging (so it gets no tables).  The grids are the
    // chunk launchers' caps.
    const bool tuned = family != DecodeFamily::Generic;
    const bool rgb = shared.colorspace == AVIFGPU_COLORSPACE_RGB;
    const DecodeFamily interior = tuned ? family
                                  : shared.hostDepth == 32 ? (rgb ? DecodeFamily::PlanarRgbF32 : DecodeFamily::YccF32)
                                                           : (rgb ? DecodeFamily::PlanarRgbInt : DecodeFamily::YccInt);
    switch (interior)
    {
    case DecodeFamily::PlanarRgbF32:
        LaunchPlanarRgbF32(WorkspaceSource<TableDecodeParams, 0>{ TableDecodeDescription(shared), workspace, maxCount }, shared, LLONG_MAX, smCount,
                           tuned ? CodeTableBytes(shared.bitDepth, shared.hasAlpha != 0) : 0, stream);
        break;
    case DecodeFamily::PlanarRgbInt:
        LaunchPlanarRgbInt(WorkspaceSource<StreamDecodeParams, 0>{ StreamDecodeDescription(shared), workspace, maxCount }, shared, LLONG_MAX, smCount, stream);
        break;
    case DecodeFamily::YccF32:
        LaunchYccF32(WorkspaceSource<FastDecodeParams, 0>{ FillF32Description(shared), workspace, maxCount }, shared,
                     static_cast<unsigned>(smCount * kDecodeBlocksPerSm), tuned ? F32TableBytesOf(shared) : 0, stream);
        break;
    default:
        LaunchYccInt(WorkspaceSource<IntDecodeParams, 0>{ IntDecodeShared(shared), workspace, maxCount }, shared,
                     static_cast<unsigned>(smCount * kYccBlocksPerSm), tuned ? YccTableBytesOf(shared) : 0, stream);
        break;
    }
    if (Launched(1) < 0)
    {
        return AVIFGPU_ERR_CUDA;
    }
    LaunchDecodeEdge(WorkspaceSource<DecodeParams, 1>{ shared, workspace, maxCount }, shared.hostDepth, static_cast<unsigned>(smCount * kStreamBlocksPerSm), stream);
    return Launched(3);
}

} // namespace avifgpu
