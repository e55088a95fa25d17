// kernels_batch_indirect.cu -- avifgpu_encode_batch_indirect and avifgpu_decode_batch_indirect: batches whose image
// records and count are read from device memory when the work runs (batch_indirect.h).  Three launches per call, whatever
// the batch holds:
//
//   PlanIndirectKernel              one CTA: routes every image (PlanIndirectEncodeImage / PlanIndirectDecodeImage), writes
//                                   its status, its records and the block-scanned first units into the workspace;
//   EncodeRgbIntIndirectKernel      the interiors, with EncodeRgbIntGroup (int_units.cuh), a warp per 256-pixel unit;
//   DecodeYccToRgbIntIndirectKernel LoadYccUnit / ExpandYccUnit / StoreYccUnit, the tables staged once per CTA;
//   EncodePlanarIndirectKernel,     the windows -- strips, and whole images the tuned kernels do not take -- with
//   DecodeIndirectKernel            EncodePlanarSite / DecodeChunkPixel (generic_units.cuh), a CTA per unit.
//
// The host does not know how much work there is, so the interior and edge grids are the batch launchers' persistent caps
// (kernels_batch.cu); a CTA with no unit returns before it stages anything.  A worker finds its unit's record with a
// warp- (CTA-) uniform binary search over the first units, starting after the record of its previous unit.
#include "batch_indirect.h"
#include "generic_units.cuh"
#include "int_units.cuh"
#include "kernel_params.h"
#include "../../include/avifgpu.h"

#include <cuda_runtime.h>

namespace avifgpu
{

namespace
{

constexpr int kWarps = kRgbThreads / 32;
constexpr int kPlanThreads = 1024;
constexpr int kDecodeBlocksPerSm = 3; // DecodeYccToRgbIntKernel's occupancy (kernels_fast_decode_int.cu)

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
    int32_t tuned;
    int32_t planeMask;
    __device__ __forceinline__ IndirectImagePlan operator()(const avifgpu_batch_image& image) const
    {
        return PlanIndirectEncodeImage(shared, hostDepth, tuned != 0, planeMask, image);
    }
};

struct DecodePlanner
{
    DecodeParams shared;
    int32_t tuned;
    int32_t planeMask;
    __device__ __forceinline__ IndirectImagePlan operator()(const avifgpu_batch_image& image) const
    {
        return PlanIndirectDecodeImage(shared, tuned != 0, planeMask, image);
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
            const IndirectImagePlan plan = planner(images[i]);
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

template <typename HostT, typename PlaneT, int CHANNELS, int XS, int YS, int PREMULTIPLY>
__global__ void __launch_bounds__(kRgbThreads) EncodeRgbIntIndirectKernel(const __grid_constant__ Rgb16Params shared, void* workspace, int maxCount)
{
    const IndirectView w(workspace, maxCount);
    const long long units = w.header->interiorUnits;
    if (static_cast<long long>(blockIdx.x) * kWarps >= units)
    {
        return; // no unit for this CTA
    }
    const int count = w.header->count;
    __shared__ float hostLut[(sizeof(HostT) == 1 && sizeof(PlaneT) == 2) ? 256 : 1];
    StageHostLut<HostT, PlaneT>(hostLut, shared.maxCode);
    const int lane = threadIdx.x & 31;
    const long long warpCount = static_cast<long long>(gridDim.x) * kWarps;
    int record = 0;
    for (long long unit = static_cast<long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5); unit < units; unit += warpCount)
    {
        record = FindRecord(w.interiorFirst, count, record, unit);
        const BatchRecord& r = w.interior[record];
        Rgb16Params p = shared;
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
            EncodeRgbIntGroup<HostT, PlaneT, CHANNELS, XS, YS, PREMULTIPLY>(p, hostLut, rowPair, column);
        }
    }
}

template <typename HostT>
__global__ void __launch_bounds__(kBatchEdgeThreads) EncodePlanarIndirectKernel(const __grid_constant__ EncodeParams shared, void* workspace, int maxCount)
{
    const IndirectView w(workspace, maxCount);
    const long long units = w.header->windowUnits;
    if (blockIdx.x >= units)
    {
        return;
    }
    const int count = 2 * w.header->count;
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();
    int record = 0;
    for (long long unit = blockIdx.x; unit < units; unit += gridDim.x)
    {
        record = FindRecord(w.windowFirst, count, record, unit);
        const BatchRecord& r = w.window[record];
        EncodeParams p = shared;
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

template <typename SampleT, int XS, int YS, int ALPHA>
__global__ void __launch_bounds__(kRgbThreads, kDecodeBlocksPerSm)
    DecodeYccToRgbIntIndirectKernel(const __grid_constant__ IntDecodeParams shared, void* workspace, int maxCount)
{
    const IndirectView w(workspace, maxCount);
    const long long units = w.header->interiorUnits;
    if (static_cast<long long>(blockIdx.x) * kWarps >= units)
    {
        return;
    }
    const int count = w.header->count;
    constexpr int kRows = YS ? 2 : 1;
    extern __shared__ __align__(16) uint8_t sharedBytes[];
    const YccTables tables = StageYccTables<SampleT, ALPHA>(sharedBytes, shared);
    __syncthreads();
    const YccFactors factors = MakeYccFactors<SampleT>(shared.matrix);
    const int lane = threadIdx.x & 31;
    const long long warpCount = static_cast<long long>(gridDim.x) * kWarps;
    int record = 0;
    for (long long unit = static_cast<long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5); unit < units; unit += warpCount)
    {
        record = FindRecord(w.interiorFirst, count, record, unit);
        const BatchRecord& r = w.interior[record];
        IntDecodeParams p = shared;
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
        LoadYccUnit<SampleT, XS, YS, ALPHA>(p, lane, unitRow, unitX, true, rawY, rawA, rawCb, rawCr);
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

template <typename PlaneT, typename HostT>
__global__ void __launch_bounds__(kBatchEdgeThreads) DecodeIndirectKernel(const __grid_constant__ DecodeParams shared, void* workspace, int maxCount)
{
    const IndirectView w(workspace, maxCount);
    const long long units = w.header->windowUnits;
    if (blockIdx.x >= units)
    {
        return;
    }
    const int count = 2 * w.header->count;
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();
    int record = 0;
    for (long long unit = blockIdx.x; unit < units; unit += gridDim.x)
    {
        record = FindRecord(w.windowFirst, count, record, unit);
        const BatchRecord& r = w.window[record];
        DecodeParams p = shared;
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

template <typename HostT, typename PlaneT, int CHANNELS, int PREMULTIPLY>
void LaunchRgbIntIndirect(const Rgb16Params& shared, int xs, int ys, unsigned grid, void* workspace, int maxCount, cudaStream_t stream)
{
    if (xs == 1 && ys == 1) EncodeRgbIntIndirectKernel<HostT, PlaneT, CHANNELS, 1, 1, PREMULTIPLY><<<grid, kRgbThreads, 0, stream>>>(shared, workspace, maxCount);
    else if (xs == 1) EncodeRgbIntIndirectKernel<HostT, PlaneT, CHANNELS, 1, 0, PREMULTIPLY><<<grid, kRgbThreads, 0, stream>>>(shared, workspace, maxCount);
    else EncodeRgbIntIndirectKernel<HostT, PlaneT, CHANNELS, 0, 0, PREMULTIPLY><<<grid, kRgbThreads, 0, stream>>>(shared, workspace, maxCount);
}

template <typename HostT, typename PlaneT>
void LaunchRgbIntIndirectChannels(const Rgb16Params& shared, int channels, bool premultiply, int xs, int ys, unsigned grid, void* workspace, int maxCount,
                                  cudaStream_t stream)
{
    if (channels == 4 && premultiply) LaunchRgbIntIndirect<HostT, PlaneT, 4, 1>(shared, xs, ys, grid, workspace, maxCount, stream);
    else if (channels == 4) LaunchRgbIntIndirect<HostT, PlaneT, 4, 0>(shared, xs, ys, grid, workspace, maxCount, stream);
    else LaunchRgbIntIndirect<HostT, PlaneT, 3, 0>(shared, xs, ys, grid, workspace, maxCount, stream);
}

template <typename SampleT, int ALPHA>
void LaunchYccIntIndirect(const IntDecodeParams& shared, int xs, int ys, unsigned grid, size_t bytes, void* workspace, int maxCount, cudaStream_t stream)
{
    if (xs == 1 && ys == 1) DecodeYccToRgbIntIndirectKernel<SampleT, 1, 1, ALPHA><<<grid, kRgbThreads, bytes, stream>>>(shared, workspace, maxCount);
    else if (xs == 1) DecodeYccToRgbIntIndirectKernel<SampleT, 1, 0, ALPHA><<<grid, kRgbThreads, bytes, stream>>>(shared, workspace, maxCount);
    else DecodeYccToRgbIntIndirectKernel<SampleT, 0, 0, ALPHA><<<grid, kRgbThreads, bytes, stream>>>(shared, workspace, maxCount);
}

int Launched(int launches)
{
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? launches : ReportLaunchFailure(static_cast<int>(e));
}

} // namespace

int LaunchEncodeIndirect(const EncodeParams& shared, int hostDepth, bool tuned, int planeMask, const avifgpu_batch_image* images,
                         const int32_t* count, int maxCount, void* workspace, int32_t* status, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const unsigned cap = static_cast<unsigned>(SmCountOrDefault(shared.smCount)) * 16; // the batch launchers' caps
    EncodePlanner planner{};
    planner.shared = shared;
    planner.hostDepth = hostDepth;
    planner.tuned = tuned ? 1 : 0;
    planner.planeMask = planeMask;
    PlanIndirectKernel<EncodePlanner><<<1, kPlanThreads, 0, stream>>>(planner, images, count, maxCount, workspace, status);
    if (Launched(1) < 0)
    {
        return AVIFGPU_ERR_CUDA;
    }
    const Rgb16Params rgb = RgbIntShared(shared);
    const bool wide = shared.imageDepth > 8;
    const bool premultiply = shared.premultiply != 0;
    if (hostDepth == 16)
    {
        if (wide) LaunchRgbIntIndirectChannels<uint16_t, uint16_t>(rgb, shared.channels, premultiply, shared.xs, shared.ys, cap, workspace, maxCount, stream);
        else LaunchRgbIntIndirectChannels<uint16_t, uint8_t>(rgb, shared.channels, premultiply, shared.xs, shared.ys, cap, workspace, maxCount, stream);
    }
    else
    {
        if (wide) LaunchRgbIntIndirectChannels<uint8_t, uint16_t>(rgb, shared.channels, premultiply, shared.xs, shared.ys, cap, workspace, maxCount, stream);
        else LaunchRgbIntIndirectChannels<uint8_t, uint8_t>(rgb, shared.channels, premultiply, shared.xs, shared.ys, cap, workspace, maxCount, stream);
    }
    if (Launched(1) < 0)
    {
        return AVIFGPU_ERR_CUDA;
    }
    EncodeParams edge = shared;
    edge.useCurveView = 0; // integer hosts: no transfer curve
    if (hostDepth == 16) EncodePlanarIndirectKernel<uint16_t><<<cap, kBatchEdgeThreads, 0, stream>>>(edge, workspace, maxCount);
    else EncodePlanarIndirectKernel<uint8_t><<<cap, kBatchEdgeThreads, 0, stream>>>(edge, workspace, maxCount);
    return Launched(3);
}

int LaunchDecodeIndirect(const DecodeParams& shared, bool tuned, int planeMask, const avifgpu_batch_image* images, const int32_t* count,
                         int maxCount, void* workspace, int32_t* status, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const int smCount = SmCountOrDefault(shared.smCount);
    DecodePlanner planner{};
    planner.shared = shared;
    planner.tuned = tuned ? 1 : 0;
    planner.planeMask = planeMask;
    PlanIndirectKernel<DecodePlanner><<<1, kPlanThreads, 0, stream>>>(planner, images, count, maxCount, workspace, status);
    if (Launched(1) < 0)
    {
        return AVIFGPU_ERR_CUDA;
    }
    IntDecodeParams ycc{};
    ycc.bitDepth = shared.bitDepth;
    ycc.maxCode = shared.maxCode;
    ycc.range = shared.range;
    ycc.matrix = shared.matrix;
    ycc.verifiedGreenDivision = shared.verifiedGreenDivision;
    // DecodeYccToRgbIntKernel's tables (at most 40 KB: no opt-in beyond the default 48 KB) and grid cap.  A description
    // the tuned kernel does not take plans no interior unit: its grid returns before staging, so it gets no tables.
    const bool host8 = shared.hostDepth == 8;
    const size_t entries = static_cast<size_t>(1) << shared.bitDepth;
    const size_t bytes = tuned ? 2 * sizeof(float) * entries + ((shared.hasAlpha && !host8) ? sizeof(uint16_t) * entries : 0) : 0;
    const unsigned grid = static_cast<unsigned>(smCount * kDecodeBlocksPerSm);
    if (host8)
    {
        if (shared.hasAlpha) LaunchYccIntIndirect<uint8_t, 1>(ycc, shared.xs, shared.ys, grid, bytes, workspace, maxCount, stream);
        else LaunchYccIntIndirect<uint8_t, 0>(ycc, shared.xs, shared.ys, grid, bytes, workspace, maxCount, stream);
    }
    else
    {
        if (shared.hasAlpha) LaunchYccIntIndirect<uint16_t, 1>(ycc, shared.xs, shared.ys, grid, bytes, workspace, maxCount, stream);
        else LaunchYccIntIndirect<uint16_t, 0>(ycc, shared.xs, shared.ys, grid, bytes, workspace, maxCount, stream);
    }
    if (Launched(1) < 0)
    {
        return AVIFGPU_ERR_CUDA;
    }
    const unsigned edgeGrid = static_cast<unsigned>(smCount * 16);
    if (shared.hostDepth == 16) DecodeIndirectKernel<uint16_t, uint16_t><<<edgeGrid, kBatchEdgeThreads, 0, stream>>>(shared, workspace, maxCount);
    else DecodeIndirectKernel<uint8_t, uint8_t><<<edgeGrid, kBatchEdgeThreads, 0, stream>>>(shared, workspace, maxCount);
    return Launched(3);
}

} // namespace avifgpu
