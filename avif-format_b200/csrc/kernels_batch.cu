// kernels_batch.cu -- many small images per launch for avifgpu_encode_batch_device and avifgpu_decode_batch_device.
// A 512 x 512 image is 2 MB of traffic, well under a microsecond of HBM time, so one launch per image is bound by the launch and the grid's ramp and
// drain.  Here one launch walks the units of every image of a chunk:
//
//   EncodeRgbIntBatchKernel    the aligned interiors, with EncodeRgbIntGroup (int_units.cuh) -- the single-image tuned
//                              kernel's own group code; a warp takes one unit (256 pixels of one row or 4:2:0 row pair,
//                              8 per lane) at a time, persistent over the chunk's concatenated unit space;
//   EncodePlanarBatchKernel    the right strips and odd last 4:2:0 rows, with EncodePlanarSite (generic_units.cuh) -- the
//                              generic kernel's own site code; a CTA takes one run of 256 chroma sites at a time;
//   DecodeYccToRgbIntBatchKernel  the decode interiors, with LoadYccUnit / ExpandYccUnit / StoreYccUnit (int_units.cuh);
//                              the unorm -> float tables are staged once per CTA for the whole chunk (one description);
//   DecodeBatchKernel          the decode edge strips, with DecodeChunkPixel (generic_units.cuh).
//
// A worker's units increase, so it finds each unit's record by walking forward through the records' first units: once per
// unit and warp- (CTA-) uniform, never per pixel.  The per-image records travel in the kernel parameter (__grid_constant__).
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

struct RgbIntBatchParams
{
    Rgb16Params shared; // pointers, strides and sizes unused
    int32_t count;
    int64_t units;
    BatchRecord image[kBatchChunkImages];
};

struct PlanarBatchParams
{
    EncodeParams shared; // pointers, strides and sizes unused
    int32_t count;
    int64_t units;
    BatchRecord window[2 * kBatchChunkImages];
};

constexpr int kDecodeBlocksPerSm = 3; // DecodeYccToRgbIntKernel's occupancy (kernels_fast_decode_int.cu)

struct YccIntBatchParams
{
    IntDecodeParams shared; // pointers, strides and sizes unused
    int32_t count;
    int64_t units;
    BatchRecord image[kBatchChunkImages];
};

struct DecodeEdgeBatchParams
{
    DecodeParams shared; // pointers, strides and sizes unused
    int32_t count;
    int64_t units;
    BatchRecord window[2 * kBatchChunkImages];
};

// CUDA 12.1+ on Volta and later: at most 32764 bytes of kernel parameters.
static_assert(sizeof(RgbIntBatchParams) <= 32764 && sizeof(PlanarBatchParams) <= 32764 && sizeof(YccIntBatchParams) <= 32764 &&
                  sizeof(DecodeEdgeBatchParams) <= 32764,
              "a chunk must fit one kernel parameter block");

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

template <typename HostT, typename PlaneT, int CHANNELS, int XS, int YS, int PREMULTIPLY>
__global__ void __launch_bounds__(kRgbThreads) EncodeRgbIntBatchKernel(const __grid_constant__ RgbIntBatchParams b)
{
    __shared__ float hostLut[(sizeof(HostT) == 1 && sizeof(PlaneT) == 2) ? 256 : 1];
    StageHostLut<HostT, PlaneT>(hostLut, b.shared.maxCode);
    const int lane = threadIdx.x & 31;
    const long long warpCount = static_cast<long long>(gridDim.x) * kWarps;
    int record = 0;
    for (long long unit = static_cast<long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5); unit < b.units; unit += warpCount)
    {
        record = RecordOfUnit(b.image, b.count, record, unit);
        const BatchRecord& r = b.image[record];
        Rgb16Params p = b.shared;
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
__global__ void __launch_bounds__(kBatchEdgeThreads) EncodePlanarBatchKernel(const __grid_constant__ PlanarBatchParams b)
{
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();
    int record = 0;
    for (long long unit = blockIdx.x; unit < b.units; unit += gridDim.x)
    {
        record = RecordOfUnit(b.window, b.count, record, unit);
        const BatchRecord& r = b.window[record];
        EncodeParams p = b.shared;
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
__global__ void __launch_bounds__(kRgbThreads, kDecodeBlocksPerSm) DecodeYccToRgbIntBatchKernel(const __grid_constant__ YccIntBatchParams b)
{
    constexpr int kRows = YS ? 2 : 1;
    extern __shared__ __align__(16) uint8_t sharedBytes[];
    const YccTables tables = StageYccTables<SampleT, ALPHA>(sharedBytes, b.shared);
    __syncthreads();
    const YccFactors factors = MakeYccFactors<SampleT>(b.shared.matrix);
    const int lane = threadIdx.x & 31;
    const long long warpCount = static_cast<long long>(gridDim.x) * kWarps;
    int record = 0;
    for (long long unit = static_cast<long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5); unit < b.units; unit += warpCount)
    {
        record = RecordOfUnit(b.image, b.count, record, unit);
        const BatchRecord& r = b.image[record];
        IntDecodeParams p = b.shared;
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
__global__ void __launch_bounds__(kBatchEdgeThreads) DecodeBatchKernel(const __grid_constant__ DecodeEdgeBatchParams b)
{
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();
    int record = 0;
    for (long long unit = blockIdx.x; unit < b.units; unit += gridDim.x)
    {
        record = RecordOfUnit(b.window, b.count, record, unit);
        const BatchRecord& r = b.window[record];
        DecodeParams p = b.shared;
        for (int k = 0; k < 4; ++k)
        {
            p.plane[k] = r.plane[k];
            p.planeStride[k] = r.planeStride[k];
        }
        p.rows = const_cast<void*>(r.rows);
        p.rowStride = r.rowStride;
        p.width = r.width;
        p.rowCount = r.rowCount;
        p.yPhase = 0; // PlanDecodeBatch: every window starts on a 4:2:0 row pair
        DecodeChunkPixel<PlaneT, HostT, kBatchEdgeThreads>(p, t, static_cast<unsigned>(unit - r.firstUnit));
    }
}

template <typename SampleT, int ALPHA>
void LaunchYccIntBatch(const YccIntBatchParams& b, int xs, int ys, unsigned grid, size_t shared, cudaStream_t stream)
{
    if (xs == 1 && ys == 1) DecodeYccToRgbIntBatchKernel<SampleT, 1, 1, ALPHA><<<grid, kRgbThreads, shared, stream>>>(b);
    else if (xs == 1) DecodeYccToRgbIntBatchKernel<SampleT, 1, 0, ALPHA><<<grid, kRgbThreads, shared, stream>>>(b);
    else DecodeYccToRgbIntBatchKernel<SampleT, 0, 0, ALPHA><<<grid, kRgbThreads, shared, stream>>>(b);
}

unsigned GridFor(long long blocks, long long cap)
{
    return static_cast<unsigned>(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

template <typename HostT, typename PlaneT, int CHANNELS, int PREMULTIPLY>
void LaunchRgbIntBatch(const RgbIntBatchParams& b, int xs, int ys, unsigned grid, cudaStream_t stream)
{
    if (xs == 1 && ys == 1) EncodeRgbIntBatchKernel<HostT, PlaneT, CHANNELS, 1, 1, PREMULTIPLY><<<grid, kRgbThreads, 0, stream>>>(b);
    else if (xs == 1) EncodeRgbIntBatchKernel<HostT, PlaneT, CHANNELS, 1, 0, PREMULTIPLY><<<grid, kRgbThreads, 0, stream>>>(b);
    else EncodeRgbIntBatchKernel<HostT, PlaneT, CHANNELS, 0, 0, PREMULTIPLY><<<grid, kRgbThreads, 0, stream>>>(b);
}

template <typename HostT, typename PlaneT>
void LaunchRgbIntBatchChannels(const RgbIntBatchParams& b, int channels, bool premultiply, int xs, int ys, unsigned grid, cudaStream_t stream)
{
    if (channels == 4 && premultiply) LaunchRgbIntBatch<HostT, PlaneT, 4, 1>(b, xs, ys, grid, stream);
    else if (channels == 4) LaunchRgbIntBatch<HostT, PlaneT, 4, 0>(b, xs, ys, grid, stream);
    else LaunchRgbIntBatch<HostT, PlaneT, 3, 0>(b, xs, ys, grid, stream);
}

} // namespace

int LaunchEncodeBatchChunk(const EncodeParams& shared, int hostDepth, const BatchChunk& chunk, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const int smCount = SmCountOrDefault(shared.smCount);
    {
        RgbIntBatchParams b{};
        b.shared = RgbIntShared(shared);
        b.count = chunk.images;
        b.units = chunk.interiorUnits;
        for (int i = 0; i < chunk.images; ++i)
        {
            b.image[i] = chunk.interior[i];
        }
        // one warp per unit; the single-image kernel's cap of 16 CTAs per SM
        const unsigned grid = GridFor((chunk.interiorUnits + kWarps - 1) / kWarps, static_cast<long long>(smCount) * 16);
        const bool wide = shared.imageDepth > 8;
        if (hostDepth == 16)
        {
            if (wide) LaunchRgbIntBatchChannels<uint16_t, uint16_t>(b, shared.channels, shared.premultiply != 0, shared.xs, shared.ys, grid, stream);
            else LaunchRgbIntBatchChannels<uint16_t, uint8_t>(b, shared.channels, shared.premultiply != 0, shared.xs, shared.ys, grid, stream);
        }
        else
        {
            if (wide) LaunchRgbIntBatchChannels<uint8_t, uint16_t>(b, shared.channels, shared.premultiply != 0, shared.xs, shared.ys, grid, stream);
            else LaunchRgbIntBatchChannels<uint8_t, uint8_t>(b, shared.channels, shared.premultiply != 0, shared.xs, shared.ys, grid, stream);
        }
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess)
        {
            return ReportLaunchFailure(static_cast<int>(e));
        }
    }
    if (chunk.windows == 0)
    {
        return BatchChunkLaunches(chunk);
    }
    PlanarBatchParams b{};
    b.shared = shared;
    b.shared.useCurveView = 0; // integer hosts: no transfer curve
    b.count = chunk.windows;
    b.units = chunk.windowUnits;
    for (int i = 0; i < chunk.windows; ++i)
    {
        b.window[i] = chunk.window[i];
    }
    const unsigned grid = GridFor(chunk.windowUnits, static_cast<long long>(smCount) * 16);
    if (hostDepth == 16) EncodePlanarBatchKernel<uint16_t><<<grid, kBatchEdgeThreads, 0, stream>>>(b);
    else EncodePlanarBatchKernel<uint8_t><<<grid, kBatchEdgeThreads, 0, stream>>>(b);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? BatchChunkLaunches(chunk) : ReportLaunchFailure(static_cast<int>(e));
}

int LaunchDecodeBatchChunk(const DecodeParams& shared, const BatchChunk& chunk, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const int smCount = SmCountOrDefault(shared.smCount);
    {
        YccIntBatchParams b{};
        b.shared.bitDepth = shared.bitDepth;
        b.shared.maxCode = shared.maxCode;
        b.shared.range = shared.range;
        b.shared.matrix = shared.matrix;
        b.shared.verifiedGreenDivision = shared.verifiedGreenDivision;
        b.count = chunk.images;
        b.units = chunk.interiorUnits;
        for (int i = 0; i < chunk.images; ++i)
        {
            b.image[i] = chunk.interior[i];
        }
        // DecodeYccToRgbIntKernel's tables (at most 40 KB: no opt-in beyond the default 48 KB) and grid cap
        const size_t entries = static_cast<size_t>(1) << shared.bitDepth;
        const bool host8 = shared.hostDepth == 8;
        const size_t bytes = 2 * sizeof(float) * entries + ((shared.hasAlpha && !host8) ? sizeof(uint16_t) * entries : 0);
        const unsigned grid = GridFor((chunk.interiorUnits + kWarps - 1) / kWarps, static_cast<long long>(smCount) * kDecodeBlocksPerSm);
        if (host8)
        {
            if (shared.hasAlpha) LaunchYccIntBatch<uint8_t, 1>(b, shared.xs, shared.ys, grid, bytes, stream);
            else LaunchYccIntBatch<uint8_t, 0>(b, shared.xs, shared.ys, grid, bytes, stream);
        }
        else
        {
            if (shared.hasAlpha) LaunchYccIntBatch<uint16_t, 1>(b, shared.xs, shared.ys, grid, bytes, stream);
            else LaunchYccIntBatch<uint16_t, 0>(b, shared.xs, shared.ys, grid, bytes, stream);
        }
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess)
        {
            return ReportLaunchFailure(static_cast<int>(e));
        }
    }
    if (chunk.windows == 0)
    {
        return BatchChunkLaunches(chunk);
    }
    DecodeEdgeBatchParams b{};
    b.shared = shared;
    b.count = chunk.windows;
    b.units = chunk.windowUnits;
    for (int i = 0; i < chunk.windows; ++i)
    {
        b.window[i] = chunk.window[i];
    }
    const unsigned grid = GridFor(chunk.windowUnits, static_cast<long long>(smCount) * 16);
    if (shared.hostDepth == 16) DecodeBatchKernel<uint16_t, uint16_t><<<grid, kBatchEdgeThreads, 0, stream>>>(b);
    else DecodeBatchKernel<uint8_t, uint8_t><<<grid, kBatchEdgeThreads, 0, stream>>>(b);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? BatchChunkLaunches(chunk) : ReportLaunchFailure(static_cast<int>(e));
}

} // namespace avifgpu
