// kernels_generic.cu -- the general kernels: every configuration of the path, one thread per pixel (decode,
// reference-layout encode) or per chroma site (planar YCbCr encode).  Correct for every combination the
// reference's twelve row shuttles accept; the tuned kernels in kernels_fast.cu take over for the layouts
// BASELINE.json measures and fall back to these for everything else.  Both sets share pixel_math.cuh, so
// they cannot disagree on arithmetic.
#include "generic_units.cuh"
#include "kernel_params.h"
#include "launch_keys.h"
#include "curve_lookup.cuh"
#include "../../include/avifgpu.h"

#include <cuda_runtime.h>

namespace avifgpu
{

using namespace avifpix;
using avifmath::LibmTables;

namespace
{

constexpr int kThreads = 256;

// Reference layout: one thread per pixel.
template <typename HostT>
__global__ void __launch_bounds__(kThreads) EncodeReferenceLayoutKernel(const EncodeParams p)
{
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();

    const int chunks = (p.width + kThreads - 1) / kThreads;
    const int x = static_cast<int>(blockIdx.x % chunks) * kThreads + threadIdx.x;
    const int y = static_cast<int>(blockIdx.x / chunks);
    if (x >= p.width || y >= p.rowCount)
    {
        return;
    }
    const HostT* px = reinterpret_cast<const HostT*>(static_cast<const uint8_t*>(p.rows) + static_cast<int64_t>(y) * p.rowStride) +
                      static_cast<int64_t>(x) * p.channels;
    uint32_t codes[4] = { 0, 0, 0, 0 };
    HostPixelToCodes<HostT>(p, px, codes, t);

    const bool wide = p.imageDepth > 8;
    if (p.channels <= 2)
    {
        StoreCode(p.plane[0], p.planeStride[0], y, x, wide, codes[0]);
        if (p.hasAlpha)
        {
            StoreCode(p.plane[3], p.planeStride[3], y, x, wide, codes[1]);
        }
    }
    else
    {
        for (int i = 0; i < p.channels; ++i)
        {
            StoreCode(p.plane[0], p.planeStride[0], y, x * p.channels + i, wide, codes[i]);
        }
    }
}

// Planar YCbCr layout: one thread per chroma site (1x1, 2x1 or 2x2 pixels).
template <typename HostT>
__global__ void __launch_bounds__(kThreads) EncodePlanarKernel(const EncodeParams p)
{
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();

    EncodePlanarSite<HostT, kThreads>(p, t, blockIdx.x);
}

// The light-level kernels (float hosts, PQ; light_level.cuh): the kernels above, every pixel's codes into the thread's tally,
// one flush per warp.  No thread leaves early: the flush needs the whole warp.
__global__ void __launch_bounds__(kThreads) EncodeReferenceLayoutLightKernel(const EncodeParams p, const LightSink light)
{
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();

    LightTally tally{ 0u, 0ull };
    const int chunks = (p.width + kThreads - 1) / kThreads;
    const int x = static_cast<int>(blockIdx.x % chunks) * kThreads + threadIdx.x;
    const int y = static_cast<int>(blockIdx.x / chunks);
    if (x < p.width && y < p.rowCount)
    {
        const float* px = reinterpret_cast<const float*>(static_cast<const uint8_t*>(p.rows) + static_cast<int64_t>(y) * p.rowStride) +
                          static_cast<int64_t>(x) * p.channels;
        uint32_t codes[4] = { 0, 0, 0, 0 };
        HostPixelToCodes<float>(p, px, codes, t);
        TallyPixel(tally, light.levels, p, codes, t);
        if (p.channels <= 2)
        {
            StoreCode(p.plane[0], p.planeStride[0], y, x, true, codes[0]);
            if (p.hasAlpha)
            {
                StoreCode(p.plane[3], p.planeStride[3], y, x, true, codes[1]);
            }
        }
        else
        {
            for (int i = 0; i < p.channels; ++i)
            {
                StoreCode(p.plane[0], p.planeStride[0], y, x * p.channels + i, true, codes[i]);
            }
        }
    }
    FlushLightTally(tally, LaunchPixelsForFirstWarp(static_cast<uint64_t>(p.width) * p.rowCount), light.acc);
}

__global__ void __launch_bounds__(kThreads) EncodePlanarLightKernel(const EncodeParams p, const LightSink light)
{
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();

    LightTally tally{ 0u, 0ull };
    EncodePlanarSite<float, kThreads, 1>(p, t, blockIdx.x, &tally, light.levels);
    FlushLightTally(tally, LaunchPixelsForFirstWarp(static_cast<uint64_t>(p.width) * p.rowCount), light.acc);
}
// ---- decode ----------------------------------------------------------------------------------------------

// PlaneT uint8_t pairs with HostT uint8_t; PlaneT uint16_t with HostT uint16_t or float.
template <typename PlaneT, typename HostT>
__global__ void __launch_bounds__(kThreads) DecodeKernel(const DecodeParams p)
{
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();

    DecodeChunkPixel<PlaneT, HostT, kThreads>(p, t, blockIdx.x);
}

// ---- primitive sweep (parity gates on the device libm) ------------------------------------------------------

__global__ void __launch_bounds__(kThreads) TransferKernel(int function, float param, const float* __restrict__ in,
                                                           float* __restrict__ out, size_t count)
{
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();
    const float luminanceForward = param / 10000.0f;  // ColorTransfer.cpp:86
    const float luminanceInverse = 10000.0f / param;  // ColorTransfer.cpp:114
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < count;
         i += static_cast<size_t>(gridDim.x) * blockDim.x)
    {
        const float v = in[i];
        float r;
        switch (function)
        {
        case AVIFGPU_FN_LINEAR_TO_PQ: r = LinearToPQ(v, luminanceForward, t); break;
        case AVIFGPU_FN_PQ_TO_LINEAR: r = PQToLinear(v, luminanceInverse, t); break;
        case AVIFGPU_FN_LINEAR_TO_SMPTE428: r = LinearToSMPTE428(v, t); break;
        case AVIFGPU_FN_SMPTE428_TO_LINEAR: r = SMPTE428ToLinear(v, t); break;
        case AVIFGPU_FN_HLG_TO_LINEAR: r = HLGToLinear(v, t); break;
        case AVIFGPU_FN_LINEAR_TO_HLG: r = LinearToHLG(v, t); break;
        case AVIFGPU_FN_POWF: r = avifmath::Powf(v, param, t); break;
        case AVIFGPU_FN_EXPF: r = avifmath::Expf(v, t); break;
        default: r = avifmath::Logf(v, t); break;
        }
        out[i] = r;
    }
}

} // namespace

EncodeParams GenericEncodeView(const EncodeParams& params, int hostDepth)
{
    EncodeParams p = params;
    p.useCurveView = 0;
    if (hostDepth == 32 && p.curveTable != nullptr && p.curveTable->compact != nullptr && p.curveTable->bandBits != nullptr &&
        (p.transfer == AVIFGPU_TRANSFER_PQ || p.transfer == AVIFGPU_TRANSFER_SMPTE428 || p.transfer == AVIFGPU_TRANSFER_HLG))
    {
        p.curveView = *p.curveTable;
        p.useCurveView = 1;
    }
    return p;
}

int LaunchEncodeGeneric(const EncodeParams& params, int hostDepth, void* streamHandle, const LightSink* light)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    if (params.width <= 0 || params.rowCount <= 0)
    {
        return 0;
    }
    const EncodeParams p = GenericEncodeView(params, hostDepth);
    if (p.planar)
    {
        const int sitesX = (p.width + p.xs) >> p.xs;
        const int sitesY = (p.rowCount + p.ys) >> p.ys;
        const unsigned grid = static_cast<unsigned>((sitesX + kThreads - 1) / kThreads) * static_cast<unsigned>(sitesY);
        if (light != nullptr)
        {
            EncodePlanarLightKernel<<<grid, kThreads, 0, stream>>>(p, *light); // float hosts only (avifgpu_encode_rows_device_light_level)
        }
        else
        {
            WithHostDepth(hostDepth, [&](auto, auto host) { EncodePlanarKernel<TypeOf<decltype(host)>><<<grid, kThreads, 0, stream>>>(p); });
        }
    }
    else
    {
        const unsigned grid = static_cast<unsigned>((p.width + kThreads - 1) / kThreads) * static_cast<unsigned>(p.rowCount);
        if (light != nullptr)
        {
            EncodeReferenceLayoutLightKernel<<<grid, kThreads, 0, stream>>>(p, *light);
        }
        else
        {
            WithHostDepth(hostDepth, [&](auto, auto host) { EncodeReferenceLayoutKernel<TypeOf<decltype(host)>><<<grid, kThreads, 0, stream>>>(p); });
        }
    }
    const cudaError_t launchError = cudaGetLastError();
    return launchError == cudaSuccess ? 1 : ReportLaunchFailure(static_cast<int>(launchError));
}

int LaunchDecodeGeneric(const DecodeParams& p, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    if (p.width <= 0 || p.rowCount <= 0)
    {
        return 0;
    }
    const unsigned grid = static_cast<unsigned>((p.width + kThreads - 1) / kThreads) * static_cast<unsigned>(p.rowCount);
    WithHostDepth(p.hostDepth, [&](auto plane, auto host) { DecodeKernel<TypeOf<decltype(plane)>, TypeOf<decltype(host)>><<<grid, kThreads, 0, stream>>>(p); });
    const cudaError_t launchError = cudaGetLastError();
    return launchError == cudaSuccess ? 1 : ReportLaunchFailure(static_cast<int>(launchError));
}

// The generic launchers return 0 for an empty strip.
int CompleteEncode(cudaError_t tuned, const EncodeParams& p, int hostDepth, int coveredWidth, int coveredRows, void* stream, const LightSink* light)
{
    if (tuned != cudaSuccess)
    {
        return ReportLaunchFailure(static_cast<int>(tuned));
    }
    const int right = LaunchEncodeGeneric(EncodeWindow(p, hostDepth, coveredWidth, 0, p.width - coveredWidth, p.rowCount), hostDepth, stream, light);
    if (right < 0)
    {
        return right;
    }
    const int bottom = LaunchEncodeGeneric(EncodeWindow(p, hostDepth, 0, coveredRows, coveredWidth, p.rowCount - coveredRows), hostDepth, stream, light);
    return bottom < 0 ? bottom : 1 + right + bottom;
}

int CompleteDecode(cudaError_t tuned, const DecodeParams& p, int coveredWidth, int coveredRows, void* stream)
{
    if (tuned != cudaSuccess)
    {
        return ReportLaunchFailure(static_cast<int>(tuned));
    }
    const int right = LaunchDecodeGeneric(DecodeWindow(p, coveredWidth, 0, p.width - coveredWidth, p.rowCount), stream);
    if (right < 0)
    {
        return right;
    }
    const int bottom = LaunchDecodeGeneric(DecodeWindow(p, 0, coveredRows, coveredWidth, p.rowCount - coveredRows), stream);
    return bottom < 0 ? bottom : 1 + right + bottom;
}

int LaunchTransfer(int function, float param, const float* in, float* out, size_t count, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    if (count == 0)
    {
        return 0;
    }
    size_t blocks = (count + kThreads - 1) / kThreads;
    if (blocks > 132u * 16u)
    {
        blocks = 132u * 16u;
    }
    TransferKernel<<<static_cast<unsigned>(blocks), kThreads, 0, stream>>>(function, param, in, out, count);
    const cudaError_t launchError = cudaGetLastError();
    return launchError == cudaSuccess ? 1 : ReportLaunchFailure(static_cast<int>(launchError));
}

namespace
{
// ColorTransfer.cpp:192-220 over `pixels` RGB triples.
__global__ void __launch_bounds__(kThreads) HlgOotfKernel(int inverse, float lumaR, float lumaG, float lumaB, float displayGamma, float peak,
                                                          const float* __restrict__ in, float* __restrict__ out, size_t pixels)
{
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < pixels; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    {
        float r = in[3 * i], g = in[3 * i + 1], b = in[3 * i + 2];
        if (inverse)
        {
            ApplyInverseHLGOOTF(r, g, b, lumaR, lumaG, lumaB, displayGamma, peak, t);
        }
        else
        {
            ApplyHLGOOTF(r, g, b, lumaR, lumaG, lumaB, displayGamma - 1.0f, peak, t);
        }
        out[3 * i] = r;
        out[3 * i + 1] = g;
        out[3 * i + 2] = b;
    }
}
} // namespace

int LaunchHlgOotf(int inverse, const float luma[3], float displayGamma, float peak, const float* in, float* out, size_t pixels, void* streamHandle)
{
    if (pixels == 0)
    {
        return 0;
    }
    size_t blocks = (pixels + kThreads - 1) / kThreads;
    if (blocks > 132 * 16)
    {
        blocks = 132 * 16;
    }
    HlgOotfKernel<<<static_cast<unsigned>(blocks), kThreads, 0, static_cast<cudaStream_t>(streamHandle)>>>(inverse, luma[0], luma[1], luma[2], displayGamma, peak, in,
                                                                                                      out, pixels);
    const cudaError_t launchError = cudaGetLastError();
    return launchError == cudaSuccess ? 1 : ReportLaunchFailure(static_cast<int>(launchError));
}

} // namespace avifgpu
