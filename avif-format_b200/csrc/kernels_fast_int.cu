// kernels_fast_int.cu -- tuned kernels for the 16-bit integer hosts (BASELINE configs 4 and 5).  Both are pure
// streaming conversions (a few float operations per sample), so the design goal is simply to keep HBM busy:
// 128-bit loads and stores, several of them in flight per thread, no integer<->float conversion instructions
// (they issue on the quarter-rate pipe and would cap config 4 just below the HBM roofline).
//
//   Gray16 -> Y plane          one 65536-entry uint16 table in shared memory (128 KB), built once per
//                              configuration by evaluating the exact per-sample formula for every input; a thread
//                              converts 8 samples per 128-bit load.
//   RGB(A)16 -> planar YCbCr   the 16-bit -> N-bit mapping is evaluated arithmetically (it is four float
//                              operations), the forward matrix and the 4:2:2 / 4:2:0 down-filter are fused, a
//                              thread converts 8 pixels (x 2 rows for 4:2:0).
#include "group_walk.cuh"
#include "int_units.cuh"
#include "kernel_params.h"
#include "launch_keys.h"
#include "packed_f32x2.cuh"
#include "../../include/avifgpu.h"

#include <cuda_runtime.h>

namespace avifgpu
{

using namespace avifpix;
using avifmath::LibmTables;

namespace
{

// ---- Gray16 --------------------------------------------------------------------------------------------------------

constexpr int kLutThreads = 1024;
constexpr int kLutEntries = 65536;

// Fills lut[v] for every 16-bit host sample with the exact code of the configuration:
//   reference LUT path   clamp((int)((v / 32768f) * max + 0.5f), 0, max)                       WriteHeifImage.cpp:140-166
//   SMPTE 428 curve      (u16)clamp(LinearToSMPTE428(v / 32768f) * max, 0, max)                 DESIGN.md "Config 5"
__global__ void __launch_bounds__(256) BuildGray16LutKernel(uint16_t* __restrict__ lut, int smpte428, uint32_t maxCode)
{
    __shared__ uint64_t libmStorage[96];
    const LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();
    const float maxCodeFloat = static_cast<float>(maxCode);
    for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < kLutEntries; v += gridDim.x * blockDim.x)
    {
        uint32_t code;
        if (smpte428)
        {
            code = FloatToCode(LinearToSMPTE428(static_cast<float>(v) / 32768.0f, t), maxCodeFloat);
        }
        else
        {
            code = DepthLutEntry(v, 32768.0f, maxCode);
        }
        lut[v] = static_cast<uint16_t>(code);
    }
}

struct Gray16Params
{
    const uint8_t* rows;
    int64_t rowStride;
    uint8_t* planeY;
    int64_t strideY;
    int32_t chunksPerRow; // 8 samples each
    int32_t rowCount;
    const uint16_t* lut;  // 65536 entries, global memory
};

__device__ __forceinline__ uint4 LookupEight(const uint16_t* __restrict__ lut, uint4 in)
{
    uint4 out;
    out.x = lut[in.x & 0xffffu] | (static_cast<uint32_t>(lut[in.x >> 16]) << 16);
    out.y = lut[in.y & 0xffffu] | (static_cast<uint32_t>(lut[in.y >> 16]) << 16);
    out.z = lut[in.z & 0xffffu] | (static_cast<uint32_t>(lut[in.z >> 16]) << 16);
    out.w = lut[in.w & 0xffffu] | (static_cast<uint32_t>(lut[in.w >> 16]) << 16);
    return out;
}

__global__ void __launch_bounds__(kLutThreads, 1) EncodeGray16LutKernel(const Gray16Params p)
{
    extern __shared__ __align__(16) uint16_t sharedLut[];
    {
        const uint4* source = reinterpret_cast<const uint4*>(p.lut);
        uint4* target = reinterpret_cast<uint4*>(sharedLut);
        for (int i = threadIdx.x; i < kLutEntries * 2 / 16; i += blockDim.x)
        {
            target[i] = source[i];
        }
    }
    __syncthreads();

    constexpr int kUnroll = 4;
    const long long chunks = static_cast<long long>(p.chunksPerRow) * p.rowCount;
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    // (measured: walking row / column incrementally, group_walk.cuh, makes THIS loop slower -- 0.86 vs 0.95 of the HBM
    // peak; the division is hidden under four loads in flight and a 16-bit look-up per sample)
    for (long long base = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; base < chunks; base += stride * kUnroll)
    {
        uint4 in[kUnroll];
        long long outOffset[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u)
        {
            const long long chunk = base + u * stride;
            if (chunk < chunks)
            {
                const long long row = chunk / p.chunksPerRow;
                const long long column = chunk - row * p.chunksPerRow;
                in[u] = __ldcs(reinterpret_cast<const uint4*>(p.rows + row * p.rowStride + column * 16));
                outOffset[u] = row * p.strideY + column * 16;
            }
            else
            {
                in[u] = make_uint4(0u, 0u, 0u, 0u);
                outOffset[u] = -1;
            }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u)
        {
            if (outOffset[u] >= 0)
            {
                __stcs(reinterpret_cast<uint4*>(p.planeY + outOffset[u]), LookupEight(sharedLut, in[u]));
            }
        }
    }
}

// ---- RGB(A) 8/16-bit hosts -> planar YCbCr (int_units.cuh) --------------------------------------------------------

__global__ void VerifyFastPremultiplyKernel(uint32_t maxCode, unsigned long long* __restrict__ counter)
{
    const float maxCodeFloat = static_cast<float>(maxCode);
    const float reciprocal = 1.0f / maxCodeFloat;
    const unsigned long long pairs = static_cast<unsigned long long>(maxCode + 1u) * (maxCode + 1u);
    unsigned long long bad = 0;
    for (unsigned long long i = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < pairs;
         i += static_cast<unsigned long long>(gridDim.x) * blockDim.x)
    {
        const uint32_t colour = static_cast<uint32_t>(i % (maxCode + 1u));
        const uint32_t alpha = static_cast<uint32_t>(i / (maxCode + 1u));
        const uint32_t expected = PremultiplyCodeGuarded(colour, alpha, maxCode);
        const uint32_t fast = __float_as_uint(FastPremultiplyBiased(static_cast<float>(colour), static_cast<float>(alpha), maxCodeFloat, reciprocal)) & 0x7fffffu;
        if (fast != expected)
        {
            ++bad;
        }
    }
    if (bad)
    {
        atomicAdd(counter, bad);
    }
}

// HostT: uint8_t / uint16_t host samples; PlaneT: uint8_t (8-bit image) / uint16_t (10 / 12-bit image) plane samples.
// PREMULTIPLY (CHANNELS == 4 only): the colour codes are multiplied by the alpha code in the image's depth before the matrix
// (WriteHeifImage.cpp:700-718, 760-778, 877-895, 947-965), through FastPremultiplyBiased.  DEST: the avifgpu_source_layout
// bits of the planes written (EncodeRgbIntGroup); 0 is libheif's planar, low-bit layout.
template <typename HostT, typename PlaneT, int CHANNELS, int XS, int YS, int PREMULTIPLY, int DEST>
__global__ void __launch_bounds__(kRgbThreads) EncodeRgbIntPlanarKernel(const Rgb16Params p)
{
    // (one copy: a copy per shared-memory bank makes the look-up conflict-free but costs every CTA 32 KB and 8192 table
    // entries to fill; computing the entry instead -- division by 255 through a verified reciprocal step -- costs six more
    // instructions per sample:
    // the look-up's shared-memory pipe is the lesser evil next to six more instructions per sample)
    __shared__ float hostLut[(sizeof(HostT) == 1 && sizeof(PlaneT) == 2) ? 256 : 1];
    StageHostLut<HostT, PlaneT>(hostLut, p.maxCode);
    const int32_t rowPairs = (p.rowCount + YS) >> YS;
    for (GroupWalk walk(static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x, static_cast<long long>(gridDim.x) * blockDim.x, p.groupsPerRow, rowPairs);
         walk.Inside(rowPairs); walk.Advance(rowPairs))
    {
        EncodeRgbIntGroup<HostT, PlaneT, CHANNELS, XS, YS, PREMULTIPLY, DEST>(p, hostLut, walk.row, walk.column);
    }
}

// ---- Gray(+A) 8/16-bit hosts -> Y (+A) planes (WriteHeifImage.cpp:169-500 without premultiplication) ------------------------
// The same depth mapping as the colour kernel, no matrix: a thread converts 8 pixels.
template <typename HostT, typename PlaneT, int CHANNELS>
__global__ void __launch_bounds__(kRgbThreads) EncodeGrayIntKernel(const Rgb16Params p)
{
    constexpr int kWordsPerRow = CHANNELS * 2 * static_cast<int>(sizeof(HostT)); // 8 pixels x CHANNELS samples / 4 bytes
    constexpr int kVectorWords = (kWordsPerRow % 4 == 0) ? 4 : 2;
    constexpr int kPlaneBytes = static_cast<int>(sizeof(PlaneT));
    __shared__ float hostLut[(sizeof(HostT) == 1 && sizeof(PlaneT) == 2) ? 256 : 1];
    if (sizeof(HostT) == 1 && sizeof(PlaneT) == 2)
    {
        for (uint32_t v = threadIdx.x; v < 256; v += blockDim.x)
        {
            hostLut[v] = __uint_as_float(0x4b000000u | DepthLutEntry(v, 255.0f, p.maxCode));
        }
        __syncthreads();
    }
    const auto loadGroup = [&](uint32_t (&words)[kWordsPerRow], long long row, long long column)
    {
        const uint8_t* source = p.rows + row * p.rowStride + column * (kWordsPerRow * 4);
#pragma unroll
        for (int q = 0; q < kWordsPerRow / kVectorWords; ++q)
        {
            if (kVectorWords == 4)
            {
                const uint4 w = __ldcs(reinterpret_cast<const uint4*>(source) + q);
                words[4 * q + 0] = w.x;
                words[4 * q + 1] = w.y;
                words[4 * q + 2] = w.z;
                words[4 * q + 3] = w.w;
            }
            else
            {
                const uint2 w = __ldcs(reinterpret_cast<const uint2*>(source) + q);
                words[2 * q + 0] = w.x;
                words[2 * q + 1] = w.y;
            }
        }
    };
    const auto convertGroup = [&](const uint32_t (&words)[kWordsPerRow], long long row, long long column)
    {
        if (sizeof(HostT) == 1 && sizeof(PlaneT) == 1 && CHANNELS == 1)
        {
            // Gray8 into an 8-bit image: the sample is the code (WriteHeifImage.cpp:224-240) -- the 8 bytes as they are
            __stcs(reinterpret_cast<uint2*>(p.plane[0] + row * p.stride[0] + column * 8), make_uint2(words[0], words[1]));
            return;
        }
        auto sample = [&](int k) -> uint32_t
        {
            if (sizeof(HostT) == 2)
            {
                const uint32_t w = words[k >> 1];
                return (k & 1) ? (w >> 16) : (w & 0xffffu);
            }
            return (words[k >> 2] >> (8 * (k & 3))) & 0xffu;
        };
        uint32_t yCodes[8], aCodes[8];
#pragma unroll
        for (int i = 0; i < 8; ++i)
        {
            yCodes[i] = BiasedToCode(SampleToBiasedCode<HostT, PlaneT>(sample(i * CHANNELS), p, hostLut));
            if (CHANNELS == 2)
            {
                aCodes[i] = BiasedToCode(SampleToBiasedCode<HostT, PlaneT>(sample(i * CHANNELS + 1), p, hostLut));
            }
        }
        StoreEight<PlaneT>(p.plane[0] + row * p.stride[0] + column * (8 * kPlaneBytes), yCodes);
        if (CHANNELS == 2)
        {
            StoreEight<PlaneT>(p.plane[3] + row * p.stride[3] + column * (8 * kPlaneBytes), aCodes);
        }
    };
    // 8-bit hosts: a group is 8 or 16 bytes -- four groups' loads in flight before the first is converted (the launch is bound
    // by memory latency otherwise: 28 % of the issue slots used, every warp on long_scoreboard); 16-bit hosts one at a time
    constexpr int kInFlight = sizeof(HostT) == 1 ? 4 : 1;
    GroupWalk walk(static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x, static_cast<long long>(gridDim.x) * blockDim.x, p.groupsPerRow, p.rowCount);
    if (kInFlight == 1)
    {
        for (; walk.Inside(p.rowCount); walk.Advance(p.rowCount))
        {
            uint32_t words[kWordsPerRow];
            loadGroup(words, walk.row, walk.column);
            convertGroup(words, walk.row, walk.column);
        }
        return;
    }
    while (walk.Inside(p.rowCount))
    {
        uint32_t wordsAll[kInFlight][kWordsPerRow];
        int rowOf[kInFlight], columnOf[kInFlight];
#pragma unroll
        for (int u = 0; u < kInFlight; ++u)
        {
            rowOf[u] = -1;
            columnOf[u] = 0;
            if (walk.Inside(p.rowCount))
            {
                rowOf[u] = walk.row;
                columnOf[u] = walk.column;
                loadGroup(wordsAll[u], walk.row, walk.column);
            }
            walk.Advance(p.rowCount);
        }
#pragma unroll
        for (int u = 0; u < kInFlight; ++u)
        {
            if (rowOf[u] >= 0)
            {
                convertGroup(wordsAll[u], rowOf[u], columnOf[u]);
            }
        }
    }
}

template <typename HostT, typename PlaneT>
cudaError_t LaunchGrayInt(const Rgb16Params& rp, int channels, int smCount, cudaStream_t stream)
{
    const long long groups = static_cast<long long>(rp.groupsPerRow) * rp.rowCount;
    const unsigned grid = GridFor((groups + kRgbThreads - 1) / kRgbThreads, static_cast<long long>(smCount) * kStreamBlocksPerSm);
    if (channels == 2) EncodeGrayIntKernel<HostT, PlaneT, 2><<<grid, kRgbThreads, 0, stream>>>(rp);
    else EncodeGrayIntKernel<HostT, PlaneT, 1><<<grid, kRgbThreads, 0, stream>>>(rp);
    return cudaGetLastError();
}

template <typename HostT, typename PlaneT, int CHANNELS, int XS, int YS, int PREMULTIPLY, int DEST>
cudaError_t LaunchRgbInt(const Rgb16Params& rp, int smCount, cudaStream_t stream)
{
    const long long groups = static_cast<long long>(rp.groupsPerRow) * ((rp.rowCount + YS) >> YS);
    const unsigned grid = GridFor((groups + kRgbThreads - 1) / kRgbThreads, static_cast<long long>(smCount) * kStreamBlocksPerSm);
    EncodeRgbIntPlanarKernel<HostT, PlaneT, CHANNELS, XS, YS, PREMULTIPLY, DEST><<<grid, kRgbThreads, 0, stream>>>(rp);
    return cudaGetLastError();
}

} // namespace

// Runs the exhaustive comparison behind FastPremultiplyBiased for one bit depth; returns the number of disagreements
// (0 = verified) or -1 on a CUDA error.  Synchronous.
long long VerifyFastPremultiply(uint32_t maxCode, void* streamHandle)
{
    return CountDisagreements(static_cast<cudaStream_t>(streamHandle), [&](unsigned long long* counter, cudaStream_t stream) {
        VerifyFastPremultiplyKernel<<<132 * 8, 256, 0, stream>>>(maxCode, counter);
    });
}

cudaError_t BuildGray16Lut(uint16_t* deviceLut, int smpte428, uint32_t maxCode, void* streamHandle)
{
    BuildGray16LutKernel<<<64, 256, 0, static_cast<cudaStream_t>(streamHandle)>>>(deviceLut, smpte428, maxCode);
    return cudaGetLastError();
}

cudaError_t LaunchEncodeGray16Lut(const EncodeParams& p, Interior inner, void* streamHandle)
{
    static std::atomic<uint64_t> configuredDevices{ 0 };
    if (const cudaError_t configured = AllowDynamicShared(EncodeGray16LutKernel, kLutEntries * 2, configuredDevices))
    {
        return configured;
    }
    Gray16Params gp{};
    gp.rows = static_cast<const uint8_t*>(p.rows);
    gp.rowStride = p.rowStride;
    gp.planeY = static_cast<uint8_t*>(p.plane[0]);
    gp.strideY = p.planeStride[0];
    gp.chunksPerRow = inner.width / 8;
    gp.rowCount = inner.rows;
    gp.lut = p.gray16Lut;
    EncodeGray16LutKernel<<<SmCountOrDefault(p.smCount), kLutThreads, kLutEntries * 2, static_cast<cudaStream_t>(streamHandle)>>>(gp);
    return cudaGetLastError();
}

// Gray(+A) hosts in the reference layout (Y plane [0], alpha plane [3]).
cudaError_t LaunchEncodeGrayInt(const EncodeParams& p, int hostDepth, Interior inner, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const int smCount = SmCountOrDefault(p.smCount);
    Rgb16Params rp{};
    rp.rows = static_cast<const uint8_t*>(p.rows);
    rp.rowStride = p.rowStride;
    for (int k = 0; k < 4; ++k)
    {
        rp.plane[k] = static_cast<uint8_t*>(p.plane[k]);
        rp.stride[k] = p.planeStride[k];
    }
    rp.groupsPerRow = inner.width / 8;
    rp.rowCount = inner.rows;
    rp.maxCodeFloat = p.maxCodeFloat;
    rp.biasedMax = 8388608.0f + p.maxCodeFloat;
    rp.maxCode = p.maxCode;
    rp.maxReciprocal = 1.0f / p.maxCodeFloat;
    const bool widePlanes = p.imageDepth > 8;
    if (hostDepth == 16)
    {
        return widePlanes ? LaunchGrayInt<uint16_t, uint16_t>(rp, p.channels, smCount, stream) : LaunchGrayInt<uint16_t, uint8_t>(rp, p.channels, smCount, stream);
    }
    return widePlanes ? LaunchGrayInt<uint8_t, uint16_t>(rp, p.channels, smCount, stream) : LaunchGrayInt<uint8_t, uint8_t>(rp, p.channels, smCount, stream);
}

cudaError_t LaunchEncodeRgbInt(const EncodeParams& p, int hostDepth, Interior inner, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const int smCount = SmCountOrDefault(p.smCount);
    Rgb16Params rp = RgbIntShared(p);
    rp.rows = static_cast<const uint8_t*>(p.rows);
    rp.rowStride = p.rowStride;
    for (int k = 0; k < 4; ++k)
    {
        rp.plane[k] = static_cast<uint8_t*>(p.plane[k]);
        rp.stride[k] = p.planeStride[k];
    }
    rp.groupsPerRow = inner.width / 8;
    rp.rowCount = inner.rows;
    return WithRgbIntKey(p, hostDepth, [&](auto host, auto plane, auto channels, auto premultiply, auto xs, auto ys, auto dest) {
        return LaunchRgbInt<TypeOf<decltype(host)>, TypeOf<decltype(plane)>, channels(), xs(), ys(), premultiply(), dest()>(rp, smCount, stream);
    });
}

} // namespace avifgpu
