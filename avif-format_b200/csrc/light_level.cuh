// light_level.cuh -- the content light level that avifgpu_encode_rows_device_light_level measures while it encodes
// (DESIGN.md section 5): the light level of a pixel is level(max(R', G', B')) of its transfer-curve codes (the Y code for
// gray hosts), level(k) = (uint32_t)(PQToLinear(k / maxCode, 1) * 2^22), truncated -- the absolute PQ scale, 2^22 = 10000
// cd/m2.  A light-level kernel keeps a running maximum code and a 64-bit level sum per thread in registers for its whole
// walk and flushes them once per warp at exit; the tuned kernels read level(k) from the context's table of the image
// depth (2^depth words, read through L1), the generic kernels evaluate it in place when there is no table yet.
#ifndef AVIFGPU_LIGHT_LEVEL_CUH
#define AVIFGPU_LIGHT_LEVEL_CUH

#include <stdint.h>

#include "pixel_math.cuh"
#include "../../include/avifgpu.h"

namespace avifgpu
{

// 2^22: level(k) is PQToLinear's absolute value (1.0 = 10000 cd/m2) in units of 2^-22.
constexpr float kLightLevelScale = 4194304.0f;

// level(k) for a code of an image whose largest code is maxCodeFloat (binary32, the glibc-identical powf).
AVIF_HD uint32_t LightLevelOf(uint32_t code, float maxCodeFloat, const avifmath::LibmTables& t)
{
    return static_cast<uint32_t>(avifpix::PQToLinear(static_cast<float>(code) / maxCodeFloat, 1.0f, t) * kLightLevelScale);
}

// Where a light-level launch adds its statistic: the caller's accumulator, and the context's level table of the image
// depth or nullptr (then only the generic kernels run, and they evaluate LightLevelOf).  The light-level kernels take it
// as a parameter of their own, so the plain kernels' parameter blocks stay as they are.
struct LightSink
{
    avifgpu_light_level* acc;
    const uint32_t* levels;
};

#if defined(__CUDACC__)
// One thread's share of the statistic, kept in registers.
struct LightTally
{
    uint32_t maxCode;
    uint64_t levelSum;
};

__device__ __forceinline__ void TallyCode(LightTally& tally, uint32_t code, uint32_t level)
{
    tally.maxCode = max(tally.maxCode, code);
    tally.levelSum += level;
}

// A tuned float kernel's lane: PIXELS pixels of R'G'B' codes (as floats, row-major, interleaved; pixels 4.. are the second
// row, taken only when it exists), max(R', G', B') of each with its level from the context's table.
template <int PIXELS, int N>
__device__ __forceinline__ void TallyLaneCodes(LightTally& tally, const float (&codeF)[N], const uint32_t* levels, bool secondRow)
{
#pragma unroll
    for (int pixel = 0; pixel < PIXELS; ++pixel)
    {
        if (pixel < 4 || secondRow)
        {
            const uint32_t k = __float2uint_rz(fmaxf(fmaxf(codeF[3 * pixel], codeF[3 * pixel + 1]), codeF[3 * pixel + 2]));
            TallyCode(tally, k, __ldg(levels + k));
        }
    }
}

// The whole warp, converged, once at exit: one atomicMax and one 64-bit atomicAdd per warp that saw a non-zero code.
// `pixels` is the launch's pixel count when this is the grid's first warp, else 0: a launch converts exactly its window,
// so the count is added once per launch instead of being tallied per pixel.
__device__ __forceinline__ void FlushLightTally(const LightTally& tally, uint64_t pixels, avifgpu_light_level* acc)
{
    const uint32_t maxCode = __reduce_max_sync(0xffffffffu, tally.maxCode);
    unsigned long long sum = tally.levelSum;
#pragma unroll
    for (int offset = 16; offset > 0; offset >>= 1)
    {
        sum += __shfl_down_sync(0xffffffffu, sum, offset);
    }
    if ((threadIdx.x & 31) == 0)
    {
        if (maxCode != 0)
        {
            atomicMax(&acc->max_code, maxCode);
            atomicAdd(reinterpret_cast<unsigned long long*>(&acc->level_sum), sum);
        }
        if (pixels != 0)
        {
            atomicAdd(reinterpret_cast<unsigned long long*>(&acc->pixels), static_cast<unsigned long long>(pixels));
        }
    }
}

// The launch's pixel count for the grid's first warp, 0 for every other warp.
__device__ __forceinline__ uint64_t LaunchPixelsForFirstWarp(uint64_t launchPixels)
{
    return (blockIdx.x == 0 && threadIdx.x < 32) ? launchPixels : 0;
}
#endif

} // namespace avifgpu

#endif
