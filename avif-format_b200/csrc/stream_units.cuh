// stream_units.cuh -- the per-group code of the streaming decodes into 8/16-bit hosts, shared by the single-image kernel
// (StreamDecodeKernel, kernels_fast_decode_int.cu) and the batched planar-RGB kernel (DecodePlanarRgbIntBatchKernel,
// kernels_batch.cu), so that both compute every output with the same instructions.
//
// A group is 8 adjacent pixels of one row: one vector load per plane (LoadStreamGroup), CHANNELS * 8 host samples stored
// as 64/128-bit words (StoreStreamGroup).  Planar RGB (ReadHeifImage.cpp:561-861) interleaves the samples as they are;
// 16-bit hosts mask them with the image's maximum (:789-792): ConvertRgbGroup.
#ifndef AVIFGPU_STREAM_UNITS_CUH
#define AVIFGPU_STREAM_UNITS_CUH

#include "int_units.cuh"
#include "kernel_params.h"

#include <cuda_runtime.h>

namespace avifgpu
{
namespace
{

constexpr int kStreamThreads = 256;

// The parameter block of the single-image kernel.  The batched kernel takes the description part (bitDepth onwards) from
// its chunk or workspace and each image's pointers, strides and width from a BatchRecord.
struct StreamDecodeParams
{
    const uint8_t* plane[4]; // RGB: R, G, B, A;  mono: Y, -, -, A
    int64_t planeStride[4];
    uint8_t* rows;
    int64_t rowStride;
    int32_t groupsPerRow; // 8 pixels each
    int32_t rowCount;
    int32_t bitDepth;
    uint32_t maxCode;
    RangeParams range;
};

// The description part of the block for `p` (pointers and sizes left zero).  Both launchers use it.
inline StreamDecodeParams StreamDecodeDescription(const DecodeParams& p)
{
    StreamDecodeParams sp{};
    sp.bitDepth = p.bitDepth;
    sp.maxCode = p.maxCode;
    sp.range = p.range;
    return sp;
}

// The group's samples at pixel `column` of row `row`: planes R, G, B (Y for monochrome), then alpha from plane 3.
template <typename SampleT, int CHANNELS, bool MONO>
__device__ __forceinline__ void LoadStreamGroup(const StreamDecodeParams& p, Raw8<SampleT> (&raw)[CHANNELS], long long row, long long column)
{
    constexpr bool kAlpha = CHANNELS > (MONO ? 1 : 3);
#pragma unroll
    for (int c = 0; c < CHANNELS; ++c)
    {
        const int planeIndex = (kAlpha && c == CHANNELS - 1) ? 3 : c;
        raw[c] = LoadEight<SampleT>(p.plane[planeIndex] + row * p.planeStride[planeIndex] + column * static_cast<long long>(sizeof(SampleT)));
    }
}

// 8 pixels of CHANNELS host samples each, packed and stored at `target`: 128-bit stores where the group is a multiple of
// 16 bytes, 64-bit ones otherwise (RGB8).
template <typename SampleT, int CHANNELS>
__device__ __forceinline__ void StoreStreamGroup(const uint32_t (&samples)[8 * CHANNELS], uint8_t* target)
{
    constexpr bool kHost8 = sizeof(SampleT) == 1;
    constexpr int kWords = 8 * CHANNELS * static_cast<int>(sizeof(SampleT)) / 4;
    uint32_t words[kWords];
#pragma unroll
    for (int w = 0; w < kWords; ++w)
    {
        if (kHost8)
        {
            words[w] = samples[4 * w] | (samples[4 * w + 1] << 8) | (samples[4 * w + 2] << 16) | (samples[4 * w + 3] << 24);
        }
        else
        {
            words[w] = samples[2 * w] | (samples[2 * w + 1] << 16);
        }
    }
    if (kWords % 4 == 0)
    {
#pragma unroll
        for (int q = 0; q < kWords / 4; ++q)
        {
            __stcs(reinterpret_cast<uint4*>(target) + q, make_uint4(words[4 * q], words[4 * q + 1], words[4 * q + 2], words[4 * q + 3]));
        }
    }
    else
    {
#pragma unroll
        for (int q = 0; q < kWords / 2; ++q)
        {
            __stcs(reinterpret_cast<uint2*>(target) + q, make_uint2(words[2 * q], words[2 * q + 1]));
        }
    }
}

// One planar-RGB group (CHANNELS 3 or 4) into the host pixels at `target`.
template <typename SampleT, int CHANNELS>
__device__ __forceinline__ void ConvertRgbGroup(const Raw8<SampleT> (&raw)[CHANNELS], uint32_t maxCode, uint8_t* target)
{
    uint32_t samples[8 * CHANNELS];
#pragma unroll
    for (int i = 0; i < 8; ++i)
    {
#pragma unroll
        for (int c = 0; c < CHANNELS; ++c)
        {
            uint32_t v = Sample<SampleT>(raw[c], i);
            if (sizeof(SampleT) != 1)
            {
                v &= maxCode;
            }
            samples[i * CHANNELS + c] = v;
        }
    }
    StoreStreamGroup<SampleT, CHANNELS>(samples, target);
}

} // namespace
} // namespace avifgpu

#endif
