// int_units.cuh -- the per-unit code of the tuned integer kernels, shared by the single-image kernels
// (kernels_fast_int.cu, kernels_fast_decode_int.cu) and their batched forms (kernels_batch.cu), so that both compute
// every output with the same instructions.
//
//   encode  EncodeRgbIntGroup converts one group: 8 pixels of a row (of a row pair for 4:2:0) of an 8/16-bit RGB(A)
//           host into planar YCbCr (+ A) codes.
//   decode  a unit is (2 rows for 4:2:0, else 1) x 256 pixels and a lane owns 8 of them per row: LoadYccUnit fetches its
//           samples, ExpandYccUnit turns them into floats through the shared-memory tables, StoreYccUnit writes pixels.
#ifndef AVIFGPU_INT_UNITS_CUH
#define AVIFGPU_INT_UNITS_CUH

#include "kernel_params.h"
#include "packed_f32x2.cuh"
#include "pixel_math.cuh"
#include "source_units.cuh"

#include <cuda_runtime.h>

namespace avifgpu
{
namespace
{

using namespace avifpix;

// ---- RGB(A) 8/16-bit hosts -> planar YCbCr ---------------------------------------------------------------------------

constexpr int kRgbThreads = 256;
constexpr float kTwo23 = 8388608.0f;

// (float)v for v < 2^23 without the conversion instruction.
__device__ __forceinline__ float UintToFloatExact(uint32_t v) { return __uint_as_float(0x4b000000u | v) - kTwo23; }

// 2^23 + min(trunc(t), maxCode) as a float, for 0 <= t < 2^23: adding 2^23 with round-toward-zero leaves floor(t) in
// the low mantissa bits.  Bit-identical to (int)t followed by the upper clamp of the reference's LUT builder.
__device__ __forceinline__ float BiasedTrunc(float t, float biasedMax) { return fminf(__fadd_rz(t, kTwo23), biasedMax); }

struct Rgb16Params
{
    const uint8_t* rows;
    int64_t rowStride;
    uint8_t* plane[4];
    int64_t stride[4];
    int32_t groupsPerRow; // 8 pixels each
    int32_t rowCount;     // even when YS == 1
    float maxCodeFloat;
    float biasedMax;      // 2^23 + maxCode
    ForwardMatrix matrix;
    float chromaOffset;
    int32_t topLeft;
    uint32_t maxCode;
    float maxReciprocal; // RN(1 / maxCode), for the verified premultiply
};

// PremultiplyColor(uint16_t, uint16_t, maxValue) (PremultipliedAlpha.cpp:62-70) behind the callers' guard
// (WriteHeifImage.cpp:947-965: alpha == max keeps the colour, alpha == 0 clears it) in six full-rate instructions:
//     product (exact: both codes < 2^12)  ->  / max by reciprocal + one residual step  ->  + 0.5, truncate.
// The division by reciprocal is not the IEEE division and trunc(x + 0.5) is not roundf(x) for every float x, but over the
// (max + 1)^2 code pairs of a bit depth it either always agrees with the reference's own sequence or it does not:
// VerifyFastPremultiplyKernel enumerates them all, and the tuned kernel is used only for depths that passed.  No special
// cases are needed: alpha == 0 gives a zero product, alpha == max gives product / max == colour exactly.
__device__ __forceinline__ float FastPremultiplyBiased(float colour, float alpha, float maxCodeFloat, float maxReciprocal)
{
    const float product = __fmul_rn(colour, alpha);
    const float quotient = DivideByConstant(product, maxCodeFloat, maxReciprocal);
    return __fadd_rz(__fadd_rn(quotient, 0.5f), kTwo23); // 2^23 + code
}

// The same six operations on two (colour, alpha) pairs at once (packed_f32x2.cuh): lane for lane the IEEE operations of
// FastPremultiplyBiased -- fma(-q, d, x) == fma(q, -d, x) -- so VerifyFastPremultiply's enumeration covers it.
__device__ __forceinline__ avifx2::F32x2 FastPremultiplyBiasedPair(avifx2::F32x2 colour, avifx2::F32x2 alpha, float maxCodeFloat, float maxReciprocal)
{
    using namespace avifx2;
    const F32x2 product = Mul2(colour, alpha);
    const F32x2 q = Mul2(product, Splat(maxReciprocal));
    const F32x2 residual = Fma2(q, Splat(-maxCodeFloat), product);
    const F32x2 quotient = Fma2(residual, Splat(maxReciprocal), q);
    return AddRz2(Add2(quotient, Splat(0.5f)), Splat(kTwo23)); // 2^23 + code
}

// Host sample -> 2^23 + code, as a float.
//   16-bit host (0..32768, or beyond: the formula is defined to continue)  WriteHeifImage.cpp:140-166:
//       (int)((v / 32768f) * max + 0.5f), clamped -- v / 32768f is exact as a multiplication;
//   8-bit host, 8-bit image   the sample is the code                        WriteHeifImage.cpp:743-747
//   8-bit host, deeper image  (int)((v / 255f) * max + 0.5f): a true division, so the 256 results are tabulated in
//                             shared memory at kernel start (the reference builds the same table, :87-112).
template <typename HostT, typename PlaneT>
__device__ __forceinline__ float SampleToBiasedCode(uint32_t v, const Rgb16Params& p, const float* __restrict__ hostLut)
{
    if (sizeof(HostT) == 2)
    {
        const float t = ((UintToFloatExact(v) * (1.0f / 32768.0f)) * p.maxCodeFloat) + 0.5f;
        return BiasedTrunc(t, p.biasedMax);
    }
    if (sizeof(PlaneT) == 1)
    {
        return __uint_as_float(0x4b000000u | v);
    }
    return hostLut[v];
}

__device__ __forceinline__ uint32_t BiasedToCode(float biased) { return __float_as_uint(biased) & 0x7fffffu; }

// 8 (4) consecutive plane samples in one vector store.
template <typename PlaneT>
__device__ __forceinline__ void StoreEight(uint8_t* address, const uint32_t (&c)[8])
{
    if (sizeof(PlaneT) == 2)
    {
        __stcs(reinterpret_cast<uint4*>(address), make_uint4(c[0] | (c[1] << 16), c[2] | (c[3] << 16), c[4] | (c[5] << 16), c[6] | (c[7] << 16)));
    }
    else
    {
        __stcs(reinterpret_cast<uint2*>(address),
               make_uint2(c[0] | (c[1] << 8) | (c[2] << 16) | (c[3] << 24), c[4] | (c[5] << 8) | (c[6] << 16) | (c[7] << 24)));
    }
}

template <typename PlaneT>
__device__ __forceinline__ void StoreFour(uint8_t* address, const uint32_t (&c)[4])
{
    if (sizeof(PlaneT) == 2)
    {
        __stcs(reinterpret_cast<uint2*>(address), make_uint2(c[0] | (c[1] << 16), c[2] | (c[3] << 16)));
    }
    else
    {
        __stcs(reinterpret_cast<uint32_t*>(address), c[0] | (c[1] << 8) | (c[2] << 16) | (c[3] << 24));
    }
}

// DEST != 0: the stores of EncodeRgbIntGroup into semi-planar and MSB-aligned planes, from the codes the planar stores
// take.  The codes are packed into words as StoreEight / StoreFour pack them (two 16-bit or four 8-bit codes a word);
// MSB-aligned words are shifted as they stand (CodesToMsbPair), and interleaved chroma is the Cb and Cr words paired by
// byte permutation into one store of twice the planar bytes -- two 128-bit stores for 16-bit 4:4:4.
template <int WORDS>
__device__ __forceinline__ void StoreWords(uint8_t* address, const uint32_t (&w)[WORDS])
{
    if constexpr (WORDS == 1)
    {
        __stcs(reinterpret_cast<uint32_t*>(address), w[0]);
    }
    else if constexpr (WORDS == 2)
    {
        __stcs(reinterpret_cast<uint2*>(address), make_uint2(w[0], w[1]));
    }
    else
    {
#pragma unroll
        for (int q = 0; q < WORDS / 4; ++q)
        {
            __stcs(reinterpret_cast<uint4*>(address) + q, make_uint4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]));
        }
    }
}

template <typename PlaneT, int DEST, int N>
__device__ __forceinline__ void PackDestWords(const uint32_t (&c)[N], uint32_t shift, uint32_t (&w)[N * sizeof(PlaneT) / 4])
{
    static_assert(sizeof(PlaneT) == 2 || !SourceMsbAligned(DEST), "8-bit planes are never MSB-aligned");
#pragma unroll
    for (int i = 0; i < N * static_cast<int>(sizeof(PlaneT)) / 4; ++i)
    {
        w[i] = sizeof(PlaneT) == 2 ? c[2 * i] | (c[2 * i + 1] << 16) : c[4 * i] | (c[4 * i + 1] << 8) | (c[4 * i + 2] << 16) | (c[4 * i + 3] << 24);
        if (SourceMsbAligned(DEST))
        {
            w[i] = CodesToMsbPair(w[i], shift);
        }
    }
}

// N (8 or 4) consecutive luma or alpha codes.
template <typename PlaneT, int DEST, int N>
__device__ __forceinline__ void StoreDestCodes(uint8_t* address, const uint32_t (&c)[N], uint32_t shift)
{
    uint32_t w[N * sizeof(PlaneT) / 4];
    PackDestWords<PlaneT, DEST>(c, shift, w);
    StoreWords(address, w);
}

// N (8 or 4) consecutive chroma sites: into plane 1 at cbAddress and plane 2 at crAddress, or, interleaved, as Cb, Cr pairs
// into plane 1 at cbAddress.
template <typename PlaneT, int DEST, int N>
__device__ __forceinline__ void StoreDestChroma(uint8_t* cbAddress, uint8_t* crAddress, const uint32_t (&cb)[N], const uint32_t (&cr)[N], uint32_t shift)
{
    constexpr int kWords = N * sizeof(PlaneT) / 4;
    uint32_t cbWords[kWords], crWords[kWords];
    PackDestWords<PlaneT, DEST>(cb, shift, cbWords);
    PackDestWords<PlaneT, DEST>(cr, shift, crWords);
    if constexpr (SourceInterleaved(DEST))
    {
        uint32_t pairs[2 * kWords];
#pragma unroll
        for (int i = 0; i < kWords; ++i)
        {
            pairs[2 * i] = sizeof(PlaneT) == 2 ? LowHalves(cbWords[i], crWords[i]) : LowPairs(cbWords[i], crWords[i]);
            pairs[2 * i + 1] = sizeof(PlaneT) == 2 ? HighHalves(cbWords[i], crWords[i]) : HighPairs(cbWords[i], crWords[i]);
        }
        StoreWords(cbAddress, pairs);
    }
    else
    {
        StoreWords(cbAddress, cbWords);
        StoreWords(crAddress, crWords);
    }
}

// The fields of the planar launch every group of `p`'s image shares; the launchers add pointers, strides and sizes.
inline Rgb16Params RgbIntShared(const EncodeParams& p)
{
    Rgb16Params rp{};
    rp.maxCodeFloat = p.maxCodeFloat;
    rp.biasedMax = 8388608.0f + p.maxCodeFloat;
    rp.matrix = p.matrix;
    rp.chromaOffset = p.chromaOffset;
    rp.topLeft = p.topLeft;
    rp.maxCode = p.maxCode;
    rp.maxReciprocal = 1.0f / p.maxCodeFloat;
    return rp;
}

// 8-bit hosts into a deeper image: the 256 biased codes SampleToBiasedCode looks up, one copy per CTA.
template <typename HostT, typename PlaneT>
__device__ __forceinline__ void StageHostLut(float* hostLut, uint32_t maxCode)
{
    if (sizeof(HostT) == 1 && sizeof(PlaneT) == 2)
    {
        for (uint32_t v = threadIdx.x; v < 256; v += blockDim.x)
        {
            hostLut[v] = __uint_as_float(0x4b000000u | DepthLutEntry(v, 255.0f, maxCode));
        }
        __syncthreads();
    }
}

// HostT: uint8_t / uint16_t host samples; PlaneT: uint8_t (8-bit image) / uint16_t (10 / 12-bit image) plane samples.
// PREMULTIPLY (CHANNELS == 4 only): the colour codes are multiplied by the alpha code in the image's depth before the matrix
// (WriteHeifImage.cpp:700-718, 760-778, 877-895, 947-965), through FastPremultiplyBiased.
// One group: pixels [8 column, 8 column + 8) of rows (rowPair << YS) .. (rowPair << YS) + YS.
// DEST: the avifgpu_source_layout bits of the planes written; 0 stores with StoreEight / StoreFour, anything else with
// StoreDestCodes / StoreDestChroma.  Nothing before the stores depends on it.
template <typename HostT, typename PlaneT, int CHANNELS, int XS, int YS, int PREMULTIPLY, int DEST = 0>
__device__ __forceinline__ void EncodeRgbIntGroup(const Rgb16Params& p, const float* __restrict__ hostLut, long long rowPair, int column)
{
    constexpr int kRows = 1 + YS;
    constexpr int kChromaPairs = SourceInterleaved(DEST) ? 2 : 1; // interleaved: Cb, Cr pairs in plane 1
    // 16 - depth == clz(maxCode) - 16 for MSB-aligned planes (the parameter block has no depth field)
    const uint32_t msbShift = SourceMsbAligned(DEST) ? static_cast<uint32_t>(__clz(p.maxCode) - 16) : 0u;
    constexpr int kWordsPerRow = CHANNELS * 2 * static_cast<int>(sizeof(HostT)); // 8 pixels x CHANNELS samples / 4 bytes
    constexpr int kVectorWords = (kWordsPerRow % 4 == 0) ? 4 : 2;                 // 128-bit loads where the row chunk allows
    constexpr int kPlaneBytes = static_cast<int>(sizeof(PlaneT));
    const long long y0 = rowPair << YS;

    uint32_t words[kRows][kWordsPerRow];
#pragma unroll
    for (int r = 0; r < kRows; ++r)
    {
        const uint8_t* source = p.rows + (y0 + r) * p.rowStride + static_cast<long long>(column) * (kWordsPerRow * 4);
#pragma unroll
        for (int q = 0; q < kWordsPerRow / kVectorWords; ++q)
        {
            if (kVectorWords == 4)
            {
                const uint4 w = __ldcs(reinterpret_cast<const uint4*>(source) + q);
                words[r][4 * q + 0] = w.x;
                words[r][4 * q + 1] = w.y;
                words[r][4 * q + 2] = w.z;
                words[r][4 * q + 3] = w.w;
            }
            else
            {
                const uint2 w = __ldcs(reinterpret_cast<const uint2*>(source) + q);
                words[r][2 * q + 0] = w.x;
                words[r][2 * q + 1] = w.y;
            }
        }
    }

    // The matrix runs on pixel pairs (2j, 2j + 1) in the two-lane FP32 instructions (packed_f32x2.cuh; its rule: a product
    // is never the operand of a packed add, so the three luma products and the chroma sums are added as scalars).  The
    // operations per pixel, and their roundings, are pixel_math.cuh's ForwardPixelFloat.
    using namespace avifx2;
    const F32x2 half2 = Splat(0.5f), bias2 = Splat(kTwo23), offset2 = Splat(p.chromaOffset);
    const F32x2 kr2 = Splat(p.matrix.kr), kg2 = Splat(p.matrix.kg), kb2 = Splat(p.matrix.kb);
    const F32x2 cbScale2 = Splat(p.matrix.cbScale), crScale2 = Splat(p.matrix.crScale);
    const F32x2 hostScale2 = Splat(p.maxCodeFloat * (1.0f / 32768.0f)); // exact: max <= 4095 times a power of two
    // 2^23 + trunc(v + 0.5) for both halves: BiasedToCode of either is the code (no upper clamp here)
    const auto biasedPair = [&](F32x2 v, float& lo, float& hi) { Unpack(AddRz2(Add2(v, half2), bias2), lo, hi); };
    const auto chromaClamp = [&](float biased) -> uint32_t { return BiasedToCode(fminf(biased, p.biasedMax)); }; // H.273: 2^depth -> 2^depth - 1

    F32x2 cb[kRows][4], cr[kRows][4]; // [row][pair]
#pragma unroll
    for (int r = 0; r < kRows; ++r)
    {
        uint32_t yCodes[8];
        uint32_t aCodes[8];
#pragma unroll
        for (int j = 0; j < 4; ++j)
        {
            // sample k of the row sits in half-word (byte) k of the loaded words
            auto sample = [&](int k) -> uint32_t
            {
                if (sizeof(HostT) == 2)
                {
                    const uint32_t w = words[r][k >> 1];
                    return (k & 1) ? (w >> 16) : (w & 0xffffu);
                }
                return (words[r][k >> 2] >> (8 * (k & 3))) & 0xffu;
            };
            // channel c of pixels 2j and 2j + 1 as 2^23-biased codes in the image's depth
            const auto biasedCodes = [&](int c) -> F32x2
            {
                const uint32_t v0 = sample((2 * j) * CHANNELS + c), v1 = sample((2 * j + 1) * CHANNELS + c);
                if (sizeof(HostT) == 2)
                {
                    // SampleToBiasedCode on the pair: (v / 32768f) * max is ONE rounding (the division is a scaling by 2^-15 and
                    // max * 2^-15 is exact), so the single packed multiply by that constant is the same number; + 0.5f follows a
                    // product and stays scalar
                    float t0, t1;
                    Unpack(Mul2(Sub2(Pack(__uint_as_float(0x4b000000u | v0), __uint_as_float(0x4b000000u | v1)), bias2), hostScale2), t0, t1);
                    float b0, b1;
                    Unpack(AddRz2(Pack(__fadd_rn(t0, 0.5f), __fadd_rn(t1, 0.5f)), bias2), b0, b1);
                    return Pack(fminf(b0, p.biasedMax), fminf(b1, p.biasedMax));
                }
                return Pack(SampleToBiasedCode<HostT, PlaneT>(v0, p, hostLut), SampleToBiasedCode<HostT, PlaneT>(v1, p, hostLut));
            };
            F32x2 red, green, blue;
            if (PREMULTIPLY)
            {
                // colour * alpha / max per channel on the pair
                const F32x2 alphaBiased = biasedCodes(3);
                const F32x2 alpha = Sub2(alphaBiased, bias2);
                red = Sub2(FastPremultiplyBiasedPair(Sub2(biasedCodes(0), bias2), alpha, p.maxCodeFloat, p.maxReciprocal), bias2);
                green = Sub2(FastPremultiplyBiasedPair(Sub2(biasedCodes(1), bias2), alpha, p.maxCodeFloat, p.maxReciprocal), bias2);
                blue = Sub2(FastPremultiplyBiasedPair(Sub2(biasedCodes(2), bias2), alpha, p.maxCodeFloat, p.maxReciprocal), bias2);
                float a0, a1;
                Unpack(alphaBiased, a0, a1);
                aCodes[2 * j] = BiasedToCode(a0);
                aCodes[2 * j + 1] = BiasedToCode(a1);
            }
            else if (sizeof(HostT) == 2)
            {
                red = Sub2(biasedCodes(0), bias2);
                green = Sub2(biasedCodes(1), bias2);
                blue = Sub2(biasedCodes(2), bias2);
                if (CHANNELS == 4)
                {
                    float a0, a1;
                    Unpack(biasedCodes(3), a0, a1);
                    aCodes[2 * j] = BiasedToCode(a0);
                    aCodes[2 * j + 1] = BiasedToCode(a1);
                }
            }
            else
            {
                float rf[2], gf[2], bf[2];
#pragma unroll
                for (int h = 0; h < 2; ++h)
                {
                    const int i = 2 * j + h;
                    if (sizeof(HostT) == 1 && sizeof(PlaneT) == 1)
                    {
                        // 8-bit host into an 8-bit image: the sample is the code.  Byte -> float is one conversion instruction
                        // (it takes the byte lane as an operand modifier).
                        rf[h] = static_cast<float>(static_cast<uint8_t>(sample(i * CHANNELS + 0)));
                        gf[h] = static_cast<float>(static_cast<uint8_t>(sample(i * CHANNELS + 1)));
                        bf[h] = static_cast<float>(static_cast<uint8_t>(sample(i * CHANNELS + 2)));
                    }
                    else
                    {
                        rf[h] = SampleToBiasedCode<HostT, PlaneT>(sample(i * CHANNELS + 0), p, hostLut) - kTwo23;
                        gf[h] = SampleToBiasedCode<HostT, PlaneT>(sample(i * CHANNELS + 1), p, hostLut) - kTwo23;
                        bf[h] = SampleToBiasedCode<HostT, PlaneT>(sample(i * CHANNELS + 2), p, hostLut) - kTwo23;
                    }
                    if (CHANNELS == 4)
                    {
                        aCodes[i] = (sizeof(HostT) == 1 && sizeof(PlaneT) == 1) ? sample(i * CHANNELS + 3)
                                                                                : BiasedToCode(SampleToBiasedCode<HostT, PlaneT>(sample(i * CHANNELS + 3), p, hostLut));
                    }
                }
                red = Pack(rf[0], rf[1]);
                green = Pack(gf[0], gf[1]);
                blue = Pack(bf[0], bf[1]);
            }
            F32x2 luma;
            if (p.matrix.identity)
            {
                luma = green;
                cb[r][j] = blue;
                cr[r][j] = red;
            }
            else
            {
                float r0, r1, g0, g1, b0, b1;
                Unpack(Mul2(red, kr2), r0, r1);
                Unpack(Mul2(green, kg2), g0, g1);
                Unpack(Mul2(blue, kb2), b0, b1);
                luma = Pack(__fadd_rn(__fadd_rn(r0, g0), b0), __fadd_rn(__fadd_rn(r1, g1), b1)); // (kr R + kg G) + kb B
                cb[r][j] = Mul2(Sub2(blue, luma), cbScale2);
                cr[r][j] = Mul2(Sub2(red, luma), crScale2);
            }
            float luma0, luma1;
            biasedPair(luma, luma0, luma1); // no upper clamp: ForwardMatrixStaysInRange (launcher)
            yCodes[2 * j] = BiasedToCode(luma0);
            yCodes[2 * j + 1] = BiasedToCode(luma1);
        }
        if constexpr (DEST == 0)
        {
            StoreEight<PlaneT>(p.plane[0] + (y0 + r) * p.stride[0] + static_cast<long long>(column) * (8 * kPlaneBytes), yCodes);
            if (CHANNELS == 4)
            {
                StoreEight<PlaneT>(p.plane[3] + (y0 + r) * p.stride[3] + static_cast<long long>(column) * (8 * kPlaneBytes), aCodes);
            }
        }
        else
        {
            StoreDestCodes<PlaneT, DEST>(p.plane[0] + (y0 + r) * p.stride[0] + static_cast<long long>(column) * (8 * kPlaneBytes), yCodes, msbShift);
            if (CHANNELS == 4)
            {
                StoreDestCodes<PlaneT, DEST>(p.plane[3] + (y0 + r) * p.stride[3] + static_cast<long long>(column) * (8 * kPlaneBytes), aCodes, msbShift);
            }
        }
    }

    // chroma: down-filter in float, then quantise (the offset is 0 for the identity matrix); chroma values are products
    // (or, for the identity matrix, plain samples): the offset is added to each half as a scalar, like the sums
    const auto addOffset = [&](F32x2 product) -> F32x2
    {
        float c0, c1;
        Unpack(product, c0, c1);
        return Pack(__fadd_rn(c0, p.chromaOffset), __fadd_rn(c1, p.chromaOffset));
    };
    if (XS == 0)
    {
#pragma unroll
        for (int r = 0; r < kRows; ++r)
        {
            uint32_t cbCode[8], crCode[8];
#pragma unroll
            for (int j = 0; j < 4; ++j)
            {
                float b0, b1, r0, r1;
                biasedPair(addOffset(cb[r][j]), b0, b1);
                biasedPair(addOffset(cr[r][j]), r0, r1);
                cbCode[2 * j] = chromaClamp(b0);
                cbCode[2 * j + 1] = chromaClamp(b1);
                crCode[2 * j] = chromaClamp(r0);
                crCode[2 * j + 1] = chromaClamp(r1);
            }
            const long long offset = static_cast<long long>(column) * (8 * kPlaneBytes);
            if constexpr (DEST == 0)
            {
                StoreEight<PlaneT>(p.plane[1] + (y0 + r) * p.stride[1] + offset, cbCode);
                StoreEight<PlaneT>(p.plane[2] + (y0 + r) * p.stride[2] + offset, crCode);
            }
            else
            {
                StoreDestChroma<PlaneT, DEST>(p.plane[1] + (y0 + r) * p.stride[1] + offset * kChromaPairs, p.plane[2] + (y0 + r) * p.stride[2] + offset,
                                              cbCode, crCode, msbShift);
            }
        }
    }
    else
    {
        // site s = pixels 2s, 2s + 1 (of both rows for 4:2:0) = the two halves of pair s; two sites per packed value
        uint32_t cbCode[4], crCode[4];
#pragma unroll
        for (int s = 0; s < 4; s += 2)
        {
            F32x2 cbBiased, crBiased; // chroma + offset for sites s, s + 1
            if (p.topLeft)
            {
                float b0, b1, r0, r1, unused;
                Unpack(cb[0][s], b0, unused);
                Unpack(cb[0][s + 1], b1, unused);
                Unpack(cr[0][s], r0, unused);
                Unpack(cr[0][s + 1], r1, unused);
                cbBiased = Pack(__fadd_rn(b0, p.chromaOffset), __fadd_rn(b1, p.chromaOffset));
                crBiased = Pack(__fadd_rn(r0, p.chromaOffset), __fadd_rn(r1, p.chromaOffset));
            }
            else
            {
                const auto siteSum = [&](const F32x2 (&plane)[kRows][4], int site) -> float
                {
                    float top0, top1;
                    Unpack(plane[0][site], top0, top1);
                    const float top = __fadd_rn(top0, top1);
                    if (YS == 0)
                    {
                        return top;
                    }
                    float bottom0, bottom1;
                    Unpack(plane[kRows - 1][site], bottom0, bottom1);
                    return __fadd_rn(top, __fadd_rn(bottom0, bottom1)); // (c00 + c01) + (c10 + c11)
                };
                // * 0.25f (0.5f) is exact, so the fused multiply-add with the offset is the two-step number
                const F32x2 scale2 = Splat(YS == 1 ? 0.25f : 0.5f);
                cbBiased = Fma2(Pack(siteSum(cb, s), siteSum(cb, s + 1)), scale2, offset2);
                crBiased = Fma2(Pack(siteSum(cr, s), siteSum(cr, s + 1)), scale2, offset2);
            }
            float b0, b1, r0, r1;
            biasedPair(cbBiased, b0, b1);
            biasedPair(crBiased, r0, r1);
            cbCode[s] = chromaClamp(b0);
            cbCode[s + 1] = chromaClamp(b1);
            crCode[s] = chromaClamp(r0);
            crCode[s + 1] = chromaClamp(r1);
        }
        const long long offset = static_cast<long long>(column) * (4 * kPlaneBytes);
        const long long chromaRow = YS ? rowPair : y0;
        if constexpr (DEST == 0)
        {
            StoreFour<PlaneT>(p.plane[1] + chromaRow * p.stride[1] + offset, cbCode);
            StoreFour<PlaneT>(p.plane[2] + chromaRow * p.stride[2] + offset, crCode);
        }
        else
        {
            StoreDestChroma<PlaneT, DEST>(p.plane[1] + chromaRow * p.stride[1] + offset * kChromaPairs, p.plane[2] + chromaRow * p.stride[2] + offset, cbCode,
                                          crCode, msbShift);
        }
    }
}

// ---- planar YCbCr -> RGB(A) 8/16-bit hosts -------------------------------------------------------------------------

constexpr int kUnitPixels = 256; // per row: 32 lanes x 8 pixels
constexpr int kYccBlocksPerSm = 3; // DecodeYccToRgbIntKernel's and its batched forms' occupancy, and their grid caps per SM
constexpr int kStreamBlocksPerSm = 16; // the grid cap per SM of the streaming kernels (no table per CTA), single-image and batched, and of the batches' edge kernels

struct IntDecodeParams
{
    const uint8_t* plane[4];
    int64_t planeStride[4];
    uint8_t* rows;
    int64_t rowStride;
    int32_t width;    // multiple of 8
    int32_t rowCount; // even when the chroma is vertically sub-sampled
    int32_t bitDepth;
    uint32_t maxCode;
    RangeParams range;
    InverseMatrix matrix;
    int32_t verifiedGreenDivision;
};

// The fields every unit of `p`'s image shares; the launchers add pointers, strides and sizes.
inline IntDecodeParams IntDecodeShared(const DecodeParams& p)
{
    IntDecodeParams fp{};
    fp.bitDepth = p.bitDepth;
    fp.maxCode = p.maxCode;
    fp.range = p.range;
    fp.matrix = p.matrix;
    fp.verifiedGreenDivision = p.verifiedGreenDivision;
    return fp;
}

// The dynamic shared memory StageYccTables fills: the Y and UV tables, plus the alpha table of 16-bit hosts with alpha.
// At most 40 KB, under the default 48 KB limit.
inline size_t YccTableBytes(int bitDepth, bool alphaTable)
{
    const size_t entries = static_cast<size_t>(1) << bitDepth;
    return 2 * sizeof(float) * entries + (alphaTable ? sizeof(uint16_t) * entries : 0);
}

// Eight (four) consecutive samples of a plane as they sit in memory, and their expansion into 32-bit codes.
template <typename SampleT>
struct Raw8
{
    uint32_t w[sizeof(SampleT) == 1 ? 2 : 4];
};

template <typename SampleT>
__device__ __forceinline__ Raw8<SampleT> LoadEight(const uint8_t* address)
{
    Raw8<SampleT> raw;
    if (sizeof(SampleT) == 1)
    {
        const uint2 v = __ldg(reinterpret_cast<const uint2*>(address));
        raw.w[0] = v.x;
        raw.w[1] = v.y;
    }
    else
    {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(address));
        raw.w[0] = v.x;
        raw.w[1] = v.y;
        raw.w[sizeof(SampleT) == 1 ? 0 : 2] = v.z;
        raw.w[sizeof(SampleT) == 1 ? 1 : 3] = v.w;
    }
    return raw;
}

// The four samples of the sub-sampled chroma under eight luma samples land in the first half of a Raw8.
template <typename SampleT>
__device__ __forceinline__ Raw8<SampleT> LoadFour(const uint8_t* address)
{
    Raw8<SampleT> raw = {};
    if (sizeof(SampleT) == 1)
    {
        raw.w[0] = __ldg(reinterpret_cast<const uint32_t*>(address));
    }
    else
    {
        const uint2 v = __ldg(reinterpret_cast<const uint2*>(address));
        raw.w[0] = v.x;
        raw.w[1] = v.y;
    }
    return raw;
}

template <typename SampleT>
__device__ __forceinline__ uint32_t Sample(const Raw8<SampleT>& raw, int i)
{
    if (sizeof(SampleT) == 1)
    {
        return (raw.w[i >> 2] >> (8 * (i & 3))) & 0xffu;
    }
    return (i & 1) ? (raw.w[i >> 1] >> 16) : (raw.w[i >> 1] & 0xffffu);
}


// 2^23 + (uint)(0.5f + (c * scale)) as a float, for c in [0, 1]: YuvDecode.cpp:314-316 / 437-439 in two instructions and
// without the conversion pipe.  The reference forms the sum with two roundings (multiply, then add); for every float c in
// [0, 1] and scale = 255 or 32768 the single-rounding fmaf(c, scale, 0.5f) truncates to the same integer -- proven by
// enumeration, tools/check_fused_quantiser.py -- so the sum is one FMA; adding 2^23 with round-toward-zero then leaves
// its integer part in the low mantissa bits, which is the truncation of the cast.
__device__ __forceinline__ uint32_t QuantiseBiased(float c, float scale) { return __float_as_uint(__fadd_rz(__fmaf_rn(c, scale, 0.5f), kTwo23)); }

// The unorm -> float tables (YuvLookupTables.cpp:115-192) in shared memory; for 16-bit hosts the alpha output
// (u16)(0.5f + a * 32768f) is tabulated whole.  The caller synchronises the CTA before reading them.
struct YccTables
{
    float* y;
    float* uv;
    uint16_t* alpha; // 16-bit hosts with alpha only
};

template <typename SampleT, int ALPHA>
__device__ __forceinline__ YccTables StageYccTables(uint8_t* sharedBytes, const IntDecodeParams& p)
{
    constexpr bool kHost8 = sizeof(SampleT) == 1;
    YccTables t;
    t.y = reinterpret_cast<float*>(sharedBytes);
    t.uv = t.y + (1u << p.bitDepth);
    t.alpha = reinterpret_cast<uint16_t*>(t.uv + (1u << p.bitDepth));
    for (uint32_t i = threadIdx.x; i <= p.maxCode; i += blockDim.x)
    {
        t.y[i] = UnormToFloatY(i, p.range);   // YuvLookupTables.cpp:157-171
        t.uv[i] = UnormToFloatUV(i, p.range); // YuvLookupTables.cpp:173-184
        if (ALPHA && !kHost8)
        {
            // YuvLookupTables.cpp:186-190 then YuvDecode.cpp:515
            t.alpha[i] = static_cast<uint16_t>(0.5f + (UnormToFloatPlain(i, p.range.maxChannelFloat) * 32768.0f));
        }
    }
    return t;
}

// YuvDecode.cpp:306-312, the pixel-independent factors (same float expressions, evaluated once)
struct YccFactors
{
    float kg, rGain, bGain, gCr, gCb, kgReciprocal, outScale;
};

template <typename SampleT>
__device__ __forceinline__ YccFactors MakeYccFactors(const InverseMatrix& matrix)
{
    YccFactors f;
    const float kr = matrix.kr, kg = matrix.kg, kb = matrix.kb;
    f.kg = kg;
    f.rGain = (2 * (1 - kr));
    f.bGain = (2 * (1 - kb));
    f.gCr = kr * (1 - kr);
    f.gCb = kb * (1 - kb);
    f.kgReciprocal = 1.0f / kg;
    f.outScale = sizeof(SampleT) == 1 ? 255.0f : 32768.0f;
    return f;
}

// The Cb and Cr samples of a lane's chroma sites from interleaved pairs at `address`, as LoadFour (XS) / LoadEight put the
// planar ones: one load of twice their bytes -- 64 or 128 bits, two 128-bit loads for 16-bit 4:4:4 -- then a byte
// permutation per word.
template <typename SampleT, int XS>
__device__ __forceinline__ void LoadInterleavedChroma(const uint8_t* address, Raw8<SampleT>& rawCb, Raw8<SampleT>& rawCr)
{
    rawCb = {};
    rawCr = {};
    if constexpr (sizeof(SampleT) == 1 && XS)
    {
        const uint2 v = __ldg(reinterpret_cast<const uint2*>(address));
        rawCb.w[0] = EvenBytes(v.x, v.y);
        rawCr.w[0] = OddBytes(v.x, v.y);
    }
    else if constexpr (sizeof(SampleT) == 1)
    {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(address));
        rawCb.w[0] = EvenBytes(v.x, v.y);
        rawCb.w[1] = EvenBytes(v.z, v.w);
        rawCr.w[0] = OddBytes(v.x, v.y);
        rawCr.w[1] = OddBytes(v.z, v.w);
    }
    else
    {
#pragma unroll
        for (int q = 0; q < (XS ? 1 : 2); ++q)
        {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(address) + q);
            rawCb.w[2 * q] = LowHalves(v.x, v.y);
            rawCb.w[2 * q + 1] = LowHalves(v.z, v.w);
            rawCr.w[2 * q] = HighHalves(v.x, v.y);
            rawCr.w[2 * q + 1] = HighHalves(v.z, v.w);
        }
    }
}

// A lane's samples of the unit at (unit row `row`, unit column `column`), as loaded; nothing is loaded for an invalid unit or a lane past the width.
// SOURCE (kernel_params.h): interleaved chroma is read in pairs from plane 1; MSB-aligned samples (16-bit planes) are
// shifted to their codes two at a time as they arrive, so the rest of the unit sees the planar, low-bit samples.
template <typename SampleT, int XS, int YS, int ALPHA, int SOURCE = 0>
__device__ __forceinline__ void LoadYccUnit(const IntDecodeParams& p, int lane, int row, int column, bool valid, Raw8<SampleT> (&rawY)[YS ? 2 : 1],
                                            Raw8<SampleT> (&rawA)[YS ? 2 : 1], Raw8<SampleT>& rawCb, Raw8<SampleT>& rawCr)
{
    constexpr int kRows = YS ? 2 : 1;
    const int x = column * kUnitPixels + lane * 8;
    const int y = row * kRows;
    if (!valid || x >= p.width)
    {
        return;
    }
    const int64_t chromaRow = YS ? row : y;
    const int64_t chromaColumn = static_cast<int64_t>(XS ? (x >> 1) : x) * sizeof(SampleT);
    if constexpr (SourceInterleaved(SOURCE))
    {
        LoadInterleavedChroma<SampleT, XS>(p.plane[1] + chromaRow * p.planeStride[1] + 2 * chromaColumn, rawCb, rawCr);
    }
    else if (XS)
    {
        rawCb = LoadFour<SampleT>(p.plane[1] + chromaRow * p.planeStride[1] + chromaColumn);
        rawCr = LoadFour<SampleT>(p.plane[2] + chromaRow * p.planeStride[2] + chromaColumn);
    }
    else
    {
        rawCb = LoadEight<SampleT>(p.plane[1] + chromaRow * p.planeStride[1] + chromaColumn);
        rawCr = LoadEight<SampleT>(p.plane[2] + chromaRow * p.planeStride[2] + chromaColumn);
    }
#pragma unroll
    for (int r = 0; r < kRows; ++r)
    {
        if (y + r < p.rowCount)
        {
            rawY[r] = LoadEight<SampleT>(p.plane[0] + static_cast<int64_t>(y + r) * p.planeStride[0] + static_cast<int64_t>(x) * sizeof(SampleT));
            if (ALPHA)
            {
                rawA[r] = LoadEight<SampleT>(p.plane[3] + static_cast<int64_t>(y + r) * p.planeStride[3] + static_cast<int64_t>(x) * sizeof(SampleT));
            }
        }
    }
    if constexpr (SourceMsbAligned(SOURCE) && sizeof(SampleT) == 2)
    {
        const uint32_t shift = 16u - static_cast<uint32_t>(p.bitDepth);
#pragma unroll
        for (int i = 0; i < 4; ++i)
        {
#pragma unroll
            for (int r = 0; r < kRows; ++r)
            {
                rawY[r].w[i] = MsbPairToCodes(rawY[r].w[i], shift);
                if (ALPHA)
                {
                    rawA[r].w[i] = MsbPairToCodes(rawA[r].w[i], shift);
                }
            }
            rawCb.w[i] = MsbPairToCodes(rawCb.w[i], shift);
            rawCr.w[i] = MsbPairToCodes(rawCr.w[i], shift);
        }
    }
}

// A lane's samples as floats through the tables; the chroma-dependent terms of YuvDecode.cpp:306-312 once per chroma
// site, reused for every luma sample the site covers (both rows of a 4:2:0 site).
template <int XS, int YS>
struct YccValues
{
    float y[YS ? 2 : 1][8];
    uint32_t alpha[YS ? 2 : 1][8];
    float rOffset[XS ? 4 : 8], bOffset[XS ? 4 : 8], gOffset[XS ? 4 : 8];
};

template <typename SampleT, int XS, int YS, int ALPHA>
__device__ __forceinline__ void ExpandYccUnit(const IntDecodeParams& p, const YccTables& tables, const YccFactors& f, const Raw8<SampleT> (&rawY)[YS ? 2 : 1],
                                              const Raw8<SampleT> (&rawA)[YS ? 2 : 1], const Raw8<SampleT>& rawCb, const Raw8<SampleT>& rawCr,
                                              YccValues<XS, YS>& values)
{
    constexpr bool kHost8 = sizeof(SampleT) == 1;
    constexpr int kRows = YS ? 2 : 1;
    constexpr int kSites = XS ? 4 : 8; // chroma sites under a lane's 8 luma samples
#pragma unroll
    for (int r = 0; r < kRows; ++r)
    {
#pragma unroll
        for (int i = 0; i < 8; ++i)
        {
            const uint32_t code = Sample<SampleT>(rawY[r], i);
            values.y[r][i] = tables.y[kHost8 ? code : min(code, p.maxCode)];
            if (ALPHA)
            {
                const uint32_t a = Sample<SampleT>(rawA[r], i);
                values.alpha[r][i] = kHost8 ? a : tables.alpha[min(a, p.maxCode)];
            }
        }
    }
#pragma unroll
    for (int s = 0; s < kSites; ++s)
    {
        const uint32_t cbCode = Sample<SampleT>(rawCb, s);
        const uint32_t crCode = Sample<SampleT>(rawCr, s);
        const float Cb = tables.uv[kHost8 ? cbCode : min(cbCode, p.maxCode)];
        const float Cr = tables.uv[kHost8 ? crCode : min(crCode, p.maxCode)];
        values.rOffset[s] = f.rGain * Cr;
        values.bOffset[s] = f.bGain * Cb;
        const float greenNumerator = 2 * ((f.gCr * Cr) + (f.gCb * Cb));
        values.gOffset[s] = p.verifiedGreenDivision ? DivideByConstant(greenNumerator, f.kg, f.kgReciprocal) : greenNumerator / f.kg;
    }
}

// The lane's pixels of the unit row starting at pixel (x0, y0); the second row of a 4:2:0 unit only when `secondRow`.
template <typename SampleT, int XS, int YS, int ALPHA>
__device__ __forceinline__ void StoreYccUnit(const IntDecodeParams& p, const YccFactors& f, const YccValues<XS, YS>& values, int x0, int y0, bool secondRow)
{
    constexpr bool kHost8 = sizeof(SampleT) == 1;
    constexpr int kRows = YS ? 2 : 1;
    constexpr int kChannels = ALPHA ? 4 : 3;
    const float outScale = f.outScale;
#pragma unroll
    for (int r = 0; r < kRows; ++r)
    {
        if (r == 1 && !secondRow)
        {
            break;
        }
        uint32_t out[8][kChannels]; // colour channels: 2^23-biased float bit patterns (the code is in the low bits)
        // Two pixels per step: the clamped sums are scalar (the saturation modifier has no packed form), the quantiser --
        // QuantiseBiased's fused multiply-add and biased truncation -- runs on the pair (packed_f32x2.cuh).
        const avifx2::F32x2 scale2 = avifx2::Splat(outScale), half2 = avifx2::Splat(0.5f), bias2 = avifx2::Splat(kTwo23);
        const auto quantisePair = [&](float c0, float c1, uint32_t& q0, uint32_t& q1)
        {
            float b0, b1;
            avifx2::Unpack(avifx2::AddRz2(avifx2::Fma2(avifx2::Pack(c0, c1), scale2, half2), bias2), b0, b1);
            q0 = __float_as_uint(b0);
            q1 = __float_as_uint(b1);
        };
        if (!kHost8)
        {
            // 16-bit hosts: one pixel at a time (the pair form measured 4 % slower there: registers)
#pragma unroll
            for (int i = 0; i < 8; ++i)
            {
                const int s = XS ? (i >> 1) : i;
                out[i][0] = QuantiseBiased(__saturatef(values.y[r][i] + values.rOffset[s]), outScale);
                out[i][1] = QuantiseBiased(__saturatef(values.y[r][i] - values.gOffset[s]), outScale);
                out[i][2] = QuantiseBiased(__saturatef(values.y[r][i] + values.bOffset[s]), outScale);
                if (ALPHA)
                {
                    out[i][3] = values.alpha[r][i];
                }
            }
        }
#pragma unroll
        for (int i = 0; kHost8 && i < 8; i += 2)
        {
            const int s0 = XS ? (i >> 1) : i, s1 = XS ? (i >> 1) : i + 1;
            // std::clamp(v, 0, 1) as the add's saturation modifier: the table entries are finite and Y >= +0, so the
            // sums are never NaN or -0.0 and the two agree for every input.
            quantisePair(__saturatef(values.y[r][i] + values.rOffset[s0]), __saturatef(values.y[r][i + 1] + values.rOffset[s1]), out[i][0], out[i + 1][0]);
            quantisePair(__saturatef(values.y[r][i] - values.gOffset[s0]), __saturatef(values.y[r][i + 1] - values.gOffset[s1]), out[i][1], out[i + 1][1]);
            quantisePair(__saturatef(values.y[r][i] + values.bOffset[s0]), __saturatef(values.y[r][i + 1] + values.bOffset[s1]), out[i][2], out[i + 1][2]);
            if (ALPHA)
            {
                out[i][3] = values.alpha[r][i];
                out[i + 1][3] = values.alpha[r][i + 1];
            }
        }
        uint8_t* target = p.rows + static_cast<int64_t>(y0 + r) * p.rowStride + static_cast<int64_t>(x0) * (kChannels * sizeof(SampleT));
        if (kHost8)
        {
            // 8 pixels x kChannels bytes: byte 0 of every value, four to a word
            uint32_t words[2 * kChannels];
#pragma unroll
            for (int w = 0; w < 2 * kChannels; ++w)
            {
                uint32_t v[4];
#pragma unroll
                for (int b = 0; b < 4; ++b)
                {
                    const int byteIndex = 4 * w + b;
                    v[b] = out[byteIndex / kChannels][byteIndex % kChannels];
                }
                words[w] = __byte_perm(__byte_perm(v[0], v[1], 0x0040), __byte_perm(v[2], v[3], 0x0040), 0x5410);
            }
            if (ALPHA)
            {
                __stcs(reinterpret_cast<uint4*>(target), make_uint4(words[0], words[1], words[2], words[3]));
                __stcs(reinterpret_cast<uint4*>(target) + 1, make_uint4(words[4], words[5], words[6], words[7]));
            }
            else
            {
#pragma unroll
                for (int q = 0; q < 3; ++q)
                {
                    __stcs(reinterpret_cast<uint2*>(target) + q, make_uint2(words[2 * q], words[2 * q + 1]));
                }
            }
        }
        else
        {
            // 8 pixels x kChannels 16-bit samples: the low half of every value, two to a word
            uint32_t words[4 * kChannels];
#pragma unroll
            for (int w = 0; w < 4 * kChannels; ++w)
            {
                const int first = 2 * w;
                words[w] = __byte_perm(out[first / kChannels][first % kChannels], out[(first + 1) / kChannels][(first + 1) % kChannels], 0x5410);
            }
#pragma unroll
            for (int q = 0; q < kChannels; ++q)
            {
                __stcs(reinterpret_cast<uint4*>(target) + q, make_uint4(words[4 * q], words[4 * q + 1], words[4 * q + 2], words[4 * q + 3]));
            }
        }
    }
}

} // namespace
} // namespace avifgpu

#endif
