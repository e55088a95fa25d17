// kernels_fast_common.cuh -- pieces shared by the tuned float-RGB(A) encode kernels (kernels_fast.cu: no curve;
// kernels_fast_flat.cu: step tables + band bitmap + bulk-copy staging; kernels_fast_rgba.cu: the same look-up for RGBA).
#ifndef AVIF_KERNELS_FAST_COMMON_CUH
#define AVIF_KERNELS_FAST_COMMON_CUH

#include "kernel_params.h"
#include "curve_lookup.cuh"
#include "packed_f32x2.cuh"
#include "source_units.cuh"

#include <cuda_runtime.h>

namespace avifgpu
{
namespace fastenc
{

using namespace avifpix;

constexpr int kTilePixels = 128;     // per row
constexpr int kValuesPerLane = 24;   // 2 rows x 4 pixels x 3 channels
constexpr int kCurveClip = 2;        // no transfer curve: code = trunc(clamp(v * max))

struct FastEncodeParams
{
    const uint8_t* rows;
    int64_t rowStride;
    uint8_t* planeY;
    int64_t strideY;
    uint8_t* planeCb;
    int64_t strideCb;
    uint8_t* planeCr;
    int64_t strideCr;
    uint8_t* planeA;  // RGBA hosts (kernels_fast_rgba.cu)
    int64_t strideA;
    int32_t premultiply;
    int32_t width;    // multiple of 4
    int32_t rowCount; // even when the chroma is vertically sub-sampled
    float pqMultiplier;
    float maxCodeFloat;
    int32_t maxCode;
    ForwardMatrix matrix;
    float chromaOffset;
    int32_t topLeft;
    CurveTableView table;
};

// The route (EncodeFamilyOf) has checked ForwardMatrixStaysInRange(): luma needs no upper clamp, chroma only the
// H.273 clip of 2^depth (a saturated red / blue) to 2^depth - 1, done on two packed codes at once.
// A lane's 2 rows x 4 pixels of R'G'B' codes (as floats, row-major, interleaved) -> Y / Cb / Cr codes in the planes:
// forward matrix, luma quantisation, chroma down-filter (the lane owns whole chroma sites, no cross-lane traffic).
// yRow / cbRow / crRow point at the lane's first sample of the tile's first row in each plane.
//
// The float arithmetic runs two pixels per instruction (packed_f32x2.cuh): pixels (0, 2) and (1, 3) of a row share a
// register pair, so the two chroma sites of a 4:2:0 / 4:2:2 lane are the two halves of one packed value.  The operation
// sequence per pixel is pixel_math.cuh's ForwardPixelFloat, rounding for rounding; see packed_f32x2.cuh for which
// operations may be packed (a product's sum is always a scalar add).
//
// DEST: the avifgpu_source_layout bits of the planes written (0: libheif's planar, low-bit layout).  Everything up to the
// stores is the same; then MSB-aligned codes are shifted two at a time as packed words (MsbWord), and with interleaved
// chroma cbRow points at the lane's first Cb, Cr pair of plane 1: the lane's Cb and Cr words are paired by byte permutation
// into one store of twice the planar bytes (crRow is not used).
template <int DEST>
__device__ __forceinline__ uint32_t MsbWord(uint32_t twoCodes, const FastEncodeParams& p)
{
    // 16 - depth == clz(maxCode) - 16 (the parameter block has no depth field)
    return SourceMsbAligned(DEST) ? CodesToMsbPair(twoCodes, static_cast<uint32_t>(__clz(p.maxCode) - 16)) : twoCodes;
}

// The Cb and Cr words of one chroma row -- two codes each, sites (0, 1) -- as a lane stores them.
template <int DEST>
__device__ __forceinline__ void StoreChromaWords(const FastEncodeParams& p, uint8_t* cbRow, uint8_t* crRow, uint32_t cbWord, uint32_t crWord)
{
    cbWord = MsbWord<DEST>(cbWord, p);
    crWord = MsbWord<DEST>(crWord, p);
    if (SourceInterleaved(DEST))
    {
        __stcs(reinterpret_cast<uint2*>(cbRow), make_uint2(LowHalves(cbWord, crWord), HighHalves(cbWord, crWord)));
    }
    else
    {
        __stcs(reinterpret_cast<uint32_t*>(cbRow), cbWord);
        __stcs(reinterpret_cast<uint32_t*>(crRow), crWord);
    }
}

// The same for 4:4:4: two words each, sites (0, 1) and (2, 3).
template <int DEST>
__device__ __forceinline__ void StoreChromaWords(const FastEncodeParams& p, uint8_t* cbRow, uint8_t* crRow, uint2 cbWords, uint2 crWords)
{
    cbWords = make_uint2(MsbWord<DEST>(cbWords.x, p), MsbWord<DEST>(cbWords.y, p));
    crWords = make_uint2(MsbWord<DEST>(crWords.x, p), MsbWord<DEST>(crWords.y, p));
    if (SourceInterleaved(DEST))
    {
        __stcs(reinterpret_cast<uint4*>(cbRow), make_uint4(LowHalves(cbWords.x, crWords.x), HighHalves(cbWords.x, crWords.x),
                                                          LowHalves(cbWords.y, crWords.y), HighHalves(cbWords.y, crWords.y)));
    }
    else
    {
        __stcs(reinterpret_cast<uint2*>(cbRow), cbWords);
        __stcs(reinterpret_cast<uint2*>(crRow), crWords);
    }
}

template <int XS, int YS, int DEST = 0>
__device__ __forceinline__ void StoreTile(const FastEncodeParams& p, const float (&codeF)[kValuesPerLane], uint8_t* yRow, uint8_t* cbRow, uint8_t* crRow,
                                          bool secondRow)
{
    using namespace avifx2;
    const F32x2 half2 = Splat(0.5f);
    const F32x2 offset2 = Splat(p.chromaOffset);
    const uint32_t maxPair = static_cast<uint32_t>(p.maxCode) * 0x00010001u;
    // cb2[r][h] / cr2[r][h]: float chroma of pixels (h, h + 2) of row r
    F32x2 cb2[2][2], cr2[2][2];
    uint32_t yWord[2][2]; // two packed 16-bit codes each: pixels (0, 1) and (2, 3)
#pragma unroll
    for (int r = 0; r < 2; ++r)
    {
        uint32_t yLow[2], yHigh[2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
        {
            const int j0 = r * 12 + h * 3;
            const int j1 = j0 + 6;
            if (p.matrix.identity)
            {
                // lossless GBR: Y = G, Cb = B, Cr = R
                cb2[r][h] = Pack(codeF[j0 + 2], codeF[j1 + 2]);
                cr2[r][h] = Pack(codeF[j0], codeF[j1]);
                yLow[h] = __float2uint_rz(codeF[j0 + 1] + 0.5f);
                yHigh[h] = __float2uint_rz(codeF[j1 + 1] + 0.5f);
                continue;
            }
            const F32x2 red = Pack(codeF[j0], codeF[j1]);
            const F32x2 green = Pack(codeF[j0 + 1], codeF[j1 + 1]);
            const F32x2 blue = Pack(codeF[j0 + 2], codeF[j1 + 2]);
            float r0, r1, g0, g1, b0, b1;
            Unpack(Mul2(red, Splat(p.matrix.kr)), r0, r1);
            Unpack(Mul2(green, Splat(p.matrix.kg)), g0, g1);
            Unpack(Mul2(blue, Splat(p.matrix.kb)), b0, b1);
            const F32x2 luma = Pack(__fadd_rn(__fadd_rn(r0, g0), b0), __fadd_rn(__fadd_rn(r1, g1), b1)); // (kr R + kg G) + kb B
            cb2[r][h] = Mul2(Sub2(blue, luma), Splat(p.matrix.cbScale));
            cr2[r][h] = Mul2(Sub2(red, luma), Splat(p.matrix.crScale));
            float q0, q1;
            Unpack(Add2(luma, half2), q0, q1);
            yLow[h] = __float2uint_rz(q0);
            yHigh[h] = __float2uint_rz(q1);
        }
        yWord[r][0] = yLow[0] | (yLow[1] << 16);   // pixels 0, 1
        yWord[r][1] = yHigh[0] | (yHigh[1] << 16); // pixels 2, 3
    }
    __stcs(reinterpret_cast<uint2*>(yRow), make_uint2(MsbWord<DEST>(yWord[0][0], p), MsbWord<DEST>(yWord[0][1], p)));
    if (secondRow)
    {
        __stcs(reinterpret_cast<uint2*>(yRow + p.strideY), make_uint2(MsbWord<DEST>(yWord[1][0], p), MsbWord<DEST>(yWord[1][1], p)));
    }

    // (chroma + offset) + 0.5 -> code, both halves; `biased` is a scalar-add result or an exact scaling, never a product
    const auto quantisePair = [&](F32x2 biased) -> uint32_t
    {
        float q0, q1;
        Unpack(Add2(biased, half2), q0, q1);
        return __vminu2(__float2uint_rz(q0) | (__float2uint_rz(q1) << 16), maxPair);
    };
    // the two halves of a product pair added to those of another, as scalars (see the header's rule)
    const auto addHalves = [](F32x2 a, F32x2 b) -> F32x2
    {
        float a0, a1, b0, b1;
        Unpack(a, a0, a1);
        Unpack(b, b0, b1);
        return Pack(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
    };
    const auto addOffset = [&](F32x2 product) -> F32x2
    {
        float c0, c1;
        Unpack(product, c0, c1);
        return Pack(__fadd_rn(c0, p.chromaOffset), __fadd_rn(c1, p.chromaOffset));
    };
    if (XS == 1 && YS == 1)
    {
        uint32_t cbWord, crWord;
        if (p.topLeft)
        {
            cbWord = quantisePair(addOffset(cb2[0][0]));
            crWord = quantisePair(addOffset(cr2[0][0]));
        }
        else
        {
            // ((c00 + c01) + (c10 + c11)) * 0.25f + offset; the scaling by 2^-2 is exact, so the fused form is the same number
            const F32x2 quarter2 = Splat(0.25f);
            const F32x2 cbSum = Add2(addHalves(cb2[0][0], cb2[0][1]), addHalves(cb2[1][0], cb2[1][1]));
            const F32x2 crSum = Add2(addHalves(cr2[0][0], cr2[0][1]), addHalves(cr2[1][0], cr2[1][1]));
            cbWord = quantisePair(Fma2(cbSum, quarter2, offset2));
            crWord = quantisePair(Fma2(crSum, quarter2, offset2));
        }
        StoreChromaWords<DEST>(p, cbRow, crRow, cbWord, crWord);
    }
    else if (XS == 1)
    {
#pragma unroll
        for (int r = 0; r < 2; ++r)
        {
            if (r == 1 && !secondRow) break;
            uint32_t cbWord, crWord;
            if (p.topLeft)
            {
                cbWord = quantisePair(addOffset(cb2[r][0]));
                crWord = quantisePair(addOffset(cr2[r][0]));
            }
            else
            {
                cbWord = quantisePair(Fma2(addHalves(cb2[r][0], cb2[r][1]), half2, offset2)); // (c0 + c1) * 0.5f + offset, exact scaling
                crWord = quantisePair(Fma2(addHalves(cr2[r][0], cr2[r][1]), half2, offset2));
            }
            StoreChromaWords<DEST>(p, cbRow + r * p.strideCb, crRow + r * p.strideCr, cbWord, crWord);
        }
    }
    else
    {
#pragma unroll
        for (int r = 0; r < 2; ++r)
        {
            if (r == 1 && !secondRow) break;
            // pairs hold pixels (0, 2) and (1, 3); the stores want (0, 1) and (2, 3)
            const uint32_t cbEven = quantisePair(addOffset(cb2[r][0])), cbOdd = quantisePair(addOffset(cb2[r][1]));
            const uint32_t crEven = quantisePair(addOffset(cr2[r][0])), crOdd = quantisePair(addOffset(cr2[r][1]));
            StoreChromaWords<DEST>(p, cbRow + r * p.strideCb, crRow + r * p.strideCr,
                                   make_uint2(__byte_perm(cbEven, cbOdd, 0x5410), __byte_perm(cbEven, cbOdd, 0x7632)),
                                   make_uint2(__byte_perm(crEven, crOdd, 0x5410), __byte_perm(crEven, crOdd, 0x7632)));
        }
    }
}

// ---- a lane's float -> code conversion through the compact step table, for the RGBA kernel (kernels_fast_rgba.cu) and
// the batched light-level kernel (kernels_batch.cu).  N is the lane's number of colour samples: 24 for 2 rows x 4 pixels,
// 12 for one row; the samples are row-major, interleaved R, G, B, and codeF always has room for 24 (StoreTile's shape).

// The compact table (one-word entries + first_k in shared memory, kernels_fast_flat.cu has the commentary) and its band
// bitmap, with the look-up's constants.
struct CompactTable
{
    const uint32_t* entries;
    const uint32_t* firstBits;
    uint32_t flatShift;
    int32_t negativeLow;
    int32_t span;
    uint32_t bandStrideLog2;
    const uint32_t* bandBits;
    uint32_t topShift;
    uint32_t codeMask;
    uint32_t magic;
};

// `entries` is where BeginTableImageCopy (table_staging.cuh) lands the table's image.
__device__ __forceinline__ CompactTable CompactTableOf(const CurveTableView& table, const uint32_t* entries)
{
    return CompactTable{ entries, entries + ((table.flatCount + 3) & ~3), table.flatShift, -static_cast<int32_t>(table.flatLow),
                         static_cast<int32_t>(table.flatHigh - table.flatLow), table.bandStrideLog2, table.bandBits, 32u - table.flatShift,
                         table.compactCodeMask, table.compactMagic };
}

// RGBA hosts: alpha, clamp / premultiplication (WriteHeifImage.cpp:1043-1077), then the colour samples the curve sees.
// raw[k] = { R, G, B, A } of the lane's pixel k; alphaCode[k] is its alpha code.
template <int PIXELS>
__device__ __forceinline__ void PrepareRgbaSamples(const FastEncodeParams& p, const uint4 (&raw)[PIXELS], uint32_t (&alphaCode)[PIXELS],
                                                   uint32_t (&colourBits)[3 * PIXELS])
{
#pragma unroll
    for (int k = 0; k < PIXELS; ++k)
    {
        const float alpha = ClampF(__uint_as_float(raw[k].w), 0.0f, 1.0f);
        float colour[3] = { __uint_as_float(raw[k].x), __uint_as_float(raw[k].y), __uint_as_float(raw[k].z) };
        if (p.premultiply && alpha < 1.0f)
        {
#pragma unroll
            for (int c = 0; c < 3; ++c)
            {
                colour[c] = (alpha == 0) ? 0.0f : PremultiplyColor(ClampF(colour[c], 0.0f, 1.0f), alpha, 1.0f);
            }
        }
        alphaCode[k] = FloatToCode(alpha, p.maxCodeFloat);
#pragma unroll
        for (int c = 0; c < 3; ++c)
        {
            colourBits[3 * k + c] = __float_as_uint(colour[c]);
        }
    }
}

// The samples are parked in the lane's staging slot (16-byte aligned, for the band-bitmap probes and the exact
// evaluations), then each goes through the table: codeF[j] is right unless bit j of bandMask is set (in or near a step's
// fuzzy band); `largest` is the max of the samples as signed integers, > 0x7f7fffff <=> a +inf / NaN is among them.
template <int N>
__device__ __forceinline__ void LookUpLaneCodes(const CompactTable& c, const uint32_t (&colourBits)[N], uint32_t* myStage, float (&codeF)[kValuesPerLane],
                                                uint32_t& bandMask, int32_t& largest)
{
#pragma unroll
    for (int q = 0; q < N / 4; ++q)
    {
        *reinterpret_cast<uint4*>(myStage + 4 * q) = make_uint4(colourBits[4 * q], colourBits[4 * q + 1], colourBits[4 * q + 2], colourBits[4 * q + 3]);
    }
    bandMask = 0;
    largest = 0;
#pragma unroll
    for (int j = 0; j < N; ++j)
    {
        bool inBand;
        uint32_t entry;
        codeF[j] = LookupCurveCompact<0>(colourBits[j], c.entries, c.flatShift, c.negativeLow, c.span, c.topShift, c.codeMask, c.magic, inBand, entry);
        asm("{ .reg .pred q; setp.ne.u32 q, %1, 0; @q or.b32 %0, %0, %2; }" : "+r"(bandMask) : "r"(static_cast<uint32_t>(inBand)), "r"(1u << j));
        largest = max(largest, static_cast<int32_t>(colourBits[j]));
    }
}

// The exact codes of the samples LookUpLaneCodes left open: an in-band sample is one below the table's code when its bit
// of the band bitmap (found through first_k) is clear; +inf / NaN take the exact evaluation, lane by lane.
template <int CURVE, int N>
__device__ __forceinline__ void ResolveLaneCodes(const FastEncodeParams& p, const avifmath::LibmTables& t,const CompactTable& c, const uint32_t* myStage,
                                                 uint32_t bandMask, int32_t largest, float (&codeF)[kValuesPerLane])
{
    uint32_t lowerMask = 0;
    {
        uint32_t pending = bandMask;
        while (pending != 0)
        {
            const int j = __ffs(static_cast<int>(pending)) - 1;
            pending &= pending - 1;
            const uint32_t bits = myStage[j];
            const int32_t bucket = __viaddmin_s32_relu(static_cast<int32_t>(bits) >> c.flatShift, c.negativeLow, c.span);
            const uint32_t entry = c.entries[bucket];
            const uint32_t k = ((entry & c.codeMask) >> kCompactLenBits) + ((entry >> c.topShift) != 0 ? 1u : 0u);
            const uint32_t distance = bits - c.firstBits[k];
            if (k != 0 && distance < (1u << c.bandStrideLog2)) // else flagged by the superset test only
            {
                const uint32_t bitIndex = (k << c.bandStrideLog2) + distance;
                const uint32_t word = __ldg(c.bandBits + (bitIndex >> 5));
                lowerMask |= (((word >> (bitIndex & 31u)) & 1u) ^ 1u) << j;
            }
        }
    }
    if (__any_sync(0xffffffffu, largest > 0x7f7fffff))
    {
        for (int j = 0; j < N; ++j)
        {
            const uint32_t bits = myStage[j];
            if (static_cast<int32_t>(bits) > 0x7f7fffff)
            {
                const float exact = CodeToFloat(ExactCurveCode<CURVE>(__uint_as_float(bits), p.pqMultiplier, p.maxCodeFloat, t));
#pragma unroll
                for (int slot = 0; slot < N; ++slot)
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
    for (int j = 0; j < N; ++j)
    {
        if (lowerMask & (1u << j))
        {
            codeF[j] -= 1.0f;
        }
    }
}

// One row of a lane's alpha plane: its 4 pixels' codes from alphaCode[first].
template <int DEST, int PIXELS>
__device__ __forceinline__ void StoreAlphaRow(const FastEncodeParams& p, uint8_t* alphaRow, const uint32_t (&alphaCode)[PIXELS], int first)
{
    __stcs(reinterpret_cast<uint2*>(alphaRow), make_uint2(MsbWord<DEST>(alphaCode[first] | (alphaCode[first + 1] << 16), p),
                                                          MsbWord<DEST>(alphaCode[first + 2] | (alphaCode[first + 3] << 16), p)));
}

} // namespace fastenc

// kernels_fast_rgba.cu; `dest` is the description's avifgpu_source_layout bits (EncodeParams::destLayout)
cudaError_t LaunchFastEncodeRgba(const fastenc::FastEncodeParams& fp, int curve, int xs, int ys, int dest, int smCount, cudaStream_t stream, const LightSink* light);

// kernels_fast_flat.cu
cudaError_t LaunchFastEncodeFlat(const fastenc::FastEncodeParams& fp, int curve, int xs, int ys, int dest, int smCount, cudaStream_t stream, const LightSink* light);
cudaError_t LaunchFastEncodeFlatInterleaved(const fastenc::FastEncodeParams& fp, int curve, int smCount, cudaStream_t stream, const LightSink* light);

} // namespace avifgpu

#endif
