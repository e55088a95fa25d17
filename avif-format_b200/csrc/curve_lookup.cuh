// curve_lookup.cuh -- device-side use of a CurveTable (see curve_tables.h): the exact curve evaluation and the
// two-level table look-up, shared by the table verifier and the conversion kernels.
#ifndef AVIF_CURVE_LOOKUP_CUH
#define AVIF_CURVE_LOOKUP_CUH

#include "curve_tables.h"
#include "pixel_math.cuh"

namespace avifgpu
{

// The exact quantised curve: WriteHeifImage.cpp:1079-1096 for one sample.
template <int CURVE>
__device__ __forceinline__ uint32_t ExactCurveCode(float x, float pqMultiplier, float maxCodeFloat, const avifmath::LibmTables& t)
{
    float curved;
    if (CURVE == kCurveLinearToPQ)
    {
        curved = avifpix::LinearToPQ(x, pqMultiplier, t);
    }
    else if (CURVE == kCurveLinearToSMPTE428)
    {
        curved = avifpix::LinearToSMPTE428(x, t);
    }
    else
    {
        curved = avifpix::LinearToHLG(x, t);
    }
    return avifpix::FloatToCode(curved, maxCodeFloat);
}

// Table look-up for the float with bit pattern `bits`.  Returns the code that is correct whenever `inBand` is
// false; when `inBand` is true the caller must evaluate ExactCurveCode instead.
// Negative floats (sign bit set; includes -0 and negative NaNs) map to code 0 like the reference: value < 0
// returns 0, and -0 / NaN quantise to 0.
__device__ __forceinline__ uint32_t LookupCurveCode(uint32_t bits, const uint2* __restrict__ octaves,
                                                    const uint32_t* __restrict__ buckets, bool& inBand)
{
    if (bits & 0x80000000u)
    {
        inBand = false;
        return 0;
    }
    const uint2 oct = octaves[bits >> 23];
    const uint32_t shift = oct.y & 0xffu;
    const uint32_t reduce = (oct.y >> 8) & 0xffu;
    const uint32_t widthQ = oct.y >> 16;
    const uint32_t mantissa = bits & 0x7fffffu;
    const uint32_t word = buckets[oct.x + (mantissa >> shift)];
    const uint32_t offsetQ = (mantissa & ((1u << shift) - 1u)) >> reduce;
    const uint32_t stepOffset = word & ((1u << kBucketOffsetBits) - 1u);
    const uint32_t distance = offsetQ - stepOffset; // wraps to a huge value below the step
    inBand = distance <= widthQ;
    return (word >> kBucketOffsetBits) + (offsetQ >= stepOffset ? 1u : 0u);
}

// Compact look-up (curve_tables.h "Compact entries").  `compact` is indexed by (bucket number - low), `span` = high - low,
// topShift = 32 - flatShift.  The bucket number is taken with an ARITHMETIC shift, so every float with the sign bit set
// (negative values, -0, negative NaNs) yields a negative index that the single add-clamp-to-[0, span] instruction (DPX)
// sends to the lowest bucket; that bucket holds no step and decodes to code 0 exactly as the reference's
// `value < 0 -> 0` / NaN -> 0 does.  +inf and the positive NaNs (bits > 0x7f7fffff) do NOT follow the steps; they land in
// the top bucket and the caller must route them to ExactCurveCode itself.
// SHIFT != 0 fixes flatShift at compile time (the shifts become immediates and entry + (bits << topShift) a single
// multiply-add on the FMA pipe); `magic` is 0x4b000000 handed in as a run-time value so that (entry & codeMask) | magic
// stays ONE three-input logic instruction.  Eleven instructions and one 32-bit shared-memory load per sample; the code
// comes out as a float (the forward matrix wants floats).
template <int SHIFT>
__device__ __forceinline__ float LookupCurveCompact(uint32_t bits, const uint32_t* __restrict__ compact, uint32_t shift, int32_t negativeLow, int32_t span,
                                                    uint32_t topShift, uint32_t codeMask, uint32_t magic, bool& inBand, uint32_t& entryOut)
{
    const uint32_t s = SHIFT != 0 ? static_cast<uint32_t>(SHIFT) : shift;
    const uint32_t top = SHIFT != 0 ? 32u - static_cast<uint32_t>(SHIFT) : topShift;
    const int32_t index = __viaddmin_s32_relu(static_cast<int32_t>(bits) >> s, negativeLow, span);
    const uint32_t entry = compact[index];
    entryOut = entry;
    const uint32_t t = entry + (bits << top);
    uint32_t biased;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(biased) : "r"(entry), "r"(codeMask), "r"(magic)); // (entry & codeMask) | magic
    // 2^23 + (field << 6) is exact in binary32; (x - 2^23) / 64 in one fma
    float code = __fmaf_rn(__uint_as_float(biased), 1.0f / 64.0f, -131072.0f);
    if (t < entry) // carry: bits >= first_k of a step bucket
    {
        code += 1.0f;
    }
    inBand = t < (entry << (32u - kCompactLenBits)); // distance from the band start < lenq units
    return code;
}

// The exact code of a sample LookupCurveCompact flagged, `fastCode` being what it returned for it.
__device__ __forceinline__ uint32_t ResolveCompactInBand(uint32_t bits, uint32_t entry, uint32_t fastCode, uint32_t topShift, uint32_t codeMask,
                                                         const uint32_t* __restrict__ firstBits, const uint32_t* __restrict__ bandBits, uint32_t strideLog2)
{
    const uint32_t k = ((entry & codeMask) >> kCompactLenBits) + ((entry >> topShift) != 0 ? 1u : 0u); // the step whose band this is
    const uint32_t distance = bits - firstBits[k];
    if (k == 0 || distance >= (1u << strideLog2))
    {
        return fastCode; // flagged by the superset test only (below first_k, wrapped): the table's answer stands
    }
    const uint32_t index = (k << strideLog2) + distance;
    const uint32_t word = __ldg(bandBits + (index >> 5));
    return ((word >> (index & 31u)) & 1u) ? k : k - 1u;
}

// Complete compact look-up for one finite sample, bitmap included (the verifier, and the generic kernel from global
// memory; the tuned kernels inline the same steps around their own batching).
__device__ __forceinline__ uint32_t LookupCurveCodeCompactResolved(uint32_t bits, const CurveTableView& table, bool& inBand)
{
    const uint32_t topShift = 32u - table.flatShift;
    uint32_t entry;
    const float code = LookupCurveCompact<0>(bits, table.compact, table.flatShift, -static_cast<int32_t>(table.flatLow),
                                             static_cast<int32_t>(table.flatHigh - table.flatLow), topShift, table.compactCodeMask, 0x4b000000u, inBand,
                                             entry);
    uint32_t result = static_cast<uint32_t>(code);
    if (inBand)
    {
        result = ResolveCompactInBand(bits, entry, result, topShift, table.compactCodeMask, table.firstBits, table.bandBits, table.bandStrideLog2);
    }
    return result;
}

} // namespace avifgpu

#endif
