// curve_tables.cu -- builds and verifies the exact float -> code tables described in curve_tables.h.
#include "curve_tables.h"
#include "curve_lookup.cuh"

#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <vector>

namespace avifgpu
{

namespace
{

constexpr int kSweepThreads = 256;
constexpr uint32_t kRunLength = 128;               // consecutive floats per thread
constexpr uint32_t kSweepEnd = 0x7f800000u;        // every non-negative finite float: bits [0, +inf)
constexpr int kMinShift = 6;                       // smallest bucket: 64 floats

// Pass 1: per code, the smallest and largest input bits that produce it.
template <int CURVE>
__global__ void __launch_bounds__(kSweepThreads) SweepKernel(float pqMultiplier, float maxCodeFloat, uint32_t* __restrict__ minBits,
                                                            uint32_t* __restrict__ maxBits)
{
    __shared__ uint64_t libmStorage[96];
    const avifmath::LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();

    const uint64_t runs = kSweepEnd / kRunLength;
    for (uint64_t run = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; run < runs;
         run += static_cast<uint64_t>(gridDim.x) * blockDim.x)
    {
        const uint32_t begin = static_cast<uint32_t>(run * kRunLength);
        uint32_t current = ExactCurveCode<CURVE>(__uint_as_float(begin), pqMultiplier, maxCodeFloat, t);
        uint32_t first = begin;
        for (uint32_t i = 1; i < kRunLength; ++i)
        {
            const uint32_t bits = begin + i;
            const uint32_t code = ExactCurveCode<CURVE>(__uint_as_float(bits), pqMultiplier, maxCodeFloat, t);
            if (code != current)
            {
                atomicMin(&minBits[current], first);
                atomicMax(&maxBits[current], bits - 1);
                current = code;
                first = bits;
            }
        }
        atomicMin(&minBits[current], first);
        atomicMax(&maxBits[current], begin + kRunLength - 1);
    }
}

// Pass 2: every input again, both tables against exact.  counters[0] = mismatches (two-level outside its bands, compact
// everywhere finite), [1] = inputs in the two-level table's bands, [2] = inputs the compact table flags.
template <int CURVE>
__global__ void __launch_bounds__(kSweepThreads) VerifyKernel(float pqMultiplier, float maxCodeFloat, CurveTableView table,
                                                             unsigned long long* __restrict__ counters)
{
    __shared__ uint64_t libmStorage[96];
    const avifmath::LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();

    unsigned long long mismatches = 0;
    unsigned long long inBandCount = 0;
    unsigned long long compactInBand = 0;
    // +inf and the positive NaNs are part of the check (bits up to 0x7fffffff): they must come out as code 0.
    const uint64_t total = 0x80000000ull;
    for (uint64_t u = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; u < total;
         u += static_cast<uint64_t>(gridDim.x) * blockDim.x)
    {
        const uint32_t bits = static_cast<uint32_t>(u);
        bool inBand;
        uint32_t fast = LookupCurveCode(bits, table.octaves, table.buckets, inBand);
        // The compact variant, band bitmap included, must reproduce the exact curve for every finite input;
        // +inf / NaN are the caller's to route to the exact evaluation (curve_lookup.cuh).
        if (table.compact != nullptr && bits <= 0x7f7fffffu)
        {
            bool inBandCompact;
            if (LookupCurveCodeCompactResolved(bits, table, inBandCompact) != ExactCurveCode<CURVE>(__uint_as_float(bits), pqMultiplier, maxCodeFloat, t))
            {
                ++mismatches;
            }
            if (inBandCompact)
            {
                ++compactInBand;
            }
        }
        if (inBand)
        {
            ++inBandCount;
        }
        else if (fast != ExactCurveCode<CURVE>(__uint_as_float(bits), pqMultiplier, maxCodeFloat, t))
        {
            ++mismatches;
        }
    }
    for (int offset = 16; offset > 0; offset >>= 1)
    {
        mismatches += __shfl_down_sync(0xffffffffu, mismatches, offset);
        inBandCount += __shfl_down_sync(0xffffffffu, inBandCount, offset);
        compactInBand += __shfl_down_sync(0xffffffffu, compactInBand, offset);
    }
    if ((threadIdx.x & 31) == 0)
    {
        if (mismatches) atomicAdd(&counters[0], mismatches);
        if (inBandCount) atomicAdd(&counters[1], inBandCount);
        if (compactInBand) atomicAdd(&counters[2], compactInBand);
    }
}

// Band bitmap: one warp per 32-bit word, lane = bit.  bands[i] = {first_k, width, k}.
template <int CURVE>
__global__ void __launch_bounds__(kSweepThreads) FillBandBitsKernel(float pqMultiplier, float maxCodeFloat, const uint3* __restrict__ bands, int bandCount,
                                                                   uint32_t strideLog2, uint32_t* __restrict__ bandBits)
{
    __shared__ uint64_t libmStorage[96];
    const avifmath::LibmTables t = avifmath::StageLibmTables(libmStorage, threadIdx.x, blockDim.x);
    __syncthreads();

    const uint32_t wordsPerBand = (1u << strideLog2) / 32u;
    const uint64_t words = static_cast<uint64_t>(bandCount) * wordsPerBand;
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warpsInGrid = static_cast<uint64_t>(gridDim.x) * (blockDim.x / 32);
    for (uint64_t w = static_cast<uint64_t>(blockIdx.x) * (blockDim.x / 32) + (threadIdx.x >> 5); w < words; w += warpsInGrid)
    {
        const uint3 band = bands[w / wordsPerBand];
        const uint32_t offset = static_cast<uint32_t>(w % wordsPerBand) * 32u + lane;
        // Every offset of the stride is answered, not only the band proper: the compact table's in-band test rounds a band
        // up to 32 floats, and past the band the exact code is k (or more) anyway.  +inf / NaN never get here (callers
        // route them to the exact evaluation), but the bitmap must not claim anything about them: left 0.
        bool atOrAbove = false;
        const uint64_t input = static_cast<uint64_t>(band.x) + offset;
        if (input <= 0x7f7fffffull)
        {
            atOrAbove = ExactCurveCode<CURVE>(__uint_as_float(static_cast<uint32_t>(input)), pqMultiplier, maxCodeFloat, t) >= band.z;
        }
        const uint32_t word = __ballot_sync(0xffffffffu, atOrAbove);
        if (lane == 0)
        {
            bandBits[((static_cast<uint64_t>(band.z) << strideLog2) >> 5) + (w % wordsPerBand)] = word;
        }
    }
}

struct Step
{
    uint32_t first; // min{bits : code >= k}
    uint32_t end;   // max(first, max{bits : code < k})
    uint32_t k;
};

bool Check(cudaError_t e, const char* what, std::string* error)
{
    if (e == cudaSuccess)
    {
        return true;
    }
    *error = std::string(what) + ": " + cudaGetErrorString(e);
    return false;
}

} // namespace

void FreeCurveTable(CurveTable* table)
{
    if (table->deviceOctaves) cudaFree(table->deviceOctaves);
    if (table->deviceBuckets) cudaFree(table->deviceBuckets);
    if (table->deviceBandBits) cudaFree(table->deviceBandBits);
    if (table->deviceCompact) cudaFree(table->deviceCompact);
    if (table->deviceFirstBits) cudaFree(table->deviceFirstBits);
    table->deviceCompact = nullptr;
    table->deviceFirstBits = nullptr;
    table->deviceOctaves = nullptr;
    table->deviceBuckets = nullptr;
    table->deviceBandBits = nullptr;
    table->valid = false;
}

bool BuildCurveTable(int curve, int param, int depth, void* streamHandle, CurveTable* table)
{
    const auto t0 = std::chrono::steady_clock::now();
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    table->curve = curve;
    table->param = param;
    table->depth = depth;
    table->valid = false;
    table->error.clear();

    const uint32_t maxCode = (1u << depth) - 1u;
    const float maxCodeFloat = static_cast<float>(maxCode);
    const float pqMultiplier = static_cast<float>(param) / 10000.0f; // ColorTransfer.cpp:86
    const size_t codeCount = static_cast<size_t>(maxCode) + 1;

    int device = 0;
    cudaDeviceProp prop{};
    if (!Check(cudaGetDevice(&device), "cudaGetDevice", &table->error) ||
        !Check(cudaGetDeviceProperties(&prop, device), "cudaGetDeviceProperties", &table->error))
    {
        return false;
    }
    const int grid = prop.multiProcessorCount * 8;

    // ---- pass 1: sweep ----------------------------------------------------------------------------------------
    uint32_t* dMin = nullptr;
    uint32_t* dMax = nullptr;
    if (!Check(cudaMalloc(&dMin, codeCount * sizeof(uint32_t)), "cudaMalloc", &table->error) ||
        !Check(cudaMalloc(&dMax, codeCount * sizeof(uint32_t)), "cudaMalloc", &table->error))
    {
        cudaFree(dMin);
        return false;
    }
    cudaMemsetAsync(dMin, 0xff, codeCount * sizeof(uint32_t), stream);
    cudaMemsetAsync(dMax, 0x00, codeCount * sizeof(uint32_t), stream);
    if (curve == kCurveLinearToPQ)
    {
        SweepKernel<kCurveLinearToPQ><<<grid, kSweepThreads, 0, stream>>>(pqMultiplier, maxCodeFloat, dMin, dMax);
    }
    else if (curve == kCurveLinearToSMPTE428)
    {
        SweepKernel<kCurveLinearToSMPTE428><<<grid, kSweepThreads, 0, stream>>>(pqMultiplier, maxCodeFloat, dMin, dMax);
    }
    else
    {
        SweepKernel<kCurveLinearToHLG><<<grid, kSweepThreads, 0, stream>>>(pqMultiplier, maxCodeFloat, dMin, dMax);
    }
    std::vector<uint32_t> minBits(codeCount), maxBits(codeCount);
    bool ok = Check(cudaMemcpyAsync(minBits.data(), dMin, codeCount * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream), "D2H", &table->error) &&
              Check(cudaMemcpyAsync(maxBits.data(), dMax, codeCount * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream), "D2H", &table->error) &&
              Check(cudaStreamSynchronize(stream), "curve sweep", &table->error);
    cudaFree(dMin);
    cudaFree(dMax);
    if (!ok)
    {
        return false;
    }
    table->stats.sweptInputs = kSweepEnd;

    // ---- thresholds -------------------------------------------------------------------------------------------
    // first_k = min over codes >= k of minBits (suffix minimum); last_k = max over codes < k of maxBits (prefix max).
    std::vector<uint32_t> first(codeCount + 1, 0xffffffffu), last(codeCount + 1, 0u);
    {
        uint32_t running = 0xffffffffu;
        for (size_t c = codeCount; c-- > 0;)
        {
            running = std::min(running, minBits[c]);
            first[c] = running;
        }
        uint32_t high = 0;
        bool any = false;
        for (size_t k = 1; k <= codeCount; ++k)
        {
            if (minBits[k - 1] != 0xffffffffu)
            {
                high = any ? std::max(high, maxBits[k - 1]) : maxBits[k - 1];
                any = true;
            }
            last[k] = high;
        }
    }
    if (first[0] != 0)
    {
        table->error = "curve sweep: code of +0 is not the minimum";
        return false;
    }
    std::vector<Step> steps;
    for (uint32_t k = 1; k <= maxCode; ++k)
    {
        if (first[k] == 0xffffffffu)
        {
            break; // codes >= k are never produced
        }
        Step s;
        s.k = k;
        s.first = first[k];
        s.end = std::max(first[k], last[k]);
        if (!steps.empty() && s.first <= steps.back().end)
        {
            table->error = "curve sweep: fuzzy bands of neighbouring codes overlap";
            return false;
        }
        if (last[k] >= first[k])
        {
            table->stats.bands++;
            table->stats.widestBand = std::max(table->stats.widestBand, last[k] - first[k] + 1);
        }
        steps.push_back(s);
    }
    table->stats.steps = static_cast<int32_t>(steps.size());

    // ---- two-level table --------------------------------------------------------------------------------------
    std::vector<uint2> octaves(256);
    std::vector<uint32_t> buckets;
    size_t cursor = 0; // first step whose end is >= the current octave start
    for (uint32_t e = 0; e < 256; ++e)
    {
        const uint64_t lo = static_cast<uint64_t>(e) << 23;
        const uint64_t hi = lo + (1u << 23);
        if (e == 255)
        {
            // +inf and NaN do not follow the step structure (LinearToPQ(inf) is NaN -> 0, LinearToSMPTE428(inf) is
            // inf -> max, NaN -> 0): one bucket whose band covers every offset, so they all take the exact path.
            octaves[e] = make_uint2(static_cast<uint32_t>(buckets.size()), 23u | (7u << 8) | (0xffffu << 16));
            buckets.push_back(0u);
            continue;
        }
        while (cursor < steps.size() && steps[cursor].end < lo)
        {
            ++cursor;
        }
        size_t stop = cursor;
        while (stop < steps.size() && steps[stop].first < hi)
        {
            ++stop;
        }
        // steps[cursor, stop) touch this octave (their [first, end] intersects it)
        int shift = 23;
        for (; shift >= kMinShift; --shift)
        {
            bool separated = true;
            for (size_t i = cursor; i + 1 < stop && separated; ++i)
            {
                const uint64_t endHere = std::min<uint64_t>(steps[i].end, hi - 1);
                const uint64_t nextFirst = std::max<uint64_t>(steps[i + 1].first, lo);
                separated = ((endHere - lo) >> shift) < ((nextFirst - lo) >> shift);
            }
            if (separated)
            {
                break;
            }
        }
        if (shift < kMinShift)
        {
            table->error = "curve table: two steps closer than the smallest bucket";
            return false;
        }
        const uint32_t reduce = shift > static_cast<int>(kOffsetResolutionBits) ? static_cast<uint32_t>(shift) - kOffsetResolutionBits : 0u;
        uint32_t widest = 0;
        for (size_t i = cursor; i < stop; ++i)
        {
            widest = std::max(widest, steps[i].end - steps[i].first);
        }
        const uint32_t widthQ = (widest >> reduce) + 2u;
        if (widthQ > 0xffffu)
        {
            table->error = "curve table: band wider than the table format allows";
            return false;
        }
        octaves[e] = make_uint2(static_cast<uint32_t>(buckets.size()), static_cast<uint32_t>(shift) | (reduce << 8) | (widthQ << 16));

        const uint32_t bucketCount = 1u << (23 - shift);
        size_t next = cursor; // first step with end >= bucket start
        for (uint32_t b = 0; b < bucketCount; ++b)
        {
            const uint64_t bLo = lo + (static_cast<uint64_t>(b) << shift);
            const uint64_t bHi = bLo + (1ull << shift);
            while (next < stop && steps[next].end < bLo)
            {
                ++next;
            }
            uint32_t word;
            if (next < stop && steps[next].first < bHi)
            {
                // this bucket meets step `next` (its start, its band, or the tail of its band)
                const uint64_t start = std::max<uint64_t>(steps[next].first, bLo);
                const uint32_t offsetQ = static_cast<uint32_t>((start - bLo) >> reduce);
                word = ((steps[next].k - 1u) << kBucketOffsetBits) | offsetQ;
            }
            else
            {
                // no step here: the code is the number of steps below the bucket
                const uint32_t code = static_cast<uint32_t>(next); // steps[0..next) all end below bLo
                word = (code << kBucketOffsetBits) | kBucketOffsetNone;
            }
            buckets.push_back(word);
        }
    }
    // Bucket words store k-1 in 12 bits: depth <= 12.
    if (depth > 12)
    {
        table->error = "curve table: depth above 12 bits";
        return false;
    }

    // ---- compact variant (curve_tables.h "Compact entries") -----------------------------------------------------
    std::vector<uint32_t> compact;
    std::vector<uint3> bands; // {first, width, k} of every step with a fuzzy band
    uint32_t flatShift = 0, flatLow = 0, flatHigh = 0, bandStrideLog2 = 5;
    if (!steps.empty())
    {
        int shift = static_cast<int>(std::min(kFlatMaxShift, 32u - static_cast<uint32_t>(depth) - kCompactLenBits));
        for (; shift >= kMinShift; --shift)
        {
            bool separated = true;
            for (size_t i = 0; i + 1 < steps.size() && separated; ++i)
            {
                separated = (steps[i].end >> shift) < (steps[i + 1].first >> shift);
            }
            if (separated)
            {
                break;
            }
        }
        bool usable = shift >= kMinShift && (steps.front().first >> shift) >= 1;
        if (usable)
        {
            flatShift = static_cast<uint32_t>(shift);
            flatLow = (steps.front().first >> shift) - 1u;
            flatHigh = (steps.back().end >> shift) + 1u;
            const uint64_t count = static_cast<uint64_t>(flatHigh) - flatLow + 1u;
            usable = count * sizeof(uint32_t) <= kFlatMaxBytes && (static_cast<uint64_t>(flatHigh + 1u) << shift) <= kSweepEnd;
            const uint32_t topShift = 32u - static_cast<uint32_t>(shift);
            const uint32_t lenMax = (1u << kCompactLenBits) - 1u;
            const uint32_t unitLog2 = static_cast<uint32_t>(shift) - kCompactLenBits; // flatShift >= kMinShift = 6
            compact.resize(usable ? count : 0);
            size_t at = 0;
            for (uint64_t b = 0; b < compact.size() && usable; ++b)
            {
                const uint64_t bLo = (static_cast<uint64_t>(flatLow) + b) << shift;
                const uint64_t bHi = bLo + (1ull << shift);
                while (at < steps.size() && steps[at].end < bLo)
                {
                    ++at;
                }
                uint32_t top = 0, field, inBandFloats = 0;
                if (at < steps.size() && steps[at].first < bHi)
                {
                    const Step& step = steps[at];
                    const bool banded = step.end > step.first;
                    if (step.first > bLo)
                    {
                        // the step starts inside this bucket: code = (k - 1) + carry
                        top = static_cast<uint32_t>((1ull << shift) - (step.first - bLo));
                        field = step.k - 1u;
                        inBandFloats = banded ? static_cast<uint32_t>(std::min<uint64_t>(step.end, bHi - 1) - step.first + 1u) : 0u;
                    }
                    else
                    {
                        // the step sits exactly on the bucket start, or this is the tail of a band that began in the
                        // previous bucket: every float here is at or above first_k
                        field = step.k;
                        inBandFloats = banded ? static_cast<uint32_t>(std::min<uint64_t>(step.end, bHi - 1) - bLo + 1u) : 0u;
                    }
                }
                else
                {
                    field = static_cast<uint32_t>(at); // no step: code = steps below
                }
                const uint32_t lenq = (inBandFloats + (1u << unitLog2) - 1u) >> unitLog2;
                usable = lenq <= lenMax && field <= maxCode;
                compact[b] = (top << topShift) | (field << kCompactLenBits) | lenq;
            }
            // the band bitmap answers bits - first_k < 2^stride for every banded step: a band rounded up to the unit (plus
            // the part of it that lies in the previous bucket) must stay inside it
            while (usable && (1u << bandStrideLog2) < table->stats.widestBand + (2u << unitLog2))
            {
                ++bandStrideLog2;
            }
            usable = usable && ((static_cast<uint64_t>(codeCount) << bandStrideLog2) / 8u) <= kBandBitmapMaxBytes;
        }
        if (usable)
        {
            for (const Step& s : steps)
            {
                if (s.end > s.first)
                {
                    bands.push_back(make_uint3(s.first, s.end - s.first + 1u, s.k));
                }
            }
        }
        else
        {
            compact.clear();
        }
    }

    // ---- upload -----------------------------------------------------------------------------------------------
    if (!Check(cudaMalloc(&table->deviceOctaves, octaves.size() * sizeof(uint2)), "cudaMalloc", &table->error) ||
        !Check(cudaMalloc(&table->deviceBuckets, buckets.size() * sizeof(uint32_t)), "cudaMalloc", &table->error))
    {
        FreeCurveTable(table);
        return false;
    }
    table->view.octaves = static_cast<const uint2*>(table->deviceOctaves);
    table->view.buckets = static_cast<const uint32_t*>(table->deviceBuckets);
    table->view.bucketCount = static_cast<int32_t>(buckets.size());
    table->view.flatCount = 0;
    table->view.bandBits = nullptr;
    table->view.bandStrideLog2 = 0;
    table->view.compact = nullptr;
    table->view.firstBits = nullptr;
    table->view.compactImageBytes = 0;
    table->view.compactCodeMask = 0;
    table->view.compactMagic = 0;
    if (!compact.empty())
    {
        // Band bitmap: the exact answer for every in-band float, one bit each, at (k << stride) + (bits - first_k).
        const size_t bitmapBytes = (codeCount << bandStrideLog2) / 8u;
        uint3* dBands = nullptr;
        bool filled = Check(cudaMalloc(&table->deviceBandBits, bitmapBytes), "cudaMalloc", &table->error) &&
                      Check(cudaMemsetAsync(table->deviceBandBits, 0, bitmapBytes, stream), "memset", &table->error);
        if (filled && !bands.empty())
        {
            filled = Check(cudaMalloc(&dBands, bands.size() * sizeof(uint3)), "cudaMalloc", &table->error) &&
                     Check(cudaMemcpyAsync(dBands, bands.data(), bands.size() * sizeof(uint3), cudaMemcpyHostToDevice, stream), "H2D", &table->error);
            if (filled)
            {
                uint32_t* bitsOut = static_cast<uint32_t*>(table->deviceBandBits);
                const int bandCount = static_cast<int>(bands.size());
                if (curve == kCurveLinearToPQ)
                {
                    FillBandBitsKernel<kCurveLinearToPQ><<<grid, kSweepThreads, 0, stream>>>(pqMultiplier, maxCodeFloat, dBands, bandCount, bandStrideLog2, bitsOut);
                }
                else if (curve == kCurveLinearToSMPTE428)
                {
                    FillBandBitsKernel<kCurveLinearToSMPTE428><<<grid, kSweepThreads, 0, stream>>>(pqMultiplier, maxCodeFloat, dBands, bandCount, bandStrideLog2, bitsOut);
                }
                else
                {
                    FillBandBitsKernel<kCurveLinearToHLG><<<grid, kSweepThreads, 0, stream>>>(pqMultiplier, maxCodeFloat, dBands, bandCount, bandStrideLog2, bitsOut);
                }
                filled = Check(cudaStreamSynchronize(stream), "band bitmap", &table->error);
            }
            cudaFree(dBands);
        }
        std::vector<uint32_t> firstBits(codeCount + 1, 0u);
        for (const Step& step : steps)
        {
            firstBits[step.k] = step.first;
        }
        // one allocation = the kernels' shared-memory image (CurveTableView::compactImageBytes)
        const size_t paddedCompact = (compact.size() + 3u) & ~static_cast<size_t>(3u);
        const size_t paddedFirst = (firstBits.size() + 3u) & ~static_cast<size_t>(3u);
        std::vector<uint32_t> image(paddedCompact + paddedFirst, 0u);
        std::copy(compact.begin(), compact.end(), image.begin());
        std::copy(firstBits.begin(), firstBits.end(), image.begin() + static_cast<std::ptrdiff_t>(paddedCompact));
        if (!filled ||
            !Check(cudaMalloc(&table->deviceCompact, image.size() * sizeof(uint32_t)), "cudaMalloc", &table->error) ||
            !Check(cudaMemcpyAsync(table->deviceCompact, image.data(), image.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, stream), "H2D", &table->error) ||
            !Check(cudaStreamSynchronize(stream), "compact table upload", &table->error))
        {
            FreeCurveTable(table);
            return false;
        }
        table->view.flatCount = static_cast<int32_t>(compact.size());
        table->view.flatShift = flatShift;
        table->view.flatLow = flatLow;
        table->view.flatHigh = flatHigh;
        table->view.bandBits = static_cast<const uint32_t*>(table->deviceBandBits);
        table->view.bandStrideLog2 = bandStrideLog2;
        table->view.compact = static_cast<const uint32_t*>(table->deviceCompact);
        table->view.firstBits = table->view.compact + paddedCompact;
        table->view.compactImageBytes = static_cast<uint32_t>(image.size() * sizeof(uint32_t));
        table->view.compactCodeMask = maxCode << kCompactLenBits;
        table->view.compactMagic = 0x4b000000u;
        table->stats.bandBitmapBytes = bitmapBytes;
        table->stats.compactBuckets = static_cast<int32_t>(compact.size());
    }
    unsigned long long* dCounters = nullptr;
    ok = Check(cudaMemcpyAsync(table->deviceOctaves, octaves.data(), octaves.size() * sizeof(uint2), cudaMemcpyHostToDevice, stream), "H2D", &table->error) &&
         Check(cudaMemcpyAsync(table->deviceBuckets, buckets.data(), buckets.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, stream), "H2D", &table->error) &&
         Check(cudaMalloc(&dCounters, 3 * sizeof(unsigned long long)), "cudaMalloc", &table->error);
    if (!ok)
    {
        FreeCurveTable(table);
        return false;
    }

    // ---- pass 2: verify every input ---------------------------------------------------------------------------
    cudaMemsetAsync(dCounters, 0, 3 * sizeof(unsigned long long), stream);
    if (curve == kCurveLinearToPQ)
    {
        VerifyKernel<kCurveLinearToPQ><<<grid, kSweepThreads, 0, stream>>>(pqMultiplier, maxCodeFloat, table->view, dCounters);
    }
    else if (curve == kCurveLinearToSMPTE428)
    {
        VerifyKernel<kCurveLinearToSMPTE428><<<grid, kSweepThreads, 0, stream>>>(pqMultiplier, maxCodeFloat, table->view, dCounters);
    }
    else
    {
        VerifyKernel<kCurveLinearToHLG><<<grid, kSweepThreads, 0, stream>>>(pqMultiplier, maxCodeFloat, table->view, dCounters);
    }
    unsigned long long counters[3] = { 0, 0, 0 };
    ok = Check(cudaMemcpyAsync(counters, dCounters, sizeof(counters), cudaMemcpyDeviceToHost, stream), "D2H", &table->error) &&
         Check(cudaStreamSynchronize(stream), "curve verify", &table->error);
    cudaFree(dCounters);
    if (!ok)
    {
        FreeCurveTable(table);
        return false;
    }
    table->stats.verifyMismatches = counters[0];
    table->stats.inBandInputs = counters[1];
    table->stats.compactInBandInputs = counters[2];
    table->stats.buildMilliseconds = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (counters[0] != 0)
    {
        table->error = "curve table: verification found inputs where the table disagrees with the exact curve";
        FreeCurveTable(table);
        return false;
    }
    table->valid = true;
    return true;
}

} // namespace avifgpu
