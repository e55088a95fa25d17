// curve_tables.h -- exact float -> code tables for the encode-side transfer curves.
//
// The headline conversion quantises code = trunc(clamp(OETF(x) * max)) with OETF = LinearToPQ (two powf) or
// LinearToSMPTE428 (one powf) -- ColorTransfer.cpp:69-92,119-127, WriteHeifImage.cpp:1093-1130.  Evaluating the
// glibc-exact powf for every sample costs ~110 issue slots per channel and caps the kernel at ~30 % of the HBM
// roofline.  But the OUTPUT is one of 2^depth codes, and as a function of the input float the code is a step
// function: outside narrow "fuzzy bands" around each step (where libm rounding noise makes the reference's own
// result non-monotone, SURVEY.md 7.3) the code is decided by comparing the input with a threshold.  So:
//
//   * a sweep kernel evaluates the EXACT curve (the same device functions the generic kernel uses) for every
//     non-negative finite float (2^31 - 2^23 inputs) and records, per code c, the
//     smallest and largest input that produced it;
//   * the host turns that into thresholds first_k = min{x : code >= k}, band ends last_k = max{x : code < k} and
//     a two-level table: per binade (octave) a bucket size 2^S chosen so that no bucket meets two steps, per
//     bucket one 32-bit word {k-1, offset of the band start};
//   * the conversion kernel does two shared-memory look-ups and a handful of integer instructions per sample;
//     samples that fall inside a (conservatively widened) band are handed to the exact evaluation (rare for the
//     curves that need this form: a single powf is monotone, so only the quantisation of the table itself widens);
//   * the compact variant (one bucket size for all binades, one 32-bit word per bucket, PQ) goes one step further:
//     inside the band of step k the exact code is k-1 or k (neighbouring bands never overlap, the builder checks), so
//     ONE BIT per in-band float records the exact answer.  A fill kernel evaluates the exact curve for every in-band
//     float (a few million) into a bitmap that lives in L2 (up to 2 MB for 12 bits); the conversion kernel resolves an
//     in-band sample with one 32-bit load instead of ~150 instructions of glibc-exact powf;
//   * a verification kernel then re-sweeps every float through both forms and checks table (+ bitmap) == exact; a
//     table that fails (it never has) is discarded and the generic kernel keeps serving that configuration.
//
// Nothing here approximates: every output is either decided by a threshold derived from the exact curve, read from
// a bit the exact curve wrote, or is the exact curve itself.
#ifndef AVIF_CURVE_TABLES_H
#define AVIF_CURVE_TABLES_H

#include <stdint.h>

#include <string>

#include <vector_types.h>

namespace avifgpu
{

enum CurveId
{
    kCurveLinearToPQ = 0,
    kCurveLinearToSMPTE428 = 1,
    kCurveLinearToHLG = 2 // the HLG save extension (ColorTransfer.cpp:141-164); served by the generic kernels only
};

constexpr uint32_t kBucketOffsetBits = 20;          // low bits of a bucket word: quantised band-start offset
constexpr uint32_t kBucketOffsetNone = 1u << 19;    // "no step in this bucket": every offset compares below it
constexpr uint32_t kOffsetResolutionBits = 19;      // offsets inside a bucket are kept to 19 bits

// Compact (single-level) variant, used when one bucket size separates the steps of every binade (true for PQ):
// buckets of 2^flatShift floats covering bit patterns [flatLow << flatShift, (flatHigh + 1) << flatShift); inputs
// outside are clamped to the end buckets, which hold no step.  flatShift is the largest shift up to kFlatMaxShift that
// separates the steps, capped at 32 - depth - kCompactLenBits so that an entry fits one word (a shift that separates
// the steps separates them at every smaller shift too).  The entries are at most kFlatMaxBytes.
constexpr uint32_t kFlatMaxShift = 16;
constexpr uint32_t kFlatMaxBytes = 132 * 1024;
constexpr uint64_t kBandBitmapMaxBytes = 8ull << 20;

// Device-resident table (global memory; kernels stage it into shared memory).
struct CurveTableView
{
    const uint2* octaves;     // 256 entries: .x = first bucket index, .y = S | r << 8 | wq << 16
    const uint32_t* buckets;  // bucketCount words: (k-1) << 20 | offset
    // flatCount / flatShift and flatLow / flatHigh are 8-byte aligned pairs: a kernel reads each pair with one load.
    int32_t flatCount;        // compact entries
    uint32_t flatShift;
    uint32_t flatLow;         // bucket number (bits >> flatShift) of compact[0]
    uint32_t flatHigh;        // bucket number of compact[flatCount - 1]
    int32_t bucketCount;
    const uint32_t* bandBits; // (maxCode + 1) << bandStrideLog2 bits: the exact answer for every in-band float
    uint32_t bandStrideLog2;  // bits reserved per step (power of two >= the widest band plus two in-band units)
    // The compact variant, one 32-bit word per bucket, or nullptr when it does not apply.  See "Compact entries" below.
    const uint32_t* compact;
    const uint32_t* firstBits; // first_k for k = 0 .. maxCode + 1 (0 for codes that no input reaches)
    // compact and firstBits are one device allocation, the shared-memory image of the kernels that use them:
    // [flatCount words, padded to a multiple of 4][maxCode + 2 words, padded to a multiple of 4] -- so one thread can
    // hand the whole table to the copy engine (cp.async.bulk wants 16-byte multiples).  firstBits == compact + (padded count).
    uint32_t compactImageBytes;
    uint32_t compactCodeMask;  // ((1 << depth) - 1) << 6
    uint32_t compactMagic;     // 0x4b000000 (the bits of 2^23), carried as data: see LookupCurveCompact
};

// Compact entries.  A random 64-bit gather from shared memory costs ~5.2 data-pipe wavefronts (two half-warp phases of
// 16 random bank pairs), a 32-bit one ~3.5, and the config-2 kernel is bound by exactly that pipe -- so a bucket is one
// word, S = flatShift, D = depth (S + D + 6 <= 32):
//     bits 31 .. 32-S   step bucket: 2^S - off, off = first_k - bucketStart in (0, 2^S);  otherwise 0
//     bits D+5 .. 6     step bucket: k - 1;  otherwise the code of every float of the bucket (before band corrections)
//     bits 5 .. 0       lenq: the in-band floats of the bucket are those less than lenq * 2^(S-6) above the band start
//                       (band start = first_k for a step bucket, the bucket start for the tail of a band that began in
//                       the previous bucket or for a step sitting exactly on the bucket start)
// With t = entry + (bits << (32 - S)): the carry out of bit 31 says bits >= first_k, so code = field + carry, and the top
// S bits of t are the distance from the band start, so in band <=> t < (entry << 26) -- the band length in units of
// 2^(S-6) floats (256 for S = 14) is what makes that a shift and ONE compare.  The test is a superset: a sample below
// first_k whose wrapped distance happens to be small is flagged too, and lenq rounds the band up to the unit; the band
// bitmap (indexed by k and bits - first_k, filled over its whole stride) gives the exact code for every flagged sample,
// and ResolveCompactInBand leaves the ones flagged by the superset alone.
constexpr uint32_t kCompactLenBits = 6;

struct CurveTableStats
{
    double buildMilliseconds = 0.0;
    uint64_t sweptInputs = 0;
    uint64_t inBandInputs = 0;     // inputs the kernel sends to the exact path (two-level table)
    uint64_t bandBitmapBytes = 0;  // size of the compact variant's band bitmap
    uint64_t compactInBandInputs = 0; // compact variant: inputs flagged in band, resolved through the band bitmap
    int32_t compactBuckets = 0;    // 0 when the compact variant does not apply
    uint64_t verifyMismatches = 0; // must be 0
    int32_t steps = 0;             // thresholds found
    int32_t bands = 0;             // thresholds with a non-empty fuzzy band
    uint32_t widestBand = 0;       // in ulps
};

struct CurveTable
{
    int32_t curve = 0;
    int32_t param = 0; // PQ: peak nits
    int32_t depth = 0;
    bool valid = false;
    CurveTableView view{};
    CurveTableStats stats;
    std::string error;
    void* deviceOctaves = nullptr;
    void* deviceBuckets = nullptr;
    void* deviceBandBits = nullptr;
    void* deviceCompact = nullptr;
    void* deviceFirstBits = nullptr;
};

// Builds (sweeps, assembles, uploads, verifies) the table on the current device.  Synchronous; uses `stream`.
// Returns true when the table is valid.  On failure table->error says why and the caller must not use it.
bool BuildCurveTable(int curve, int param, int depth, void* stream, CurveTable* table);
void FreeCurveTable(CurveTable* table);

} // namespace avifgpu

#endif
