// tests/native/launch_route_check.cpp -- host-side check of the direct-call route (EncodeFamilyOf / DecodeFamilyOf,
// host_params.cpp, then EncodeBlockInterior / DecodeBlockInterior, kernel_params.h) against an independent statement of
// the decision chain it replaced: the tuned launchers tried in turn, each checking its description and then its block and
// declining the call when either fails, the generic kernel taking whatever none of them takes.
//
// Over every description ValidateEncodeDesc / ValidateDecodeDesc accepts (host depths, channels, alpha states, depths,
// curves, layouts, chroma, destination / source layouts, Gray16 curves, HLG extensions, the row matrix, nclx matrices and
// ranges), context states (no step table, two-level only, compact with and without its bitmap, compact too large for each
// kernel, two-level too large, Gray16 LUT present or absent, verified shortcuts 0 or 1) and blocks (aligned; rows, each
// plane or a stride misaligned; unequal chroma strides; widths 1 / 3 / 7 / 8 / 9 / 130; one row; an odd 4:2:0 first row),
// the route must give the same family and the same interior as the chain.  For the batched families it must also give
// the same interior in the per-image plan (PlanBatchEncodeImage / PlanBatchDecodeImage) of the same block.
// Prints "encode descriptions=N calls=K tuned=T" and "decode ..."; exit code 1 on the first failure.
#include "batch_plan.h"
#include "host_params.h"

#include <cstdio>
#include <cstdlib>
#include <type_traits>
#include <vector>

using namespace avifgpu;

namespace
{

const Interior kNone = { 0, 0 };

// ---- the chain: block rules -----------------------------------------------------------------------------------------

bool At(const void* p, int64_t stride, int alignment) { return (reinterpret_cast<uintptr_t>(p) % alignment) == 0 && (stride % alignment) == 0; }
bool Pairs(int layout) { return (layout & AVIFGPU_SOURCE_CHROMA_INTERLEAVED) != 0; }

Interior ChainRgbIntBlock(const EncodeParams& p, int hostDepth)
{
    const int planeBytes = p.imageDepth > 8 ? 2 : 1;
    const int rowAlign = (8 * p.channels * (hostDepth / 8)) % 16 == 0 ? 16 : 8;
    const int chromaAlign = (p.xs ? 4 : 8) * planeBytes;
    const bool chroma = Pairs(p.destLayout) ? At(p.plane[1], p.planeStride[1], 2 * chromaAlign > 16 ? 16 : 2 * chromaAlign)
                                            : At(p.plane[1], p.planeStride[1], chromaAlign) && At(p.plane[2], p.planeStride[2], chromaAlign);
    if (p.width < 8 || !At(p.rows, p.rowStride, rowAlign) || !At(p.plane[0], p.planeStride[0], 8 * planeBytes) || !chroma ||
        (p.channels == 4 && !At(p.plane[3], p.planeStride[3], 8 * planeBytes)))
        return kNone;
    const int rows = p.ys ? (p.rowCount & ~1) : p.rowCount;
    return rows < 1 ? kNone : Interior{ p.width & ~7, rows };
}

Interior ChainRgbF32Block(const EncodeParams& p)
{
    const int chromaAlign = p.xs ? 4 : 8;
    const bool chroma = Pairs(p.destLayout) ? At(p.plane[1], p.planeStride[1], 2 * chromaAlign)
                                            : At(p.plane[1], p.planeStride[1], chromaAlign) && At(p.plane[2], p.planeStride[2], chromaAlign);
    if (!At(p.rows, p.rowStride, 16) || !At(p.plane[0], p.planeStride[0], 8) || !chroma || (p.channels == 4 && p.hasAlpha && !At(p.plane[3], p.planeStride[3], 8)))
        return kNone;
    const int rows = p.ys ? (p.rowCount & ~1) : p.rowCount;
    return (p.width & ~3) < 4 || rows < 1 ? kNone : Interior{ p.width & ~3, rows };
}

// The step-table fits, with the kernels' shared-memory layouts written out: 227 KiB per CTA; the flat kernel's libm
// tables, barriers and 28 warps' two-row staging; the RGBA kernel's libm tables, barrier and 16 warps' 28 words per lane.
const size_t kLimit = 227 * 1024;
const size_t kFlatFixed = 768 + 256 + 28 * 2 * 128 * 12;
const size_t kRgbaFixed = 768 + 16 + 16 * 32 * 28 * 4;
bool ChainCompactFits(const CurveTableView& t) { return t.compact && t.firstBits && t.bandBits && kFlatFixed + t.compactImageBytes <= kLimit; }
bool ChainTwoLevelFits(const CurveTableView& t) { return t.buckets && t.octaves && kFlatFixed + 2048 + static_cast<size_t>(t.bucketCount) * 4 <= kLimit; }

// ---- the chain: the encode launchers in their order ------------------------------------------------------------------

bool ChainEncodeFloatRgb(const EncodeParams& p, int hostDepth, EncodeFamily* f, Interior* in)
{
    const bool rgba = p.channels == 4 && p.hasAlpha;
    if (p.rowMatrixEnabled) return false;
    if (hostDepth == 32 && !p.planar && p.channels == 3 && !p.hasAlpha && p.imageDepth > 8 && !p.hlgInverseOotf &&
        (p.transfer == AVIFGPU_TRANSFER_PQ || p.transfer == AVIFGPU_TRANSFER_SMPTE428) && p.curveTable && p.curveTable->buckets)
    {
        const int width4 = p.width & ~3;
        if (width4 < 4 || p.rowCount < 1 || !At(p.rows, p.rowStride, 16) || !At(p.plane[0], p.planeStride[0], 8)) return false;
        if (!ChainCompactFits(*p.curveTable) && !ChainTwoLevelFits(*p.curveTable)) return false;
        *f = EncodeFamily::RgbF32Interleaved;
        *in = Interior{ width4, p.rowCount };
        return true;
    }
    if (hostDepth != 32 || !p.planar || (p.channels != 3 && !rgba) || (p.channels == 3 && p.hasAlpha) || p.imageDepth <= 8) return false;
    const bool pq = p.transfer == AVIFGPU_TRANSFER_PQ;
    const bool clip = p.transfer == AVIFGPU_TRANSFER_CLIP;
    if (!pq && !clip && p.transfer != AVIFGPU_TRANSFER_SMPTE428) return false;
    if (!clip && (!p.curveTable || !p.curveTable->buckets)) return false;
    if (!ForwardMatrixStaysInRange(p.matrix, p.chromaOffset, static_cast<int>(p.maxCode))) return false;
    if (rgba && (clip || !p.curveTable->compact || !p.curveTable->bandBits)) return false;
    const Interior inner = ChainRgbF32Block(p);
    if (inner.width == 0) return false;
    if (rgba)
    {
        const CurveTableView& t = *p.curveTable;
        if (!p.plane[3] || !t.compact || !t.firstBits || !t.bandBits || kRgbaFixed + t.compactImageBytes > kLimit) return false;
        *f = EncodeFamily::RgbaF32Flat;
    }
    else if (!clip)
    {
        const CurveTableView& t = *p.curveTable;
        if (!(ChainCompactFits(t) || ChainTwoLevelFits(t)) || !(p.destLayout == AVIFGPU_SOURCE_PLANAR || !pq || ChainCompactFits(t))) return false;
        *f = EncodeFamily::RgbF32Flat;
    }
    else
    {
        *f = EncodeFamily::RgbF32Clip;
    }
    *in = inner;
    return true;
}

bool ChainEncodeInteger(const EncodeParams& p, int hostDepth, EncodeFamily* f, Interior* in)
{
    if (hostDepth != 16 && hostDepth != 8) return false;
    if (hostDepth == 16 && p.imageDepth > 8 && p.channels == 1 && !p.planar)
    {
        if (!p.gray16Lut || p.width < 8 || !At(p.rows, p.rowStride, 16) || !At(p.plane[0], p.planeStride[0], 16)) return false;
        *f = EncodeFamily::Gray16Lut;
        *in = Interior{ p.width / 8 * 8, p.rowCount };
        return true;
    }
    if (!p.planar && (p.channels == 1 || p.channels == 2) && !p.premultiply && !p.gray16Smpte428 && p.imageDepth <= 12)
    {
        const int planeBytes = p.imageDepth > 8 ? 2 : 1;
        const int rowAlign = (8 * p.channels * (hostDepth / 8)) % 16 == 0 ? 16 : 8;
        if (p.width < 8 || p.rowCount < 1 || !At(p.rows, p.rowStride, rowAlign) || !At(p.plane[0], p.planeStride[0], 8 * planeBytes) ||
            (p.channels == 2 && !At(p.plane[3], p.planeStride[3], 8 * planeBytes)))
            return false;
        *f = EncodeFamily::GrayInt;
        *in = Interior{ p.width & ~7, p.rowCount };
        return true;
    }
    const avifpix::ForwardMatrix& m = p.matrix;
    if (!p.planar || (p.channels != 3 && p.channels != 4) || (p.premultiply && !(p.channels == 4 && p.verifiedPremultiply)) || p.imageDepth > 12 ||
        !(m.identity || (m.kr >= 0.0f && m.kg >= 0.0f && m.kb >= 0.0f && m.kr < 1.0f && m.kb < 1.0f)) ||
        !ForwardMatrixStaysInRange(m, p.chromaOffset, static_cast<int>(p.maxCode)))
        return false;
    *in = ChainRgbIntBlock(p, hostDepth);
    *f = EncodeFamily::RgbInt;
    return in->width > 0;
}

bool ChainEncodeGrayFloat(const EncodeParams& p, int hostDepth, EncodeFamily* f, Interior* in)
{
    if (hostDepth != 32 || p.planar || p.channels > 2 || p.imageDepth <= 8 || p.hlgInverseOotf || p.rowMatrixEnabled) return false;
    const bool pq = p.transfer == AVIFGPU_TRANSFER_PQ;
    if (!pq && p.transfer != AVIFGPU_TRANSFER_CLIP) return false;
    if (pq && (!p.curveTable || !p.curveTable->compact || !p.curveTable->firstBits || !p.curveTable->bandBits)) return false;
    const int width4 = p.width & ~3;
    if (width4 < 4 || p.rowCount < 1 || !At(p.rows, p.rowStride, 16) || !At(p.plane[0], p.planeStride[0], 8) || (p.channels == 2 && !At(p.plane[3], p.planeStride[3], 8)))
        return false;
    if (pq && 768 + 16 + static_cast<size_t>(p.curveTable->compactImageBytes) > 100 * 1024) return false;
    *f = EncodeFamily::GrayF32;
    *in = Interior{ width4, p.rowCount };
    return true;
}

void ChainEncode(const EncodeParams& p, int hostDepth, EncodeFamily* f, Interior* in)
{
    if (ChainEncodeFloatRgb(p, hostDepth, f, in) || ChainEncodeInteger(p, hostDepth, f, in) || ChainEncodeGrayFloat(p, hostDepth, f, in)) return;
    *f = EncodeFamily::Generic;
    *in = kNone;
}

// ---- the chain: the decode launchers in their order ------------------------------------------------------------------

bool ChainSumsNormal(int bitDepth, const F32DecodeFactors& f, float kg)
{
    const auto moderate = [](float v) { return v >= 1.0f / 65536.0f && v <= 4.0f; };
    return bitDepth <= 12 && moderate(f.rGain) && moderate(f.bGain) && moderate(f.gCr) && moderate(f.gCb) && moderate(kg) &&
           moderate(f.kgReciprocal / 65536.0f * 4.0f);
}

bool ChainDecodeYccFloat(const DecodeParams& p, DecodeFamily* f, Interior* in)
{
    if (p.colorspace != AVIFGPU_COLORSPACE_YCBCR || p.hostDepth != 32 || (p.hasAlpha && p.premultiplied) || p.bitDepth > 12 || p.bitDepth <= 8) return false;
    const bool hlg = p.transfer == AVIFGPU_TRANSFER_HLG;
    if (p.transfer != AVIFGPU_TRANSFER_PQ && !hlg && p.transfer != AVIFGPU_TRANSFER_SMPTE428) return false;
    if (hlg && !p.verifiedHlgDivisions) return false;
    if (hlg && p.applyOotf && !avifmath::PowfStraightLineCovers(p.gammaMinusOne, false)) return false;
    if (hlg && p.applyOotf && !(p.lumaR >= 0.0f && p.lumaG >= 0.0f && p.lumaB >= 0.0f && p.lumaR + p.lumaG + p.lumaB <= 2.5f)) return false;
    if (!hlg && !ChainSumsNormal(p.bitDepth, F32DecodeFactorsOf(p.matrix), p.matrix.kg)) return false;
    const int chromaAlign = p.xs ? 4 : 8;
    const bool pairs = Pairs(p.sourceLayout);
    const bool chroma = pairs ? At(p.plane[1], p.planeStride[1], 2 * chromaAlign) : At(p.plane[1], p.planeStride[1], chromaAlign) && At(p.plane[2], p.planeStride[2], chromaAlign);
    if (p.yPhase != 0 || !At(p.plane[0], p.planeStride[0], 8) || !chroma || !At(p.rows, p.rowStride, 16) || (p.hasAlpha && !At(p.plane[3], p.planeStride[3], 8))) return false;
    if (!pairs && p.planeStride[1] != p.planeStride[2]) return false;
    const int rows = p.ys ? (p.rowCount & ~1) : p.rowCount;
    if ((p.width & ~3) < 4 || rows < 1) return false;
    *f = DecodeFamily::YccF32;
    *in = Interior{ p.width & ~3, rows };
    return true;
}

Interior ChainPlanarRgbBlock(const DecodeParams& p)
{
    const int planeAlign = p.hostDepth == 8 ? 8 : 16;
    const int rowAlign = (8 * (p.hasAlpha ? 4 : 3) * (p.hostDepth / 8)) % 16 == 0 ? 16 : 8;
    for (int c = 0; c < 3; ++c)
        if (!At(p.plane[c], p.planeStride[c], planeAlign)) return kNone;
    if ((p.hasAlpha && !At(p.plane[3], p.planeStride[3], planeAlign)) || !At(p.rows, p.rowStride, rowAlign) || (p.width & ~7) < 8 || p.rowCount < 1) return kNone;
    return Interior{ p.width & ~7, p.rowCount };
}

bool ChainDecodeInteger(const DecodeParams& p, DecodeFamily* f, Interior* in)
{
    if ((p.hostDepth != 8 && p.hostDepth != 16) || p.bitDepth > 12 || (p.hasAlpha && p.premultiplied)) return false;
    const bool narrow = (p.hostDepth == 8) == (p.bitDepth <= 8);
    if (p.colorspace == AVIFGPU_COLORSPACE_MONOCHROME)
    {
        const int sampleBytes = p.hostDepth == 8 ? 1 : 2;
        const int rowAlign = (8 * (p.hasAlpha ? 2 : 1) * sampleBytes) % 16 == 0 ? 16 : 8;
        if (!narrow || !At(p.plane[0], p.planeStride[0], 8 * sampleBytes) || (p.hasAlpha && !At(p.plane[3], p.planeStride[3], 8 * sampleBytes)) ||
            !At(p.rows, p.rowStride, rowAlign) || (p.width & ~7) < 8 || p.rowCount < 1)
            return false;
        *f = DecodeFamily::MonoInt;
        *in = Interior{ p.width & ~7, p.rowCount };
        return true;
    }
    if (p.colorspace == AVIFGPU_COLORSPACE_RGB)
    {
        *f = DecodeFamily::PlanarRgbInt;
        *in = narrow ? ChainPlanarRgbBlock(p) : kNone;
        return in->width > 0;
    }
    if (p.colorspace != AVIFGPU_COLORSPACE_YCBCR || p.yPhase != 0 || !narrow) return false;
    const int sampleBytes = p.hostDepth == 8 ? 1 : 2;
    const int chromaAlign = (p.xs ? 4 : 8) * sampleBytes;
    const int rowAlign = p.hasAlpha ? 16 : 8 * sampleBytes;
    const bool chroma = Pairs(p.sourceLayout) ? At(p.plane[1], p.planeStride[1], 2 * chromaAlign > 16 ? 16 : 2 * chromaAlign)
                                              : At(p.plane[1], p.planeStride[1], chromaAlign) && At(p.plane[2], p.planeStride[2], chromaAlign);
    if (!At(p.plane[0], p.planeStride[0], 8 * sampleBytes) || !chroma || (p.hasAlpha && !At(p.plane[3], p.planeStride[3], 8 * sampleBytes)) ||
        !At(p.rows, p.rowStride, rowAlign))
        return false;
    const int rows = p.ys ? (p.rowCount & ~1) : p.rowCount;
    if ((p.width & ~7) < 8 || rows < 1) return false;
    *f = DecodeFamily::YccInt;
    *in = Interior{ p.width & ~7, rows };
    return true;
}

bool ChainDecodeTable(const DecodeParams& p, DecodeFamily* f, Interior* in)
{
    const bool mono = p.colorspace == AVIFGPU_COLORSPACE_MONOCHROME;
    if (p.hostDepth != 32 || (!mono && p.colorspace != AVIFGPU_COLORSPACE_RGB) || p.bitDepth <= 8 || p.bitDepth > 12) return false;
    if (mono)
    {
        if (p.transfer != AVIFGPU_TRANSFER_PQ || !At(p.plane[0], p.planeStride[0], 16) || (p.hasAlpha && !At(p.plane[3], p.planeStride[3], 16)) ||
            !At(p.rows, p.rowStride, 16) || (p.width & ~7) < 8 || p.rowCount < 1)
            return false;
        *f = DecodeFamily::MonoF32;
        *in = Interior{ p.width & ~7, p.rowCount };
        return true;
    }
    if (p.transfer != AVIFGPU_TRANSFER_PQ && p.transfer != AVIFGPU_TRANSFER_HLG && p.transfer != AVIFGPU_TRANSFER_SMPTE428) return false;
    *f = DecodeFamily::PlanarRgbF32;
    *in = ChainPlanarRgbBlock(p); // premultiplied alpha too
    return in->width > 0;
}

void ChainDecode(const DecodeParams& p, DecodeFamily* f, Interior* in)
{
    if (ChainDecodeYccFloat(p, f, in) || ChainDecodeInteger(p, f, in) || ChainDecodeTable(p, f, in)) return;
    *f = DecodeFamily::Generic;
    *in = kNone;
}

// ---- the grid ---------------------------------------------------------------------------------------------------------

[[noreturn]] void Fail(const char* what, int descriptions, int block)
{
    std::printf("FAIL: %s (description %d, block %d)\n", what, descriptions, block);
    std::exit(1);
}

// A block's buffers: `misalign` picks one defect -- 0 none, 1 / 2 rows by 4 / 8 bytes, 3 the row stride by 4, 4 + 2k / 5 + 2k
// plane k by 2 / 8 bytes, 12 plane k's stride by 4 for k = 0..3 (13..15), 16 Cb and Cr strides unequal but aligned.
struct Block
{
    int width, rows, misalign;
};

std::vector<Block> Blocks()
{
    std::vector<Block> b;
    for (int width : { 1, 3, 7, 8, 9, 130 })
        for (int rows : { 1, 2, 5 }) b.push_back({ width, rows, 0 });
    for (int misalign = 1; misalign <= 16; ++misalign) b.push_back({ 130, 5, misalign });
    return b;
}

template <typename Params>
void PlaceBlock(Params& p, const Block& b, const bool present[4])
{
    p.width = b.width;
    p.rowCount = b.rows;
    p.rows = reinterpret_cast<void*>(static_cast<uintptr_t>(0x1000000 + (b.misalign == 1 ? 4 : b.misalign == 2 ? 8 : 0)));
    p.rowStride = 4096 + (b.misalign == 3 ? 4 : 0);
    for (int k = 0; k < 4; ++k)
    {
        const uintptr_t offset = b.misalign == 4 + 2 * k ? 2 : b.misalign == 5 + 2 * k ? 8 : 0;
        using Plane = typename std::remove_reference<decltype(p.plane[k])>::type;
        p.plane[k] = present[k] ? reinterpret_cast<Plane>(static_cast<uintptr_t>(0x2000000 + 0x1000000 * k) + offset) : nullptr;
        p.planeStride[k] = present[k] ? 2048 + (b.misalign == 12 + k ? 4 : 0) + (b.misalign == 16 && k == 2 ? 256 : 0) : 0;
    }
}

template <typename Params>
avifgpu_batch_image ImageOf(const Params& p)
{
    avifgpu_batch_image image{};
    image.width = p.width;
    image.height = p.rowCount;
    image.rows = const_cast<void*>(static_cast<const void*>(p.rows));
    image.row_stride_bytes = p.rowStride;
    for (int k = 0; k < 4; ++k)
    {
        image.planes.data[k] = const_cast<void*>(static_cast<const void*>(p.plane[k]));
        image.planes.stride[k] = p.planeStride[k];
    }
    return image;
}

// Context states of the step table: none; two-level only; compact with its bitmap (+ two-level); compact without its bitmap;
// compact only (no two-level); compact too large for the gray kernel, for the flat kernel, for the RGBA kernel; two-level too
// large for the flat kernel.
std::vector<CurveTableView> Tables()
{
    static const uint32_t word = 0;
    static const uint2 octave{};
    const auto make = [](bool twoLevel, int bucketCount, bool compact, bool bitmap, uint32_t compactBytes) {
        CurveTableView t{};
        if (twoLevel)
        {
            t.octaves = &octave;
            t.buckets = &word;
            t.bucketCount = bucketCount;
        }
        if (compact)
        {
            t.compact = &word;
            t.firstBits = &word;
            t.compactImageBytes = compactBytes;
        }
        t.bandBits = bitmap ? &word : nullptr;
        return t;
    };
    return { make(true, 4096, false, false, 0),        make(true, 4096, true, true, 60000),  make(true, 4096, true, false, 60000),
             make(false, 0, true, true, 60000),         make(true, 4096, true, true, 120000), make(true, 4096, true, true, 160000),
             make(true, 4096, true, true, 200000),      make(true, 40000, false, true, 0) };
}

} // namespace

int main()
{
    const std::vector<Block> blocks = Blocks();
    const std::vector<CurveTableView> tables = Tables();
    static const uint16_t lut = 0;
    long long calls = 0, tuned = 0;
    int descriptions = 0;

    const avifgpu_nclx nclxs[] = { { 1, 9, 16, 9, 1 }, { 1, 1, 1, 1, 1 }, { 1, 1, 13, 0, 1 }, { 1, 10, 1, 12, 1 }, { 0, 0, 0, 0, 0 } };
    for (int hostDepth : { 8, 16, 32 })
    for (int channels = 1; channels <= 4; ++channels)
    for (int alpha = 0; alpha <= 2; ++alpha)
    for (int depth : { 8, 10, 12 })
    for (int transfer = 0; transfer <= 3; ++transfer)
    for (int layout = 0; layout <= 1; ++layout)
    for (int chroma = 1; chroma <= 3; ++chroma)
    for (int dest = 0; dest <= 3; ++dest)
    for (int gray16 = 0; gray16 <= 1; ++gray16)
    for (int hlg = 0; hlg <= 2; ++hlg)
    for (int rowMatrix = 0; rowMatrix <= 1; ++rowMatrix)
    for (const avifgpu_nclx& nclx : nclxs)
    {
        if ((hostDepth != 32 && (transfer != 0 || hlg != 0 || rowMatrix)) || (hostDepth != 16 && gray16) || (layout == 0 && (chroma != 1 || dest != 0)))
            continue; // fields the description ignores there
        avifgpu_encode_desc d{};
        d.struct_size = sizeof(d);
        d.width = 130;
        d.height = 5;
        d.host_depth = hostDepth;
        d.host_channels = channels;
        d.alpha_state = alpha;
        d.image_bit_depth = depth;
        d.transfer = transfer;
        d.pq_peak_nits = 10000;
        d.layout = layout;
        d.chroma = chroma;
        d.gray16_curve = gray16;
        d.nclx = nclx;
        d.hlg_extension = hlg;
        d.hlg_display_gamma = 1.2f;
        d.hlg_peak_nits = 1000;
        d.row_matrix_enabled = rowMatrix;
        d.row_matrix[0] = d.row_matrix[4] = d.row_matrix[8] = 1.0f;
        d.dest_layout = dest;
        if (ValidateEncodeDesc(&d, nullptr) != AVIFGPU_OK) continue;
        ++descriptions;
        EncodeParams base;
        FillEncodeParams(d, &base);
        bool present[4];
        int planeMask = 0;
        for (int k = 0; k < 4; ++k)
        {
            present[k] = EncodePlaneGeometry(d, k).present;
            planeMask |= present[k] ? 1 << k : 0;
        }
        for (int table = -1; table < static_cast<int>(tables.size()); ++table)
        for (int withLut = 0; withLut <= 1; ++withLut)
        for (int verified = 0; verified <= 1; ++verified)
        {
            EncodeParams shared = base;
            shared.curveTable = table < 0 ? nullptr : &tables[table];
            shared.gray16Lut = withLut ? &lut : nullptr;
            shared.verifiedPremultiply = verified;
            const EncodeFamily family = EncodeFamilyOf(shared, hostDepth);
            const EncodeFamily batchFamily = EncodeBatchFamilyOf(shared, hostDepth);
            for (size_t b = 0; b < blocks.size(); ++b)
            {
                EncodeParams p = shared;
                PlaceBlock(p, blocks[b], present);
                EncodeFamily expected;
                Interior expectedInner;
                ChainEncode(p, hostDepth, &expected, &expectedInner);
                const Interior inner = EncodeBlockInterior(family, p, hostDepth);
                const EncodeFamily got = inner.width > 0 ? family : EncodeFamily::Generic;
                if (got != expected || inner.width != expectedInner.width || (inner.width > 0 && inner.rows != expectedInner.rows))
                {
                    std::printf("encode: family %d interior %d x %d, the chain %d, %d x %d\n", static_cast<int>(got), inner.width, inner.rows,
                                static_cast<int>(expected), expectedInner.width, expectedInner.rows);
                    Fail("encode route", descriptions, static_cast<int>(b));
                }
                const BatchImagePlan plan = PlanBatchEncodeImage(shared, hostDepth, batchFamily, planeMask, ImageOf(p));
                const bool batched = expected == EncodeFamily::RgbInt;
                if (plan.status != AVIFGPU_OK || plan.interior.width != (batched ? expectedInner.width : 0) ||
                    (batched && plan.interior.rowCount != expectedInner.rows))
                    Fail("encode plan interior", descriptions, static_cast<int>(b));
                ++calls;
                tuned += got != EncodeFamily::Generic;
            }
        }
    }
    std::printf("encode descriptions=%d calls=%lld tuned=%lld\n", descriptions, calls, tuned);

    descriptions = 0;
    calls = tuned = 0;
    const avifgpu_nclx decodeNclx[] = { { 1, 9, 16, 9, 1 }, { 1, 9, 18, 9, 0 }, { 1, 1, 17, 1, 1 }, { 1, 9, 1, 9, 1 }, { 1, 1, 16, 0, 1 },
                                        { 1, 22, 18, 12, 1 }, { 0, 0, 0, 0, 0 } };
    for (int hostDepth : { 8, 16, 32 })
    for (int colorspace = 0; colorspace <= 2; ++colorspace)
    for (int chroma = 1; chroma <= 3; ++chroma)
    for (int bitDepth : { 8, 10, 12, 16 })
    for (int alpha = 0; alpha <= 2; ++alpha)
    for (int source = 0; source <= 3; ++source)
    for (int ootf = 0; ootf <= 1; ++ootf)
    for (float gamma : { 1.2f, 9.0f })
    for (const avifgpu_nclx& nclx : decodeNclx)
    {
        if ((colorspace != AVIFGPU_COLORSPACE_YCBCR && (chroma != 1 || source != 0)) || (hostDepth != 32 && (ootf || gamma != 1.2f)))
            continue;
        avifgpu_decode_desc d{};
        d.struct_size = sizeof(d);
        d.width = 130;
        d.height = 5;
        d.colorspace = colorspace;
        d.chroma = chroma;
        d.bit_depth = bitDepth;
        d.alpha_state = alpha;
        d.host_depth = hostDepth;
        d.nclx = nclx;
        d.hlg_apply_ootf = ootf;
        d.hlg_display_gamma = gamma;
        d.hlg_peak_nits = 1000;
        d.pq_peak_nits = 10000;
        d.source_layout = source;
        int32_t transfer;
        DecodeParams base;
        if (ValidateDecodeDesc(&d, &transfer, nullptr) != AVIFGPU_OK || !FillDecodeParams(d, transfer, &base, nullptr)) continue;
        ++descriptions;
        bool present[4];
        int planeMask = 0;
        for (int k = 0; k < 4; ++k)
        {
            present[k] = DecodePlaneGeometry(d, k).present;
            planeMask |= present[k] ? 1 << k : 0;
        }
        for (int verified = 0; verified < 8; ++verified)
        {
            DecodeParams shared = base;
            shared.verifiedHlgDivisions = verified & 1;
            shared.verifiedGreenDivision = (verified >> 1) & 1;
            shared.verifiedPqRatio = (verified >> 2) & 1;
            const DecodeFamily family = DecodeFamilyOf(shared);
            const DecodeFamily batchFamily = DecodeBatchFamilyOf(shared);
            for (size_t b = 0; b < blocks.size(); ++b)
            for (int phase = 0; phase <= shared.ys; ++phase)
            {
                DecodeParams p = shared;
                PlaceBlock(p, blocks[b], present);
                p.yPhase = phase;
                DecodeFamily expected;
                Interior expectedInner;
                ChainDecode(p, &expected, &expectedInner);
                const Interior inner = DecodeBlockInterior(family, p);
                const DecodeFamily got = inner.width > 0 ? family : DecodeFamily::Generic;
                if (got != expected || inner.width != expectedInner.width || (inner.width > 0 && inner.rows != expectedInner.rows))
                {
                    std::printf("decode: family %d interior %d x %d, the chain %d, %d x %d\n", static_cast<int>(got), inner.width, inner.rows,
                                static_cast<int>(expected), expectedInner.width, expectedInner.rows);
                    Fail("decode route", descriptions, static_cast<int>(b));
                }
                if (phase == 0)
                {
                    const BatchImagePlan plan = PlanBatchDecodeImage(shared, batchFamily, planeMask, ImageOf(p));
                    const bool batched = (expected == DecodeFamily::YccF32 || expected == DecodeFamily::YccInt || expected == DecodeFamily::PlanarRgbInt ||
                                          expected == DecodeFamily::PlanarRgbF32) && !(p.hasAlpha && p.premultiplied);
                    if (plan.status != AVIFGPU_OK || plan.interior.width != (batched ? expectedInner.width : 0) ||
                        (batched && plan.interior.rowCount != expectedInner.rows))
                        Fail("decode plan interior", descriptions, static_cast<int>(b));
                }
                ++calls;
                tuned += got != DecodeFamily::Generic;
            }
        }
    }
    std::printf("decode descriptions=%d calls=%lld tuned=%lld\n", descriptions, calls, tuned);
    return 0;
}
