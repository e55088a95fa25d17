// tests/native/batch_plan_check.cpp -- the batch planning of both batch APIs (csrc/batch_plan.h, csrc/host_params.cpp) on
// the CPU, slice by slice.  Every description of a slice runs seeded batches through the three checks of plan_harness.h
// (the per-image step, its layout and FindRecord, the host-described plan); a slice adds the statements that only hold
// for its descriptions, each restated independently of the library:
//   encode        every valid encode description (both layouts; integer and float hosts), verified premultiply off and on;
//                 a chunk's kernel parameters fit the 32764-byte limit;
//   encode_dest   8/16-bit RGB(A) into planar YCbCr in every destination layout (avifgpu_encode_desc.dest_layout):
//                 validation of every layout bit set, the API-10-sized description against an inaccessible page, plane
//                 geometry and EncodeWindow, the block halves against the stores' alignment, routing independent of the
//                 layout, the plane mask, and the interleaved plane's alignment on every image;
//   decode_int    YCbCr into 8/16-bit hosts;
//   decode_f32    YCbCr into 32-bit hosts (PQ, HLG with and without the OOTF, SMPTE 428), verified divisions off and on:
//                 which descriptions the float family takes;
//   decode_rgb    planar RGB into 8/16/32-bit hosts: which descriptions its families take, their unit width, and every
//                 image's interior against the kernels' alignment; YCbCr and monochrome descriptions route as they did;
//   decode_source YCbCr in every source layout (avifgpu_decode_desc.source_layout): validation of every layout bit set,
//                 the API-9-sized description against an inaccessible page, plane geometry, routing, the plane mask, and
//                 the interleaved plane's alignment on every image;
//   indirect      the workspace of the device-described batch, then planar encodes and YCbCr decodes into 8/16-bit hosts.
// Prints one line per slice, "<slice> descriptions=N images=K units=U" and the slice's own counters; exit code 1 on any
// failure.
#include "plan_harness.h"

#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

using namespace avifgpu;

namespace
{

avifgpu_encode_desc EncodeDesc(int hostDepth, int channels, int alphaState, int imageDepth, int layout, int chroma, int dest)
{
    avifgpu_encode_desc d{};
    d.struct_size = sizeof(d);
    d.width = 64;
    d.height = 8;
    d.host_depth = hostDepth;
    d.host_channels = channels;
    d.alpha_state = alphaState;
    d.image_bit_depth = imageDepth;
    d.transfer = AVIFGPU_TRANSFER_PQ;
    d.pq_peak_nits = 10000;
    d.layout = layout;
    d.chroma = chroma;
    d.nclx = avifgpu_nclx{ 1, 9, 16, 9, 1 };
    d.hlg_display_gamma = 1.2f;
    d.hlg_peak_nits = 1000;
    d.dest_layout = dest;
    return d;
}

avifgpu_decode_desc DecodeDesc(int colorspace, int chroma, int bitDepth, int alpha, int hostDepth, int layout, int transferCharacteristics)
{
    avifgpu_decode_desc d{};
    d.struct_size = sizeof(d);
    d.width = 64;
    d.height = 8;
    d.colorspace = colorspace;
    d.chroma = chroma;
    d.bit_depth = bitDepth;
    d.alpha_state = alpha;
    d.host_depth = hostDepth;
    d.nclx = avifgpu_nclx{ 1, 9, transferCharacteristics, 9, 1 };
    d.hlg_apply_ootf = 1;
    d.hlg_display_gamma = 1.2f;
    d.hlg_peak_nits = 1000;
    d.pq_peak_nits = 1000;
    d.source_layout = layout;
    return d;
}

int AlphaFor(int channels) { return (channels == 2 || channels == 4) ? AVIFGPU_ALPHA_STRAIGHT : AVIFGPU_ALPHA_NONE; }

bool IsPlanarRgb(DecodeFamily family) { return family == DecodeFamily::PlanarRgbInt || family == DecodeFamily::PlanarRgbF32; }

// The interleaved plane's alignment, restated (PairAlignment), against the route of every accepted image of a batch: a
// misaligned plane never takes the tuned family, the generator's misaligned ones have no interior, and (for a description
// the tuned family takes) an aligned image of at least 8 x 2 pixels keeps its interior.
template <typename Params>
void CheckInterleavedRoute(const Case<Params>& c, const std::vector<FakeImage<Params>>& images, bool tuned, int batch)
{
    for (const FakeImage<Params>& im : images)
    {
        const Params& p = im.p;
        if (im.rejected || !Interleaved(p))
        {
            continue;
        }
        const Interior inner = RouteInterior(p, c.hostDepth);
        if (inner.width > 0 && !Aligned(p.plane[1], p.planeStride[1], PairAlignment(p)))
        {
            Fail("a misaligned interleaved plane took the tuned route", c.index, batch);
        }
        if ((im.shape == kPairPointer || im.shape == kPairStride) && inner.width > 0)
        {
            Fail("a misaligned interleaved plane has an interior", c.index, batch);
        }
        if (tuned && im.shape == kAligned && p.width >= 8 && p.rowCount >= 2 && inner.width == 0)
        {
            Fail("an aligned interleaved image lost its interior", c.index, batch);
        }
    }
}

// ---- encode ----

void EncodeSlice()
{
    static_assert(sizeof(EncodeParams) + 16 + 2 * kBatchChunkImages * sizeof(BatchRecord) <= 32764, "edge parameters");
    std::mt19937_64 rng(1234);
    Counts n;
    int batch = 0;
    for (int hostDepth : { 8, 16, 32 })
        for (int channels = 1; channels <= 4; ++channels)
            for (int alpha : { 0, 1, 2 })
                for (int depth : { 8, 10, 12 })
                    for (int layout : { 0, 1 })
                        for (int chroma : { 1, 2, 3 })
                            for (int matrix : { 1, 0, 9 })
                            {
                                avifgpu_encode_desc d{};
                                d.struct_size = sizeof(d);
                                d.width = 16;
                                d.height = 16;
                                d.host_depth = hostDepth;
                                d.host_channels = channels;
                                d.alpha_state = alpha;
                                d.image_bit_depth = depth;
                                d.transfer = AVIFGPU_TRANSFER_CLIP;
                                d.pq_peak_nits = 80;
                                d.layout = layout;
                                d.chroma = chroma;
                                d.nclx = avifgpu_nclx{ 1, 1, 13, matrix, 1 };
                                if ((layout == 0 && (chroma != 3 || matrix != 1)) || ValidateEncodeDesc(&d, nullptr) != AVIFGPU_OK)
                                {
                                    continue;
                                }
                                ++n.descriptions;
                                for (int verified : { 0, 1 })
                                {
                                    EncodeParams shared;
                                    FillEncodeParams(d, &shared);
                                    shared.verifiedPremultiply = verified;
                                    const Case<EncodeParams> c = CaseOf(d, shared, n.descriptions);
                                    for (int trial = 0; trial < 3; ++trial)
                                    {
                                        CheckBatch(rng, d, c, trial == 2 ? 300 : 20, batch++, n);
                                    }
                                }
                            }
    std::printf("encode descriptions=%d images=%lld units=%lld batches=%d\n", n.descriptions, n.images, n.units, batch);
}

// ---- encode_dest ----

int EncodeDestValidations()
{
    int checked = 0;
    for (int dest : { 0, 1, 2, 3, 4, 5, 8, -1 })
        for (int hostDepth : { 8, 16, 32 })
            for (int channels : { 1, 2, 3, 4 })
                for (int layout : { AVIFGPU_LAYOUT_REFERENCE, AVIFGPU_LAYOUT_PLANAR_YCBCR })
                    for (int imageDepth : { 8, 10, 12 })
                    {
                        avifgpu_encode_desc d = EncodeDesc(hostDepth, channels, AlphaFor(channels), imageDepth, layout, AVIFGPU_CHROMA_420, 0);
                        const int base = ValidateEncodeDesc(&d, nullptr);
                        d.dest_layout = dest;
                        const int status = ValidateEncodeDesc(&d, nullptr);
                        int expected = base;
                        if (base == AVIFGPU_OK && dest != 0)
                        {
                            if (dest & ~3)
                            {
                                expected = AVIFGPU_ERR_BAD_PARAM;
                            }
                            else if (layout != AVIFGPU_LAYOUT_PLANAR_YCBCR)
                            {
                                expected = AVIFGPU_ERR_UNSUPPORTED;
                            }
                            else if ((dest & AVIFGPU_SOURCE_MSB_ALIGNED) && imageDepth == 8)
                            {
                                expected = AVIFGPU_ERR_BAD_PARAM;
                            }
                        }
                        if (status != expected)
                        {
                            std::printf("FAIL validation dest %d host %d channels %d layout %d depth %d: %d, expected %d\n", dest, hostDepth, channels, layout,
                                        imageDepth, status, expected);
                            ++g_failures;
                        }
                        ++checked;
                    }

    // An API-10-sized description as the last bytes before an inaccessible page: whatever would lie past it cannot be read.
    const avifgpu_encode_desc current = EncodeDesc(16, 4, AVIFGPU_ALPHA_STRAIGHT, 10, AVIFGPU_LAYOUT_PLANAR_YCBCR, AVIFGPU_CHROMA_420, 3);
    avifgpu_encode_desc* old = EndingAtGuardPage(current, AVIFGPU_ENCODE_DESC_V10_SIZE);
    if (old == nullptr)
    {
        std::printf("FAIL guard page\n");
        ++g_failures;
        return checked;
    }
    old->struct_size = AVIFGPU_ENCODE_DESC_V10_SIZE;
    avifgpu_encode_desc full;
    const avifgpu_encode_desc* widened = WidenEncodeDesc(old, &full);
    EncodeParams fromOld;
    FillEncodeParams(*widened, &fromOld);
    const PlaneGeometry g1 = EncodePlaneGeometry(*widened, 1), g2 = EncodePlaneGeometry(*widened, 2);
    if (AVIFGPU_ENCODE_DESC_V10_SIZE != 124 || sizeof(avifgpu_encode_desc) != 128 || ValidateEncodeDesc(old, nullptr) != AVIFGPU_OK ||
        DestLayoutOf(*old) != 0 || widened != &full || full.struct_size != sizeof(avifgpu_encode_desc) || full.dest_layout != 0 ||
        ValidateEncodeDesc(widened, nullptr) != AVIFGPU_OK || full.image_bit_depth != 10 || full.pq_peak_nits != 10000 ||
        std::memcmp(full.row_matrix, current.row_matrix, sizeof(full.row_matrix)) != 0 || EncodeHostColBytes(*widened) != 8 ||
        fromOld.destLayout != 0 || !g1.present || g1.widthSamples != 32 || !g2.present)
    {
        std::printf("FAIL API-10-sized description\n");
        ++g_failures;
    }
    if (WidenEncodeDesc(&current, &full) != &current || DestLayoutOf(current) != 3)
    {
        std::printf("FAIL current-sized description\n");
        ++g_failures;
    }
    avifgpu_encode_desc odd = current;
    for (uint32_t size : { 0u, 40u, 120u, 126u, 132u })
    {
        odd.struct_size = size;
        if (ValidateEncodeDesc(&odd, nullptr) != AVIFGPU_ERR_BAD_PARAM || WidenEncodeDesc(&odd, &full) != &odd)
        {
            std::printf("FAIL description size %u\n", size);
            ++g_failures;
        }
    }
    checked += 3;

    // geometry: 7 x 5 -> 4 x 3 sites (4:2:0), 4 x 5 (4:2:2), 7 x 5 (4:4:4); and EncodeWindow's move of plane 1
    for (int chroma : { AVIFGPU_CHROMA_420, AVIFGPU_CHROMA_422, AVIFGPU_CHROMA_444 })
        for (int dest : { 0, 1, 2, 3 })
        {
            avifgpu_encode_desc d = EncodeDesc(16, 4, AVIFGPU_ALPHA_STRAIGHT, 12, AVIFGPU_LAYOUT_PLANAR_YCBCR, chroma, dest);
            d.width = 7;
            d.height = 5;
            const int xs = chroma == AVIFGPU_CHROMA_444 ? 0 : 1, ys = chroma == AVIFGPU_CHROMA_420 ? 1 : 0;
            const int sites = (7 + xs) >> xs, chromaRows = (5 + ys) >> ys;
            const bool interleaved = dest & 1;
            const PlaneGeometry g0 = EncodePlaneGeometry(d, 0), c1 = EncodePlaneGeometry(d, 1), c2 = EncodePlaneGeometry(d, 2), g3 = EncodePlaneGeometry(d, 3);
            if (!g0.present || g0.widthSamples != 7 || !g3.present || g3.widthSamples != 7 || !c1.present || c1.height != chromaRows ||
                c1.bytesPerSample != 2 || c1.widthSamples != (interleaved ? 2 * sites : sites) || c2.present == interleaved ||
                (!interleaved && (c2.widthSamples != sites || c2.height != chromaRows)) || (interleaved && c2.bytesPerSample != 0))
            {
                std::printf("FAIL geometry chroma %d dest %d\n", chroma, dest);
                ++g_failures;
            }
            EncodeParams p;
            FillEncodeParams(d, &p);
            for (int k = 0; k < 4; ++k)
            {
                p.plane[k] = (k == 2 && interleaved) ? nullptr : reinterpret_cast<void*>(static_cast<uintptr_t>(k + 1) << 32);
                p.planeStride[k] = 1024 * (k + 1);
            }
            p.rows = reinterpret_cast<const void*>(static_cast<uintptr_t>(1) << 40);
            p.rowStride = 4096;
            p.width = 7;
            p.rowCount = 5;
            const int x0 = 4, y0 = 2;
            const EncodeParams w = EncodeWindow(p, 16, x0, y0, 3, 3);
            const int64_t expected1 = static_cast<int64_t>(y0 >> ys) * p.planeStride[1] + static_cast<int64_t>(x0 >> xs) * (interleaved ? 2 : 1) * 2;
            const int64_t expected0 = static_cast<int64_t>(y0) * p.planeStride[0] + x0 * 2;
            if (static_cast<uint8_t*>(w.plane[1]) - static_cast<uint8_t*>(p.plane[1]) != expected1 ||
                static_cast<uint8_t*>(w.plane[0]) - static_cast<uint8_t*>(p.plane[0]) != expected0 || (interleaved && w.plane[2] != nullptr) ||
                static_cast<uint8_t*>(w.plane[3]) - static_cast<uint8_t*>(p.plane[3]) != static_cast<int64_t>(y0) * p.planeStride[3] + x0 * 2)
            {
                std::printf("FAIL EncodeWindow chroma %d dest %d\n", chroma, dest);
                ++g_failures;
            }
            ++checked;
        }
    return checked;
}

// The block halves against the restated alignment rule on random buffers, both kernel families, every layout.
void BlockHalves(std::mt19937_64& rng)
{
    for (int hostDepth : { 8, 16, 32 })
        for (int imageDepth : { 8, 10, 12 })
            for (int chroma : { 1, 2, 3 })
                for (int dest : { 0, 1, 2, 3 })
                    for (int channels : { 3, 4 })
                    {
                        const avifgpu_encode_desc d = EncodeDesc(hostDepth, channels, AlphaFor(channels), imageDepth, AVIFGPU_LAYOUT_PLANAR_YCBCR, chroma, dest);
                        if (ValidateEncodeDesc(&d, nullptr) != AVIFGPU_OK)
                        {
                            continue;
                        }
                        EncodeParams p;
                        FillEncodeParams(d, &p);
                        const bool floatHost = hostDepth == 32;
                        const int planeBytes = imageDepth > 8 ? 2 : 1;
                        for (int trial = 0; trial < 200; ++trial)
                        {
                            const auto pointer = [&](int k) { return reinterpret_cast<void*>((static_cast<uintptr_t>(k + 1) << 32) + 2 * (rng() % 16)); };
                            p.rows = pointer(4);
                            p.rowStride = 4096 + 4 * static_cast<int64_t>(rng() % 8);
                            for (int k = 0; k < 4; ++k)
                            {
                                p.plane[k] = (k == 2 && (dest & 1)) || (k == 3 && channels == 3) ? nullptr : pointer(k);
                                p.planeStride[k] = 2048 + 2 * static_cast<int64_t>(rng() % 16);
                            }
                            p.width = 1 + static_cast<int>(rng() % 40);
                            p.rowCount = 1 + static_cast<int>(rng() % 5);
                            const bool chromaOk = (dest & 1) ? Aligned(p.plane[1], p.planeStride[1], PairAlignment(p, floatHost))
                                                             : Aligned(p.plane[1], p.planeStride[1], floatHost ? (p.xs ? 4 : 8) : (p.xs ? 4 : 8) * planeBytes) &&
                                                                   Aligned(p.plane[2], p.planeStride[2], floatHost ? (p.xs ? 4 : 8) : (p.xs ? 4 : 8) * planeBytes);
                            const int evenRows = p.ys ? (p.rowCount & ~1) : p.rowCount;
                            Interior expected{ 0, 0 }, got;
                            if (floatHost)
                            {
                                const bool ok = chromaOk && Aligned(p.rows, p.rowStride, 16) && Aligned(p.plane[0], p.planeStride[0], 8) &&
                                                (channels == 3 || Aligned(p.plane[3], p.planeStride[3], 8)) && p.width >= 4 && evenRows >= 1;
                                expected = ok ? Interior{ p.width & ~3, evenRows } : Interior{ 0, 0 };
                                got = EncodeRgbF32BlockInterior(p);
                            }
                            else
                            {
                                const int rowAlign = (8 * channels * hostDepth / 8) % 16 == 0 ? 16 : 8;
                                const bool ok = chromaOk && Aligned(p.rows, p.rowStride, rowAlign) && Aligned(p.plane[0], p.planeStride[0], 8 * planeBytes) &&
                                                (channels == 3 || Aligned(p.plane[3], p.planeStride[3], 8 * planeBytes)) && p.width >= 8 && evenRows >= 1;
                                expected = ok ? Interior{ p.width & ~7, evenRows } : Interior{ 0, 0 };
                                got = EncodeRgbIntBlockInterior(p, hostDepth);
                            }
                            if (got.width != expected.width || got.rows != expected.rows)
                            {
                                Fail("block half against the restated alignment rule", hostDepth * 1000 + imageDepth * 10 + dest, trial);
                            }
                        }
                    }
}

void EncodeDestSlice()
{
    const int validations = EncodeDestValidations();
    std::mt19937_64 rng(20261018);
    BlockHalves(rng);
    Counts n;
    for (int hostDepth : { 8, 16 })
        for (int imageDepth : { 8, 10, 12 })
            for (int alphaCase : { 0, 1, 2 })
                for (int chroma : { 1, 2, 3 })
                    for (int dest : { 0, 1, 2, 3 })
                    {
                        const int channels = alphaCase == 0 ? 3 : 4;
                        const int alphaState = alphaCase == 0 ? AVIFGPU_ALPHA_NONE : alphaCase == 1 ? AVIFGPU_ALPHA_STRAIGHT : AVIFGPU_ALPHA_PREMULTIPLIED;
                        const avifgpu_encode_desc d = EncodeDesc(hostDepth, channels, alphaState, imageDepth, AVIFGPU_LAYOUT_PLANAR_YCBCR, chroma, dest);
                        if (ValidateEncodeDesc(&d, nullptr) != AVIFGPU_OK)
                        {
                            continue;
                        }
                        EncodeParams probe;
                        FillEncodeParams(d, &probe);
                        probe.verifiedPremultiply = 1;
                        if (probe.destLayout != dest)
                        {
                            Fail("FillEncodeParams does not carry the layout", n.descriptions, -1);
                        }
                        const bool tuned = EncodeBatchFamilyOf(probe, hostDepth) == EncodeFamily::RgbInt;
                        EncodeParams planarProbe = probe;
                        planarProbe.destLayout = 0;
                        if (!tuned || (EncodeBatchFamilyOf(planarProbe, hostDepth) == EncodeFamily::RgbInt) != tuned)
                        {
                            Fail("description routing depends on the layout", n.descriptions, -1);
                        }
                        ++n.descriptions;
                        const Case<EncodeParams> c = CaseOf(d, probe, n.descriptions);
                        if (((c.planeMask >> 2) & 1) == (dest & 1) || (c.planeMask & 3) != 3 || ((c.planeMask >> 3) & 1) != (channels == 4 ? 1 : 0))
                        {
                            Fail("plane mask", n.descriptions, -1);
                        }
                        for (int trial = 0; trial < 3; ++trial)
                        {
                            CheckInterleavedRoute(c, CheckBatch(rng, d, c, trial == 2 ? 200 : 24, trial, n), tuned, trial);
                        }
                    }
    std::printf("encode_dest descriptions=%d images=%lld units=%lld validations=%d\n", n.descriptions, n.images, n.units, validations);
}

// ---- decode_int ----

void DecodeIntSlice()
{
    std::mt19937_64 rng(1234);
    Counts n;
    for (int hostDepth : { 8, 16 })
        for (int bitDepth : { 8, 10, 12 })
            for (int alpha : { 0, 1, 2 })
                for (int chroma : { 1, 2, 3 })
                {
                    avifgpu_decode_desc d{};
                    d.struct_size = sizeof(d);
                    d.width = 16;
                    d.height = 16;
                    d.colorspace = AVIFGPU_COLORSPACE_YCBCR;
                    d.chroma = chroma;
                    d.bit_depth = bitDepth;
                    d.alpha_state = alpha;
                    d.host_depth = hostDepth;
                    d.nclx = avifgpu_nclx{ 1, 1, 13, 1, 1 };
                    d.pq_peak_nits = 80;
                    int32_t transfer = 0;
                    DecodeParams probe{};
                    if (ValidateDecodeDesc(&d, &transfer, nullptr) != AVIFGPU_OK || !FillDecodeParams(d, transfer, &probe, nullptr))
                    {
                        continue;
                    }
                    ++n.descriptions;
                    const Case<DecodeParams> c = CaseOf(d, probe, n.descriptions);
                    for (int trial = 0; trial < 3; ++trial)
                    {
                        CheckBatch(rng, d, c, trial == 2 ? 300 : 20, trial, n);
                    }
                }
    std::printf("decode_int descriptions=%d images=%lld units=%lld\n", n.descriptions, n.images, n.units);
}

// ---- decode_f32 ----

struct Curve
{
    int transferCharacteristics, ootf;
};

void DecodeF32Slice()
{
    std::mt19937_64 rng(20261016);
    Counts n;
    for (int bitDepth : { 8, 10, 12, 16 })
        for (int alpha : { 0, 1, 2 })
            for (int chroma : { 1, 2, 3 })
                for (Curve curve : { Curve{ 16, 0 }, Curve{ 18, 1 }, Curve{ 18, 0 }, Curve{ 17, 0 } })
                    for (int verified : { 0, 1 })
                    {
                        avifgpu_decode_desc d{};
                        d.struct_size = sizeof(d);
                        d.colorspace = AVIFGPU_COLORSPACE_YCBCR;
                        d.chroma = chroma;
                        d.bit_depth = bitDepth;
                        d.alpha_state = alpha;
                        d.host_depth = 32;
                        d.nclx = avifgpu_nclx{ 1, 9, curve.transferCharacteristics, n.descriptions % 2 ? 9 : 1, (n.descriptions / 2) % 2 };
                        d.hlg_apply_ootf = curve.ootf;
                        d.hlg_display_gamma = 1.2f;
                        d.hlg_peak_nits = 1000;
                        d.pq_peak_nits = 1000;
                        int32_t transfer = 0;
                        DecodeParams probe{};
                        if (ValidateDecodeDesc(&d, &transfer, nullptr) != AVIFGPU_OK || !FillDecodeParams(d, transfer, &probe, nullptr))
                        {
                            continue;
                        }
                        probe.verifiedHlgDivisions = verified;
                        probe.verifiedGreenDivision = verified;
                        probe.verifiedPqRatio = verified;
                        const bool tuned = DecodeBatchFamilyOf(probe) != DecodeFamily::Generic;
                        if (tuned != (DecodeFamilyOf(probe) == DecodeFamily::YccF32))
                        {
                            Fail("DecodeBatchFamilyOf is not the float family for 32-bit hosts", n.descriptions, -1);
                        }
                        const bool expectTuned = bitDepth >= 10 && bitDepth <= 12 && alpha != 2 && (curve.transferCharacteristics != 18 || verified);
                        if (tuned != expectTuned)
                        {
                            Fail("description routing", n.descriptions, -1);
                        }
                        ++n.descriptions;
                        const Case<DecodeParams> c = CaseOf(d, probe, n.descriptions);
                        for (int trial = 0; trial < 3; ++trial)
                        {
                            CheckBatch(rng, d, c, trial == 2 ? 300 : 24, trial, n);
                        }
                    }
    std::printf("decode_f32 descriptions=%d images=%lld units=%lld\n", n.descriptions, n.images, n.units);
}

// ---- decode_rgb ----

// The kernels' block conditions, restated: StreamDecodeKernel reads 8 samples per plane with one 64-bit (8-bit planes) or
// 128-bit load and stores 8 pixels with 64-bit stores (RGB8) or 128-bit ones; TableDecodeF32Kernel reads 128 bits per
// plane and stores 128-bit words.  Width rounded down to 8 pixels, at least 8; every row.
Interior ExpectedInterior(const DecodeParams& p)
{
    const bool tuned = p.colorspace == AVIFGPU_COLORSPACE_RGB && !(p.hasAlpha && p.premultiplied) && p.bitDepth <= 12 &&
                       (p.hostDepth == 8 ? p.bitDepth == 8 : p.bitDepth >= 10);
    const int planeAlign = p.bitDepth > 8 ? 16 : 8;
    const int rowAlign = (p.hostDepth == 8 && !p.hasAlpha) ? 8 : 16;
    bool aligned = Aligned(p.rows, p.rowStride, rowAlign);
    for (int k = 0; k < 4; ++k)
    {
        if (k < 3 || p.hasAlpha)
        {
            aligned = aligned && Aligned(p.plane[k], p.planeStride[k], planeAlign);
        }
    }
    if (!tuned || !aligned || p.width < 8 || p.rowCount < 1)
    {
        return Interior{ 0, 0 };
    }
    return Interior{ p.width & ~7, p.rowCount };
}

// YCbCr and monochrome descriptions route as they did before planar RGB was batched: DecodeBatchFamilyOf is the float
// YCbCr family for 32-bit hosts and the integer one otherwise, with 128- and 256-pixel units; monochrome is never batched.
int YccRoutingCensus()
{
    int ycbcr = 0;
    for (int colorspace : { AVIFGPU_COLORSPACE_YCBCR, AVIFGPU_COLORSPACE_MONOCHROME })
        for (int hostDepth : { 8, 16, 32 })
            for (int bitDepth : { 8, 10, 12, 16 })
                for (int alpha : { 0, 1, 2 })
                    for (int chroma : { 1, 2, 3 })
                        for (Curve curve : { Curve{ 16, 0 }, Curve{ 18, 1 }, Curve{ 17, 0 } })
                            for (int verified : { 0, 1 })
                            {
                                avifgpu_decode_desc d{};
                                d.struct_size = sizeof(d);
                                d.colorspace = colorspace;
                                d.chroma = colorspace == AVIFGPU_COLORSPACE_MONOCHROME ? AVIFGPU_CHROMA_MONOCHROME : chroma;
                                d.bit_depth = bitDepth;
                                d.alpha_state = alpha;
                                d.host_depth = hostDepth;
                                d.nclx = avifgpu_nclx{ 1, 9, curve.transferCharacteristics, 9, 1 };
                                d.hlg_apply_ootf = curve.ootf;
                                d.hlg_display_gamma = 1.2f;
                                d.hlg_peak_nits = 1000;
                                d.pq_peak_nits = 1000;
                                int32_t transfer = 0;
                                DecodeParams p{};
                                if (ValidateDecodeDesc(&d, &transfer, nullptr) != AVIFGPU_OK || !FillDecodeParams(d, transfer, &p, nullptr))
                                {
                                    continue;
                                }
                                p.verifiedHlgDivisions = verified;
                                p.verifiedGreenDivision = verified;
                                p.verifiedPqRatio = verified;
                                ++ycbcr;
                                const bool before = hostDepth == 32 ? (DecodeFamilyOf(p) == DecodeFamily::YccF32) : (DecodeFamilyOf(p) == DecodeFamily::YccInt);
                                if ((DecodeBatchFamilyOf(p) != DecodeFamily::Generic) != before || IsPlanarRgb(DecodeBatchFamilyOf(p)))
                                {
                                    Fail("YCbCr / monochrome description routing changed", ycbcr, -1);
                                }
                                if (colorspace == AVIFGPU_COLORSPACE_MONOCHROME && before)
                                {
                                    Fail("monochrome batched", ycbcr, -1);
                                }
                                if (DecodeBatchUnitPixels(hostDepth == 32 ? DecodeFamily::YccF32 : DecodeFamily::YccInt) != (hostDepth == 32 ? 128 : 256))
                                {
                                    Fail("YCbCr / monochrome unit width changed", ycbcr, -1);
                                }
                            }
    return ycbcr;
}

void DecodeRgbSlice()
{
    const int ycbcr = YccRoutingCensus();
    std::mt19937_64 rng(20261016);
    Counts n;
    for (int hostDepth : { 8, 16, 32 })
        for (int bitDepth : { 8, 10, 12, 16 })
            for (int alpha : { 0, 1, 2 })
                for (int fullRange : { 0, 1 })
                    for (Curve curve : { Curve{ 16, 0 }, Curve{ 18, 1 }, Curve{ 18, 0 }, Curve{ 17, 0 } })
                    {
                        if (hostDepth != 32 && curve.transferCharacteristics != 16)
                        {
                            continue; // integer hosts have no transfer curve: enumerate each description once
                        }
                        avifgpu_decode_desc d{};
                        d.struct_size = sizeof(d);
                        d.colorspace = AVIFGPU_COLORSPACE_RGB;
                        d.chroma = AVIFGPU_CHROMA_444;
                        d.bit_depth = bitDepth;
                        d.alpha_state = alpha;
                        d.host_depth = hostDepth;
                        d.nclx = avifgpu_nclx{ 1, 9, curve.transferCharacteristics, 0, fullRange };
                        d.hlg_apply_ootf = curve.ootf;
                        d.hlg_display_gamma = 1.2f;
                        d.hlg_peak_nits = 1000;
                        d.pq_peak_nits = 1000;
                        int32_t transfer = 0;
                        DecodeParams probe{};
                        if (ValidateDecodeDesc(&d, &transfer, nullptr) != AVIFGPU_OK || !FillDecodeParams(d, transfer, &probe, nullptr))
                        {
                            continue;
                        }
                        const bool tuned = DecodeBatchFamilyOf(probe) != DecodeFamily::Generic;
                        if (tuned != IsPlanarRgb(DecodeBatchFamilyOf(probe)))
                        {
                            Fail("DecodeBatchFamilyOf is not the planar-RGB family for RGB", n.descriptions, -1);
                        }
                        const bool expectTuned = alpha != 2 && bitDepth <= 12 && (hostDepth == 8 ? bitDepth == 8 : bitDepth >= 10);
                        if (tuned != expectTuned)
                        {
                            Fail("description routing", n.descriptions, -1);
                        }
                        if (DecodeBatchUnitPixels(hostDepth == 32 ? DecodeFamily::PlanarRgbF32 : DecodeFamily::PlanarRgbInt) != 256)
                        {
                            Fail("planar-RGB unit width", n.descriptions, -1);
                        }
                        ++n.descriptions;
                        const Case<DecodeParams> c = CaseOf(d, probe, n.descriptions);
                        for (int trial = 0; trial < 3; ++trial)
                        {
                            for (const FakeImage<DecodeParams>& im : CheckBatch(rng, d, c, trial == 2 ? 300 : 24, trial, n))
                            {
                                if (im.rejected)
                                {
                                    continue;
                                }
                                const Interior expected = ExpectedInterior(im.p);
                                const Interior inner = RouteInterior(im.p, hostDepth);
                                const Interior split = IsPlanarRgb(DecodeBatchFamilyOf(im.p)) ? DecodePlanarRgbBlockInterior(im.p) : Interior{ 0, 0 };
                                if (inner.width != expected.width || inner.rows != expected.rows || split.width != inner.width || split.rows != inner.rows)
                                {
                                    Fail("interior against the kernels' restated conditions", n.descriptions, trial);
                                }
                            }
                        }
                    }
    std::printf("decode_rgb descriptions=%d images=%lld units=%lld ycbcr=%d\n", n.descriptions, n.images, n.units, ycbcr);
}

// ---- decode_source ----

int DecodeSourceValidations()
{
    int checked = 0;
    for (int layout : { 0, 1, 2, 3, 4, 5, 8, -1 })
        for (int colorspace : { AVIFGPU_COLORSPACE_YCBCR, AVIFGPU_COLORSPACE_RGB, AVIFGPU_COLORSPACE_MONOCHROME })
            for (int bitDepth : { 8, 10, 12, 16 })
            {
                const avifgpu_decode_desc d = DecodeDesc(colorspace, AVIFGPU_CHROMA_420, bitDepth, 0, bitDepth == 8 ? 8 : 16, layout, 16);
                int32_t transfer = 0;
                const int status = ValidateDecodeDesc(&d, &transfer, nullptr);
                int expected = AVIFGPU_OK;
                if (layout & ~3)
                {
                    expected = AVIFGPU_ERR_BAD_PARAM;
                }
                else if (layout != 0 && colorspace != AVIFGPU_COLORSPACE_YCBCR)
                {
                    expected = AVIFGPU_ERR_UNSUPPORTED;
                }
                else if ((layout & AVIFGPU_SOURCE_MSB_ALIGNED) && bitDepth != 10 && bitDepth != 12)
                {
                    expected = AVIFGPU_ERR_BAD_PARAM;
                }
                if (status != expected)
                {
                    std::printf("FAIL validation layout %d colorspace %d depth %d: %d, expected %d\n", layout, colorspace, bitDepth, status, expected);
                    ++g_failures;
                }
                ++checked;
            }
    // An API-9-sized description as the last bytes before an inaccessible page: accepted, planar, and widened with
    // source_layout 0 without a read past its end.
    const avifgpu_decode_desc current = DecodeDesc(AVIFGPU_COLORSPACE_YCBCR, AVIFGPU_CHROMA_420, 10, 0, 16, 3, 16);
    avifgpu_decode_desc* old = EndingAtGuardPage(current, AVIFGPU_DECODE_DESC_V9_SIZE);
    if (old == nullptr)
    {
        std::printf("FAIL guard page\n");
        ++g_failures;
        return checked;
    }
    old->struct_size = AVIFGPU_DECODE_DESC_V9_SIZE;
    int32_t transfer = 0;
    avifgpu_decode_desc full;
    const avifgpu_decode_desc* widened = WidenDecodeDesc(old, &full);
    if (AVIFGPU_DECODE_DESC_V9_SIZE != 68 || ValidateDecodeDesc(old, &transfer, nullptr) != AVIFGPU_OK || SourceLayoutOf(*old) != 0 ||
        widened != &full || full.struct_size != sizeof(avifgpu_decode_desc) || full.source_layout != 0 || full.bit_depth != 10 || full.pq_peak_nits != 1000)
    {
        std::printf("FAIL API-9-sized description\n");
        ++g_failures;
    }
    if (WidenDecodeDesc(&current, &full) != &current || SourceLayoutOf(current) != 3)
    {
        std::printf("FAIL current-sized description\n");
        ++g_failures;
    }
    avifgpu_decode_desc odd = current;
    odd.struct_size = 40;
    if (ValidateDecodeDesc(&odd, &transfer, nullptr) != AVIFGPU_ERR_BAD_PARAM || WidenDecodeDesc(&odd, &full) != &odd)
    {
        std::printf("FAIL other description size\n");
        ++g_failures;
    }
    // geometry: 4:2:0 of 7 x 5 -> 4 x 3 sites
    for (int layout : { 0, 1, 2, 3 })
    {
        avifgpu_decode_desc d = DecodeDesc(AVIFGPU_COLORSPACE_YCBCR, AVIFGPU_CHROMA_420, 10, 1, 16, layout, 16);
        d.width = 7;
        d.height = 5;
        const PlaneGeometry g1 = DecodePlaneGeometry(d, 1), g2 = DecodePlaneGeometry(d, 2), g0 = DecodePlaneGeometry(d, 0), g3 = DecodePlaneGeometry(d, 3);
        const bool interleaved = layout & 1;
        if (!g0.present || g0.widthSamples != 7 || !g3.present || !g1.present || g1.height != 3 || g1.bytesPerSample != 2 ||
            g1.widthSamples != (interleaved ? 8 : 4) || g2.present == interleaved || (!interleaved && g2.widthSamples != 4))
        {
            std::printf("FAIL geometry layout %d\n", layout);
            ++g_failures;
        }
        ++checked;
    }
    return checked;
}

void DecodeSourceSlice()
{
    const int validations = DecodeSourceValidations();
    std::mt19937_64 rng(20261017);
    Counts n;
    for (int hostDepth : { 8, 16, 32 })
        for (int bitDepth : { 8, 10, 12 })
            for (int alpha : { 0, 1, 2 })
                for (int chroma : { 1, 2, 3 })
                    for (int layout : { 0, 1, 2, 3 })
                        for (int transferCharacteristics : { 16, 18, 17 })
                        {
                            if (hostDepth != 32 && transferCharacteristics != 16)
                            {
                                continue; // integer hosts have no curve
                            }
                            const avifgpu_decode_desc d = DecodeDesc(AVIFGPU_COLORSPACE_YCBCR, chroma, bitDepth, alpha, hostDepth, layout, transferCharacteristics);
                            int32_t transfer = 0;
                            DecodeParams probe{};
                            if (ValidateDecodeDesc(&d, &transfer, nullptr) != AVIFGPU_OK || !FillDecodeParams(d, transfer, &probe, nullptr))
                            {
                                continue;
                            }
                            probe.verifiedHlgDivisions = probe.verifiedGreenDivision = probe.verifiedPqRatio = 1;
                            if (probe.sourceLayout != layout)
                            {
                                Fail("FillDecodeParams does not carry the layout", n.descriptions, -1);
                            }
                            const bool tuned = DecodeBatchFamilyOf(probe) != DecodeFamily::Generic;
                            const bool expectTuned = alpha != 2 && (hostDepth == 32 ? bitDepth > 8 : true);
                            if (tuned != expectTuned)
                            {
                                Fail("description routing", n.descriptions, -1);
                            }
                            ++n.descriptions;
                            const Case<DecodeParams> c = CaseOf(d, probe, n.descriptions);
                            if (((c.planeMask >> 2) & 1) == (layout & 1))
                            {
                                Fail("plane mask", n.descriptions, -1);
                            }
                            for (int trial = 0; trial < 3; ++trial)
                            {
                                CheckInterleavedRoute(c, CheckBatch(rng, d, c, trial == 2 ? 200 : 24, trial, n), tuned, trial);
                            }
                        }
    std::printf("decode_source descriptions=%d images=%lld units=%lld validations=%d\n", n.descriptions, n.images, n.units, validations);
}

// ---- indirect ----

void IndirectSlice()
{
    // the workspace sections are 256-byte aligned, in order, and large enough
    for (int m : { 1, 2, 63, 64, 1000, kIndirectMaxImages })
    {
        const IndirectLayout l = IndirectWorkspaceLayout(m);
        const size_t offsets[5] = { l.interiorFirst, l.windowFirst, l.interior, l.window, l.bytes };
        const size_t need[4] = { 8u * m, 16u * m, sizeof(BatchRecord) * m, 2 * sizeof(BatchRecord) * m };
        if (l.interiorFirst < sizeof(IndirectHeader)) Fail("layout header", m, 0);
        for (int k = 0; k < 4; ++k)
            if (offsets[k] % 256 || offsets[k + 1] < offsets[k] + need[k]) Fail("layout", m, k);
    }

    std::mt19937_64 rng(4321);
    Counts encode;
    for (int hostDepth : { 8, 16 })
        for (int channels : { 3, 4 })
            for (int alpha : { 0, 1, 2 })
                for (int depth : { 8, 10, 12 })
                    for (int chroma : { 1, 2, 3 })
                        for (int matrix : { 1, 0, 9 })
                        {
                            avifgpu_encode_desc d{};
                            d.struct_size = sizeof(d);
                            d.host_depth = hostDepth;
                            d.host_channels = channels;
                            d.alpha_state = alpha;
                            d.image_bit_depth = depth;
                            d.transfer = AVIFGPU_TRANSFER_CLIP;
                            d.pq_peak_nits = 80;
                            d.layout = AVIFGPU_LAYOUT_PLANAR_YCBCR;
                            d.chroma = chroma;
                            d.nclx = avifgpu_nclx{ 1, 1, 13, matrix, 1 };
                            if (ValidateEncodeDesc(&d, nullptr) != AVIFGPU_OK)
                            {
                                continue;
                            }
                            ++encode.descriptions;
                            for (int verified : { 0, 1 })
                            {
                                EncodeParams shared;
                                FillEncodeParams(d, &shared);
                                shared.verifiedPremultiply = verified;
                                CheckBatch(rng, d, CaseOf(d, shared, encode.descriptions), 120, verified, encode);
                            }
                        }

    Counts decode;
    for (int hostDepth : { 8, 16 })
        for (int bitDepth : { 8, 10, 12, 16 })
            for (int alpha : { 0, 1 })
                for (int chroma : { 1, 2, 3 })
                {
                    avifgpu_decode_desc d{};
                    d.struct_size = sizeof(d);
                    d.colorspace = AVIFGPU_COLORSPACE_YCBCR;
                    d.chroma = chroma;
                    d.bit_depth = bitDepth;
                    d.alpha_state = alpha;
                    d.host_depth = hostDepth;
                    d.nclx = avifgpu_nclx{ 1, 1, 13, 1, 1 };
                    d.pq_peak_nits = 80;
                    int32_t transfer = 0;
                    DecodeParams shared{};
                    if (ValidateDecodeDesc(&d, &transfer, nullptr) != AVIFGPU_OK || !FillDecodeParams(d, transfer, &shared, nullptr))
                    {
                        continue;
                    }
                    ++decode.descriptions;
                    for (int trial = 0; trial < 4; ++trial)
                    {
                        CheckBatch(rng, d, CaseOf(d, shared, decode.descriptions), 120, trial, decode);
                    }
                }
    std::printf("indirect descriptions=%d images=%lld units=%lld encode_descriptions=%d encode_images=%lld decode_descriptions=%d decode_images=%lld\n",
                encode.descriptions + decode.descriptions, encode.images + decode.images, encode.units + decode.units, encode.descriptions, encode.images,
                decode.descriptions, decode.images);
}

} // namespace

int main()
{
    EncodeSlice();
    EncodeDestSlice();
    DecodeIntSlice();
    DecodeF32Slice();
    DecodeRgbSlice();
    DecodeSourceSlice();
    IndirectSlice();
    return g_failures == 0 ? 0 : 1;
}
