// tests/native/semiplanar_plan_check.cpp -- host-side check of the semi-planar and MSB-aligned decode sources
// (avifgpu_decode_desc.source_layout) in csrc/host_params.cpp and csrc/batch_plan.h:
//   validation   every layout bit set x colour space x bit depth: non-zero layouts for YCbCr only (UNSUPPORTED otherwise),
//                MSB-aligned for 10/12 bits only, unknown bits BAD_PARAM; an API-9-sized description is accepted, reads as
//                the planar layout and widens to a full one;
//   geometry     interleaved chroma is one plane 1 of 2 * ((width + xs) >> xs) samples and no plane 2;
//   batches      for every YCbCr description into 8-, 16- and 32-bit hosts in each layout, seeded batches of mixed sizes
//                (odd widths, one-row images, misaligned rows, Y and interleaved chroma planes): every pixel covered exactly
//                once; an image batched exactly when the block half (DecodeBlockInterior of DecodeBatchFamilyOf) takes it;
//                the interleaved plane's alignment restated; records' planes where DecodeWindow puts them (two samples per
//                interleaved site); interior units of 256 (128 for 32-bit hosts) pixels; one or two launches per chunk.
// Prints "semiplanar validations=V descriptions=N images=K units=U"; exit code 1 on any failure.
#include "batch_plan.h"
#include "host_params.h"

#include <cstddef>
#include <cstdio>
#include <random>
#include <vector>

using namespace avifgpu;

namespace
{

long long g_failures = 0;

void Fail(const char* what, int description, int batch)
{
    if (++g_failures <= 20)
    {
        std::printf("FAIL %s: description %d, batch %d\n", what, description, batch);
    }
}

avifgpu_decode_desc Desc(int colorspace, int chroma, int bitDepth, int alpha, int hostDepth, int layout, int transferCharacteristics)
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

avifgpu_batch_image BatchImageOf(const DecodeParams& p)
{
    avifgpu_batch_image image{};
    image.width = p.width;
    image.height = p.rowCount;
    image.rows = p.rows;
    image.row_stride_bytes = p.rowStride;
    for (int k = 0; k < 4; ++k)
    {
        image.planes.data[k] = const_cast<void*>(p.plane[k]);
        image.planes.stride[k] = p.planeStride[k];
    }
    return image;
}

void Cover(std::vector<int>& count, const DecodeParams& p, const BatchRecord& r, int colBytes, int description, int batch)
{
    const int64_t offset = static_cast<int64_t>(reinterpret_cast<uintptr_t>(r.rows) - reinterpret_cast<uintptr_t>(p.rows));
    const int y0 = static_cast<int>(offset / p.rowStride);
    const int x0 = static_cast<int>(offset % p.rowStride) / colBytes;
    if (offset < 0 || r.width <= 0 || r.rowCount <= 0 || x0 + r.width > p.width || y0 + r.rowCount > p.rowCount || (y0 & p.ys) != 0)
    {
        Fail("record outside its image or off a row pair", description, batch);
        return;
    }
    const DecodeParams w = DecodeWindow(p, x0, y0, r.width, r.rowCount);
    for (int k = 0; k < 4; ++k)
    {
        if (r.plane[k] != w.plane[k] || r.planeStride[k] != p.planeStride[k])
        {
            Fail("record plane not where DecodeWindow puts it", description, batch);
        }
    }
    // the interleaved plane moves by two samples per chroma site
    if (SourceInterleaved(p.sourceLayout) && p.plane[1] != nullptr)
    {
        const int64_t expected = static_cast<int64_t>(y0 >> p.ys) * p.planeStride[1] + static_cast<int64_t>(x0 >> p.xs) * 2 * (p.bitDepth > 8 ? 2 : 1);
        if (static_cast<const uint8_t*>(r.plane[1]) - static_cast<const uint8_t*>(p.plane[1]) != expected)
        {
            Fail("interleaved chroma window offset", description, batch);
        }
    }
    for (int y = y0; y < y0 + r.rowCount; ++y)
    {
        for (int x = x0; x < x0 + r.width; ++x)
        {
            ++count[static_cast<size_t>(y) * p.width + x];
        }
    }
}

bool CoveredOnce(const std::vector<int>& count)
{
    for (int v : count)
    {
        if (v != 1)
        {
            return false;
        }
    }
    return true;
}

Interior BlockHalfInterior(const DecodeParams& p) { return DecodeBlockInterior(DecodeBatchFamilyOf(p), p); }

// The alignment the tuned kernels' pair loads need of the interleaved plane, restated from the loads: twice the planar
// chroma's bytes per lane, at most 16 (the integer kernels read 16-bit 4:4:4 in two 128-bit loads).
int InterleavedAlignment(const DecodeParams& p)
{
    const int planar = (p.xs ? 4 : 8) * (p.hostDepth == 8 ? 1 : 2);
    if (p.hostDepth == 32)
    {
        return 2 * (p.xs ? 4 : 8);
    }
    return 2 * planar > 16 ? 16 : 2 * planar;
}

int Validations()
{
    int checked = 0;
    for (int layout : { 0, 1, 2, 3, 4, 5, 8, -1 })
        for (int colorspace : { AVIFGPU_COLORSPACE_YCBCR, AVIFGPU_COLORSPACE_RGB, AVIFGPU_COLORSPACE_MONOCHROME })
            for (int bitDepth : { 8, 10, 12, 16 })
            {
                const avifgpu_decode_desc d = Desc(colorspace, AVIFGPU_CHROMA_420, bitDepth, 0, bitDepth == 8 ? 8 : 16, layout, 16);
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
    // an API-9-sized description: accepted, planar, widened with source_layout 0 whatever lies past its end
    avifgpu_decode_desc old = Desc(AVIFGPU_COLORSPACE_YCBCR, AVIFGPU_CHROMA_420, 10, 0, 16, 3, 16);
    old.struct_size = AVIFGPU_DECODE_DESC_V9_SIZE;
    int32_t transfer = 0;
    avifgpu_decode_desc full;
    const avifgpu_decode_desc* widened = WidenDecodeDesc(&old, &full);
    if (AVIFGPU_DECODE_DESC_V9_SIZE != 68 || ValidateDecodeDesc(&old, &transfer, nullptr) != AVIFGPU_OK || SourceLayoutOf(old) != 0 ||
        widened != &full || full.struct_size != sizeof(avifgpu_decode_desc) || full.source_layout != 0 || full.bit_depth != 10 || full.pq_peak_nits != 1000)
    {
        std::printf("FAIL API-9-sized description\n");
        ++g_failures;
    }
    avifgpu_decode_desc current = Desc(AVIFGPU_COLORSPACE_YCBCR, AVIFGPU_CHROMA_420, 10, 0, 16, 3, 16);
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
        avifgpu_decode_desc d = Desc(AVIFGPU_COLORSPACE_YCBCR, AVIFGPU_CHROMA_420, 10, 1, 16, layout, 16);
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

} // namespace

int main()
{
    const int validations = Validations();
    std::mt19937_64 rng(20261017);
    int descriptions = 0;
    long long images = 0, units = 0;
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
                            const avifgpu_decode_desc d = Desc(AVIFGPU_COLORSPACE_YCBCR, chroma, bitDepth, alpha, hostDepth, layout, transferCharacteristics);
                            int32_t transfer = 0;
                            DecodeParams probe{};
                            if (ValidateDecodeDesc(&d, &transfer, nullptr) != AVIFGPU_OK || !FillDecodeParams(d, transfer, &probe, nullptr))
                            {
                                continue;
                            }
                            probe.verifiedHlgDivisions = probe.verifiedGreenDivision = probe.verifiedPqRatio = 1;
                            if (probe.sourceLayout != layout)
                            {
                                Fail("FillDecodeParams does not carry the layout", descriptions, -1);
                            }
                            const DecodeFamily family = DecodeBatchFamilyOf(probe);
                        const bool tuned = family != DecodeFamily::Generic;
                            const bool expectTuned = alpha != 2 && (hostDepth == 32 ? bitDepth > 8 : true);
                            if (tuned != expectTuned)
                            {
                                Fail("description routing", descriptions, -1);
                            }
                            ++descriptions;
                            int planeMask = 0;
                            for (int k = 0; k < 4; ++k)
                            {
                                planeMask |= DecodePlaneGeometry(d, k).present ? 1 << k : 0;
                            }
                            if (((planeMask >> 2) & 1) == (layout & 1))
                            {
                                Fail("plane mask", descriptions, -1);
                            }
                            const int colBytes = DecodeHostColBytes(d);
                            for (int trial = 0; trial < 3; ++trial)
                            {
                                const int n = 1 + static_cast<int>(rng() % (trial == 2 ? 200 : 24));
                                std::vector<DecodeParams> params(n);
                                std::vector<int> shapes(n);
                                for (int i = 0; i < n; ++i)
                                {
                                    avifgpu_decode_desc di = d;
                                    const int shape = shapes[i] = static_cast<int>(rng() % 8);
                                    di.width = shape == 0 ? 1 + static_cast<int>(rng() % 9) : 1 + static_cast<int>(rng() % 600);
                                    di.height = shape == 1 ? 1 : 1 + static_cast<int>(rng() % 9);
                                    DecodeParams& p = params[i];
                                    FillDecodeParams(di, transfer, &p, nullptr);
                                    p.verifiedHlgDivisions = p.verifiedGreenDivision = p.verifiedPqRatio = 1;
                                    const uintptr_t base = static_cast<uintptr_t>(i + 1) << 36;
                                    p.rows = reinterpret_cast<void*>(base + (shape == 2 ? 4 : 0));
                                    p.rowStride = (static_cast<int64_t>(di.width) * colBytes + 63) / 64 * 64 + 64;
                                    p.rowCount = di.height;
                                    for (int k = 0; k < 4; ++k)
                                    {
                                        const PlaneGeometry g = DecodePlaneGeometry(di, k);
                                        if (g.present)
                                        {
                                            p.plane[k] = reinterpret_cast<const void*>(base + (static_cast<uintptr_t>(k + 1) << 30) + (shape == 3 && k == 0 ? 2 : 0));
                                            p.planeStride[k] = (static_cast<int64_t>(g.widthSamples) * g.bytesPerSample + 63) / 64 * 64 + 128;
                                        }
                                    }
                                    // misalign plane 1 by half the interleaved load (shape 4) or just its stride (shape 5)
                                    if ((shape == 4 || shape == 5) && (layout & 1))
                                    {
                                        const int half = InterleavedAlignment(p) / 2;
                                        if (shape == 4)
                                        {
                                            p.plane[1] = static_cast<const uint8_t*>(p.plane[1]) + half;
                                        }
                                        else
                                        {
                                            p.planeStride[1] += half;
                                        }
                                    }
                                }
                                std::vector<avifgpu_batch_image> batch(n);
                                for (int i = 0; i < n; ++i)
                                {
                                    batch[i] = BatchImageOf(params[i]);
                                }
                                images += n;

                                // ---- the host plan ----
                                BatchPlan plan;
                                PlanDecodeBatch(probe, planeMask, batch.data(), n, &plan);
                                std::vector<std::vector<int>> count(n);
                                std::vector<int> batched(n, 0);
                                for (int i = 0; i < n; ++i)
                                {
                                    count[i].assign(static_cast<size_t>(params[i].width) * params[i].rowCount, 0);
                                }
                                const int unitPixels = DecodeBatchUnitPixels(hostDepth == 32 ? DecodeFamily::YccF32 : DecodeFamily::YccInt);
                                int last = -1;
                                for (const BatchChunk& c : plan.chunks)
                                {
                                    if (c.images < 1 || c.images > kBatchChunkImages)
                                    {
                                        Fail("chunk size", descriptions, trial);
                                    }
                                    bool edges = false;
                                    int64_t first = 0;
                                    for (int j = 0; j < c.images; ++j)
                                    {
                                        const int i = c.imageIndex[j];
                                        if (i <= last)
                                        {
                                            Fail("image order", descriptions, trial);
                                        }
                                        last = i;
                                        batched[i] = 1;
                                        const Interior inner = BlockHalfInterior(params[i]);
                                        if (c.interior[j].width != inner.width || c.interior[j].rowCount != inner.rows || c.interior[j].firstUnit != first)
                                        {
                                            Fail("chunk interior", descriptions, trial);
                                        }
                                        first += BatchInteriorUnits(inner.width, inner.rows, params[i].ys, unitPixels);
                                        edges = edges || inner.width < params[i].width || inner.rows < params[i].rowCount;
                                        Cover(count[i], params[i], c.interior[j], colBytes, descriptions, trial);
                                    }
                                    if (first != c.interiorUnits)
                                    {
                                        Fail("chunk unit total", descriptions, trial);
                                    }
                                    for (int j = 0; j < c.windows; ++j)
                                    {
                                        Cover(count[c.windowImage[j]], params[c.windowImage[j]], c.window[j], colBytes, descriptions, trial);
                                    }
                                    if (BatchChunkLaunches(c) != (edges ? 2 : 1))
                                    {
                                        Fail("chunk launches", descriptions, trial);
                                    }
                                }
                                for (const int32_t i : plan.fallback)
                                {
                                    batched[i] = 2;
                                    for (int& v : count[i])
                                    {
                                        ++v;
                                    }
                                }
                                for (int i = 0; i < n; ++i)
                                {
                                    const DecodeParams& p = params[i];
                                    const Interior inner = BlockHalfInterior(p);
                                    if ((inner.width > 0) != (batched[i] == 1))
                                    {
                                        Fail("image routing", descriptions, trial);
                                    }
                                    if (!CoveredOnce(count[i]))
                                    {
                                        Fail("host plan: pixel not covered exactly once", descriptions, trial);
                                    }
                                    if ((layout & 1) && inner.width > 0 && !Aligned(p.plane[1], p.planeStride[1], InterleavedAlignment(p)))
                                    {
                                        Fail("a misaligned interleaved plane took the tuned route", descriptions, trial);
                                    }
                                    if ((layout & 1) && (shapes[i] == 4 || shapes[i] == 5) && inner.width > 0)
                                    {
                                        Fail("a misaligned interleaved plane has an interior", descriptions, trial);
                                    }
                                    if ((layout & 1) && tuned && shapes[i] >= 6 && p.width >= 8 && p.rowCount >= 2 && inner.width == 0)
                                    {
                                        Fail("an aligned interleaved image lost its interior", descriptions, trial);
                                    }
                                }

                                // ---- the per-image step, as the plan kernel runs it ----
                                std::vector<int64_t> interiorFirst(n), interiorUnits(n);
                                int64_t total = 0;
                                for (int i = 0; i < n; ++i)
                                {
                                    const BatchImagePlan step = PlanBatchDecodeImage(probe, family, planeMask, batch[i]);
                                    std::vector<int> covered(static_cast<size_t>(params[i].width) * params[i].rowCount, 0);
                                    const Interior inner = BlockHalfInterior(params[i]);
                                    if (step.status != AVIFGPU_OK || step.interior.width != inner.width || (inner.width > 0 && step.interior.rowCount != inner.rows))
                                    {
                                        Fail("step interior", descriptions, trial);
                                    }
                                    if (step.interior.width > 0)
                                    {
                                        Cover(covered, params[i], step.interior, colBytes, descriptions, trial);
                                        const int64_t expected = static_cast<int64_t>((inner.width + unitPixels - 1) / unitPixels) * (inner.rows >> params[i].ys);
                                        if (step.interiorUnits != expected)
                                        {
                                            Fail("step interior units", descriptions, trial);
                                        }
                                    }
                                    for (int k = 0; k < step.windows; ++k)
                                    {
                                        Cover(covered, params[i], step.window[k], colBytes, descriptions, trial);
                                        if (step.windowUnits[k] != BatchEdgeUnits(step.window[k].width, step.window[k].rowCount, 0, 0))
                                        {
                                            Fail("step window units", descriptions, trial);
                                        }
                                    }
                                    if (!CoveredOnce(covered))
                                    {
                                        Fail("step: pixel not covered exactly once", descriptions, trial);
                                    }
                                    interiorFirst[i] = total;
                                    interiorUnits[i] = step.interiorUnits;
                                    total += step.interiorUnits;
                                }
                                int record = 0;
                                for (int64_t u = 0; u < total; ++u)
                                {
                                    record = FindRecord(interiorFirst.data(), n, record, u);
                                    if (u < interiorFirst[record] || u >= interiorFirst[record] + interiorUnits[record])
                                    {
                                        Fail("FindRecord", descriptions, trial);
                                        break;
                                    }
                                }
                                units += total;
                            }
                        }
    std::printf("semiplanar validations=%d descriptions=%d images=%lld units=%lld\n", validations, descriptions, images, units);
    return g_failures == 0 ? 0 : 1;
}
