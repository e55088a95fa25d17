// tests/native/rgb_batch_plan_check.cpp -- host-side check of the planar-RGB decode planning (csrc/batch_plan.h,
// csrc/host_params.cpp): PlanDecodeBatch behind avifgpu_decode_batch_device, and the per-image step PlanBatchDecodeImage
// that the plan kernel of avifgpu_decode_batch_indirect runs.  For every valid planar-RGB description (host depths 8 / 16 /
// 32, bit depths 8 / 10 / 12 / 16, alpha none / straight / premultiplied, full and limited range, and for 32-bit hosts PQ,
// HLG with and without the OOTF and SMPTE 428) and seeded random batches of 1 to 300 images of mixed sizes -- widths 1 to
// 7, 8, 9, 255, 256, 257 and random ones, one-row images, some with rows misaligned by 4 or 8 bytes, some with an R, G, B
// or alpha plane misaligned by 2 or 8 bytes -- on fake padded planes:
//   description    DecodeBatchFamilyOf is a planar-RGB family, and takes exactly the descriptions with no or straight alpha
//                  and a depth its kernel reads;
//   host plans     every pixel of every image is covered exactly once by an interior, a window or a direct call; an
//                  image is batched exactly when the route (DecodeBatchFamilyOf, DecodeBlockInterior) of its own block
//                  take it, with that interior, which is also the one an independent statement of the kernels' alignment
//                  rules gives; chunks keep image order and hold at most kBatchChunkImages images; first units are running
//                  sums of 256-pixel units; the only window of a batched image is its right strip; a chunk has a second
//                  launch exactly when one of its images has a width that is not a multiple of 8;
//   per-image step every pixel covered exactly once by the interior and windows; every record's planes where DecodeWindow
//                  puts them; interior units counted with the 256-pixel unit, window units as BatchEdgeUnits; FindRecord
//                  over the concatenated interior units finds the record that owns each unit.
// YCbCr and monochrome descriptions route as they did: DecodeBatchFamilyOf is the float YCbCr family for 32-bit hosts and
// the integer one otherwise, with 128- and 256-pixel units; monochrome is never batched.
// Prints "rgb descriptions=N images=K units=U ycbcr=Y"; exit code 1 on any failure.
#include "batch_plan.h"
#include "host_params.h"

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

// The window of `p` a record's rows pointer starts, or false when it is not inside the image.
bool Origin(const DecodeParams& p, const BatchRecord& r, int colBytes, int& x0, int& y0)
{
    const int64_t offset = static_cast<int64_t>(reinterpret_cast<uintptr_t>(r.rows) - reinterpret_cast<uintptr_t>(p.rows));
    if (offset < 0)
    {
        return false;
    }
    y0 = static_cast<int>(offset / p.rowStride);
    x0 = static_cast<int>(offset % p.rowStride) / colBytes;
    return r.width > 0 && r.rowCount > 0 && x0 + r.width <= p.width && y0 + r.rowCount <= p.rowCount;
}

void Cover(std::vector<int>& count, const DecodeParams& p, const BatchRecord& r, int colBytes, int description, int batch)
{
    int x0, y0;
    if (!Origin(p, r, colBytes, x0, y0))
    {
        Fail("record outside its image", description, batch);
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

bool AlignedTo(const void* p, int64_t stride, int alignment)
{
    return reinterpret_cast<uintptr_t>(p) % alignment == 0 && stride % alignment == 0;
}

// The kernels' block conditions, restated: StreamDecodeKernel reads 8 samples per plane with one 64-bit (8-bit planes) or
// 128-bit load and stores 8 pixels with 64-bit stores (RGB8) or 128-bit ones; TableDecodeF32Kernel reads 128 bits per
// plane and stores 128-bit words.  Width rounded down to 8 pixels, at least 8; every row.
bool IsPlanarRgb(DecodeFamily family) { return family == DecodeFamily::PlanarRgbInt || family == DecodeFamily::PlanarRgbF32; }

Interior ExpectedInterior(const DecodeParams& p)
{
    const bool tuned = p.colorspace == AVIFGPU_COLORSPACE_RGB && !(p.hasAlpha && p.premultiplied) && p.bitDepth <= 12 &&
                       (p.hostDepth == 8 ? p.bitDepth == 8 : p.bitDepth >= 10);
    const int planeAlign = p.bitDepth > 8 ? 16 : 8;
    const int rowAlign = (p.hostDepth == 8 && !p.hasAlpha) ? 8 : 16;
    bool aligned = AlignedTo(p.rows, p.rowStride, rowAlign);
    for (int k = 0; k < 4; ++k)
    {
        if (k < 3 || p.hasAlpha)
        {
            aligned = aligned && AlignedTo(p.plane[k], p.planeStride[k], planeAlign);
        }
    }
    if (!tuned || !aligned || p.width < 8 || p.rowCount < 1)
    {
        return Interior{ 0, 0 };
    }
    return Interior{ p.width & ~7, p.rowCount };
}

constexpr int kWidths[] = { 1, 2, 3, 7, 8, 9, 255, 256, 257, 512, 513 };

} // namespace

int main()
{
    std::mt19937_64 rng(20261016);
    int descriptions = 0, ycbcr = 0;
    long long images = 0, units = 0;
    struct Curve
    {
        int transferCharacteristics, ootf;
    };

    // ---- YCbCr and monochrome descriptions route as before ----
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

    // ---- planar RGB ----
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
                        const DecodeFamily family = DecodeBatchFamilyOf(probe);
                        const bool tuned = family != DecodeFamily::Generic;
                        if (tuned != IsPlanarRgb(DecodeBatchFamilyOf(probe)))
                        {
                            Fail("DecodeBatchFamilyOf is not the planar-RGB family for RGB", descriptions, -1);
                        }
                        const bool expectTuned = alpha != 2 && bitDepth <= 12 && (hostDepth == 8 ? bitDepth == 8 : bitDepth >= 10);
                        if (tuned != expectTuned)
                        {
                            Fail("description routing", descriptions, -1);
                        }
                        if (DecodeBatchUnitPixels(hostDepth == 32 ? DecodeFamily::PlanarRgbF32 : DecodeFamily::PlanarRgbInt) != 256)
                        {
                            Fail("planar-RGB unit width", descriptions, -1);
                        }
                        ++descriptions;
                        int planeMask = 0;
                        for (int k = 0; k < 4; ++k)
                        {
                            planeMask |= DecodePlaneGeometry(d, k).present ? 1 << k : 0;
                        }
                        const int colBytes = DecodeHostColBytes(d);
                        for (int trial = 0; trial < 3; ++trial)
                        {
                            const int n = 1 + static_cast<int>(rng() % (trial == 2 ? 300 : 24));
                            std::vector<DecodeParams> params(n);
                            for (int i = 0; i < n; ++i)
                            {
                                avifgpu_decode_desc di = d;
                                const int shape = static_cast<int>(rng() % 10);
                                di.width = shape < 4 ? kWidths[rng() % (sizeof(kWidths) / sizeof(kWidths[0]))] : 1 + static_cast<int>(rng() % 600);
                                di.height = shape == 4 ? 1 : 1 + static_cast<int>(rng() % 9);
                                DecodeParams& p = params[i];
                                FillDecodeParams(di, transfer, &p, nullptr);
                                const uintptr_t base = static_cast<uintptr_t>(i + 1) << 36;
                                p.rows = reinterpret_cast<void*>(base + (shape == 5 ? 4 : shape == 6 ? 8 : 0));
                                p.rowStride = (static_cast<int64_t>(di.width) * colBytes + 63) / 64 * 64 + 64;
                                p.rowCount = di.height;
                                const int oddPlane = static_cast<int>(rng() % 4);
                                for (int k = 0; k < 4; ++k)
                                {
                                    const PlaneGeometry g = DecodePlaneGeometry(di, k);
                                    if (g.present)
                                    {
                                        const uintptr_t off = (k == oddPlane && shape == 7) ? 2 : (k == oddPlane && shape == 8) ? 8 : 0;
                                        p.plane[k] = reinterpret_cast<const void*>(base + (static_cast<uintptr_t>(k + 1) << 30) + off);
                                        p.planeStride[k] = (static_cast<int64_t>(g.widthSamples) * g.bytesPerSample + 63) / 64 * 64 + 128;
                                    }
                                }
                            }
                            std::vector<avifgpu_batch_image> batch(n);
                            for (int i = 0; i < n; ++i)
                            {
                                batch[i] = BatchImageOf(params[i]);
                                const Interior expected = ExpectedInterior(params[i]);
                                const Interior inner = DecodeBlockInterior(DecodeBatchFamilyOf(params[i]), params[i]);
                                const Interior split = IsPlanarRgb(DecodeBatchFamilyOf(params[i])) ? DecodePlanarRgbBlockInterior(params[i]) : Interior{ 0, 0 };
                                if (inner.width != expected.width || inner.rows != expected.rows || split.width != inner.width || split.rows != inner.rows)
                                {
                                    Fail("interior against the kernels' restated conditions", descriptions, trial);
                                }
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
                                    const Interior inner = DecodeBlockInterior(DecodeBatchFamilyOf(params[i]), params[i]);
                                    if (c.interior[j].width != inner.width || c.interior[j].rowCount != inner.rows || c.interior[j].firstUnit != first)
                                    {
                                        Fail("chunk interior", descriptions, trial);
                                    }
                                    first += BatchInteriorUnits(inner.width, inner.rows, 0, 256);
                                    edges = edges || params[i].width % 8 != 0;
                                    Cover(count[i], params[i], c.interior[j], colBytes, descriptions, trial);
                                }
                                if (first != c.interiorUnits)
                                {
                                    Fail("chunk unit total", descriptions, trial);
                                }
                                for (int j = 0; j < c.windows; ++j)
                                {
                                    const DecodeParams& p = params[c.windowImage[j]];
                                    const BatchRecord& w = c.window[j];
                                    if (w.width != p.width % 8 || w.rowCount != p.rowCount || w.rows != static_cast<const uint8_t*>(p.rows) + (p.width & ~7) * colBytes)
                                    {
                                        Fail("a window that is not the right strip", descriptions, trial);
                                    }
                                    Cover(count[c.windowImage[j]], p, w, colBytes, descriptions, trial);
                                }
                                if (BatchChunkLaunches(c) != (edges ? 2 : 1))
                                {
                                    Fail("chunk launches", descriptions, trial);
                                }
                            }
                            int batchedImages = 0;
                            for (int i = 0; i < n; ++i)
                            {
                                batchedImages += DecodeBlockInterior(DecodeBatchFamilyOf(params[i]), params[i]).width > 0 ? 1 : 0;
                            }
                            if (static_cast<int>(plan.chunks.size()) != (batchedImages + kBatchChunkImages - 1) / kBatchChunkImages)
                            {
                                Fail("chunk count", descriptions, trial);
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
                                if ((DecodeBlockInterior(DecodeBatchFamilyOf(params[i]), params[i]).width > 0) != (batched[i] == 1))
                                {
                                    Fail("image routing", descriptions, trial);
                                }
                                if (!CoveredOnce(count[i]))
                                {
                                    Fail("host plan: pixel not covered exactly once", descriptions, trial);
                                }
                            }

                            // ---- the per-image step, as the plan kernel runs it ----
                            std::vector<int64_t> interiorFirst(n);
                            std::vector<int64_t> interiorUnits(n);
                            int64_t total = 0;
                            for (int i = 0; i < n; ++i)
                            {
                                const BatchImagePlan step = PlanBatchDecodeImage(probe, family, planeMask, batch[i]);
                                std::vector<int> covered(static_cast<size_t>(params[i].width) * params[i].rowCount, 0);
                                const Interior inner = DecodeBlockInterior(DecodeBatchFamilyOf(params[i]), params[i]);
                                if (step.status != AVIFGPU_OK || step.interior.width != inner.width || (inner.width > 0 && step.interior.rowCount != inner.rows))
                                {
                                    Fail("step interior", descriptions, trial);
                                }
                                if (step.interior.width > 0)
                                {
                                    Cover(covered, params[i], step.interior, colBytes, descriptions, trial);
                                    const int64_t expected = static_cast<int64_t>((inner.width + 255) / 256) * inner.rows;
                                    if (step.interiorUnits != expected)
                                    {
                                        Fail("step interior units", descriptions, trial);
                                    }
                                    if (step.windows != (params[i].width % 8 != 0 ? 1 : 0))
                                    {
                                        Fail("step windows", descriptions, trial);
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
                                if (FindRecord(interiorFirst.data(), n, 0, u) != record)
                                {
                                    Fail("FindRecord from record 0", descriptions, trial);
                                    break;
                                }
                            }
                            units += total;
                        }
                    }
    std::printf("rgb descriptions=%d images=%lld units=%lld ycbcr=%d\n", descriptions, images, units, ycbcr);
    return g_failures == 0 ? 0 : 1;
}
